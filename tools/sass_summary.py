#!/usr/bin/env python
"""Static evidence for the hot kernels (no GPU needed): registers / shared memory / spills
from the ptxas logs and the SASS instruction mix of each kernel from `cuobjdump -sass`.

    python tools/sass_summary.py [tag]     -> profiles/<tag>_sass_summary.json,
                                              profiles/<tag>_ptxas_{pv,wind,heat,plan}.log

The mix counts every SASS instruction of the function body (loop bodies once; it is an
instruction MIX, not a dynamic count -- the dynamic count per step comes from ncu's
smsp__inst_executed in the same profiles/ directory).  Two mnemonic groups are listed separately:
Blackwell-only instructions (packed FP32, tcgen05 / tensor memory), which an sm_90a build must not
contain, and Hopper's asynchronous-copy / barrier / cluster instructions (TMA, mbarrier), which
are legitimate on sm_90a and listed so their use is on record."""
import collections
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "atlite_b200", "csrc")
TAG = sys.argv[1] if len(sys.argv) > 1 else "r2"

KERNELS = {
    "pv_fused (shuffle reduce, ERA5 default, solar position in-kernel)": ("pv.o", r"k_fused_reduceINS_6PvPhysILi1ELb1EEELi2ELi5E"),
    "pv_fused_stored_solar_f64": ("pv.o", r"k_fused_reduceINS_6PvPhysILi2ELb1EEELi2ELi4E"),
    "pv_fused_era5_inputs_runtime_switches (mode 4)": ("pv.o", r"k_fused_reduceINS_6PvPhysILi4ELb1EEELi2ELi4E"),
    "pv_fused_general (mode 0)": ("pv.o", r"k_fused_reduceINS_6PvPhysILi0ELb1EEELi1ELi4E"),
    "pv_fused_era5_raw (mode 5: raw ssrd/ssr/tisr/fdir, ERA5 default)": ("pv.o", r"k_fused_reduceINS_6PvPhysILi5ELb1EEELi2ELi5E"),
    "pv_fused_era5_raw_general (mode 6)": ("pv.o", r"k_fused_reduceINS_6PvPhysILi6ELb1EEELi1ELi4E"),
    "wind_fused_log_lattice_folded (shuffle reduce, resident weights, L2 prefetch)": ("wind.o", r"k_fused_reduceINS_8WindPhysILb1ELi1ELi1EEELi2ELi6E"),
    "wind_raw_fused_log_lattice_folded (u100, v100, fsr)": ("wind.o", r"k_fused_reduceINS_11WindRawPhysILb1ELi1ELi1EEELi2ELi6E"),
    "wind_fused_log_saturating_table (ATL_WIND_TABLE=3)": ("wind.o", r"k_fused_reduceINS_8WindPhysILb1ELi1ELi4EEELi2ELi6E"),
    "heat_fused (staged reduce)": ("heat.o", r"k_heatILi0ELb1"),
    "spmm_fused": ("plan.o", r"k_fused_reduceINS_12IdentityPhysILb1EEELi4"),
    "pv_cells_timesum": ("pv.o", r"7k_cellsINS_6PvPhysILi1ELb1EEELi1"),
    "line_rating (128-bit lanes, solar position in-kernel)": ("line_rating.o", r"k_line_ratingILb1ELi0ELb0E"),
    "line_rating_raw (t2m, u100, v100, fdir; solar position in-kernel)": ("line_rating.o", r"k_line_ratingILb1ELi0ELb1E"),
    "line_rating_stored_solar_f64": ("line_rating.o", r"k_line_ratingILb1ELi2ELb0E"),
    "line_rating_raw_stored_solar_f64": ("line_rating.o", r"k_line_ratingILb1ELi2ELb1E"),
    "line_rating_raw_scalar (solar position in-kernel)": ("line_rating.o", r"k_line_ratingILb0ELi0ELb1E"),
}
CLASSES = [
    ("fp32_packed", r"^(FFMA2|FMUL2|FADD2)"),
    ("fp32_fma", r"^(FFMA|FMUL|FADD|FMNMX|FSEL|FSETP|FCHK|FSET)"),
    ("mufu", r"^MUFU"),
    ("convert", r"^(F2I|I2F|F2F|I2FP|F2FP)"),
    ("int_alu", r"^(IADD3|IADD|IMAD|LOP3|SHF|LEA|ISETP|SEL|VIADD|VIMNMX|VIADDMNMX|IMNMX|PRMT|LOP|IABS|MOV|HFMA2|SGXT|BMSK|PLOP3|P2R|R2P|POPC|FLO)"),
    ("global_load", r"^LDG"),
    ("global_store_atomic", r"^(STG|REDG|ATOMG|RED|ATOM)"),
    ("shared_load", r"^LDS"),
    ("shared_store", r"^STS"),
    ("const_uniform", r"^(LDC|LDCU|ULDC|UMOV|UIADD3|ULEA|UISETP|UIMAD|USHF|ULOP3|S2UR|S2R|R2UR|UPRMT|USEL|UFLO|UPOPC|CS2R)"),
    ("shuffle_vote", r"^(SHFL|VOTE|MATCH|REDUX)"),
    ("l2_prefetch", r"^CCTL\.E\.PF2"),
    ("control", r"^(BRA|BSSY|BSYNC|EXIT|CALL|RET|WARPSYNC|BAR|NOP|YIELD|BREAK|BMOV|DEPBAR|ERRBAR|MEMBAR|CCTL|NANOSLEEP|BPT|KILL|RPCMOV|ENDCOLLECTIVE)"),
    ("local_mem", r"^(LDL|STL)"),
]
BLACKWELL_ONLY = r"^(FFMA2|FMUL2|FADD2|TCGEN|UTC|STTM|LDTM|UGETNEXT)"
HOPPER_ASYNC = r"^(UTMA|UBLKCP|SYNCS|FENCE\.VIEW|ACQBULK|CLUSTER|ELECT)"


def functions(obj):
    out = subprocess.run(["cuobjdump", "-sass", os.path.join(CSRC, obj)], capture_output=True, text=True).stdout
    cur, res = None, {}
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            res[cur] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if m and cur:
            ins = re.sub(r"^@!?U?P\d+\s+", "", m.group(1).strip())
            res[cur].append(ins)
    return res


def ptxas(obj):
    log = os.path.join(CSRC, obj.replace(".o", ".ptxas.log"))
    info, cur = {}, None
    if not os.path.exists(log):
        return info
    for line in open(log):
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            info[cur] = {}
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            info[cur].update(stack_bytes=int(m.group(1)), spill_store_bytes=int(m.group(2)), spill_load_bytes=int(m.group(3)))
        m = re.search(r"Used (\d+) registers", line)
        if m and cur:
            info[cur]["registers"] = int(m.group(1))
            s = re.search(r"(\d+) bytes smem", line)
            info[cur]["static_smem_bytes"] = int(s.group(1)) if s else 0
    return info


def main():
    os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
    summary = {"how": "cuobjdump -sass + ptxas -v of the in-tree objects (nvcc -gencode arch=compute_90a,code=sm_90a "
                      "-O3 -lineinfo -ftz=true -prec-div=false -prec-sqrt=false); static instruction mix per kernel",
               "kernels": {}}
    cache_f, cache_p = {}, {}
    for name, (obj, pat) in KERNELS.items():
        fs = cache_f.setdefault(obj, functions(obj))
        ps = cache_p.setdefault(obj, ptxas(obj))
        hits = [f for f in fs if re.search(pat, f)]
        if not hits:
            summary["kernels"][name] = {"error": f"no function matches {pat}"}
            continue
        for f in hits:
            ins = fs[f]
            mix = collections.Counter()
            other = collections.Counter()
            for i in ins:
                op = i.split()[0]
                for cls, rx in CLASSES:
                    if re.match(rx, op):
                        mix[cls] += 1
                        break
                else:
                    other[op.split(".")[0]] += 1
            bw = collections.Counter(i.split()[0].split(".")[0] for i in ins if re.match(BLACKWELL_ONLY, i.split()[0]))
            hop = collections.Counter(i.split()[0].split(".")[0] for i in ins if re.match(HOPPER_ASYNC, i.split()[0]))
            wide = collections.Counter(re.match(r"(LDG|LDS|STS|STG)\S*", i).group(0) for i in ins
                                       if re.match(r"(LDG|LDS|STS|STG)", i))
            ts = re.search(r"Li(\d+)EEEvT_", f)
            key = name if len(hits) == 1 else f"{name}_stage{ts.group(1) if ts else len(summary['kernels'])}"
            summary["kernels"][key] = {"function": f, "instructions": len(ins), "mix": dict(mix),
                                       "unclassified": dict(other), "blackwell_only_mnemonics": dict(bw),
                                       "hopper_async_mnemonics": dict(hop),
                                       "memory_ops_by_width": dict(wide), **ps.get(f, {})}
    with open(os.path.join(ROOT, "profiles", f"{TAG}_sass_summary.json"), "w") as fh:
        json.dump(summary, fh, indent=1)
    for obj in ("pv", "wind", "heat", "plan"):
        src = os.path.join(CSRC, f"{obj}.ptxas.log")
        if os.path.exists(src):
            with open(src) as a, open(os.path.join(ROOT, "profiles", f"{TAG}_ptxas_{obj}.log"), "w") as b:
                b.write(a.read())
    for k, v in summary["kernels"].items():
        print(k, {x: v.get(x) for x in ("instructions", "registers", "spill_store_bytes")}, v.get("mix"))


if __name__ == "__main__":
    main()
