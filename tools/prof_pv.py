#!/usr/bin/env python
"""Kernel-only timing / ncu target for the fused kernels on device-resident data.

    ATL_TB=<tb> python tools/prof_pv.py [pv|wind|heat|spmm|pvsum|pvcube|windsum|windcube] [small|big|odd|oddpad|c5] [reps]

small = 200x200x8760 -> 100 shapes (bench workload); big = 1440x720x438 -> 3000 shapes;
odd = 201x199x8760 unpadded (scalar lanes); oddpad = the same with rows padded to 204.
Prints one JSON line with the median CUDA-event time and achieved GB/s.
"""
import json
import os
import sys
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import atlite_b200 as ab  # noqa: E402
from bench import hbm_peak  # noqa: E402
from atlite_b200 import _lib, engine, synthetic as syn  # noqa: E402

if os.environ.get("ATL_LIB_PATH"):  # A/B timing: another build of the library, e.g. another commit's
    _lib.LIB_PATH = os.path.abspath(os.environ["ATL_LIB_PATH"])
from atlite_b200.convert import _HeatSpec, _PvSpec, _WindSpec  # noqa: E402

warnings.simplefilter("ignore")
kind = sys.argv[1] if len(sys.argv) > 1 else "pv"
size = sys.argv[2] if len(sys.argv) > 2 else "small"
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 7
dev = torch.device("cuda", 0)
if size == "small":
    nx, ny, nt, nbus, x0, y0 = 200, 200, 8760, 100, 0.0, 30.0
elif size == "c5":  # BASELINE configs[4]: Europe-scale 1000 x 800 at 0.05 deg, per-cell outputs
    nx, ny, nt, nbus, x0, y0 = 1000, 800, 240, 100, -12.0, 33.0
elif size in ("odd", "oddpad"):  # nx % 4 != 0: SCALAR lane layout / rows padded to pitch 204 (VEC)
    nx, ny, nt, nbus, x0, y0 = 201, 199, 8760, 100, 0.0, 30.0
else:
    nx, ny, nt, nbus, x0, y0 = 1440, 720, 432, 3000, -180.0, -90.0
nt = int(os.environ.get("ATL_NT", nt))  # e.g. ATL_NT=8760 with size big: the full year (wind / heat / spmm only)
x, y = syn.make_coords(nx, ny, x0, y0, *((0.05, 0.05) if size == "c5" else ()))
tm = syn.make_time(nt + 24 * 170)[24 * 170:] if size == "big" else syn.make_time(nt)
need = None if kind.startswith("pv") else (["temperature"] if kind in ("heat", "spmm") else [])
f = syn.make_pv_fields_device(tm, x, y, dev, seed=7, **({} if need is None else {"names": need})) if need != [] else {}
wf = syn.make_wind_fields_device(nt, ny, nx, dev, seed=7) if kind.startswith("wind") else None
pitch = nx
if size == "oddpad":  # what Cutout.to_device() does
    pitch = nx + (-nx) % 4
    f = {k: torch.nn.functional.pad(v, (0, pitch - nx)).contiguous() for k, v in f.items()}
    if wf is not None:
        wf = {k: torch.nn.functional.pad(v, (0, pitch - nx)).contiguous() for k, v in wf.items()}
plan = engine.get_plan(syn.make_shapes(nx, ny, nbus), ny, nx, pitch=pitch)
coords = dict(time=tm, x=x, y=y, lon=x, lat=y)
out_b = 0.0
if kind in ("pvsum", "pvcube"):  # no-matrix branch (convert.py:200-211): per-cell time sum / cube
    spec = _PvSpec(ab.Dataset(f, coords=coords), ab.get_solarpanelconfig("CSi"), ab.get_orientation("latitude_optimal"))
    fn, bpc = (lambda: spec.cells(timesum=kind == "pvsum")), 20
    out_b = 0.0 if kind == "pvsum" else 4.0
elif kind in ("windsum", "windcube"):
    ws = _WindSpec(ab.Dataset(wf, coords=coords), ab.get_windturbineconfig("Vestas_V112_3MW"))
    fn, bpc = (lambda: ws.cells(timesum=kind == "windsum")), 8
    out_b = 0.0 if kind == "windsum" else 4.0
elif kind == "pv":
    spec = _PvSpec(ab.Dataset(f, coords=coords), ab.get_solarpanelconfig("CSi"), ab.get_orientation("latitude_optimal"))
    fn, bpc = (lambda: spec.op.reduce(plan, spec.fields)), 20
elif kind == "spmm":  # aggregate_matrix on a pre-computed (time, y, x) field (atl_spmm)
    out = torch.zeros((nt, nbus), dtype=torch.float32, device=dev)
    fld = f["temperature"]
    fn, bpc = (lambda: _lib.check(_lib.load().atl_spmm(plan.handle, fld.data_ptr(), nt, out.data_ptr(), engine._stream_ptr()))), 4
elif kind == "wind":
    ws = _WindSpec(ab.Dataset(wf, coords=coords), ab.get_windturbineconfig("Vestas_V112_3MW"))
    fn, bpc = (lambda: ws.op.reduce(plan, ws.wnd, ws.aux)), 8
else:
    hs = _HeatSpec(ab.Dataset({"temperature": f["temperature"]}, coords=coords), 15.0, 1.0, 0.0, 0.0)
    fn, bpc = (lambda: hs.op.reduce(plan, hs.temp, hs.day_start)), 4
for _ in range(3):
    fn()
torch.cuda.synchronize()
ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
for a, b in ev:
    a.record()
    fn()
    b.record()
torch.cuda.synchronize()
ms = float(np.median([a.elapsed_time(b) for a, b in ev]))
cts = float(nx) * ny * nt
# PV: the sun gate loads the inputs of lit (lane, step) pairs only; "GBs" stays the algorithmic
# figure (every cell-step), "GBs_read" counts the input bytes actually requested
lit = 1.0
if kind.startswith("pv"):
    n_lit, n_all = syn.lit_lane_steps(tm, x, y, vec=pitch % 4 == 0)
    lit = n_lit / n_all
print(json.dumps({"kind": kind, "size": size, "tb": os.environ.get("ATL_TB", "auto"), "nt": nt,
                  "lib": os.path.basename(os.environ.get("ATL_LIB_PATH", "")) or "default", "ms": round(ms, 4),
                  "cell_ts_per_s": cts / ms * 1e3, "GBs": round(cts * (bpc + out_b) / ms / 1e6, 1),
                  "frac_of_hbm_peak": round(cts * (bpc + out_b) / ms / 1e6 / hbm_peak()[0], 4),
                  "lit_lane_share": round(lit, 4), "GBs_read": round(cts * (bpc * lit + out_b) / ms / 1e6, 1),
                  "plan": plan.info["slots_per_active_tile"]}))
