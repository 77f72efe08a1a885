#!/usr/bin/env python
"""gis.reproject on the GPU: kernel times of the cross-CRS warp and of the same-CRS path.

    python tools/prof_reproject.py [--cases abc] [--repeat 7] [--nt 744] [--out FILE]

Cases (every source generated on the device from a seed, float32):
  (a) an EPSG:3035 100 m raster of 4000 x 4000 km (40000 x 40000 = 1.6e9 pixels, 6.4 GB) averaged onto
      the 0.25 deg EPSG:4326 Europe grid (-12..45 E, 33..72 N, 228 x 156, south-up like a cutout);
  (b) a 0.25 deg EPSG:4326 (nt, 156, 228) field onto a 5 km EPSG:3035 grid (800 x 800), nearest and
      average;
  (c) the SARAH-like case of tools/prof_regrid.py (0.05 deg (nt, 900, 1400) onto 0.25 deg), within
      EPSG:4326: through k_regrid on regrid_axis(pad=0) tables (what gis.reproject runs) and through
      the cross-CRS kernel forced onto the identity pair, alternated, with the largest difference.
Kernel time: CUDA events around one launch, one warm-up first, median and min of --repeat.  Bytes:
the source once plus the destination once, over the median, against the H100 SXM's 3.35 TB/s
data-sheet HBM3 bandwidth.  Prints one JSON line per case with the card's name and power limit,
read in the same run, and writes them to --out if given.
"""
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from atlite_b200 import engine, gis  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
EUROPE = (0.25, 0.0, -12.0, 0.0, 0.25, 33.0), (156, 228)  # south-up 0.25 deg grid


def arg(name, default):
    return type(default)(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def timed(fn, repeat):
    out = fn()  # warm-up
    times = []
    for _ in range(repeat):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) * 1e-3)
    return out, times


def report(name, workload, times, src, out, **extra):
    med = float(np.median(times))
    moved = src.numel() * src.element_size() + out.numel() * out.element_size()
    return dict(case=name, workload=workload, kernel_ms_median=round(med * 1e3, 3),
                kernel_ms_min=round(min(times) * 1e3, 3), repeat=len(times), bytes_moved_GB=round(moved / 1e9, 3),
                achieved_TB_per_s=round(moved / med / 1e12, 3),
                share_of_3_35_TB_per_s=round(moved / med / HBM_BYTES_PER_S, 3), **extra)


def main():
    cases, repeat, nt = arg("--cases", "abc"), arg("--repeat", 7), arg("--nt", 744)
    out_path = arg("--out", "")
    if not torch.cuda.is_available():
        raise SystemExit("prof_reproject.py needs a CUDA device")
    card = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(0)
    lines = []

    if "a" in cases:
        n = 40000
        st = (100.0, 0.0, 2.5e6, 0.0, -100.0, 5.4e6)
        src = torch.rand((1, n, n), generator=gen, device=dev, dtype=torch.float32)
        op = engine.ReprojectOp((st, (n, n), 3035), (EUROPE[0], EUROPE[1], 4326), 5, device=0)
        out, times = timed(lambda: op(src), repeat)
        lines.append(report("a", f"float32 3035 100 m {n}x{n} -> 4326 0.25 deg 228x156, average", times, src, out,
                            tile=[op.desc.tile_y, op.desc.tile_x],
                            valid_cells=int((~torch.isnan(out)).sum())))
        del src, out

    if "b" in cases:
        (ny, nx) = EUROPE[1]
        src = torch.rand((nt, ny, nx), generator=gen, device=dev, dtype=torch.float32)
        dt = (5000.0, 0.0, 2.5e6, 0.0, -5000.0, 5.4e6)
        for resampling, what in ((0, "nearest"), (5, "average")):
            op = engine.ReprojectOp((EUROPE[0], (ny, nx), 4326), (dt, (800, 800), 3035), resampling, device=0)
            out, times = timed(lambda: op(src), repeat)
            lines.append(report(f"b-{what}", f"float32 4326 0.25 deg ({nt}, {ny}, {nx}) -> 3035 5 km 800x800, {what}",
                                times, src, out, tile=[op.desc.tile_y, op.desc.tile_x]))
            del out

        del src

    if "c" in cases:
        ny, nx = 900, 1400
        st = (0.05, 0.0, -12.0, 0.0, 0.05, 33.0)
        dt, dshape = (0.25, 0.0, -12.0, 0.0, 0.25, 33.0), (ny // 5, nx // 5)
        src = torch.rand((nt, ny, nx), generator=gen, device=dev, dtype=torch.float32)
        ytab, xtab = gis._same_crs_tables(st, (ny, nx), dt, dshape, False)
        rop = engine.RegridOp((ny, nx), ytab, xtab, device=0)
        iop = engine.ReprojectOp((st, (ny, nx), 4326), (dt, dshape, 4326), 5, device=0)
        rt, it = [], []
        for _ in range(2):  # alternated
            a, t = timed(lambda: rop(src, nodata=None, empty=np.nan), repeat)
            rt += t
            b, t = timed(lambda: iop(src), repeat)
            it += t
        diff = float(((a.double() - b.double()).abs() / b.double().abs()).max())
        wl = f"float32 4326 0.05 deg ({nt}, {ny}, {nx}) -> 0.25 deg {dshape[1]}x{dshape[0]}, average"
        lines.append(report("c-k_regrid", wl, rt, src, a, launch=rop.info))
        lines.append(report("c-identity", wl, it, src, b, tile=[iop.desc.tile_y, iop.desc.tile_x],
                            max_rel_diff_to_k_regrid=diff))
        del src, a, b

    with_card = [json.dumps(dict(card=card, power_limit_and_max_sm_clock=power, **ln)) for ln in lines]
    for ln in with_card:
        print(ln)
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as fh:
            fh.write("\n".join(with_card) + "\n")


if __name__ == "__main__":
    main()
