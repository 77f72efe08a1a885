#!/usr/bin/env python
"""gis.regrid on a SARAH-like case: 0.05 deg irradiance over Europe averaged onto a 0.25 deg cutout.

    python tools/prof_regrid.py [--nx 1400 --ny 900 --nt 2920 --repeat 9] [--host-steps N] [--out FILE]

Workload: a device-resident float32 source of nx x ny x nt at 0.05 deg (1400 x 900 x 2920 = 14.7 GB,
generated on the GPU) resampled with Resampling.average onto the 0.25 deg grid it nests in
(280 x 180).  Kernel: CUDA events around one atl_regrid_f32 launch, one warm-up first, median and
min of --repeat (default 9).  Bytes: the source once plus the destination once, over the median
kernel time, against the H100 SXM's 3.35 TB/s data-sheet HBM3 bandwidth.  Public call: ``ab.regrid``
on the same values held in host memory (the first --host-steps steps, default all that fit in half
the free host memory), host clock around the call, which ends in a device synchronise and the copy
back.  Prints one JSON line with the card's name and power limit, and writes it to --out if given.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import pandas as pd

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import atlite_b200 as ab  # noqa: E402
from atlite_b200 import engine, gis  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def arg(name, default):
    return type(default)(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def main():
    nx, ny, nt, repeat = arg("--nx", 1400), arg("--ny", 900), arg("--nt", 2920), arg("--repeat", 9)
    out_path = arg("--out", "")
    if not torch.cuda.is_available():
        raise SystemExit("prof_regrid.py needs a CUDA device")
    card = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    xs, ys = -12.0 + 0.025 + 0.05 * np.arange(nx), 33.0 + 0.025 + 0.05 * np.arange(ny)
    dimx = pd.Index(-12.0 + 0.125 + 0.25 * np.arange(nx // 5), name="x")
    dimy = pd.Index(33.0 + 0.125 + 0.25 * np.arange(ny // 5), name="y")

    # the tables and plan regrid builds for this grid pair
    t0 = time.perf_counter()
    sx0, sdx = gis.regular_axis(xs, "x")
    sy0, sdy = gis.regular_axis(ys, "y")
    dx0, ddx = gis._transform_axis(dimx, "x")
    dy0, ddy = gis._transform_axis(dimy, "y")
    pad = int(abs(ddx) // min(sdx, sdy) * 1.1)
    op = engine.RegridOp((ny, nx), gis.regrid_axis(sy0, sdy, ny, dy0, ddy, len(dimy), pad),
                         gis.regrid_axis(sx0, sdx, nx, dx0, ddx, len(dimx), pad), device=0)
    plan_ms = (time.perf_counter() - t0) * 1e3

    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(0)
    src = torch.rand((nt, ny, nx), generator=gen, device=dev, dtype=torch.float32)
    out = op(src)  # warm-up
    times = []
    for _ in range(repeat):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = op(src)
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) * 1e-3)
    med = float(np.median(times))
    moved = src.numel() * 4 + out.numel() * 4

    # the public call on host-resident values
    free = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    host_steps = min(nt, arg("--host-steps", max(1, int(free // 2 // (nx * ny * 4 + out[0].numel() * 4)))))
    host = src[:host_steps].cpu().numpy()
    da = ab.DataArray(host, {"time": np.arange(host_steps), "y": ys, "x": xs}, ("time", "y", "x"))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = ab.regrid(da, dimx, dimy, resampling=5)
    torch.cuda.synchronize()
    host_s = time.perf_counter() - t0
    same = bool(np.array_equal(res.values, out[:host_steps].cpu().numpy()))

    result = {
        "card": card, "power_limit_and_max_sm_clock": power,
        "workload": f"float32 {nx}x{ny}x{nt} at 0.05 deg -> {len(dimx)}x{len(dimy)} at 0.25 deg, average",
        "launch": op.info, "plan_build_ms": round(plan_ms, 2),
        "kernel_ms_median": round(med * 1e3, 3), "kernel_ms_min": round(min(times) * 1e3, 3), "repeat": repeat,
        "bytes_moved_GB": round(moved / 1e9, 3), "achieved_TB_per_s": round(moved / med / 1e12, 3),
        "share_of_3.35_TB_per_s": round(moved / med / HBM_BYTES_PER_S, 3),
        "host_call_steps": host_steps, "host_call_s": round(host_s, 3),
        "host_call_GB_per_s": round(host_steps * nx * ny * 4 / host_s / 1e9, 2),
        "host_result_equals_device_result": same,
    }
    line = json.dumps(result)
    print(line)
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
