#!/usr/bin/env python
"""gis.reproject statistics on the GPU: kernel times of each statistic against the average on the
cross-CRS case (a) of tools/prof_reproject.py.

    python tools/prof_reproject_stats.py [--resampling 5,13,8,10,6] [--repeat 7] [--n 40000] [--out FILE]

Case (a): an EPSG:3035 100 m raster of 4000 x 4000 km (n x n = 1.6e9 pixels, 6.4 GB, float32, generated
on the device) onto the 0.25 deg EPSG:4326 Europe grid (228 x 156, south-up like a cutout).  Each
statistic is timed alternately with the average (5) in the same run: CUDA events around one call, one
warm-up first, median and min of --repeat.  Bytes: the source once over the median, against the H100
SXM's 3.35 TB/s data-sheet HBM3 bandwidth.  Prints one JSON line per statistic with the card's name,
power limit, read in the same run, and writes them to --out if given.
"""
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from atlite_b200 import engine  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
EUROPE = (0.25, 0.0, -12.0, 0.0, 0.25, 33.0), (156, 228)  # south-up 0.25 deg grid
NAMES = {5: "average", 6: "mode", 8: "max", 9: "min", 10: "med", 11: "q1", 12: "q3", 13: "sum", 14: "rms"}


def arg(name, default):
    return type(default)(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def timed(fn, repeat):
    times = []
    for _ in range(repeat):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) * 1e-3)
    return times


def main():
    codes = [int(c) for c in arg("--resampling", "5,13,8,10,6").split(",")]
    repeat, n, out_path = arg("--repeat", 7), arg("--n", 40000), arg("--out", "")
    if not torch.cuda.is_available():
        raise SystemExit("prof_reproject_stats.py needs a CUDA device")
    card = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(0)
    st = (100.0, 0.0, 2.5e6, 0.0, -100.0, 5.4e6)
    src = torch.rand((1, n, n), generator=gen, device=dev, dtype=torch.float32)
    ops = {c: engine.ReprojectOp((st, (n, n), 3035), (EUROPE[0], EUROPE[1], 4326), c, device=0) for c in set(codes) | {5}}
    for c in ops:  # warm-up
        ops[c](src)
    torch.cuda.synchronize()
    lines = []
    for c in codes:
        ts, avg = [], []
        for _ in range(max(1, repeat // 2 + 1)):  # alternated with the average
            ts += timed(lambda: ops[c](src), 2)
            avg += timed(lambda: ops[5](src), 2)
        ts, avg = ts[:repeat], avg[:repeat]
        med, amed = float(np.median(ts)), float(np.median(avg))
        moved = src.numel() * src.element_size()
        lines.append(dict(card=card, power_limit_and_max_sm_clock=power, case="a", resampling=NAMES[c],
                          workload=f"float32 3035 100 m {n}x{n} -> 4326 0.25 deg 228x156",
                          kernel_ms_median=round(med * 1e3, 3), kernel_ms_min=round(min(ts) * 1e3, 3),
                          average_ms_median=round(amed * 1e3, 3), ratio_to_average=round(med / amed, 3),
                          repeat=len(ts), source_GB=round(moved / 1e9, 3),
                          source_TB_per_s=round(moved / med / 1e12, 3),
                          share_of_3_35_TB_per_s=round(moved / med / HBM_BYTES_PER_S, 3),
                          tile=[ops[c].desc.tile_y, ops[c].desc.tile_x]))
    with_json = [json.dumps(ln) for ln in lines]
    for ln in with_json:
        print(ln)
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as fh:
            fh.write("\n".join(with_json) + "\n")


if __name__ == "__main__":
    main()
