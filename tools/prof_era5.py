#!/usr/bin/env python
"""Streaming rate of the ERA5 derivation kernels (csrc/era5.cu) on device-resident raw fields."""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import atlite_b200 as ab  # noqa: E402
from bench import hbm_peak  # noqa: E402
from atlite_b200 import era5, synthetic as syn  # noqa: E402

nx, ny, nt = 1440, 720, 96
dev = torch.device("cuda", 0)
x, y = syn.make_coords(nx, ny, -180.0, -90.0)
t = syn.make_time(nt)
g = torch.Generator(device=dev).manual_seed(1)
f = {k: torch.rand((nt, ny, nx), device=dev, generator=g) * 10 + 0.1 for k in ("u100", "v100", "u10", "v10", "fsr", "ssrd", "ssr", "tisr", "fdir")}
ds = ab.Dataset({k: (("time", "y", "x"), v) for k, v in f.items()}, coords=dict(time=t, x=x, y=y, lon=x, lat=y))


def timeit(fn, n=5):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
    for a, b in ev:
        a.record(); fn(); b.record()
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


cells = float(nx) * ny * nt
out = {}
for name, fn, bpc in (("wind", lambda: era5.get_data_wind(ds), 36), ("influx", lambda: era5.get_data_influx(ds, solar_position_vars=False), 32),
                      ("solar_position", lambda: era5.solar_position(t, x, y), 16)):
    ms = timeit(fn)
    out[name] = {"ms": round(ms, 3), "GBs": round(cells * bpc / ms / 1e6, 1), "frac_of_hbm_peak": round(cells * bpc / ms / 1e6 / hbm_peak()[0], 3)}
print(json.dumps(out))
