#!/usr/bin/env python
"""GEBCO on the GPU: the int16 window average (atl_regrid_window) and gebco.get_data end to end, for a
Europe-sized window at 15 arc-seconds.

    python tools/prof_gebco.py [--repeat 20] [--out FILE]

Fixture: a GEBCO-like NetCDF-3 file (int16 ``elevation``, ascending lat / lon centres at 15'') over
lon -12.5..42.5, lat 32.5..72.5, written to a temporary directory and read once, so it sits in the
page cache.  The cutouts span x -12..42, y 33..72 at 0.25 and 0.05 deg: their window is about 1.2e8
int16 pixels.  For each cutout:

* kernel: the window uploaded to the device once, then one atl_regrid_window launch over all bands,
  timed with CUDA events (one warm-up, median and min of --repeat); bytes = window read once plus the
  int16 output, against the H100 SXM's 3.35 TB/s data-sheet HBM3 bandwidth;
* H2D: one copy of the whole window from pinned memory, CUDA events;
* file read: copying the window out of the memory-mapped file into native int16 (host clock);
* get_data: host clock around ``gebco.get_data`` (after a warm-up call), which reads, streams in
  bands (``RegridOp.WINDOW_SLAB_BYTES``) and averages.

Prints one JSON line with the card's name and power limit, read in the same run.
"""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import pandas as pd

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import atlite_b200 as ab  # noqa: E402
from atlite_b200 import gebco, ingest  # noqa: E402
from atlite_b200.engine import RegridOp  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
RES = 1 / 240


def arg(name, default):
    return type(default)(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def events(fn, repeat):
    fn()  # warm-up
    times = []
    for _ in range(repeat):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) * 1e-3)
    return float(np.median(times)), float(min(times))


def write_grid(path):
    from scipy.io import netcdf_file

    lon = -12.5 + (np.arange(round(55 / RES)) + 0.5) * RES
    lat = 32.5 + (np.arange(round(40 / RES)) + 0.5) * RES
    f = netcdf_file(path, "w")
    f.createDimension("lat", len(lat))
    f.createDimension("lon", len(lon))
    for n, c in (("lat", lat), ("lon", lon)):
        f.createVariable(n, "f8", (n,))[:] = c
    v = f.createVariable("elevation", "i2", ("lat", "lon"))
    rng = np.random.default_rng(0)
    wave = np.cos(np.radians(lon * 20))[None, :]
    for r in range(0, len(lat), 960):  # row blocks: the fixture is never held whole as int64 noise
        rows = slice(r, min(len(lat), r + 960))
        g = 3000 * np.sin(np.radians(lat[rows] * 30))[:, None] * wave
        v[rows] = (g + rng.integers(-300, 300, g.shape)).astype(np.int16)
    f.close()
    return lon, lat


def main():
    repeat, out_path = arg("--repeat", 20), arg("--out", "")
    if not torch.cuda.is_available():
        raise SystemExit("prof_gebco.py needs a CUDA device")
    card = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    result = {"card": card, "power_limit_and_max_sm_clock": power, "repeat": repeat,
              "window_slab_MiB": RegridOp.WINDOW_SLAB_BYTES >> 20}
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "gebco.nc")
        t0 = time.perf_counter()
        write_grid(path)
        result["fixture_write_s"] = round(time.perf_counter() - t0, 2)
        result["file_GB"] = round(os.path.getsize(path) / 1e9, 3)
        for res in (0.25, 0.05):
            x = np.round(-12.0 + res * np.arange(round(54 / res) + 1), 6)
            y = np.round(33.0 + res * np.arange(round(39 / res) + 1), 6)
            lon, lat, var = ingest.open_grid(path)
            win = gebco._cutout_window(x, y, gebco.grid_transform(lon, lat), var.shape)
            (r0, r1), (c0, c1), ytab, xtab = gebco._tables(win, len(x), len(y), var.shape, True)
            window = var.window(r0, r1, c0, c1)
            t0 = time.perf_counter()
            host = np.asarray(window)  # page cache -> native int16
            read_s = time.perf_counter() - t0
            pinned = torch.empty(host.shape, dtype=torch.int16, pin_memory=True)
            pinned.numpy()[...] = host
            dev = torch.empty(host.shape, dtype=torch.int16, device="cuda:0")
            h2d = events(lambda: dev.copy_(pinned, non_blocking=True), repeat)
            op = RegridOp((r1 - r0, c1 - c0), ytab, xtab, device=0)
            holder = {}
            k_med, k_min = events(lambda: holder.__setitem__("o", op.window(dev)), repeat)
            assert np.array_equal(holder["o"].cpu().numpy(), op.window(host))
            k_bytes = host.nbytes + holder["o"].numel() * 2
            time_ax = pd.date_range("2013-01-01", periods=1, freq="h")
            cut = ab.Cutout(data=ab.Dataset(coords=dict(time=time_ax, x=x, y=y, lon=x, lat=y)))
            gebco.get_data(cut, "height", None, gebco_path=path)  # warm-up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ds = gebco.get_data(cut, "height", None, gebco_path=path)
            torch.cuda.synchronize()
            total = time.perf_counter() - t0
            assert np.array_equal(ds.raw("height"), holder["o"].cpu().numpy())
            key = f"{res}deg"
            result[key] = {
                "cutout": f"{len(x)}x{len(y)}", "window_px": f"{c1 - c0}x{r1 - r0}",
                "window_MB": round(host.nbytes / 1e6, 1), "kernel_info": op.info,
                "kernel_ms_median": round(k_med * 1e3, 3), "kernel_ms_min": round(k_min * 1e3, 3),
                "kernel_TB_per_s": round(k_bytes / k_med / 1e12, 3),
                "kernel_share_of_3.35_TB_per_s": round(k_bytes / k_med / HBM_BYTES_PER_S, 3),
                "h2d_pinned_ms_median": round(h2d[0] * 1e3, 3),
                "h2d_GB_per_s": round(host.nbytes / h2d[0] / 1e9, 2),
                "file_read_ms": round(read_s * 1e3, 1),
                "get_data_ms": round(total * 1e3, 1),
            }
            del dev, pinned, host, holder
            torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
