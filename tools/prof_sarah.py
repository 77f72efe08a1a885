#!/usr/bin/env python
"""SARAH on the GPU: the gap-fill + hourly-mean kernel, the regrid launch after it, and sarah.get_data
end to end, over Europe at 0.05 deg.

    python tools/prof_sarah.py [--nx 1080 --ny 780 --days 4 --repeat 9] [--out FILE]

Kernel: SIS and SID of --days days of 48 half-hours (nx x ny cells, generated on the GPU with dawn /
dusk NaN runs and 2 % scattered NaNs), one block per day, interpolated and pair-averaged by one
atl_sarah_fill launch; CUDA events, one warm-up, median and min of --repeat.  Bytes: both inputs read
once plus both hourly outputs written once, over the median kernel time, against the H100 SXM's
3.35 TB/s data-sheet HBM3 bandwidth.  Regrid: the same for one RegridOp launch on the hourly SIS onto
the 0.25 deg grid.  get_data: --days synthetic int16 NetCDF-3 day files per variable (the SARAH
layout, scale_factor + _FillValue) written to a temporary directory and read for a 0.25 deg hourly
cutout; host clock around the call, split into file reading (``sarah._cf_field``) and the rest
(GPU work and copies).  Prints one JSON line with the card's name and power limit.
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
from atlite_b200 import gis, sarah  # noqa: E402
from atlite_b200.engine import SarahOp  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def arg(name, default):
    return type(default)(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def timed(fn, repeat):
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


def fields(nt, ny, nx, seed, dev):
    gen = torch.Generator(device=dev).manual_seed(seed)
    v = torch.rand((nt, ny, nx), generator=gen, device=dev) * 900
    t = (torch.arange(nt, device=dev) % 48).view(-1, 1, 1)
    dawn = torch.randint(8, 16, (1, ny, nx), generator=gen, device=dev)
    dusk = torch.randint(32, 42, (1, ny, nx), generator=gen, device=dev)
    gaps = torch.rand((nt, ny, nx), generator=gen, device=dev) < 0.02
    return torch.where((t < dawn) | (t >= dusk) | gaps, torch.full_like(v, float("nan")), v)


def write_day(path, var, day, lon, lat, raw):
    from scipy.io import netcdf_file

    f = netcdf_file(path, "w")
    f.createDimension("time", raw.shape[0])
    f.createDimension("lat", len(lat))
    f.createDimension("lon", len(lon))
    t = f.createVariable("time", "f8", ("time",))
    t[:] = np.arange(raw.shape[0]) * 30.0
    t.units = f"minutes since {day:%Y-%m-%d} 00:00:00"
    for name, c in (("lat", lat), ("lon", lon)):
        f.createVariable(name, "f8", (name,))[:] = c
    v = f.createVariable(var, "i2", ("time", "lat", "lon"))
    v.scale_factor = 0.1
    v._FillValue = np.int16(-999)
    v[:] = raw
    f.close()


def main():
    nx, ny, days, repeat = arg("--nx", 1080), arg("--ny", 780), arg("--days", 4), arg("--repeat", 9)
    out_path = arg("--out", "")
    if not torch.cuda.is_available():
        raise SystemExit("prof_sarah.py needs a CUDA device")
    card = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    dev = torch.device("cuda", 0)
    nt = 48 * days
    sis, sid = fields(nt, ny, nx, 0, dev), fields(nt, ny, nx, 1, dev)
    op = SarahOp(ny, nx, 0)
    starts = list(range(0, nt, 48))
    holder = {}

    def fill():
        holder["out"] = op(sis, sid, starts)

    k_med, k_min = timed(fill, repeat)
    k_bytes = 2 * sis.numel() * 4 + 2 * holder["out"][0].numel() * 4

    lon = np.round(-12.0 + 0.025 + 0.05 * np.arange(nx), 4)
    lat = np.round(33.0 + 0.025 + 0.05 * np.arange(ny), 4)
    dlon = pd.Index(-12.0 + 0.125 + 0.25 * np.arange(nx // 5), name="lon")
    dlat = pd.Index(33.0 + 0.125 + 0.25 * np.arange(ny // 5), name="lat")
    rop = gis.regrid_op(lon, lat, dlon, dlat, gis.RESAMPLING_AVERAGE, 0)
    hsis = holder["out"][0]

    def regrid():
        holder["r"] = rop(hsis)

    r_med, r_min = timed(regrid, repeat)
    r_bytes = hsis.numel() * 4 + holder["r"].numel() * 4
    del sis, sid, holder
    torch.cuda.empty_cache()

    # get_data end to end on files
    rng = np.random.default_rng(0)
    day0 = pd.Timestamp("2013-06-01")
    with tempfile.TemporaryDirectory() as d:
        t0 = time.perf_counter()
        for k in range(days):
            day = day0 + pd.Timedelta(days=k)
            for var in ("SIS", "SID"):
                raw = rng.integers(0, 9000, (48, ny, nx), dtype=np.int16)
                raw[:10] = -999
                raw[40:] = -999
                write_day(os.path.join(d, f"{var}in{day:%Y%m%d}0000.nc"), var, day, lon, lat, raw)
        write_s = time.perf_counter() - t0
        time_ax = pd.date_range(day0, periods=24 * days, freq="h")
        x, y = np.asarray(dlon), np.asarray(dlat)
        cut = ab.Cutout(data=ab.Dataset(coords=dict(time=time_ax, x=x, y=y, lon=x, lat=y)))
        read = [0.0]
        inner = sarah._cf_field

        def counted(*a, **kw):
            t = time.perf_counter()
            r = inner(*a, **kw)
            read[0] += time.perf_counter() - t
            return r

        sarah._cf_field = counted
        sarah.get_data(cut, "influx", None, sarah_dir=d)  # warm-up (tables, modules)
        read[0] = 0.0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ds = sarah.get_data(cut, "influx", None, sarah_dir=d)
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
        sarah._cf_field = inner
        assert ds.raw("influx_direct").shape == (24 * days, len(y), len(x))

    result = {
        "card": card, "power_limit_and_max_sm_clock": power,
        "workload": f"SIS + SID float32 {nx}x{ny}x{nt} (0.05 deg, {days} days, one block per day), interpolate + hourly",
        "kernel_ms_median": round(k_med * 1e3, 3), "kernel_ms_min": round(k_min * 1e3, 3), "repeat": repeat,
        "kernel_bytes_GB": round(k_bytes / 1e9, 3), "kernel_TB_per_s": round(k_bytes / k_med / 1e12, 3),
        "kernel_share_of_3.35_TB_per_s": round(k_bytes / k_med / HBM_BYTES_PER_S, 3),
        "regrid_ms_median": round(r_med * 1e3, 3), "regrid_ms_min": round(r_min * 1e3, 3),
        "regrid_TB_per_s": round(r_bytes / r_med / 1e12, 3),
        "get_data_days": days, "get_data_s": round(total, 3), "get_data_s_per_day": round(total / days, 3),
        "get_data_file_read_s_per_day": round(read[0] / days, 3),
        "get_data_other_s_per_day": round((total - read[0]) / days, 3),
        "fixture_write_s": round(write_s, 2),
    }
    line = json.dumps(result)
    print(line)
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
