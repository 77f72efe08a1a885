#!/usr/bin/env python
"""Separate conversion calls against one Cutout.convert_many, on a Europe-sized raw ERA5 cutout.

    python tools/prof_convert_many.py [--days 365 --lazy-days 30 --repeat 3] [--out FILE]

Cutout: 281 x 201 cells at 0.25 deg, --days of hourly raw ERA5 variables (tisr, fdir, ssrd, ssr, t2m,
u100, v100, fsr, u10, v10; float32), one seeded week of values tiled over the period, as a pageable
NumPy cutout, as its pin_host() copy, and (--lazy-days, to keep the file small) as an uncompressed
chunk-container cutout (ingest.write_chunked, 100-step chunks) in a temporary directory.  Requests:
PV, dual-tracking PV, wind by the log law and by the power law, heat demand and temperature, each
reduced to 300 regions with aggregate_time=None.

For each cutout: one warm-up of both, then --repeat rounds that time the six separate calls and one
convert_many in turn (host clock; every call returns host arrays, so it has synchronised).  Reports
the median wall times, the host -> device bytes (convert_many's from the stats of its shared passes;
the separate calls' as the sum of each request's own pass), the loader calls of the lazy cutout, and
the largest relative difference between the two results.  Prints one JSON line with the card's name
and power limit.
"""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import atlite_b200 as ab  # noqa: E402
from atlite_b200 import engine, ingest, synthetic as syn  # noqa: E402

NX, NY = 281, 201
RAW = ("tisr", "fdir", "ssrd", "ssr", "t2m", "u100", "v100", "fsr", "u10", "v10")


def arg(name, default):
    return type(default)(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def raw_fields(nt, seed=11):
    """(nt, NY, NX) float32 raw ERA5 variables: a seeded week, tiled."""
    rng = np.random.default_rng(seed)
    week = min(nt, 168)
    lo_hi = dict(tisr=(0, 4.5e6), ssrd=(0, 3.0e6), t2m=(250, 305), u100=(-15, 15), v100=(-15, 15),
                 fsr=(1e-4, 1.5), u10=(-8, 8), v10=(-8, 8))
    base = {k: rng.uniform(lo, hi, (week, NY, NX)).astype(np.float32) for k, (lo, hi) in lo_hi.items()}
    base["ssr"] = (base["ssrd"] * np.float32(0.8)).astype(np.float32)
    base["fdir"] = (base["ssrd"] * np.float32(0.6)).astype(np.float32)
    out = {}
    for k in RAW:
        a = np.empty((nt, NY, NX), dtype=np.float32)
        for t in range(0, nt, week):
            a[t:t + week] = base[k][:min(week, nt - t)]
        out[k] = a
    return out


def dataset(fields, time, x, y):
    return ab.Dataset({k: (("time", "y", "x"), v) for k, v in fields.items()},
                      coords=dict(time=time, x=x, y=y, lon=x, lat=y), attrs={"module": "era5"})


def requests(m):
    base = dict(matrix=m, aggregate_time=None)
    return {
        "pv": dict(method="pv", panel="CSi", orientation="latitude_optimal", **base),
        "pv_dual": dict(method="pv", panel="CSi", orientation="latitude_optimal", tracking="dual", **base),
        "wind_log": dict(method="wind", turbine="Vestas_V112_3MW", **base),
        "wind_power": dict(method="wind", turbine="Vestas_V112_3MW", interpolation_method="power", **base),
        "heat": dict(method="heat_demand", **base),
        "temperature": dict(method="temperature", **base),
    }


class Counted:
    """engine.reduce_host_many with its pass statistics summed."""

    def __init__(self):
        self.fn, self.bytes, self.slabs = engine.reduce_host_many, 0, 0

    def __call__(self, jobs, chunk_units=0):
        outs, st = self.fn(jobs, chunk_units)
        self.bytes += st["h2d_bytes"]
        self.slabs += st["n_slabs"]
        return outs, st


def separate(c, req):
    return {n: getattr(c, r["method"])(**{k: v for k, v in r.items() if k != "method"}) for n, r in req.items()}


def measure(c, req, repeat, loads=None):
    counted = Counted()
    engine.reduce_host_many = counted
    try:
        for r in req:  # each request's own pass: the bytes its separate call copies
            c.convert_many({r: req[r]})
        sep_bytes, counted.bytes = counted.bytes, 0
        a = separate(c, req)  # warm-up
        b = c.convert_many(req)
        many_bytes = counted.bytes
        rel = max(float(np.nanmax(np.abs(np.asarray(a[n].values) - np.asarray(b[n].values)) /
                                  np.maximum(np.abs(np.asarray(a[n].values)), 1e-6))) for n in req)
        t_sep, t_many, n_sep, n_many = [], [], [], []
        for _ in range(repeat):
            n0 = sum(loads.values()) if loads is not None else 0
            t = time.perf_counter()
            separate(c, req)
            t_sep.append(time.perf_counter() - t)
            n1 = sum(loads.values()) if loads is not None else 0
            t = time.perf_counter()
            c.convert_many(req)
            t_many.append(time.perf_counter() - t)
            n2 = sum(loads.values()) if loads is not None else 0
            n_sep.append(n1 - n0)
            n_many.append(n2 - n1)
    finally:
        engine.reduce_host_many = counted.fn
    out = dict(separate_s=float(np.median(t_sep)), convert_many_s=float(np.median(t_many)),
               speedup=float(np.median(t_sep) / np.median(t_many)),
               separate_h2d_gb=sep_bytes / 1e9, convert_many_h2d_gb=many_bytes / 1e9, max_rel_diff=rel)
    if loads is not None:
        out.update(separate_loader_calls=n_sep[0], convert_many_loader_calls=n_many[0])
    return out


def main():
    days, lazy_days, repeat = arg("--days", 365), arg("--lazy-days", 30), arg("--repeat", 3)
    x, y = syn.make_coords(NX, NY, -12.0, 33.0, 0.25, 0.25)
    m = syn.make_shapes(NX, NY, 300)
    req = requests(m)
    res = dict(card=card(), grid=[NY, NX], requests=list(req))
    nt = 24 * days
    host = ab.Cutout(data=dataset(raw_fields(nt), syn.make_time(nt), x, y))
    res["days"] = days
    res["host"] = measure(host, req, repeat)
    print(json.dumps(dict(partial="host", **res["host"])), flush=True)
    pinned = host.pin_host()
    res["pinned"] = measure(pinned, req, repeat)
    print(json.dumps(dict(partial="pinned", **res["pinned"])), flush=True)
    del pinned, host
    nl = 24 * lazy_days
    with tempfile.TemporaryDirectory() as tmp:
        coords = dict(time=syn.make_time(nl), x=x, y=y, lon=x, lat=y)
        p = ingest.write_chunked(os.path.join(tmp, "cut.bin"), raw_fields(nl), coords, chunk=(100, None, None),
                                 complevel=0, shuffle=False, attrs={"module": "era5"})
        lazy = ab.Cutout(data=ingest.open_cutout(p))
        loads = {}
        for name, load in list(lazy.data._loaders.items()):
            def counted(lo, hi, load=load, name=name):
                loads[name] = loads.get(name, 0) + 1
                return load(lo, hi)
            lazy.data._loaders[name] = counted
        res["lazy_days"] = lazy_days
        res["lazy"] = measure(lazy, req, repeat, loads)
    line = json.dumps(res)
    print(line)
    out = arg("--out", "")
    if out:
        with open(out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
