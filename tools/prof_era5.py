#!/usr/bin/env python
"""Streaming rate of the ERA5 derivation kernels (csrc/era5.cu) on device-resident raw fields.

    python tools/prof_era5.py           the derivation kernels (96 steps)
    python tools/prof_era5.py --fused   raw ERA5 fields converted directly by the fused PV and wind
                                        kernels, against the prepared routes (1460 steps -> 3000 shapes)"""
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
FUSED = "--fused" in sys.argv
x, y = syn.make_coords(nx, ny, -180.0, -90.0)
t = syn.make_time(nt)


def timeit(fn, n=5):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
    for a, b in ev:
        a.record(); fn(); b.record()
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def derivations():
    g = torch.Generator(device=dev).manual_seed(1)
    f = {k: torch.rand((nt, ny, nx), device=dev, generator=g) * 10 + 0.1 for k in ("u100", "v100", "u10", "v10", "fsr", "ssrd", "ssr", "tisr", "fdir")}
    ds = ab.Dataset({k: (("time", "y", "x"), v) for k, v in f.items()}, coords=dict(time=t, x=x, y=y, lon=x, lat=y))
    cells = float(nx) * ny * nt
    out = {}
    for name, fn, bpc in (("wind", lambda: era5.get_data_wind(ds), 36), ("influx", lambda: era5.get_data_influx(ds, solar_position_vars=False), 32),
                          ("solar_position", lambda: era5.solar_position(t, x, y), 16)):
        ms = timeit(fn)
        out[name] = {"ms": round(ms, 3), "GBs": round(cells * bpc / ms / 1e6, 1), "frac_of_hbm_peak": round(cells * bpc / ms / 1e6 / hbm_peak()[0], 3)}
    return out


def fused(steps=1460, nbus=3000):
    """cell-ts/s and requested bytes of each route from ERA5 data to PV / wind time series.  The
    PV inputs a lane requests are the lit share of its steps (the sun gate) times 20 B per
    cell-step; the stored-solar route is not gated (36 B)."""
    import subprocess
    import warnings

    from atlite_b200 import convert, engine

    warnings.simplefilter("ignore")
    card = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    tt = syn.make_time(steps)
    co = dict(time=tt, x=x, y=y, lon=x, lat=y)
    plan = engine.get_plan(syn.make_shapes(nx, ny, nbus), ny, nx)
    cells = float(nx) * ny * steps
    g = torch.Generator(device=dev).manual_seed(2)

    def rnd(lo, hi, n=steps):
        return torch.empty((n, ny, nx), device=dev).uniform_(lo, hi, generator=g)

    lit, total = syn.lit_lane_steps(tt[::4], x, y, time_shift="-30min")  # every 4th step: the lit share
    share = lit / total
    pv = dict(panel=ab.get_solarpanelconfig("CSi"), orientation=ab.get_orientation("latitude_optimal"))
    turb = ab.get_windturbineconfig("Vestas_V112_3MW")  # hub 80 m: log law from 100 m
    out = {"card": card, "power_limit_and_max_sm_clock": power, "grid": [steps, ny, nx], "shapes": nbus,
           "lit_share_of_lane_steps": round(share, 4)}

    def row(name, ms, bpc):
        out[name] = {"ms": round(ms, 2), "cell_ts_per_s": f"{cells / ms * 1e3:.3e}",
                     "requested_GB": round(cells * bpc / 1e9, 2), "GBs": round(cells * bpc / ms / 1e6, 1)}

    # raw fields: PV (ssrd, ssr, tisr, fdir, t2m) and wind (u100, v100, fsr)
    raw = dict(ssrd=rnd(0, 3e6), tisr=rnd(0, 4.5e6), t2m=rnd(250, 305))
    raw["ssr"] = raw["ssrd"] * 0.8
    raw["fdir"] = raw["ssrd"] * 0.6
    raw.update(u100=rnd(-15, 15), v100=rnd(-15, 15), fsr=rnd(-0.05, 2.0))
    ds = ab.Dataset({k: (("time", "y", "x"), v) for k, v in raw.items()}, coords=dict(co))
    spec = convert._PvSpec(ds, **pv)
    row("pv_raw_fused", timeit(lambda: spec.reduce(plan)), 20 * share)
    spec = convert._WindSpec(ds, turb)
    row("wind_raw_fused_log", timeit(lambda: spec.reduce(plan)), 12)
    wp = ab.Dataset({"wnd100m": (("time", "y", "x"), torch.sqrt(raw["u100"] ** 2 + raw["v100"] ** 2)),
                     "roughness": (("time", "y", "x"), raw["fsr"].clamp(min=2e-4))}, coords=dict(co))
    spec = convert._WindSpec(wp, turb)
    row("wind_prepared_log", timeit(lambda: spec.reduce(plan)), 8)
    del raw, ds, wp, spec
    torch.cuda.empty_cache()

    # prepared PV with the solar position stored as float64 (what era5.prepare writes): MODE 2
    alt, az = era5.solar_position(tt, x, y, "-30min")
    prep = {k: rnd(0, 800) for k in ("influx_toa", "influx_direct", "influx_diffuse")}
    prep.update(albedo=rnd(0, 0.5), temperature=rnd(250, 305), solar_altitude=alt, solar_azimuth=az)
    ds = ab.Dataset({k: (("time", "y", "x"), v) for k, v in prep.items()}, coords=dict(co))
    spec = convert._PvSpec(ds, **pv)
    row("pv_prepared_stored_solar_f64", timeit(lambda: spec.reduce(plan)), 36)
    del prep, alt, az, ds, spec
    torch.cuda.empty_cache()

    # era5.prepare (influx + solar position) followed by PV: half the steps fit next to the raw fields
    half = steps // 2
    tt2 = tt[:half]
    raw = dict(ssrd=rnd(0, 3e6, half), tisr=rnd(0, 4.5e6, half), t2m=rnd(250, 305, half))
    raw["ssr"] = raw["ssrd"] * 0.8
    raw["fdir"] = raw["ssrd"] * 0.6
    ds = ab.Dataset({k: (("time", "y", "x"), v) for k, v in raw.items()}, coords=dict(co, time=tt2))

    def prepare_and_pv():
        p = era5.get_data_influx(ds)
        p["temperature"] = (("time", "y", "x"), raw["t2m"])
        return convert._PvSpec(p, **pv).reduce(plan)

    ms = timeit(prepare_and_pv, n=3)
    out["era5_prepare_then_pv"] = {"steps": half, "ms": round(ms, 2), "cell_ts_per_s": f"{float(nx) * ny * half / ms * 1e3:.3e}"}
    return out



print(json.dumps(fused() if FUSED else derivations()))
