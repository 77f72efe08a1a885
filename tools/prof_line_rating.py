#!/usr/bin/env python
"""Wall time of the public dynamic-line-rating call (Cutout.line_rating) on a Europe-sized year,
split into the stages the call runs, and of the same call on the host-resident copy of the cutout.

    python tools/prof_line_rating.py [--nt 8760] [--repeat 5]
    python tools/prof_line_rating.py --raw [--nt 8760] [--repeat 5]

Workload: a device-resident cutout of 220 x 160 cells at 0.25 degree over --nt hourly steps
(temperature, wnd100m, wnd_azimuth, influx_direct as float32 fields generated on the device, ~4.9 GB
for a year, plus the static height; the solar position is computed in-kernel), and
synthetic.make_line_network(x, y, 2000), about 6000 lines.  The public call is timed with a host
clock (it ends in the device-to-host copy of the result), warm-up first, median of --repeat; the
kernel alone with CUDA events around LineRatingOp.reduce, median of --repeat after a warm-up; the
other stages each on their own with a host clock (ending in a device synchronise), in the order the
call runs them: per-line parameters (azimuths, the parameter table), intersection matrix, the plan
(a cache hit inside the call; its cold build is shown apart), operator set-up (almanac tables,
per-line constants), the result (float64, (line, time), to the host) and the labelled array.  The
host-resident call streams the float32 fields to the device part by part; it is timed once after a
warm-up.
Bytes requested: 16 B per cell-step of every active tile (4 float32 fields, 128 cells per tile,
out-of-grid lanes included), against 3.35 TB/s (H100 SXM data sheet).  Prints one JSON line with
the card's name, power limit and max SM clock.

--raw: the kernel alone on a raw ERA5 cutout of the same grid (t2m, u100, v100, fdir as float32
fields and a static geopotential z; the kernel derives wind speed, wind azimuth and direct influx
and computes the solar position at -30 min), next to the prepared kernel with the position computed
in-kernel and the prepared kernel reading a stored float64 position, which is what era5.prepare
stores.  CUDA events around the reduce, the three variants interleaved, median of --repeat rounds
after a warm-up.  Bytes requested per cell-step: 16 (raw), 16 (prepared, computed position), 32
(prepared, stored float64 position)."""
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import atlite_b200 as ab  # noqa: E402
from atlite_b200 import _lib, convert, engine, era5, gis, synthetic as syn  # noqa: E402
from atlite_b200.labelled import make_dataarray  # noqa: E402


def arg(name, default):
    return int(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def raw_main(nt, repeat, card, power):
    nx, ny = 220, 160
    x, y = syn.make_coords(nx, ny, -10.0, 35.0)
    time_ax = syn.make_time(nt)
    g = torch.Generator(device="cuda").manual_seed(7)
    sh = (nt, ny, nx)
    u = lambda lo, hi, s=sh: torch.rand(s, generator=g, device="cuda") * (hi - lo) + lo  # noqa: E731
    co = dict(time=time_ax, x=x, y=y, lon=x, lat=y)
    raw = {"t2m": u(255.0, 305.0), "u100": u(-15.0, 15.0), "v100": u(-15.0, 15.0), "fdir": u(0.0, 900.0 * 3600.0),
           "z": u(0.0, 2000.0 * 9.80665, (ny, nx))}
    prep = {"temperature": raw["t2m"], "wnd100m": u(0.0, 20.0), "wnd_azimuth": u(0.0, 2 * np.pi),
            "influx_direct": u(0.0, 900.0), "height": u(0.0, 2000.0, (ny, nx))}
    lines = syn.make_line_network(x, y, 2000)
    I = gis.compute_intersectionmatrix(x, y, lines)
    _, _, df = convert._line_parameters(lines, 1e-4, {})
    lp = {k: df[k].to_numpy(np.float64) for k in _lib.LINE_PARAMS}
    plan = engine.get_plan(I, ny, nx, entries=True)
    specs = {"raw_computed_position": convert._LineRatingSpec(ab.Dataset(raw, coords=co), lp),
             "prepared_computed_position": convert._LineRatingSpec(ab.Dataset(prep, coords=co), lp)}
    alt, az = era5.solar_position(time_ax, x, y, "-30min")
    specs["prepared_stored_f64_position"] = convert._LineRatingSpec(
        ab.Dataset(dict(prep, solar_altitude=alt, solar_azimuth=az), coords=co), lp)
    assert specs["raw_computed_position"].raw and not specs["prepared_computed_position"].raw
    for sp_ in specs.values():
        sp_.reduce(plan)
    ks = {k: [] for k in specs}
    for _ in range(repeat):
        for k, sp_ in specs.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            sp_.reduce(plan)
            b.record()
            b.synchronize()
            ks[k].append(a.elapsed_time(b))
    info = plan.info
    per_cell = {"raw_computed_position": 16, "prepared_computed_position": 16, "prepared_stored_f64_position": 32}
    ms = {k: float(np.median(v)) for k, v in ks.items()}
    out = {"card": card, "power_limit_and_max_sm_clock": power, "mode": "raw", "grid": [ny, nx], "nt": nt,
           "lines": len(lines), "nnz": int(I.nnz), "active_tiles": info["n_active_tiles"], "repeat": repeat,
           "kernel_ms_median": {k: round(v, 3) for k, v in ms.items()},
           "kernel_ms_min_max": {k: [round(min(v), 3), round(max(v), 3)] for k, v in ks.items()},
           "raw_over_prepared_computed": round(ms["raw_computed_position"] / ms["prepared_computed_position"], 4),
           "kernel_bytes_requested_GB": {k: round(info["n_active_tiles"] * 128 * b * nt / 1e9, 3)
                                         for k, b in per_cell.items()}}
    print(json.dumps(out))


def main():
    nt, repeat = arg("--nt", 8760), arg("--repeat", 5)
    if not torch.cuda.is_available():
        raise SystemExit("prof_line_rating.py needs a CUDA device")
    warnings.simplefilter("ignore")
    card = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    if "--raw" in sys.argv:
        return raw_main(nt, repeat, card, power)
    nx, ny = 220, 160
    x, y = syn.make_coords(nx, ny, -10.0, 35.0)
    time_ax = syn.make_time(nt)
    g = torch.Generator(device="cuda").manual_seed(7)
    sh = (nt, ny, nx)
    u = lambda lo, hi: torch.rand(sh, generator=g, device="cuda") * (hi - lo) + lo  # noqa: E731
    fields = {"temperature": u(255.0, 305.0), "wnd100m": u(0.0, 20.0), "wnd_azimuth": u(0.0, 2 * np.pi),
              "influx_direct": u(0.0, 900.0), "height": torch.rand((ny, nx), generator=g, device="cuda") * 2000.0}
    ds = ab.Dataset(fields, coords=dict(time=time_ax, x=x, y=y, lon=x, lat=y))
    cut = ab.Cutout(data=ds)
    lines = syn.make_line_network(x, y, 2000)

    def wall(fn):
        fn()
        ts = []
        for _ in range(repeat):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
        return float(np.median(ts))

    t_public = wall(lambda: cut.line_rating(lines, 1e-4))
    t_params = wall(lambda: convert._line_parameters(lines, 1e-4, {}))
    s, dim, df = convert._line_parameters(lines, 1e-4, {})
    lp = {k: df[k].to_numpy(np.float64) for k in _lib.LINE_PARAMS}
    t_inter = wall(lambda: gis.compute_intersectionmatrix(x, y, list(s.values)))
    I = gis.compute_intersectionmatrix(x, y, lines)
    t_plan = wall(lambda: engine.Plan(I, ny, nx, entries=True))
    t_plan_hit = wall(lambda: engine.get_plan(I, ny, nx, entries=True))
    plan = engine.get_plan(I, ny, nx, entries=True)
    t_setup = wall(lambda: convert._LineRatingSpec(ds, lp))
    spec = convert._LineRatingSpec(ds, lp)
    res = spec.reduce(plan)
    t_result = wall(lambda: res.to(torch.float64).T.contiguous().cpu().numpy())
    vals = res.to(torch.float64).T.contiguous().cpu().numpy()
    t_label = wall(lambda: make_dataarray(vals, (dim, "time"), {dim: df.index, "time": spec.time_labels},
                                                      {"units": "A"}))
    torch.cuda.synchronize()
    ks = []
    for _ in range(repeat):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        spec.reduce(plan)
        b.record()
        b.synchronize()
        ks.append(a.elapsed_time(b))
    t_kernel = float(np.median(ks))
    host = ab.Cutout(data=ab.Dataset({k: v.cpu().numpy() for k, v in fields.items()},
                                     coords=dict(time=time_ax, x=x, y=y, lon=x, lat=y)))
    host.line_rating(lines, 1e-4)
    t0 = time.perf_counter()
    host.line_rating(lines, 1e-4)
    t_host = (time.perf_counter() - t0) * 1e3
    parts = {"line_parameters": t_params, "intersection_matrix": t_inter, "plan_cache_hit": t_plan_hit,
             "operator_setup": t_setup, "kernel": t_kernel, "result_to_host_f64": t_result,
             "labelled_array": t_label}
    info = plan.info
    cell_steps = ny * nx * nt
    entry_steps = int(I.nnz) * nt
    bytes_req = info["n_active_tiles"] * 128 * 16 * nt
    out = {"card": card, "power_limit_and_max_sm_clock": power, "grid": [ny, nx], "nt": nt, "lines": len(lines),
           "nnz": int(I.nnz), "active_tiles": info["n_active_tiles"], "slots": info["n_slots"],
           "slots_per_active_tile": round(info["slots_per_active_tile"], 2), "fused_plan": bool(info["fused"]),
           "repeat": repeat,
           "ms": {"public_call": round(t_public, 2), **{k: round(v, 3) for k, v in parts.items()},
                  "unattributed": round(t_public - sum(parts.values()), 2), "plan_build_cold": round(t_plan, 2),
                  "public_call_host_resident": round(t_host, 1)},
           "kernel_cell_steps_per_s": float(f"{cell_steps / (t_kernel * 1e-3):.3e}"),
           "kernel_entry_steps_per_s": float(f"{entry_steps / (t_kernel * 1e-3):.3e}"),
           "kernel_bytes_requested_GB": round(bytes_req / 1e9, 3),
           "kernel_share_of_3.35TBps": round(bytes_req / (t_kernel * 1e-3) / 3.35e12, 3)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
