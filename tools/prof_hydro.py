#!/usr/bin/env python
"""Cutout.hydro on a Europe-sized synthetic case: the shift-and-sum kernel (atl_hydro_shift_sum)
timed with CUDA events, its bytes over that time, and the end-to-end wall time split into the
host steps, the indicator matrix, the runoff reduce and the shift.

    python tools/prof_hydro.py [--repeat N] [--nx 1440 --ny 720 --nt 8760 --basins 10000 --plants 2000]

Workload: a device-resident float32 runoff cutout of nx x ny x nt (generated on the GPU), the
basins of synthetic.make_basins over it (HydroBASINS-like Voronoi basins in one drainage tree) and
plants at the sites of the basins whose upstream sets hold 400-600 basins, dealt round-robin (the
synthetic trees are shallow, so several plants share a basin; the summed upstream sizes are about
500 per plant, 1e6 in all, and the rows that plants share are served from L2).  Kernel: CUDA events around one launch, warm-up
first, median and min of N (default 7).  Bytes: "walked" counts every entry's row segment (what
the kernel reads, from L2 or HBM), "unique" each basin row once plus the output.  Prints one JSON
line with the card's name and power limit."""
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
from atlite_b200 import engine, hydro, synthetic as syn  # noqa: E402


def arg(name, default):
    return type(default)(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def main():
    repeat, nx, ny, nt = arg("--repeat", 7), arg("--nx", 1440), arg("--ny", 720), arg("--nt", 8760)
    n_basins, n_plants = arg("--basins", 10_000), arg("--plants", 2000)
    if not torch.cuda.is_available():
        raise SystemExit("prof_hydro.py needs a CUDA device")
    card = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    x, y = syn.make_coords(nx, ny, -180.0 + 0.125, -90.0 + 0.125)
    t0 = time.perf_counter()
    basins = syn.make_basins(x, y, n_basins, seed=8)
    nd = pd.Index(basins["HYBAS_ID"]).get_indexer(basins["NEXT_DOWN"])
    ptr, up = hydro.upstream_basins(nd, np.arange(len(basins)))
    sizes = np.diff(ptr)
    on = ((basins["site_lon"] < x[-1]) & (basins["site_lat"] < y[-1])).to_numpy()
    cand = np.flatnonzero(on)
    near = cand[np.argsort(np.abs(sizes[cand] - 500), kind="stable")]
    k = max(1, int((np.abs(sizes[near] - 500) <= 100).sum()))
    pick = near[np.arange(n_plants) % k]  # several plants on one river, as on real ones
    plants = basins.iloc[pick][["site_lon", "site_lat"]].set_axis(["lon", "lat"], axis=1)
    plants.index = [f"plant{i}" for i in range(len(plants))]
    setup_s = time.perf_counter() - t0

    dev = torch.device("cuda", 0)
    ro = torch.empty((nt, ny, nx), dtype=torch.float32, device=dev)
    g = torch.Generator(device=dev)
    g.manual_seed(14)
    for lo in range(0, nt, 73):
        hi = min(nt, lo + 73)
        ro[lo:hi] = -torch.log1p(-torch.rand((hi - lo, ny, nx), device=dev, generator=g)) * 2e-4
    nxp = -(-nx // 4) * 4
    if nxp != nx:
        ro = torch.nn.functional.pad(ro, (0, nxp - nx))
    co = dict(time=syn.make_time(nt), x=x, y=y, lon=x, lat=y)
    cut = ab.Cutout(data=ab.Dataset({"runoff": (("time", "y", "x"), ro)}, coords=co))

    def sync_ms(fn):
        torch.cuda.synchronize()
        t = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return r, (time.perf_counter() - t) * 1e3

    # the steps of convert.hydro, one by one
    r, host_route = sync_ms(lambda: hydro.route(plants, basins))
    b = r.basins
    ind, t_ind = sync_ms(lambda: cut.indicatormatrix(b.shapes))
    m, t_norm = sync_ms(lambda: hydro.normalise_rows(ind))
    res, t_runoff = sync_ms(lambda: cut.runoff(matrix=m, index=b.shapes.index, weight_with_height=False,
                                               aggregate_time=None))
    R = np.asarray(res.transpose("hid", "time").values, dtype=np.float64)
    area, t_area = sync_ms(lambda: hydro.basin_areas(b.shapes))
    dist = b.meta["DIST_MAIN"].to_numpy(dtype=np.float64)
    plant_of = np.repeat(np.arange(len(r.ptr) - 1), np.diff(r.ptr))
    shifts, t_shift_host = sync_ms(lambda: hydro.travel_steps(dist[r.rows], dist[r.rows[r.ptr[:-1]]][plant_of], 1))
    out, t_shift = sync_ms(lambda: engine.hydro_shift_sum(R, r.ptr, r.rows, shifts, area[r.rows]).cpu().numpy())

    # the kernel alone, on device-resident inputs
    Rd = torch.from_numpy(R).to(dev)
    ptr_d = torch.from_numpy(r.ptr).to(dev)
    rows_d = torch.from_numpy(r.rows.astype(np.int32)).to(dev)
    sh_d = torch.from_numpy(shifts).to(dev)
    w_d = torch.from_numpy(area[r.rows]).to(dev)
    o = torch.empty((len(plants), nt), dtype=torch.float64, device=dev)
    lib = ab._lib.load()

    def launch():
        ab._lib.check(lib.atl_hydro_shift_sum(0, R.shape[0], nt, engine._dptr(Rd), len(plants), engine._dptr(ptr_d),
                                              engine._dptr(rows_d), engine._dptr(sh_d), engine._dptr(w_d),
                                              engine._dptr(o), engine._stream_ptr()))

    launch()
    ts = []
    for _ in range(repeat):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        launch()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    assert np.array_equal(o.cpu().numpy(), out)
    k_med, k_min = float(np.median(ts)), float(min(ts))
    n_ent = int(r.ptr[-1])
    walked = n_ent * nt * 8 + len(plants) * nt * 8
    unique = R.shape[0] * nt * 8 + len(plants) * nt * 8

    _, e2e = sync_ms(lambda: cut.hydro(plants, basins, aggregate_time=None))
    _, e2e2 = sync_ms(lambda: cut.hydro(plants, basins, aggregate_time=None))
    ms = lambda v: round(v, 2)  # noqa: E731
    print(json.dumps({
        "card": card, "power_limit_and_max_sm_clock": power, "grid": [ny, nx], "nt": nt,
        "basins": len(basins), "plants": len(plants), "unique_basins": int(R.shape[0]), "entries": n_ent,
        "setup_s": round(setup_s, 1),
        "kernel_ms_median_min": [ms(k_med), ms(k_min)], "repeat": repeat,
        "kernel_bytes_walked_GB": round(walked / 1e9, 2), "kernel_bytes_unique_GB": round(unique / 1e9, 3),
        "walked_TBps": round(walked / (k_med * 1e-3) / 1e12, 2),
        "unique_TBps_of_3.35": round(unique / (k_med * 1e-3) / 1e12, 3),
        "steps_ms": {"host_route": ms(host_route), "indicator": ms(t_ind), "normalise": ms(t_norm),
                     "runoff": ms(t_runoff), "area": ms(t_area), "travel_steps": ms(t_shift_host),
                     "shift_with_copies": ms(t_shift)},
        "end_to_end_ms": [ms(e2e), ms(e2e2)],
    }))


if __name__ == "__main__":
    main()
