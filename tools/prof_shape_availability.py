"""Time ExclusionContainer.compute_shape_availability with dst_transform / dst_crs / dst_shape.

One Europe-sized shape in an EPSG:3035 container at 100 m: an irregular polygon over a --km-wide
square window (default 4200 km: 1.76e9 pixels, more than one band under the default
``_Session.BAND_BYTES``), with a synthetic uint8 land-cover raster (200 m, 10 excluded codes, 300 m
buffer).  The shape goes onto a 0.25 deg EPSG:4326 grid and onto a 1 km EPSG:3035 grid, both
covering the window.  For each it prints the whole call's wall time (best of --repeat, after a
warm-up call), then, from a separate profiled call, the device time of the box pass (k_avail_rect),
the band kernels (k_avail_average), the finalize (k_avail_finalize) and the window's own kernels,
and the window bytes the band kernels read over their time.  For context, the same shape through
Cutout.availabilitymatrix on the 0.25 deg grid (the pixel-centre counts path).  The card's name and
power limit are read in the same run.  JSON on stdout, and in --out when given.

    python tools/prof_shape_availability.py [--km 4200] [--repeat 3] [--out PATH]
"""

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import atlite_b200 as ab  # noqa: E402
from atlite_b200 import availability, gis, proj  # noqa: E402
from atlite_b200 import synthetic as syn  # noqa: E402


def case(km, res=100.0):
    x0, y0 = 2.4e6, 1.2e6
    side = km * 1e3
    rng = np.random.default_rng(0)
    a = np.linspace(0, 2 * np.pi, 4000, endpoint=False)
    r = 0.5 * side * (0.8 + 0.1 * np.sin(7 * a) + 0.05 * np.sin(31 * a) + 0.02 * rng.standard_normal(len(a)))
    r = np.minimum(r, 0.499 * side)
    shape = np.c_[x0 + side / 2 + r * np.cos(a), y0 + side / 2 + r * np.sin(a)]
    lres = 2 * res
    n = int(side / lres) + 2
    patch = 10  # land-cover classes in 2 km patches
    coarse = rng.integers(0, 44, (-(-n // patch), -(-n // patch)), dtype=np.uint8)
    lc = np.empty((n, n), dtype=np.uint8)
    for k in range(0, n, 4000):
        rows = np.arange(k, min(k + 4000, n)) // patch
        lc[k:k + 4000] = np.repeat(coarse[rows], patch, axis=1)[:, :n]
    ex = gis.ExclusionContainer(3035, res=res)
    ex.add_raster(gis.Raster(lc, (lres, 0, x0 - lres, 0, -lres, y0 + side + lres), 3035),
                  codes=[1, 2, 3, 5, 8, 13, 21, 34, 40, 43], buffer=300)
    return ex, shape, (x0, y0, side)


def grids(x0, y0, side):
    t = np.linspace(0, 1, 201)
    bx = np.r_[x0 + side * t, np.full_like(t, x0 + side), x0 + side * t, np.full_like(t, x0)]
    by = np.r_[np.full_like(t, y0), y0 + side * t, np.full_like(t, y0 + side), y0 + side * t]
    lon, lat = proj.transform(bx, by, 3035, 4326)
    lo0, lo1 = np.floor(lon.min() * 4) / 4, np.ceil(lon.max() * 4) / 4
    la0, la1 = np.floor(lat.min() * 4) / 4, np.ceil(lat.max() * 4) / 4
    g4326 = ((0.25, 0.0, lo0, 0.0, -0.25, la1), (int(round((la1 - la0) * 4)), int(round((lo1 - lo0) * 4))), 4326)
    n1 = int(side / 1000.0)
    g3035 = ((1000.0, 0.0, x0, 0.0, -1000.0, y0 + side), (n1, n1), 3035)
    cut = ab.Cutout(data=syn.make_dataset(g4326[1][1], g4326[1][0], 2, x0=lo0 + 0.125, y0=la0 + 0.125, kinds=()))
    return {"EPSG:4326 0.25 deg": g4326, "EPSG:3035 1 km": g3035}, cut


def device_ms(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        t = getattr(ev, "self_device_time_total", None)
        if t is None:
            t = getattr(ev, "self_cuda_time_total", 0)
        if t:
            kern[ev.key[:70]] = round(t / 1e3, 3)
    return dict(sorted(kern.items(), key=lambda kv: -kv[1]))


def best_wall(fn, repeat):
    fn()
    torch.cuda.synchronize()
    walls = []
    for _ in range(repeat):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        walls.append(time.perf_counter() - t0)
    return out, walls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--km", type=float, default=4200)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--out", help="also write the JSON result to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ex, shape, (x0, y0, side) = case(a.km)
    gs, cut = grids(x0, y0, side)
    _, (ny, nx) = gis.padded_transform_and_shape((shape[:, 0].min(), shape[:, 1].min(), shape[:, 0].max(),
                                                  shape[:, 1].max()), 100.0)
    bands = []
    orig = availability._Session.bands

    def counting(self, parts):
        for b in orig(self, parts):
            bands.append(b[2])
            yield b

    availability._Session.bands = counting
    out = dict(gpu=gpu, km=a.km, window=[ny, nx], window_pixels=nx * ny, grids={})
    for name, (t, dshape, dcrs) in gs.items():
        bands.clear()
        call = lambda: ex.compute_shape_availability(shape, t, dcrs, dshape)[0]  # noqa: E731
        v, walls = best_wall(call, a.repeat)
        n_bands = len(bands) // (a.repeat + 1)
        kern = device_ms(call)
        band_ms = sum(ms for k, ms in kern.items() if "k_avail_average" in k)
        out["grids"][name] = dict(
            dst_shape=list(dshape), bands=n_bands, wall_s=[round(w, 3) for w in walls],
            box_pass_ms=sum(ms for k, ms in kern.items() if "k_avail_rect" in k), band_kernels_ms=round(band_ms, 3),
            finalize_ms=sum(ms for k, ms in kern.items() if "k_avail_finalize" in k),
            band_read_GBps=round(nx * ny / (band_ms * 1e-3) / 1e9, 1) if band_ms else None,
            cells_nonzero=int((v > 0).sum()), eligible_share_mean=float(v[v > 0].mean()),
            device_ms_by_kernel=kern)
    Acall = lambda: cut.availabilitymatrix([shape], ex, shapes_crs=3035)  # noqa: E731
    _, walls = best_wall(Acall, a.repeat)
    out["counts_path_0.25deg"] = dict(wall_s=[round(w, 3) for w in walls], device_ms_by_kernel=device_ms(Acall))
    print(json.dumps(out, indent=1))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
