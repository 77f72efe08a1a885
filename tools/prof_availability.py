"""Time Cutout.availabilitymatrix on a Europe-sized synthetic case.

EPSG:3035 container at 100 m over a 4000 x 4000 km box, ``--regions`` Voronoi regions
(synthetic.make_voronoi_shapes), a uint8 land-cover raster (3035, 100 m) with a 10-code list and an
800 m buffer, a float depth-like raster (4326, 0.01 deg) with a callable, and one buffered coastline
polyline; cutout on the 0.25 deg EPSG:4326 grid around the box.  Prints the end-to-end wall time
(best of --repeat, after a warm-up call), then, in a separate profiled call, the device time per
kernel; with --oracle, the NumPy oracle's time for one region (only as a scale).  The JSON result
is printed, and written to --out when given.

--crs ESRI:54009 or EPSG:3857 runs the same case in that container CRS: the regions and the
coastline projected into it, the 3035 land cover and the 4326 depth then both sampled across CRSs.
--band-mb lowers the per-band device memory budget (``_Session.BAND_BYTES``), so that windows run
in row bands; --dump writes the (region, y, x) matrix as a .npy file.

    python tools/prof_availability.py [--regions 300] [--km 4000] [--repeat 2] [--oracle] [--out PATH]
                                      [--crs {3035,ESRI:54009,EPSG:3857}] [--band-mb MB] [--dump PATH]
"""

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import atlite_b200 as ab  # noqa: E402
from atlite_b200 import gis, proj  # noqa: E402
from atlite_b200 import synthetic as syn  # noqa: E402


def case(n_regions, km, res=100.0, crs=3035):
    x0, y0 = 2.0e6, 1.0e6
    side = km * 1e3
    gx = np.linspace(x0 + 5e3, x0 + side - 5e3, 400)
    gy = np.linspace(y0 + 5e3, y0 + side - 5e3, 400)
    regions = syn.make_voronoi_shapes(gx, gy, n_regions, seed=11)
    rng = np.random.default_rng(0)
    n = int(side / res)
    patch = 20  # land-cover classes in 2 km patches, so that buffers widen their borders
    coarse = rng.integers(0, 44, (-(-n // patch), -(-n // patch)), dtype=np.uint8)
    lc = np.empty((n, n), dtype=np.uint8)
    for k in range(0, n, 4000):  # in row blocks: bounded temporaries
        rows = np.arange(k, min(k + 4000, n)) // patch
        lc[k:k + 4000] = np.repeat(coarse[rows], patch, axis=1)[:, :n]
    land = gis.Raster(lc, (res, 0, x0, 0, -res, y0 + side), 3035)
    corners = np.array([[x0, y0], [x0 + side, y0], [x0, y0 + side], [x0 + side, y0 + side],
                        [x0 + side / 2, y0], [x0 + side / 2, y0 + side]])
    lon, lat = proj.laea_inverse(corners[:, 0], corners[:, 1])
    lo0, lo1, la0, la1 = np.floor(lon.min()) - 1, np.ceil(lon.max()) + 1, np.floor(lat.min()) - 1, np.ceil(lat.max()) + 1
    dres = 0.01
    dny, dnx = int((la1 - la0) / dres), int((lo1 - lo0) / dres)
    depth = np.repeat(np.repeat(rng.normal(40.0, 60.0, (-(-dny // 10), -(-dnx // 10))), 10, 0), 10, 1)
    depth = np.ascontiguousarray(depth[:dny, :dnx] + rng.normal(0, 5.0, (dny, dnx)), dtype=np.float32)
    sea = gis.Raster(depth, (dres, 0, lo0, 0, -dres, la1), 4326)
    t = np.linspace(0, 1, 20000)
    coast = np.c_[x0 + side * t, y0 + side * (0.5 + 0.3 * np.sin(9 * t) + 0.01 * np.cumsum(rng.normal(0, 0.2, len(t))))]
    if crs != 3035:
        regions = [np.stack(proj.transform(r[:, 0], r[:, 1], 3035, crs), axis=1) for r in regions]
        coast = np.stack(proj.transform(coast[:, 0], coast[:, 1], 3035, crs), axis=1)
    ex = gis.ExclusionContainer(crs, res=res)
    ex.add_raster(land, codes=[1, 2, 3, 5, 8, 13, 21, 34, 40, 43], buffer=800)
    ex.add_raster(sea, codes=lambda d: d < -50.0)
    ex.add_geometry([{"type": "LineString", "coordinates": coast.tolist()}], buffer=2000)
    nxc, nyc = int((lo1 - lo0) / 0.25), int((la1 - la0) / 0.25)
    cut = ab.Cutout(data=syn.make_dataset(nxc, nyc, 2, x0=lo0 + 0.125, y0=la0 + 0.125, kinds=()))
    return cut, regions, ex


def cut_area(cut, crs):
    x, y = np.asarray(cut.coords["x"]), np.asarray(cut.coords["y"])
    area = proj.laea_cell_area if crs == 3035 else lambda *b: proj.cell_area(crs, *b)
    return area(x[None] - 0.125, x[None] + 0.125, y[:, None] - 0.125, y[:, None] + 0.125)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--regions", type=int, default=300)
    ap.add_argument("--km", type=float, default=4000)
    ap.add_argument("--repeat", type=int, default=2)
    ap.add_argument("--oracle", action="store_true")
    ap.add_argument("--out", help="also write the JSON result to this file")
    ap.add_argument("--crs", default="3035", choices=["3035", "ESRI:54009", "EPSG:3857"])
    ap.add_argument("--band-mb", type=float, help="per-band device memory budget in MiB")
    ap.add_argument("--dump", help="write the availability matrix to this .npy file")
    a = ap.parse_args()
    crs = proj.epsg(int(a.crs) if a.crs.isdigit() else a.crs)
    if a.band_mb:
        from atlite_b200 import availability

        availability._Session.BAND_BYTES = int(a.band_mb * 2 ** 20)
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    cut, regions, ex = case(a.regions, a.km, crs=crs)
    pixels, largest = 0, 0
    for r in regions:
        _, (ny, nx) = gis.padded_transform_and_shape((r[:, 0].min(), r[:, 1].min(), r[:, 0].max(), r[:, 1].max()), 100.0)
        pixels += nx * ny
        largest = max(largest, nx * ny)
    A = cut.availabilitymatrix(regions, ex, shapes_crs=crs)  # warm-up
    torch.cuda.synchronize()
    walls = []
    for _ in range(a.repeat):
        t0 = time.perf_counter()
        B = cut.availabilitymatrix(regions, ex, shapes_crs=crs)
        torch.cuda.synchronize()
        walls.append(time.perf_counter() - t0)
    assert np.array_equal(np.asarray(A.values), np.asarray(B.values)), "not repeatable"
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        cut.availabilitymatrix(regions, ex, shapes_crs=crs)
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        if ev.device_type.name == "CUDA" or getattr(ev, "self_device_time_total", 0):
            t = getattr(ev, "self_device_time_total", None)
            if t is None:
                t = ev.self_cuda_time_total
            if t:
                kern[ev.key[:60]] = round(t / 1e3, 2)
    out = dict(gpu=gpu, crs=a.crs, regions=a.regions, km=a.km, window_pixels=int(pixels),
               largest_window_bytes=11 * int(largest), band_mb=a.band_mb, wall_s=[round(w, 3) for w in walls],
               device_ms_by_kernel=dict(sorted(kern.items(), key=lambda kv: -kv[1])),
               eligible_share=float((np.asarray(A.values) * cut_area(cut, crs)).sum() / (pixels * 1e4)))
    if a.dump:
        np.save(a.dump, np.asarray(A.values))
    if a.oracle:
        import availability_oracle as AO

        r = regions[0]
        sub = gis.ExclusionContainer(3035, res=100.0)
        sub.add_raster(ex.rasters[0]["raster"], codes=ex.rasters[0]["codes"], buffer=800)
        t0 = time.perf_counter()
        gis.shape_availability(r, sub)
        torch.cuda.synchronize()
        tg = time.perf_counter() - t0
        lr = ex.rasters[0]["raster"]
        t0 = time.perf_counter()
        AO.shape_availability([(r, False)], 3035, 100.0, [dict(raster=dict(array=lr.array, transform=lr.transform,
                                                                           epsg=3035),
                                                                codes=ex.rasters[0]["codes"], buffer=800, res=100.0)])
        out["one_region_landcover_only_s"] = dict(gpu=round(tg, 3), numpy_oracle=round(time.perf_counter() - t0, 3))
    print(json.dumps(out, indent=1))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
