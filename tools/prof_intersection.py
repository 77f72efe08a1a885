#!/usr/bin/env python
"""Wall time of the public intersection-matrix call (gis.compute_intersectionmatrix), per
geometry kind and for all of them in one call, next to compute_indicatormatrix on the
same regions.

    python tools/prof_intersection.py [--repeat N]

Workload: 1440 x 720 grid at 0.25 degree, 3000 Voronoi regions (synthetic.make_voronoi_shapes),
the line network between their sites (synthetic.make_line_network, ~9000 polylines of 2-50
vertices) and 100 000 random points.  Host clock around the call, which ends in a device
synchronise and returns the host CSR; warm-up call first, median of N (default 7).  The host-side
reading of the geometries (gis.pack_geometries) is timed on its own too.  Prints one JSON line
with the card's name and power limit."""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from atlite_b200 import gis, synthetic as syn  # noqa: E402


def wall_ms(fn, repeat):
    fn()  # warm-up: module load, allocator
    ts = []
    for _ in range(repeat):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return round(float(np.median(ts)), 2), round(float(min(ts)), 2)


def main():
    repeat = int(sys.argv[sys.argv.index("--repeat") + 1]) if "--repeat" in sys.argv else 7
    if not torch.cuda.is_available():
        raise SystemExit("prof_intersection.py needs a CUDA device")
    card = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    x, y = syn.make_coords(1440, 720, -180.0 + 0.125, -90.0 + 0.125)
    regions = syn.make_voronoi_shapes(x, y, 3000)
    lines = syn.make_line_network(x, y, 3000)
    rng = np.random.default_rng(3)
    pts = np.c_[rng.uniform(x[0] - 0.125, x[-1] + 0.125, 100_000), rng.uniform(y[0] - 0.125, y[-1] + 0.125, 100_000)]
    points = [{"type": "Point", "coordinates": p} for p in pts]
    out = {"card": card, "power_limit_and_max_sm_clock": power, "grid": [720, 1440],
           "regions": len(regions), "lines": len(lines),
           "line_segments": int(sum(len(a["coordinates"]) - 1 for a in lines)), "points": len(points),
           "repeat": repeat, "ms_median_min": {}}
    cases = {"regions": regions, "lines": lines, "points": points, "all": regions + lines + points}
    for name, shapes in cases.items():
        out["ms_median_min"][f"intersection_{name}"] = wall_ms(lambda: gis.compute_intersectionmatrix(x, y, shapes),
                                                               repeat)
        # of which: reading the geometries into the packed arrays on the host
        out["ms_median_min"][f"pack_geometries_{name}"] = wall_ms(lambda: gis.pack_geometries(shapes), repeat)
    out["ms_median_min"]["indicator_regions"] = wall_ms(lambda: gis.compute_indicatormatrix(x, y, regions), repeat)
    m = gis.compute_intersectionmatrix(x, y, cases["all"])
    out["nnz_all"] = int(m.nnz)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
