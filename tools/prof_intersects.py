#!/usr/bin/env python
"""Wall time of the general form of the intersection matrix (gis.compute_intersectionmatrix(orig, dest)).

    python tools/prof_intersects.py [--repeat N]

Workloads, all in EPSG:4326 over the Europe extent of the 0.25 degree grid (220 x 160 cells):
  * cells: 3 000 Voronoi regions (synthetic.make_voronoi_shapes) as ``dest`` against the cells given
    as polygons (gis.cell_edges boxes) as ``orig``; next to it the grid form
    ``compute_intersectionmatrix(x, y, regions)`` on the same input, which gives the same matrix.
  * lines: the 3 000 regions as ``orig`` against a line network (synthetic.make_line_network) of
    about 20 000 lines as ``dest``.
  * points: 10^5 random points as ``orig`` against the 3 000 regions as ``dest``.
  * regions: the 3 000 regions against themselves, where neighbours share borders.
Host clock around the call, which returns the host CSR (the device is synchronised inside), warm-up
call first, then the median and minimum of N (default 7).  The host-side reading of the geometries
(gis.pack_geometries, both sides) is timed on its own too, and the candidate pairs (closed boxes
that meet) are counted on the host.  Prints one JSON line with the card's name and power limit."""
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
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return round(float(np.median(ts)), 2), round(float(min(ts)), 2)


def boxes(shapes):
    """(n, 4) closed bounding boxes (xlo, ylo, xhi, yhi); empty shapes never meet."""
    spp, pp, _, xy = gis.pack_geometries(shapes)
    out = np.tile([np.inf, np.inf, -np.inf, -np.inf], (len(spp) - 1, 1))
    for s in range(len(spp) - 1):
        v = xy[pp[spp[s]]:pp[spp[s + 1]]]
        if len(v):
            out[s] = (*v.min(0), *v.max(0))
    return out


def candidate_pairs(orig, dest):
    """Pairs of closed boxes that meet: the pairs the pair test runs on."""
    o, d = boxes(orig), boxes(dest)
    order = np.argsort(o[:, 0], kind="stable")
    xs = o[order, 0]
    n = 0
    for b in d:
        k = order[:np.searchsorted(xs, b[2], side="right")]
        q = o[k]
        n += int(((b[0] <= q[:, 2]) & (q[:, 1] <= b[3]) & (b[1] <= q[:, 3])).sum())
    return n


def main():
    repeat = int(sys.argv[sys.argv.index("--repeat") + 1]) if "--repeat" in sys.argv else 7
    if not torch.cuda.is_available():
        raise SystemExit("prof_intersects.py needs a CUDA device")
    card = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    x, y = syn.make_coords(220, 160, -12.0 + 0.125, 33.0 + 0.125)
    xlo, xhi = gis.cell_edges(x)
    ylo, yhi = gis.cell_edges(y)
    cells = [np.array([[xlo[i], ylo[j]], [xhi[i], ylo[j]], [xhi[i], yhi[j]], [xlo[i], yhi[j]]])
             for j in range(len(y)) for i in range(len(x))]
    regions = syn.make_voronoi_shapes(x, y, 3000)
    lines = syn.make_line_network(x, y, 6700)
    rng = np.random.default_rng(1)
    points = [{"type": "Point", "coordinates": p} for p in
              np.c_[rng.uniform(x[0], x[-1], 100_000), rng.uniform(y[0], y[-1], 100_000)].tolist()]
    cases = {"cells": (cells, regions), "lines": (regions, lines), "points": (points, regions),
             "regions": (regions, regions)}
    out = {"card": card, "power_limit_and_max_sm_clock": power, "grid": [len(y), len(x)], "regions": len(regions),
           "lines": len(lines), "line_segments": int(sum(len(s["coordinates"]) - 1 for s in lines)),
           "points": len(points), "repeat": repeat, "ms_median_min": {}, "nnz": {}, "candidate_pairs": {}}
    out["ms_median_min"]["grid_form_cells"] = wall_ms(lambda: gis.compute_intersectionmatrix(x, y, regions), repeat)
    for name, (orig, dest) in cases.items():
        out["ms_median_min"][name] = wall_ms(lambda: gis.compute_intersectionmatrix(orig, dest), repeat)
        out["ms_median_min"][f"pack_geometries_{name}"] = wall_ms(
            lambda: (gis.pack_geometries(orig), gis.pack_geometries(dest)), repeat)
        out["nnz"][name] = int(gis.compute_intersectionmatrix(orig, dest).nnz)
        out["candidate_pairs"][name] = candidate_pairs(orig, dest)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
