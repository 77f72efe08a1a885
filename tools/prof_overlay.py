#!/usr/bin/env python
"""Wall time of the overlay form of the indicator matrix (gis.compute_indicatormatrix(orig, dest)).

    python tools/prof_overlay.py [--repeat N]

Workloads, all in EPSG:4326 over a Europe-sized extent:
  * population_layout: 1 500 Voronoi regions (synthetic.make_voronoi_shapes) with every edge cut
    into equal pieces, about 10^6 vertices in all, as ``orig``; the cell polygons of the 0.25 degree
    grid (gis.cell_edges boxes, 216 x 156 cells) as ``dest``.  PyPSA-Eur's population layout has
    this shape (NUTS3 regions against grid cells).
  * population_layout_T: the same with ``orig`` and ``dest`` swapped.
  * regions: the 1 500 densified regions against 3 000 other densified regions (about 10^6
    vertices as well), as region-to-region keys are.
Host clock around the call, which returns the host CSR; warm-up call first, then the median and
minimum of N (default 5).  The host-side reading of the geometries (gis.pack_shapes, both sides) is
timed on its own too.  Prints one JSON line with the card's name and power limit."""
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


def densify(rings, vertices):
    """Every edge cut into k equal pieces, k chosen so that the rings hold about ``vertices`` in all."""
    k = max(1, round(vertices / sum(len(r) for r in rings)))
    t = np.arange(k)[:, None] / k
    out = []
    for r in rings:
        a, b = r, np.roll(r, -1, axis=0)
        out.append(np.ascontiguousarray((a[:, None, :] + t[None] * (b - a)[:, None, :]).reshape(-1, 2)))
    return out


def main():
    repeat = int(sys.argv[sys.argv.index("--repeat") + 1]) if "--repeat" in sys.argv else 5
    if not torch.cuda.is_available():
        raise SystemExit("prof_overlay.py needs a CUDA device")
    card = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    x, y = syn.make_coords(216, 156, -12.0 + 0.125, 33.0 + 0.125)
    xlo, xhi = gis.cell_edges(x)
    ylo, yhi = gis.cell_edges(y)
    cells = [np.array([[xlo[i], ylo[j]], [xhi[i], ylo[j]], [xhi[i], yhi[j]], [xlo[i], yhi[j]]])
             for j in range(len(y)) for i in range(len(x))]
    regions = densify(syn.make_voronoi_shapes(x, y, 1500, seed=8), 1_000_000)
    others = densify(syn.make_voronoi_shapes(x, y, 3000, seed=9), 1_000_000)
    cases = {"population_layout": (regions, cells), "population_layout_T": (cells, regions),
             "regions": (regions, others)}
    out = {"card": card, "power_limit_and_max_sm_clock": power, "grid": [len(y), len(x)], "cells": len(cells),
           "regions": len(regions), "region_vertices": int(sum(len(r) for r in regions)),
           "other_regions": len(others), "other_vertices": int(sum(len(r) for r in others)),
           "repeat": repeat, "ms_median_min": {}, "nnz": {}}
    for name, (orig, dest) in cases.items():
        out["ms_median_min"][name] = wall_ms(lambda: gis.compute_indicatormatrix(orig, dest), repeat)
        # of which: reading the geometries of both sides into the packed arrays on the host
        out["ms_median_min"][f"pack_shapes_{name}"] = wall_ms(lambda: (gis.pack_shapes(orig), gis.pack_shapes(dest)),
                                                              repeat)
        out["nnz"][name] = int(gis.compute_indicatormatrix(orig, dest).nnz)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
