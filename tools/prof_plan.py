#!/usr/bin/env python
"""Aggregation-plan build times, and a "many layouts" PV workflow that needs a new plan per call.

    python tools/prof_plan.py [--tree DIR] [--reps 9] [--steps 730] [--out FILE]

Matrices: 1440 x 720 -> 3000 Voronoi shapes (synthetic.make_shapes, 1.2 M entries) and a 1 x S
layout row.  Times, median (and min / max) of --reps after a warm-up:

  host_reference   the CPU tiling (atl_plan_tiling_host), host clock
  create_pitched   atl_plan_create_pitched from host arrays, host clock (the call returns with the
                   plan complete on the device)
  create_device    atl_plan_create_device from device arrays, CUDA events on the build stream
  pv_new_layout    Cutout.pv(matrix=M, layout=L_k, aggregate_time=None) on a device-resident
                   1440 x 720 x --steps cutout, with a new layout L_k every call (a new matrix,
                   so a new plan), host clock around the call (its result is copied to the host)

--tree imports atlite_b200 from another checkout (e.g. the parent commit, built), so that two
builds can be timed alternately in separate processes; entry points a tree lacks are skipped.
The card's name and power limit are read in the same run and written beside the numbers.
"""

from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def stats(xs):
    xs = sorted(xs)
    return {"median_ms": xs[len(xs) // 2] * 1e3, "min_ms": xs[0] * 1e3, "max_ms": xs[-1] * 1e3, "n": len(xs)}


def timed(fn, reps, warm=2):
    for _ in range(warm):
        fn()
    out = []
    for _ in range(reps):
        out.append(fn())
    return stats(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", default=ROOT)
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--steps", type=int, default=730)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.tree))
    import scipy.sparse as sp
    import torch

    import atlite_b200 as ab
    from atlite_b200 import _lib, synthetic as syn

    assert os.path.dirname(os.path.dirname(os.path.abspath(ab.__file__))) == os.path.abspath(args.tree)
    lib = _lib.load()
    nx, ny = 1440, 720
    shapes = syn.make_shapes(nx, ny, 3000)
    lay0 = syn.make_layout(nx, ny)
    row = sp.csr_matrix(lay0.reshape(1, -1))
    res = {"tree": os.path.abspath(args.tree), "card": card(), "torch": torch.__version__}
    stream = torch.cuda.current_stream()

    for name, m in (("shapes_3000", shapes), ("layout_row", row)):
        indptr = np.ascontiguousarray(m.indptr, np.int64)
        idx = np.ascontiguousarray(m.indices, np.int32)
        dat = np.ascontiguousarray(m.data, np.float64)
        n_bus = m.shape[0]
        hargs = (_lib.ptr(indptr), _lib.ptr(idx), _lib.ptr(dat))
        r = {"nnz": int(m.nnz), "n_bus": n_bus}

        def host_ref():
            info = _lib.PlanInfo()
            t = time.perf_counter()
            _lib.check(lib.atl_plan_tiling_host(ny, nx, n_bus, *hargs, C.byref(info), None, None, None, 0))
            return time.perf_counter() - t

        def create_pitched():
            h = C.c_void_p()
            torch.cuda.synchronize()
            t = time.perf_counter()
            _lib.check(lib.atl_plan_create_pitched(0, ny, nx, nx, n_bus, *hargs, C.byref(h)))
            torch.cuda.synchronize()
            dt = time.perf_counter() - t
            lib.atl_plan_destroy(h)
            return dt

        r["host_reference"] = timed(host_ref, args.reps)
        r["create_pitched"] = timed(create_pitched, args.reps)
        if hasattr(lib, "atl_plan_create_device"):
            d = [torch.from_numpy(a).cuda() for a in (indptr, idx, dat)]

            def create_device():
                h = C.c_void_p()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                _lib.check(lib.atl_plan_create_device(0, ny, nx, nx, n_bus, len(dat),
                                                      *(C.c_void_p(t.data_ptr()) for t in d), 0,
                                                      C.c_void_p(stream.cuda_stream), C.byref(h)))
                e1.record(stream)
                e1.synchronize()
                lib.atl_plan_destroy(h)
                return e0.elapsed_time(e1) / 1e3

            r["create_device"] = timed(create_device, args.reps)
        res[name] = r

    # the many-layouts workflow on a resident cutout
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ds = syn.make_dataset(nx, ny, args.steps, -180.0, -90.0, kinds=("pv",), t_offset=24 * 150)
        cut = ab.Cutout(data=ds).to_device()
        del ds
        coords = cut.data.coords
        k = [0]

        def layout():
            k[0] += 1
            return ab.DataArray(lay0 * (1.0 + 1e-3 * k[0]), {"y": coords["y"], "x": coords["x"]}, ("y", "x"))

        mats = {"scipy": shapes}
        if hasattr(ab.engine, "device_csr"):
            mats["cuda_csr"] = torch.sparse_csr_tensor(torch.from_numpy(shapes.indptr.astype(np.int64)),
                                                       torch.from_numpy(shapes.indices.astype(np.int64)),
                                                       torch.from_numpy(shapes.data), shapes.shape).cuda()
        for mname, M in mats.items():
            def call():
                L = layout()
                torch.cuda.synchronize()
                t = time.perf_counter()
                cut.pv(panel="CSi", orientation="latitude_optimal", matrix=M, layout=L, aggregate_time=None)
                return time.perf_counter() - t

            res[f"pv_new_layout_{args.steps}steps_{mname}"] = timed(call, args.reps)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "a") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
