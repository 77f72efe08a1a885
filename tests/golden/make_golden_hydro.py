#!/usr/bin/env python
"""Generate ``reference_hydro.npz``: the REFERENCE'S OWN ``convert.hydro`` (convert.py:1087-1149)
with its ``determine_basins``, ``find_upstream_basins`` and ``shift_and_aggregate_runoff_for_plants``
(hydro.py), loaded from the reference's source files under the stand-ins of ``xr_shim.py`` and
``xr_shim_hydro.py``, on a
fixed synthetic basin tree.

Three things the reference takes from shapely / geopandas / a cutout are stood in for here:
  * ``find_basin`` (shapely point-in-polygon): a fixed plant -> basin assignment;
  * ``shapes.to_crs(dict(proj="cea")).area`` (pyproj): fixed areas per basin;
  * the cutout: ``indicatormatrix`` returns a fixed lil_matrix (as the reference's gis does), with
    an all-zero row for a basin off the grid, and ``runoff`` returns the normalised matrix it is
    handed times fixed per-cell series.
Everything in between -- the upstream walk, the unique-basin order, the normalisation, the area
scaling, the travel steps and the rolls -- is the reference's source executing.  The tree has
shifts < 0 (a basin whose DIST_MAIN is smaller than its plant's), shifts >= T, a plant downstream
of two other plants, two plants in one basin and a basin no plant drains.

    python tests/golden/make_golden_hydro.py     # writes tests/golden/reference_hydro.npz
"""

import io
import os
import sys
import types
import warnings
import zipfile

import numpy as np
import pandas as pd
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import xr_shim_hydro  # noqa: E402

warnings.simplefilter("ignore")
conv, hydrom = xr_shim_hydro.load_reference_hydro()

T, S = 40, 30
# HYBAS_ID, NEXT_DOWN, DIST_MAIN (km): frame order is not id order, nor walk order
BASINS = [
    (117, 111, 260.0),  # far up the main stem: 260 km from 111 -> 72 steps at 1 m/s (>= T)
    (111, 0, 0.0),      # outlet
    (121, 111, 30.0),
    (113, 112, 95.0),
    (112, 111, 40.0),
    (131, 121, 12.0),   # DIST_MAIN below its plant's (121 at 30 km): a negative shift
    (114, 113, 150.0),
    (122, 121, 61.0),
    (141, 0, 5.0),      # another outlet: no plant drains it
    (115, 113, 180.5),
    (116, 114, 205.0),
    (132, 122, 88.0),
    (133, 122, 99.9),
    (118, 117, 330.0),
]
# plant label -> basin id (what shapely's find_basin would return)
PLANTS = [("dam_a", 113), ("ror_b", 121), ("ror_c", 111), ("ror_d", 113), ("head_e", 118)]


class _GeoSeries(pd.Series):
    @property
    def _constructor(self):
        return _GeoSeries

    def to_crs(self, crs):
        assert crs == {"proj": "cea"}
        return types.SimpleNamespace(area=pd.Series([AREA[h] for h in self.index], index=self.index))


class _Frame(pd.DataFrame):
    @property
    def _constructor(self):
        return _Frame

    @property
    def _constructor_sliced(self):
        return _GeoSeries


class _Cutout:
    """indicatormatrix and runoff as the reference's hydro() calls them."""

    def __init__(self, rows, cells, time):
        self.rows, self.cells, self.time = rows, cells, time
        self.seen = {}

    def indicatormatrix(self, shapes):
        m = sp.lil_matrix((len(shapes), S), dtype=float)
        for i, h in enumerate(shapes.index):
            m[i] = self.rows[h]
        return m

    def runoff(self, matrix, index, weight_with_height, show_progress, **kw):
        # dense (older scipy: sparse / dense is dense) or sparse (newer: it keeps the stored entries)
        m = matrix.toarray() if sp.issparse(matrix) else np.asarray(matrix, dtype=np.float64)
        self.seen.update(matrix=m, index=np.asarray(index), nnz=np.count_nonzero(m) if not sp.issparse(matrix)
                         else sp.csr_matrix(matrix).nnz)
        return xr_shim_hydro.DataArray(m @ self.cells.T, {"hid": index, "time": self.time}, ("hid", "time"))


rng = np.random.default_rng(23)
ids = [b[0] for b in BASINS]
AREA = {h: float(a) for h, a in zip(ids, rng.uniform(1e8, 5e9, len(ids)))}
ROWS = {}
for h in ids:
    r = np.where(rng.uniform(size=S) < 0.35, rng.uniform(0.05, 1.0, S), 0.0)
    ROWS[h] = r
ROWS[133] = np.zeros(S)  # off the grid: covers no cell
CELLS = rng.exponential(2e-4, (T, S)).astype(np.float32).astype(np.float64)
TIME = pd.date_range("2013-01-01", periods=T, freq="h")


def main():
    hb = _Frame({"HYBAS_ID": ids, "NEXT_DOWN": [b[1] for b in BASINS], "DIST_MAIN": [b[2] for b in BASINS],
                 "geometry": [f"basin {h}" for h in ids]})
    where = dict(PLANTS)
    hydrom.find_basin = lambda shapes, lon, lat: where[lon]
    sys.modules["geopandas"].GeoDataFrame = _Frame
    plants = pd.DataFrame({"lon": [p for p, _ in PLANTS], "lat": 0.0}, index=pd.Index([p for p, _ in PLANTS]))
    basins = hydrom.determine_basins(plants, hb)  # the reference's own walk and unique-basin order
    out = {"ids": np.array(ids), "next_down": np.array([b[1] for b in BASINS]),
           "dist_main": np.array([b[2] for b in BASINS]), "area": np.array([AREA[h] for h in ids]),
           "rows": np.array([ROWS[h] for h in ids]), "cells": CELLS, "time_ns": TIME.as_unit("ns").asi8,
           "plant_names": np.array([p for p, _ in PLANTS]), "plant_hids": np.array([h for _, h in PLANTS]),
           "upstream_ptr": np.cumsum([0] + [len(u) for u in basins.plants["upstream"]]),
           "upstream": np.concatenate([np.asarray(u) for u in basins.plants["upstream"]]),
           "unique": np.asarray(basins.shapes.index)}
    flowspeeds = [1.0, 0.5, 2.7]
    for k, fs in enumerate(flowspeeds):
        cut = _Cutout(ROWS, CELLS, TIME)
        res = conv.hydro(cut, plants, hb, flowspeed=fs)  # the reference's own hydro()
        assert res.dims == ("plant", "time")
        out[f"inflow_{k}"] = np.asarray(res.values, dtype=np.float64)
        out["normalised"] = cut.seen["matrix"]
        out["normalised_nnz"] = np.array(cut.seen["nnz"])
        assert np.array_equal(cut.seen["index"], out["unique"])
    out["flowspeeds"] = np.array(flowspeeds)
    buf = io.BytesIO()
    np.savez_compressed(buf, **out)
    # rewrite the zip without timestamps, so the file's bytes depend only on its contents
    src = zipfile.ZipFile(io.BytesIO(buf.getvalue()))
    with zipfile.ZipFile(os.path.join(HERE, "reference_hydro.npz"), "w", zipfile.ZIP_DEFLATED) as dst:
        for name in sorted(src.namelist()):
            zi = zipfile.ZipInfo(name, date_time=(1980, 1, 1, 0, 0, 0))
            zi.compress_type = zipfile.ZIP_DEFLATED
            dst.writestr(zi, src.read(name))
    print("wrote reference_hydro.npz:", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
