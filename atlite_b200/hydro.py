"""Host logic of ``Cutout.hydro`` (the reference's hydro.py): which basin each plant lies in, the
basins upstream of it, the basin areas and the travel steps.  NumPy only; the per-plant sum of the
rolled basin runoff runs on the GPU (``engine.hydro_shift_sum``, csrc/hydro.cu).

``hydrobasins`` is one level of the HydroBASINS dataset: a (Geo)DataFrame with the columns
``HYBAS_ID``, ``DIST_MAIN`` (km to the outlet along the main stem), ``NEXT_DOWN`` (the basin the
water flows to) and ``geometry`` (any polygon form ``gis.geometry_parts(polygonal=True)`` reads,
in lon / lat degrees), or a path that ``geopandas.read_file`` reads.
"""

from __future__ import annotations

import logging
import os
from collections import namedtuple

import numpy as np
import pandas as pd
import scipy.sparse as sp

from . import gis

logger = logging.getLogger(__name__)

Basins = namedtuple("Basins", ["plants", "meta", "shapes"])

# GRS80, PROJ's default ellipsoid for proj=cea
GRS80_A = 6378137.0
GRS80_F = 1.0 / 298.257222101
_EPS = np.finfo(np.float64).eps
_ORIENT_ERR = (3.0 + 16.0 * _EPS) * _EPS  # Shewchuk's orient2d error bound factor


def read_hydrobasins(hydrobasins):
    """The basin table as a DataFrame (a path goes through ``geopandas.read_file``), with the
    reference's checks of its type and columns (hydro.py:43-59)."""
    if isinstance(hydrobasins, (str, os.PathLike)):
        try:
            import geopandas as gpd
        except ImportError as e:
            raise ImportError(f"reading hydrobasins from the file {str(hydrobasins)!r} needs geopandas; "
                              "pass the basins as a (Geo)DataFrame instead") from e
        hydrobasins = gpd.read_file(hydrobasins)
    assert isinstance(hydrobasins, pd.DataFrame), (
        "hydrobasins should be passed as a filename or a GeoDataFrame, "
        f"but received `type(hydrobasins) = {type(hydrobasins)}`"
    )
    missing_columns = pd.Index(["HYBAS_ID", "DIST_MAIN", "NEXT_DOWN", "geometry"]).difference(hydrobasins.columns)
    assert missing_columns.empty, (
        "Couldn't find the column(s) {} in the hydrobasins dataset.".format(", ".join(missing_columns))
    )
    return hydrobasins


# --------------------------------------------------------------------------
# point -> basin
# --------------------------------------------------------------------------


class _Edges:
    """Every ring edge of every basin, flat, with the per-basin edge ranges and bounding boxes."""

    def __init__(self, shapes):
        x1, y1, x2, y2, counts = [], [], [], [], []
        box = np.full((len(shapes), 4), np.nan)  # xmin, xmax, ymin, ymax; NaN: no rings, never a candidate
        for i, g in enumerate(shapes):
            rings = [ring for _, ring in gis.geometry_parts(g, polygonal=True)]
            for ring in rings:
                nxt = np.roll(ring, -1, axis=0)  # the closing edge; a closed ring's is a point
                x1.append(ring[:, 0]), y1.append(ring[:, 1]), x2.append(nxt[:, 0]), y2.append(nxt[:, 1])
            counts.append(sum(len(r) for r in rings))
            if rings:
                v = np.concatenate(rings)
                box[i] = v[:, 0].min(), v[:, 0].max(), v[:, 1].min(), v[:, 1].max()
        cat = (lambda a: np.concatenate(a) if a else np.zeros(0))
        self.x1, self.y1, self.x2, self.y2 = cat(x1), cat(y1), cat(x2), cat(y2)
        self.ptr = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        self.box = box

    def candidates(self, px, py):
        b = self.box
        return np.flatnonzero((b[:, 0] <= px) & (px <= b[:, 1]) & (b[:, 2] <= py) & (py <= b[:, 3]))

    def contains(self, cand, px, py):
        """Boolean per candidate basin: the closed polygon (edges and vertices included, holes
        excluded, their boundary included) contains the point.  Even-odd rule over all rings with
        exact orientation signs (a float filter, exact rational arithmetic when it is inconclusive)."""
        cnt = self.ptr[cand + 1] - self.ptr[cand]
        tot = int(cnt.sum())
        if tot == 0:
            return np.zeros(len(cand), dtype=bool)
        owner = np.repeat(np.arange(len(cand)), cnt)
        e = np.repeat(self.ptr[cand] - np.cumsum(cnt) + cnt, cnt) + np.arange(tot)
        x1, y1, x2, y2 = self.x1[e], self.y1[e], self.x2[e], self.y2[e]
        left = (x1 - px) * (y2 - py)
        right = (y1 - py) * (x2 - px)
        det = left - right
        sign = np.sign(det)
        unsure = np.abs(det) <= _ORIENT_ERR * (np.abs(left) + np.abs(right))
        for k in np.flatnonzero(unsure):
            sign[k] = _exact_orient_sign(x1[k], y1[k], x2[k], y2[k], px, py)
        on_edge = (sign == 0) & (np.minimum(x1, x2) <= px) & (px <= np.maximum(x1, x2)) \
            & (np.minimum(y1, y2) <= py) & (py <= np.maximum(y1, y2))
        cross = ((y1 <= py) & (py < y2) & (sign > 0)) | ((y2 <= py) & (py < y1) & (sign < 0))
        boundary = np.bincount(owner, weights=on_edge, minlength=len(cand)) > 0
        odd = np.bincount(owner, weights=cross, minlength=len(cand)).astype(np.int64) % 2 == 1
        return boundary | odd


def _exact_orient_sign(x1, y1, x2, y2, px, py):
    from fractions import Fraction as Fr

    a, b, c, d, u, v = (Fr(float(q)) for q in (x1, y1, x2, y2, px, py))
    det = (a - u) * (d - v) - (b - v) * (c - u)
    return float((det > 0) - (det < 0))


def find_basins(plants, shapes):
    """Position in ``shapes`` of the basin each plant lies in (hydro.py:23-30): shapely's
    ``intersects`` of the point and the polygon, so a point on an edge or a vertex is inside, a
    point in a hole outside, on a hole's boundary inside.  Several matches: the reference's warning
    and the first in frame order; none: ``IndexError``."""
    edges = _Edges(list(shapes.values))
    out = np.empty(len(plants), dtype=np.int64)
    lon = plants["lon"].to_numpy(dtype=np.float64)
    lat = plants["lat"].to_numpy(dtype=np.float64)
    for i in range(len(plants)):
        cand = edges.candidates(lon[i], lat[i])
        hit = cand[edges.contains(cand, lon[i], lat[i])] if len(cand) else cand
        if len(hit) == 0:
            raise IndexError(f"plant {plants.index[i]!r} at ({lon[i]}, {lat[i]}) lies in no basin")
        if len(hit) > 1:
            hids = shapes.index[hit]
            logger.warning(f"The point ({lon[i]}, {lat[i]}) is in several basins: {hids}. Assuming the first one.")
        out[i] = hit[0]
    return out


# --------------------------------------------------------------------------
# upstream walk
# --------------------------------------------------------------------------


def upstream_basins(next_down, roots):
    """Per root, the basin itself and every basin upstream of it, in the reference's breadth-first
    order (hydro.py:33-39): the root, then the basins draining into it in frame order, then theirs.
    ``next_down``: position of each basin's downstream basin (-1: none in the table).  Returns
    (ptr, basins) in CSR form; all roots are walked together, one tree level per step."""
    next_down = np.asarray(next_down, dtype=np.int64)
    n = len(next_down)
    has = np.flatnonzero(next_down >= 0)
    child = has[np.argsort(next_down[has], kind="stable")]  # children grouped by parent, frame order
    cptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(next_down[has], minlength=n), out=cptr[1:])
    owner = np.arange(len(roots), dtype=np.int64)
    node = np.asarray(roots, dtype=np.int64)
    owners, nodes = [owner], [node]
    for _ in range(n + 1):
        cnt = cptr[node + 1] - cptr[node]
        tot = int(cnt.sum())
        if tot == 0:
            break
        rep = np.repeat(np.arange(len(node)), cnt)
        node = child[cptr[node][rep] + np.arange(tot) - np.repeat(np.cumsum(cnt) - cnt, cnt)]
        owner = owner[rep]
        owners.append(owner)
        nodes.append(node)
    else:
        raise ValueError("NEXT_DOWN links the basins in a cycle")
    owner, node = np.concatenate(owners), np.concatenate(nodes)
    order = np.argsort(owner, kind="stable")  # per root: level by level, each in walk order
    ptr = np.zeros(len(roots) + 1, dtype=np.int64)
    np.cumsum(np.bincount(owner, minlength=len(roots)), out=ptr[1:])
    return ptr, node[order]


Routing = namedtuple("Routing", ["basins", "ptr", "rows"])


def route(plants, hydrobasins):
    """``determine_basins`` plus the walk in CSR form: ``ptr`` (n_plants + 1) and, per walked
    basin, its ``rows`` position on the basin axis (the rows of ``basins.meta``)."""
    hb = read_hydrobasins(hydrobasins).set_index("HYBAS_ID")
    meta = hb[hb.columns.difference(("geometry",))]
    shapes = hb["geometry"]
    pos = find_basins(plants, shapes)
    nd = meta.index.get_indexer(pd.Index(meta["NEXT_DOWN"]))
    ptr, up = upstream_basins(nd, pos)
    ids = meta.index.to_numpy()
    upstream = [list(ids[up[ptr[i]:ptr[i + 1]]]) for i in range(len(pos))]
    plant_basins = pd.DataFrame({"hid": ids[pos], "upstream": upstream}, index=plants.index)
    _, first = np.unique(up, return_index=True)
    unique = up[np.sort(first)]  # order of first appearance
    hid = pd.Index(ids[unique], name="hid")
    where = np.full(len(ids), -1, dtype=np.int64)
    where[unique] = np.arange(len(unique))
    basins = Basins(plant_basins, meta.iloc[unique].set_axis(hid), shapes.iloc[unique].set_axis(hid))
    return Routing(basins, ptr, where[up])


def determine_basins(plants, hydrobasins, show_progress=False):
    """The reference's ``determine_basins`` (hydro.py:42-78): returns ``Basins(plants, meta,
    shapes)`` with ``plants`` a DataFrame of ``hid`` and ``upstream`` (a list of basin ids) per
    plant, and ``meta`` / ``shapes`` the non-geometry columns and the geometries of the basins any
    plant drains, in order of first appearance, indexed by ``hid``.  ``show_progress`` is accepted
    and unused."""
    return route(plants, hydrobasins).basins


# --------------------------------------------------------------------------
# areas and travel steps
# --------------------------------------------------------------------------


def authalic_q(lat_deg, e2=None):
    """q(phi) of the ellipsoidal equal-area projections: (1 - e^2) (sin phi / (1 - e^2 sin^2 phi)
    - ln((1 - e sin phi) / (1 + e sin phi)) / (2 e)), GRS80 by default."""
    e2 = GRS80_F * (2.0 - GRS80_F) if e2 is None else e2
    e = np.sqrt(e2)
    s = np.sin(np.radians(np.asarray(lat_deg, dtype=np.float64)))
    return (1.0 - e2) * (s / (1.0 - e2 * s * s) - np.log((1.0 - e * s) / (1.0 + e * s)) / (2.0 * e))


def cea_xy(lon_deg, lat_deg):
    """PROJ's ``+proj=cea`` forward on GRS80 with lat_ts = 0: x = a lambda, y = a q(phi) / 2."""
    return GRS80_A * np.radians(np.asarray(lon_deg, dtype=np.float64)), GRS80_A * authalic_q(lat_deg) / 2.0


def _ring_area(x, y):
    """|shoelace area| of a ring, closed or not, shifted by its first vertex as GEOS does."""
    if len(x) < 3:
        return 0.0
    x = x - x[0]
    return abs(float(np.dot(x, np.roll(y, -1)) - np.dot(np.roll(x, -1), y))) / 2.0


def basin_areas(shapes):
    """Area in m^2 of each shape in the cylindrical equal-area projection (the reference's
    ``shapes.to_crs(dict(proj="cea")).area``): every vertex projected, then the planar area of the
    projected polygon, exterior minus holes, summed over the polygons of a MultiPolygon."""
    out = np.zeros(len(shapes))
    for i, g in enumerate(shapes):
        for kind, ring in gis.geometry_parts(g, polygonal=True):
            a = _ring_area(*cea_xy(ring[:, 0], ring[:, 1]))
            out[i] += -a if kind == gis.PART_HOLE else a
    return out


def travel_steps(dist_main, dist_plant, flowspeed):
    """``int(distance / (flowspeed * 3.6) + 0.5)`` per upstream basin, truncated toward zero as
    ``astype(int)`` does (hydro.py:95-99): the time steps the water needs at ``flowspeed`` m/s over
    the difference of ``DIST_MAIN`` (km)."""
    n = (np.asarray(dist_main, dtype=np.float64) - dist_plant) / (flowspeed * 3.6) + 0.5
    if not np.isfinite(n).all():
        raise ValueError("Cannot convert non-finite travel times (NaN DIST_MAIN?) to integer steps")
    return np.trunc(n).astype(np.int64)


def normalise_rows(matrix):
    """Each row divided by its sum, NaN and +-inf set to 0 (convert.py:1132-1134), as CSR without
    stored zeros: a basin that covers no cell has an empty row."""
    m = sp.csr_matrix(matrix, dtype=np.float64, copy=True)
    m.sum_duplicates()
    s = np.asarray(m.sum(axis=1)).ravel()
    with np.errstate(divide="ignore", invalid="ignore"):
        m.data = np.nan_to_num(m.data / np.repeat(s, np.diff(m.indptr)), nan=0.0, posinf=0.0, neginf=0.0)
    m.eliminate_zeros()
    return m
