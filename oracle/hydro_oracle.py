"""CPU oracle for ``Cutout.hydro`` (TEST INFRASTRUCTURE ONLY -- never imported by atlite_b200).

float64 NumPy restatement of the reference's hydro path (atlite/hydro.py, convert.py:1087-1149):

  * ``find_basin``: shapely's ``intersects`` of a point and a (Multi)Polygon, decided in EXACT
    rational arithmetic (every float64 coordinate converted exactly with ``fractions``): on a ring
    edge or vertex -> inside, else the even-odd rule over all rings (holes excluded).  Basins are
    tested one by one in frame order, by a different method than the vectorised float filter of
    atlite_b200/hydro.py.
  * ``upstream``: the breadth-first walk over ``NEXT_DOWN`` as a Python list, one basin at a time.
  * ``determine_basins``: plant basins, upstream lists and the unique basins in order of first
    appearance.
  * ``normalise``: dense row normalisation, NaN / inf -> 0.
  * ``cea_area``: GRS80 cylindrical equal-area projection of the vertices, then the shoelace area,
    exterior minus holes (what ``shapes.to_crs(dict(proj="cea")).area`` gives: ``to_crs`` moves
    vertices and does not densify).
  * ``shift_and_aggregate``: per plant and upstream basin ``np.roll`` of the area-scaled runoff by
    ``int(dDIST_MAIN / (flowspeed * 3.6) + 0.5)`` steps, added in walk order.

tests/golden/make_golden_hydro.py runs the reference's own ``find_upstream_basins``,
``determine_basins`` (its point location replaced by a fixed assignment), ``hydro``'s
normalisation and ``shift_and_aggregate_runoff_for_plants``; tests/test_hydro.py pins this oracle to
its output (tests/golden/reference_hydro.npz).  Pure Python loops: small cases only.
"""

from __future__ import annotations

from fractions import Fraction as Fr

import numpy as np
import scipy.sparse as sp

EXTERIOR, HOLE = 0, 1
A = 6378137.0  # GRS80
F = 1.0 / 298.257222101


def _orient(a, b, c):
    return (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0])


def point_in_parts(parts, px, py):
    """Closed (Multi)Polygon given as ``gis.geometry_parts`` (kind, ring) parts contains the point?"""
    p = (Fr(float(px)), Fr(float(py)))
    crossings = 0
    for _, ring in parts:
        pts = [(Fr(float(u)), Fr(float(v))) for u, v in np.asarray(ring, dtype=np.float64)[:, :2]]
        for i in range(len(pts)):
            a, b = pts[i], pts[(i + 1) % len(pts)]
            o = _orient(a, b, p)
            if o == 0 and min(a[0], b[0]) <= p[0] <= max(a[0], b[0]) and min(a[1], b[1]) <= p[1] <= max(a[1], b[1]):
                return True
            if (a[1] <= p[1] < b[1] and o > 0) or (b[1] <= p[1] < a[1] and o < 0):
                crossings += 1
    return crossings % 2 == 1


def find_basin(parts_by_basin, px, py):
    """Frame positions of every basin containing the point (the caller takes the first)."""
    return [i for i, parts in enumerate(parts_by_basin) if point_in_parts(parts, px, py)]


def upstream(ids, next_down, hid):
    """hydro.py:33-39 on lists."""
    hids = [hid]
    i = 0
    while i < len(hids):
        hids.extend(b for b, d in zip(ids, next_down) if d == hids[i])
        i += 1
    return hids


def determine_basins(ids, next_down, plant_hids):
    """(upstream list per plant, unique basins in order of first appearance)."""
    ups = [upstream(list(ids), list(next_down), h) for h in plant_hids]
    seen, unique = set(), []
    for u in ups:
        for b in u:
            if b not in seen:
                seen.add(b)
                unique.append(b)
    return ups, unique


def normalise(matrix):
    """Row-normalised dense matrix, NaN and +-inf -> 0 (convert.py:1132-1134)."""
    m = np.asarray(sp.csr_matrix(matrix).todense(), dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.nan_to_num(m / m.sum(axis=1, keepdims=True), nan=0.0, posinf=0.0, neginf=0.0)


def authalic_q(lat_deg):
    e2 = F * (2 - F)
    e = np.sqrt(e2)
    s = np.sin(np.deg2rad(np.asarray(lat_deg, dtype=np.float64)))
    return (1 - e2) * (s / (1 - e2 * s ** 2) - 1 / (2 * e) * np.log((1 - e * s) / (1 + e * s)))


def cea_area(parts):
    """Area in m^2 of a (Multi)Polygon in +proj=cea (GRS80, lat_ts=0)."""
    total = 0.0
    for kind, ring in parts:
        r = np.asarray(ring, dtype=np.float64)
        x = A * np.deg2rad(r[:, 0])
        y = A * authalic_q(r[:, 1]) / 2
        s = 0.0
        for i in range(len(x)):
            j = (i + 1) % len(x)
            s += x[i] * y[j] - x[j] * y[i]
        total += -abs(s) / 2 if kind == HOLE else abs(s) / 2
    return total


def travel_steps(dist, flowspeed):
    return int(np.trunc(dist / (flowspeed * 3.6) + 0.5))


def shift_and_aggregate(ups, plant_hids, dist_main, runoff, flowspeed):
    """hydro.py:81-104: ``runoff`` maps basin id -> (T,) float64 series (already area-scaled),
    ``dist_main`` basin id -> DIST_MAIN.  Returns (n_plants, T)."""
    T = len(next(iter(runoff.values()))) if runoff else 0
    out = np.zeros((len(ups), T))
    for p, (u, h) in enumerate(zip(ups, plant_hids)):
        for b in u:
            out[p] += np.roll(runoff[b], travel_steps(dist_main[b] - dist_main[h], flowspeed))
    return out


def hydro(od, x, y, plants_lonlat, table, flowspeed=1, weight_with_height=False, indicator=None, post=None):
    """Inflow (n_plants, T) of the plants at ``plants_lonlat`` ((P, 2) lon, lat), from the basin
    ``table`` (dict of HYBAS_ID, DIST_MAIN, NEXT_DOWN lists and ``parts``: the ``geometry_parts``
    of each basin).  ``od``: the oracle dataset (atlite_oracle form, runoff and height); the runoff
    aggregation is atlite_oracle's convert_and_aggregate with convert_runoff.  ``indicator``:
    callable (x, y, parts list) -> (n, S) indicator matrix, default indicator_oracle's.
    ``post``: callable on the (T, B) basin runoff (the smoothing / quantile cut of ``runoff``)."""
    import atlite_oracle as O
    import indicator_oracle as IO

    ids, nd, dist = list(table["HYBAS_ID"]), list(table["NEXT_DOWN"]), list(table["DIST_MAIN"])
    parts = table["parts"]
    plant_hids = []
    for lon, lat in plants_lonlat:
        hit = find_basin(parts, lon, lat)
        if not hit:
            raise IndexError(f"({lon}, {lat}) lies in no basin")
        plant_hids.append(ids[hit[0]])
    ups, unique = determine_basins(ids, nd, plant_hids)
    pos = {b: i for i, b in enumerate(ids)}
    uparts = [parts[pos[b]] for b in unique]
    if indicator is None:
        rings = [[(r, k == HOLE) for k, r in p] for p in uparts]
        indicator = (lambda x_, y_, _: IO.indicatormatrix(x_, y_, rings))
    m = normalise(indicator(x, y, uparts))
    R = O.convert_and_aggregate(od, O.convert_runoff, matrix=m, aggregate_time=None,
                                weight_with_height=weight_with_height)  # (T, B)
    if post is not None:
        R = post(R)
    area = np.array([cea_area(p) for p in uparts])
    scaled = {b: R[:, i] * area[i] for i, b in enumerate(unique)}
    return shift_and_aggregate(ups, plant_hids, {b: dist[pos[b]] for b in ids}, scaled, flowspeed), \
        dict(ups=ups, unique=unique, area=area, plant_hids=plant_hids)
