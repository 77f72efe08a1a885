"""EXACT checker for the overlay form of the indicator matrix (TEST INFRASTRUCTURE ONLY).

``compute_indicatormatrix(orig, dest)`` (atlite/gis.py:104-145) gives I[i, j] =
area(dest_i ∩ orig_j) / area(orig_j).  The reference delegates the areas to shapely / GEOS, which
cannot run in this image; this module computes them in exact rational arithmetic
(``fractions.Fraction``; every float64 input converts exactly), by a method that shares nothing
with the kernel's boundary integral: a slab decomposition.

The plane is cut at the y of every vertex of both shapes and of every crossing of two of their
edges.  Inside a slab no edge starts, ends or crosses another, so the edges that span it keep
their order along x, the weights between neighbouring edges stay the same, and the length

    L(y) = ∫ w_D(x, y) w_O(x, y) dx

is linear in y; the slab contributes ``h * L(y_mid)`` exactly.  w_S is the winding number of
shape S with exteriors counter-clockwise and holes clockwise: 1 inside a valid polygon, 0 outside,
2 where two parts of one multipolygon overlap (which then count twice, as in the kernels).

``intersection_area`` is the definition: it tests every pair of edges for a crossing and every
edge against every slab, so it takes seconds at a few hundred edges.  ``intersection_area_sweep``
returns the same Fraction with the same slabs, found by sweeps in y: only edges that meet the
pair's y window, crossings only between edges whose boxes meet, and an active-edge set per slab.
It handles shapes of several hundred edges each in about a second.
"""

from __future__ import annotations

from fractions import Fraction as Fr


def _fr(v):
    """Exact value of a float (any float64 is a dyadic rational), an int or a Fraction."""
    return v if isinstance(v, (Fr, int)) else Fr(float(v))


def _rings(shape):
    """[(ring, is_hole)] -> [[(Fr x, Fr y), ...]] oriented: exteriors CCW, holes CW; degenerate rings dropped.
    Coordinates may be floats or exact Fractions."""
    out = []
    for ring, hole in shape:
        pts = [(_fr(p[0]), _fr(p[1])) for p in ring]
        if len(pts) > 1 and pts[0] == pts[-1]:
            pts = pts[:-1]
        a2 = _area2(pts)
        if len(pts) < 3 or a2 == 0:
            continue
        if (a2 > 0) == bool(hole):
            pts = pts[::-1]
        out.append(pts)
    return out


def _area2(pts):
    n = len(pts)
    return sum(pts[k][0] * pts[(k + 1) % n][1] - pts[(k + 1) % n][0] * pts[k][1] for k in range(n))


def _edges(rings):
    return [(r[k], r[(k + 1) % len(r)]) for r in rings for k in range(len(r)) if r[k] != r[(k + 1) % len(r)]]


def _cross_y(e, f):
    """y of the single crossing point of segments e and f, or None (parallel or apart)."""
    (ax, ay), (bx, by) = e
    (cx, cy), (dx, dy) = f
    den = (bx - ax) * (dy - cy) - (by - ay) * (dx - cx)
    if den == 0:
        return None
    t = ((cx - ax) * (dy - cy) - (cy - ay) * (dx - cx)) / den
    u = ((cx - ax) * (by - ay) - (cy - ay) * (bx - ax)) / den
    if 0 <= t <= 1 and 0 <= u <= 1:
        return ay + t * (by - ay)
    return None


def shape_area(shape):
    """Exact area of one shape given as [(ring, is_hole)]: exteriors minus holes."""
    return sum(_area2(r) for r in _rings(shape)) / 2


def intersection_area(d, o):
    """Exact ∫ w_D w_O dA of two shapes given as [(ring, is_hole)] (``gis.geometry_rings``)."""
    ed, eo = _edges(_rings(d)), _edges(_rings(o))
    if not ed or not eo:
        return Fr(0)
    lo = max(min(min(p[1], q[1]) for p, q in ed), min(min(p[1], q[1]) for p, q in eo))
    hi = min(max(max(p[1], q[1]) for p, q in ed), max(max(p[1], q[1]) for p, q in eo))
    if not lo < hi:
        return Fr(0)
    ys = {lo, hi}
    ys.update(p[1] for e in ed + eo for p in e if lo < p[1] < hi)
    alle = ed + eo
    for i in range(len(alle)):
        for j in range(i + 1, len(alle)):
            y = _cross_y(alle[i], alle[j])
            if y is not None and lo < y < hi:
                ys.add(y)
    ys = sorted(ys)
    tagged = [(e, 0) for e in ed] + [(e, 1) for e in eo]
    total = Fr(0)
    for y0, y1 in zip(ys, ys[1:]):
        ym = (y0 + y1) / 2
        events = []
        for ((ax, ay), (bx, by)), side in tagged:
            if min(ay, by) <= y0 and max(ay, by) >= y1:  # spans the slab (horizontal edges never do)
                x = ax + (ym - ay) * (bx - ax) / (by - ay)
                events.append((x, side, 1 if by > ay else -1))
        events.sort(key=lambda ev: ev[0])
        w = [0, 0]  # winding numbers left of everything: the signed crossings of a closed ring sum to 0
        length, prev = Fr(0), None
        for x, side, up in events:
            if prev is not None and w[0] and w[1]:
                length += w[0] * w[1] * (x - prev)
            w[side] -= up
            prev = x
        total += (y1 - y0) * length
    return total


def intersection_area_sweep(d, o):
    """``intersection_area(d, o)``, bit for bit, by sweeps in y instead of all pairs."""
    return edges_intersection_area(_edges(_rings(d)), _edges(_rings(o)))


def edges_intersection_area(ed, eo):
    """∫ w_D w_O dA from the oriented edges of D and O (exteriors CCW, holes CW), each edge a pair
    of (Fraction x, Fraction y) points.  An edge whose y range misses the window [lo, hi] of the
    pair may be left out: it adds no slab boundary and spans no slab."""
    if not ed or not eo:
        return Fr(0)
    lo = max(min(min(p[1], q[1]) for p, q in ed), min(min(p[1], q[1]) for p, q in eo))
    hi = min(max(max(p[1], q[1]) for p, q in ed), max(max(p[1], q[1]) for p, q in eo))
    if not lo < hi:
        return Fr(0)
    # (ymin, ymax, xmin, xmax, edge, side) of the edges with a point strictly inside the window
    recs = []
    for side, es in ((0, ed), (1, eo)):
        for e in es:
            (ax, ay), (bx, by) = e
            ylo, yhi = (ay, by) if ay <= by else (by, ay)
            if yhi > lo and ylo < hi:
                recs.append((ylo, yhi, min(ax, bx), max(ax, bx), e, side))
    recs.sort(key=lambda r: r[0])
    ys = {lo, hi}
    ys.update(p[1] for r in recs for p in r[4] if lo < p[1] < hi)
    # crossings: every pair whose y ranges meet is seen once, when the later-starting edge enters
    active = []
    for r in recs:
        active = [a for a in active if a[1] >= r[0]]
        for a in active:
            if a[3] >= r[2] and r[3] >= a[2]:
                y = _cross_y(a[4], r[4])
                if y is not None and lo < y < hi:
                    ys.add(y)
        active.append(r)
    ys = sorted(ys)
    # slabs in y order: an edge spans [y0, y1] iff ymin <= y0 and ymax >= y1 (horizontal ones never)
    spanning = [r for r in recs if r[0] < r[1]]
    total, active, k = Fr(0), [], 0
    for y0, y1 in zip(ys, ys[1:]):
        while k < len(spanning) and spanning[k][0] <= y0:
            active.append(spanning[k])
            k += 1
        active = [a for a in active if a[1] >= y1]
        ym = (y0 + y1) / 2
        events = []
        for a in active:
            (ax, ay), (bx, by) = a[4]
            events.append((ax + (ym - ay) * (bx - ax) / (by - ay), a[5], 1 if by > ay else -1))
        events.sort(key=lambda ev: ev[0])  # ties have no length between them: their order is free
        w = [0, 0]
        length, prev = Fr(0), None
        for x, side, up in events:
            if prev is not None and w[0] and w[1]:
                length += w[0] * w[1] * (x - prev)
            w[side] -= up
            prev = x
        total += (y1 - y0) * length
    return total


def _box(shape):
    pts = [p for ring, _ in shape for p in ring]
    if not pts:
        return None
    xs, ys = [_fr(p[0]) for p in pts], [_fr(p[1]) for p in pts]
    return min(xs), min(ys), max(xs), max(ys)


def overlay_fractions(orig, dest):
    """{(dest index, orig index): Fraction area(dest ∩ orig) / area(orig)}, non-zero entries only.
    ``orig`` and ``dest``: lists of shapes, each a list of (ring, is_hole)."""
    areas = [shape_area(o) for o in orig]
    oboxes, out = [_box(o) for o in orig], {}
    for i, d in enumerate(dest):
        bd = _box(d)
        if bd is None:
            continue
        for j, o in enumerate(orig):
            bo = oboxes[j]
            if bo is None or bo[0] >= bd[2] or bd[0] >= bo[2] or bo[1] >= bd[3] or bd[1] >= bo[3]:
                continue
            a = intersection_area_sweep(d, o)
            if a:
                out[(i, j)] = a / areas[j]
    return out
