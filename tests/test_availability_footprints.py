"""The land-eligibility kernels at production footprints, against exact integer references.

Every case is dyadic: the container's ``res`` is a power of two (128 m or 16 m in EPSG:3035,
2^-4 or 2^-7 degrees in EPSG:4326), and every vertex, raster origin, raster pixel size, buffer and
cutout edge lies on a lattice of 1/8 container pixel.  Then pixel centres, ``floor((x - c) / a)``
of raster sampling and counting, ``k = int(buffer / res) + 1`` and the orientation signs are all
exact in float64, and same-CRS ``proj.transform`` is the identity, so the kernels must match the
references here bit for bit with no tie excused.  The references work in int64 on that lattice
(coordinates times 8 / res):

* polygon mask: a centre is inside by the crossings of the edges whose y range [min, max) holds
  its row, counted when the centre is strictly left of the upward edge (orient2d > 0); even-odd
  for shapes, nonzero winding with oriented weights for geometry exclusions;
* raster buffers: ``scipy.ndimage.distance_transform_cdt(taxicab) <= k``;
* raster sampling: integer pixel lookup, with the shape's mask on raster-pixel centres;
* geometry buffers: exact (rational) distances from centres to segments; only where the kernel's
  float ``seg_dist2`` is not exact, a pixel whose distance lies within 1e-12 b of b is excused;
* counts: ``np.bincount`` of exact cell indices.

The GPU cases reach the kernels' rare branches: dilation halos longer than a 64-row chunk and
taller than the window, a window taller than the 65 535-row launch grid, count tiles that span
more cells than the shared histogram, tiles binned thousands of segments, every kind of exact
tie in the polygon mask, rows of more than 1000 crossings, and bands thinner than their halo.
On the CPU, the references are checked against ``oracle/availability_oracle.py`` on small cases,
and a branch table recomputes each case's deciding quantity with the kernels' constants.
"""

import ctypes as C
from fractions import Fraction
from types import SimpleNamespace as NS

import numpy as np
import pytest
import scipy.ndimage as ndi
from scipy.spatial import cKDTree

import availability_oracle as AO
import atlite_b200 as ab
from atlite_b200 import _lib, availability, gis
from atlite_b200 import synthetic as syn

# csrc/availability.cu, restated
K_CHUNK, COUNT_TILE, HIST, GRID_Y = 64, 64, 8, 65535
TILE = _lib.AVAIL_TILE
TIE = Fraction(1, 10 ** 12)  # geometry buffers: |distance - b| <= TIE * b may be decided either way


# ---------------------------------------------------------------- dyadic frames
class Frame:
    """A container CRS and ``res``; geometry is given in integer units of res / 8 from ``origin``
    (a pixel corner, in the same units)."""

    def __init__(self, crs, res, origin=(0, 0)):
        self.crs, self.res, self.unit = crs, float(res), float(res) / 8
        self.origin = np.asarray(origin, dtype=np.int64)
        assert (self.origin % 8 == 0).all()

    def xy(self, a):
        return (np.asarray(a, dtype=np.int64) + self.origin) * self.unit

    def transform(self, ra, ru0, rv0):
        """North-up transform of a raster with pixels of ``ra`` units and top-left corner (ru0, rv0)."""
        return (ra * self.unit, 0.0, float((self.origin[0] + ru0) * self.unit), 0.0, -ra * self.unit,
                float((self.origin[1] + rv0) * self.unit))


F128 = Frame(3035, 128.0, (250000, 187496))  # (4 000 000, 2 999 936) m
F16 = Frame(3035, 16.0, (2000000, 1499968))
F4 = Frame(4326, 2.0 ** -4)
F7 = Frame(4326, 2.0 ** -7)


class Win:
    """Pixel window: left / top pixel edges L, T (in pixels from the origin), nx, ny; centre of
    (i, j) at (cu0 + 8 i, cv0 - 8 j) units."""

    def __init__(self, L, T, nx, ny):
        self.L, self.T, self.nx, self.ny = L, T, nx, ny
        self.cu0, self.cv0 = 8 * L + 4, 8 * T - 4


def window_of(polys):
    """The padded window of the shape's bounds (gis.py:186-194 on the lattice)."""
    v = np.concatenate([r for p in polys for r in p])
    L, R = int(v[:, 0].min()) // 8, int(v[:, 0].max()) // 8 + 1
    B, T = int(v[:, 1].min()) // 8, int(v[:, 1].max()) // 8 + 1
    return Win(L, T, R - L, T - B)


def bounds_of(polys):
    v = np.concatenate([r for p in polys for r in p])
    return int(v[:, 0].min()), int(v[:, 1].min()), int(v[:, 0].max()), int(v[:, 1].max())


def inset_box(nx, ny, u0=0, v0=0):
    """A box whose window is exactly nx x ny pixels from pixel corner (u0, v0), every centre inside."""
    return [[np.array([[u0 + 2, v0 + 2], [u0 + 8 * nx - 2, v0 + 2], [u0 + 8 * nx - 2, v0 + 8 * ny - 2],
                       [u0 + 2, v0 + 8 * ny - 2]], dtype=np.int64)]]


# ---------------------------------------------------------------- exact references
def edges_of(polys, orient=False):
    """(n, 4) int64 ring edges (closing edges included) and weights: 1, or with ``orient`` +1 for a
    counter-clockwise exterior or clockwise hole and -1 otherwise."""
    e, w = [], []
    for poly in polys:
        for k, r in enumerate(poly):
            r = np.asarray(r, dtype=np.int64)
            nxt = np.roll(r, -1, axis=0)
            e.append(np.c_[r, nxt])
            s = 1
            if orient:
                area2 = int((r[:, 0] * nxt[:, 1] - nxt[:, 0] * r[:, 1]).sum())
                s = 1 if (area2 > 0) != (k > 0) else -1
            w.append(np.full(len(r), s, dtype=np.int64))
    if not e:
        return np.zeros((0, 4), np.int64), np.zeros(0, np.int64)
    return np.concatenate(e), np.concatenate(w)


def crossings(edges, cu0, cv0, step, nx, ny):
    """Every (edge, row) pair whose row centre lies in [min v, max v) of the edge: edge index, row,
    the number of centres strictly left of the upward edge, K and D (orient2d at centre u of the
    row is K - u D, in units relative to the first centre) and the edge's direction."""
    e = np.asarray(edges, dtype=np.int64)
    up = e[:, 3] > e[:, 1]
    au, av = np.where(up, e[:, 0], e[:, 2]) - cu0, np.where(up, e[:, 1], e[:, 3]) - cv0
    bu, bv = np.where(up, e[:, 2], e[:, 0]) - cu0, np.where(up, e[:, 3], e[:, 1]) - cv0
    # row j's centre is at v = -step j: av <= -step j < bv
    j0 = np.maximum(-bv // step + 1, 0)
    j1 = np.minimum(-av // step, ny - 1)
    n = np.maximum(j1 - j0 + 1, 0)
    idx = np.repeat(np.arange(len(e)), n)
    j = j0[idx] + np.arange(int(n.sum())) - np.repeat(np.cumsum(n) - n, n)
    cv = -step * j
    D = (bv - av)[idx]
    K = au[idx] * (bv[idx] - cv) - bu[idx] * (av[idx] - cv)
    i = np.clip(-(-K // (step * D)), 0, nx)  # #{i >= 0 : step i D < K}
    return idx, j, i, K, D, up[idx]


def mask_of(edges, w, cu0, cv0, step, nx, ny, nonzero=False):
    """bool (ny, nx): even-odd (or nonzero winding) over the edges, centre (i, j) at
    (cu0 + step i, cv0 - step j)."""
    acc = np.zeros(ny * (nx + 1), dtype=np.int64)
    if len(edges):
        idx, j, i, _, _, up = crossings(edges, cu0, cv0, step, nx, ny)
        wt = np.where(up, w[idx], -w[idx])
        acc = np.rint(np.bincount(j * (nx + 1) + i, weights=wt, minlength=ny * (nx + 1))).astype(np.int64)
    s = np.cumsum(acc.reshape(ny, nx + 1)[:, ::-1], axis=1)[:, ::-1][:, 1:]  # pixel p: edges with i > p
    return (s != 0) if nonzero else (s % 2 == 1)


def dilate(m, k):
    """Pixels within L1 distance k of a set pixel (k dilations with the 4-connected cross)."""
    if k == 0 or not m.any():
        return m.copy()
    return ndi.distance_transform_cdt(~m, metric="taxicab") <= k


def rule(codes, values):
    """ExclusionContainer.add_raster's ``codes`` rule."""
    if callable(codes):
        return np.asarray(codes(values)).astype(bool)
    if codes is not None and np.size(codes) > 0 and (np.ndim(codes) > 0 or bool(codes)):
        return np.isin(values, codes)
    return values.astype(bool)


def raster_excl(win, polys, r):
    """Exclusion of one raster on the window: the pixel under each centre, the shape's mask on
    raster-pixel centres, the nodata rule elsewhere, ``invert``, then the dilation by k."""
    arr = np.asarray(r["array"])
    if arr.dtype == bool:
        arr = arr.astype(np.uint8)
    rny, rnx = arr.shape
    RA, RU, RV = r["ra"], r["ru0"], r["rv0"]
    keep = np.zeros((rny, rnx), dtype=bool)
    bu0, bv0, bu1, bv1 = bounds_of(polys)
    if bu0 < RU + rnx * RA and bu1 > RU and bv0 < RV and bv1 > RV - rny * RA:
        i0, i1 = max((bu0 - RU) // RA, 0), min((bu1 - RU) // RA + 1, rnx)
        j0, j1 = max((RV - bv1) // RA, 0), min((RV - bv0) // RA + 1, rny)
        if i1 > i0 and j1 > j0:
            e, w = edges_of(polys)
            keep[j0:j1, i0:i1] = mask_of(e, w, RU + RA * i0 + RA // 2, RV - RA * j0 - RA // 2, RA, i1 - i0, j1 - j0)
    col = (win.cu0 + 8 * np.arange(win.nx) - RU) // RA
    row = (RV - (win.cv0 - 8 * np.arange(win.ny))) // RA
    cin, rin = (col >= 0) & (col < rnx), (row >= 0) & (row < rny)
    cc, rr = np.where(cin, col, 0), np.where(rin, row, 0)
    ok = rin[:, None] & cin[None, :] & keep[rr[:, None], cc[None, :]]
    ex = np.where(ok, rule(r["codes"], arr)[rr[:, None], cc[None, :]],
                  rule(r["codes"], np.asarray([r["nodata"]]).astype(arr.dtype))[0])
    if r["invert"]:
        ex = ~ex
    return dilate(ex, r["k"])


def segments_of(g):
    """The segments a geometry buffer measures: ring edges, line pieces, points (int64 units)."""
    s = [edges_of(g["polys"])[0]] + [np.c_[a[:-1], a[1:]] for a in g["lines"]]
    s.append(np.c_[g["points"], g["points"]])
    return np.concatenate([np.asarray(x, dtype=np.int64).reshape(-1, 4) for x in s])


def exact_d2(px, py, s):
    """Squared distance from the point to the segment, exact (a Fraction)."""
    x1, y1, x2, y2 = (int(v) for v in s)
    dx, dy, ax, ay = x2 - x1, y2 - y1, px - x1, py - y1
    l2, dot = dx * dx + dy * dy, ax * dx + ay * dy
    if l2 == 0 or dot <= 0:
        return Fraction(ax * ax + ay * ay)
    if dot >= l2:
        return Fraction((px - x2) ** 2 + (py - y2) ** 2)
    cr = ax * dy - ay * dx
    return Fraction(cr * cr, l2)


def near_of(segs, win, B):
    """(near, tie, exact_tie): centres within B (units) of a segment, decided exactly; ``tie``:
    the distance lies within TIE * B of B, ``exact_tie``: it is B.  A KD-tree of points every half
    pixel along the segments bounds the distance d by the nearest sample's ds (d <= ds and
    ds^2 <= d^2 + 2^2); only the centres that bound leaves undecided are computed exactly."""
    segs = np.asarray(segs, dtype=np.int64) - [win.cu0, win.cv0, win.cu0, win.cv0]
    length = np.hypot(segs[:, 2] - segs[:, 0], segs[:, 3] - segs[:, 1])
    m = np.ceil(length / 4).astype(np.int64) + 1
    owner = np.repeat(np.arange(len(segs)), m)
    t = (np.arange(int(m.sum())) - np.repeat(np.cumsum(m) - m, m)) / np.maximum(np.repeat(m, m) - 1, 1)
    sx = segs[owner, 0] + t * (segs[owner, 2] - segs[owner, 0])
    sy = segs[owner, 1] + t * (segs[owner, 3] - segs[owner, 1])
    tree = cKDTree(np.c_[sx, sy])
    gx, gy = np.meshgrid(8.0 * np.arange(win.nx), -8.0 * np.arange(win.ny))
    ds, _ = tree.query(np.c_[gx.ravel(), gy.ravel()], distance_upper_bound=B + 8)
    near = ds <= B * (1 - 1e-9)
    unsure = np.flatnonzero((ds > B * (1 - 1e-9)) & (ds <= np.sqrt(B * B + 4.0) * (1 + 1e-9)))
    tie, exact = np.zeros_like(near), np.zeros_like(near)
    B2, lo, hi = Fraction(B * B), Fraction(B * B) * (1 - TIE) ** 2, Fraction(B * B) * (1 + TIE) ** 2
    for p in unsure:
        px, py = 8 * int(p % win.nx), -8 * int(p // win.nx)
        cand = np.unique(owner[tree.query_ball_point((px, py), ds[p] + 4.0)])
        d2 = min(exact_d2(px, py, segs[c]) for c in cand)
        near[p], tie[p], exact[p] = d2 <= B2, lo <= d2 <= hi, d2 == B2
    shape = (win.ny, win.nx)
    return near.reshape(shape), tie.reshape(shape), exact.reshape(shape)


def geometry_excl(win, g):
    """(excluded, tie, exact_tie) of one geometry collection."""
    e, w = edges_of(g["polys"], orient=True)
    inside = mask_of(e, w, win.cu0, win.cv0, 8, win.nx, win.ny, nonzero=True)
    z = np.zeros_like(inside)
    B = g["buffer"]
    if B == 0:
        ex, tie, exact = inside, z, z
    else:
        near, tie, exact = near_of(segments_of(g), win, abs(B))
        ex = (inside | near) if B > 0 else (inside & ~near)
    return (~ex if g["invert"] else ex), tie, exact


def reference(case):
    """(eligible, window, tie, exact_tie) of the case's shape."""
    win = window_of(case.shape)
    e, w = edges_of(case.shape)
    excl = ~mask_of(e, w, win.cu0, win.cv0, 8, win.nx, win.ny)
    tie, exact = np.zeros_like(excl), np.zeros_like(excl)
    for r in case.rasters:
        excl |= raster_excl(win, case.shape, r)
    for g in case.geoms:
        ex, t, x = geometry_excl(win, g)
        excl |= ex
        tie |= t
        exact |= x
    return ~excl, win, tie, exact


def counts_of(eligible, win, grid):
    """(gny, gnx) eligible centres per cutout cell; grid = (gx0, gdx, gy0, gdy, gnx, gny) in units."""
    gx0, gdx, gy0, gdy, gnx, gny = grid
    ix = (win.cu0 + 8 * np.arange(win.nx) - gx0) // gdx
    iy = (win.cv0 - 8 * np.arange(win.ny) - gy0) // gdy
    IX, IY = np.broadcast_to(ix[None, :], eligible.shape), np.broadcast_to(iy[:, None], eligible.shape)
    ok = eligible & (IX >= 0) & (IX < gnx) & (IY >= 0) & (IY < gny)
    return np.bincount((IY[ok] * gnx + IX[ok]), minlength=gny * gnx).reshape(gny, gnx).astype(np.int64)


# ---------------------------------------------------------------- the API
def poly_json(frame, poly):
    return {"type": "Polygon", "coordinates": [frame.xy(r).tolist() for r in poly]}


def shape_json(frame, polys):
    return {"type": "MultiPolygon", "coordinates": [[frame.xy(r).tolist() for r in p] for p in polys]}


def container(case):
    f = case.frame
    ex = gis.ExclusionContainer(f.crs, f.res)
    for r in case.rasters:
        ras = gis.Raster(r["array"], f.transform(r["ra"], r["ru0"], r["rv0"]), f.crs)
        ex.add_raster(ras, codes=r["codes"], buffer=float((8 * (r["k"] - 1) + 4) * f.unit) if r["k"] else 0,
                      invert=r["invert"], nodata=r["nodata"])
    for g in case.geoms:
        parts = [poly_json(f, p) for p in g["polys"]] + [
            {"type": "LineString", "coordinates": f.xy(a).tolist()} for a in g["lines"]]
        if len(g["points"]):
            parts.append({"type": "MultiPoint", "coordinates": f.xy(g["points"]).tolist()})
        ex.add_geometry(parts, buffer=float(g["buffer"] * f.unit), invert=g["invert"])
    return ex


def run_shape(case):
    """(eligible, transform) from gis.shape_availability."""
    return gis.shape_availability(shape_json(case.frame, case.shape), container(case))


def check_shape(case, pinned=False):
    """Run the case and compare with the reference: bit for bit, except (unless ``pinned``) the
    geometry-buffer pixels within TIE * b of b.  Returns (excused pixels, window size)."""
    got, t = run_shape(case)
    want, win, tie, exact = reference(case)
    f = case.frame
    assert tuple(t)[:6] == (f.res, 0, float((f.origin[0] + 8 * win.L) * f.unit), 0, -f.res,
                            float((f.origin[1] + 8 * win.T) * f.unit))
    assert got.shape == want.shape == (win.ny, win.nx)
    assert 0 < want.sum() < want.size
    bad = got != want
    if not pinned:
        bad &= ~tie
    assert not bad.any(), (f"{case.name}: {int(bad.sum())} of {bad.size} pixels differ, first at "
                           f"{np.argwhere(bad)[0]}, {int(tie.sum())} near-tie pixels")
    return int((tie & (got != want)).sum()), int(tie.sum()), int(exact.sum()), got.size


def raster(arr, ra, ru0, rv0, codes=None, k=0, invert=False, nodata=255):
    return dict(array=arr, ra=ra, ru0=ru0, rv0=rv0, codes=codes, k=k, invert=invert, nodata=nodata)


def geometry(polys=(), lines=(), points=(), buffer=0, invert=False):
    return dict(polys=[[np.asarray(r, dtype=np.int64) for r in p] for p in polys],
                lines=[np.asarray(a, dtype=np.int64) for a in lines],
                points=np.asarray(points, dtype=np.int64).reshape(-1, 2), buffer=buffer, invert=invert)


def case(name, frame, shape, rasters=(), geoms=(), **kw):
    return NS(name=name, frame=frame, shape=[[np.asarray(r, dtype=np.int64) for r in p] for p in shape],
              rasters=list(rasters), geoms=list(geoms), **kw)


# ---------------------------------------------------------------- cases: polygon mask
def random_rings(rng, nx, ny, n_rings, n_vert):
    """Rings with vertices on quarter-pixel columns and half-pixel rows (one in eight on a centre),
    spanning the window [0, nx) x [0, ny) exactly: ties of every kind."""
    rings = []
    for k in range(n_rings):
        u = 2 * rng.integers(0, 4 * nx, n_vert)
        v = 4 * rng.integers(0, 2 * ny, n_vert)
        if k == 0:
            u[:2], v[:2] = (0, 8 * nx - 2), (0, 8 * ny - 4)
        rings.append(np.c_[u, v])
    return [[r] for r in rings]


def mask_width_case(nx):
    return case(f"mask_nx{nx}", F128, random_rings(np.random.default_rng(nx), nx, 24, 6, 11), branch="nx",
                nx=nx)


def staircase(u, v):
    """Step-shaped boundary: vertical edges meeting horizontal ones on centre rows (v = 8 m + 4)."""
    return [np.array([[0, 0], [40, 0], [40, 20], [60, 20], [60, 44], [84, 44], [84, 68], [0, 68]]) + [u, v]]


def ties_case():
    """One of every exact tie, each in its own part of the window (even-odd over all parts)."""
    parts = [
        staircase(0, 0),  # horizontal edges on centre rows between vertical steps
        [np.array([[0, 0], [-20, 20], [4, 44], [28, 20]]) + [140, 4]],  # a diamond with vertices on centres
        [np.array([[0, -4], [64, 60], [-24, 60]]) + [204, 8]],  # edges through centres (slopes 1 and -1)
        [np.array([[0, 0], [32, 0], [32, 64], [0, 64]]) + [300, 0],  # a hole sharing a vertex with its exterior
         np.array([[0, 0], [12, 28], [24, 12]]) + [300, 0]],
        [np.array([[0, 0], [20, 0], [20, 4], [20, 36], [20, 68], [0, 68]]) + [352, 0]],  # collinear edges meeting
        [np.array([[20, 0], [44, 0], [44, 68], [20, 68]]) + [352, 0]],  # a part touching it along a centre column
        [np.array([[0, 4], [36, 4], [36, 36], [0, 36]]) + [420, 0],  # parts touching along a centre row
         ],
        [np.array([[0, 36], [36, 36], [36, 68], [0, 68]]) + [420, 0]],
        [np.array([[0, 0], [4, 0], [4, 68], [0, 68]]) + [476, 0]],  # a sliver whose right edge is a centre column
    ]
    return case("mask_ties", F128, parts, branch="ties")


def steep_flat_case():
    """Steep and flat edges whose exact crossing of a centre row is the centre itself or 1 / D
    units from it (D: the edge's height), so the float estimate sits on the boundary of ceil."""
    polys, x = [], 4
    for E, D in ((5, 1003), (3, 997), (-7, 1021), (997, 3), (1021, 5), (-1003, 7), (61, 3), (3, 61)):
        for delta in (-1, 0, 1):
            cu, cv = x + 8 * (abs(E) // 4 + 4), 4 + 8 * (D // 4 + 4)
            # a = (au, cv - t) with (cv - av) E / D = cu - au + delta / D  <=>  t E = delta (mod D)
            t = (delta * pow(E % D, -1, D)) % D if delta else D
            au = cu + (delta - t * E) // D
            assert (delta - t * E) % D == 0
            a = np.array([au, cv - t])
            b = a + (1 if delta else 2) * np.array([E, D])  # D: the edge's height when delta != 0
            W = 8 * 3 + 3
            polys.append([np.array([a, b, b + [W, 0], a + [W, 0]])])
            x += 8 * (2 * abs(E) // 8 + 10)
    return case("mask_steep_flat", F128, polys, branch="steep_flat")


def sawtooth_case():
    """A 12 000-pixel row crossed by a 2000-edge sawtooth: more than 1000 crossings per row."""
    k = np.arange(2001)
    top = np.c_[48 * k, 8 * 10 + np.where(k % 2 == 1, 8 * 40 + 4 * (k % 3 == 0), 4 * (k % 5 == 0))]
    top[-1, 0] = 8 * 12000 - 4
    ring = np.r_[[[0, 0]], top, [[8 * 12000 - 4, 0]]]
    return case("mask_sawtooth", F128, [[ring]], branch="crossings")


def mask_cases():
    return [mask_width_case(n) for n in (1, 31, 32, 33)] + [ties_case(), steep_flat_case(), sawtooth_case()]


def winding_case(invert):
    """Geometry exclusions by nonzero winding: opposite orientations overlapping, a polygon nested
    in another's hole, and a polygon reaching past the window's right edge."""
    ccw = np.array([[40, 40], [400, 40], [400, 300], [40, 300]])
    cw = np.array([[200, 100], [200, 500], [600, 500], [600, 100]])  # clockwise, overlapping ccw
    outer = [np.array([[700, 40], [1200, 40], [1200, 500], [700, 500]]),
             np.array([[780, 100], [780, 444], [1100, 444], [1100, 100]])]  # its hole, clockwise
    nested = np.array([[850, 150], [1000, 150], [1000, 380], [850, 380]])
    past = np.array([[1300, 4], [3000, 4], [3000, 600], [1300, 604]])
    g = geometry(polys=[[ccw], [cw], outer, [nested], [past]], invert=invert)
    return case(f"geom_winding_{'invert' if invert else 'plain'}", F128, inset_box(180, 80), geoms=[g],
                branch="winding")


# ---------------------------------------------------------------- cases: dilation and raster sampling
DILATE_K = (1, 9, 63, 64, 65, 79, 157)


def dilation_raster(nx, ny, seed):
    """Sparse set pixels: random ones, the four window corners, pixels on chunk borders (rows
    64 m - 1 and 64 m); most rows hold none."""
    rng = np.random.default_rng(seed)
    a = np.zeros((ny, nx), dtype=np.uint8)
    a[rng.integers(0, ny, 40), rng.integers(0, nx, 40)] = 7
    a[[0, 0, ny - 1, ny - 1], [0, nx - 1, 0, nx - 1]] = 1
    for m, c in ((1, 500), (6, 1700), (17, 2700), (30, 100)):
        a[64 * m - 1, c] = a[64 * m, c + 700] = 3
    return a


def dilation_case(ny, nx=3500):
    arr = dilation_raster(nx, ny, ny)
    return case(f"dilate_ny{ny}", F128, inset_box(nx, ny), rasters=[raster(arr, 8, 0, 8 * ny, nodata=0)],
                branch="dilate", ks=DILATE_K)


def thin_case(ny, ks):
    arr = np.zeros((ny, 300), dtype=np.uint8)
    arr[ny // 2, 5] = arr[ny - 1, 290] = 1
    return case(f"dilate_thin_ny{ny}", F128, inset_box(300, ny), rasters=[raster(arr, 8, 0, 8 * ny, nodata=0)],
                branch="thin", ks=ks)


CONCAVE = [np.array([[6, 4], [2400, 90], [1500, 1300], [2700, 2300], [60, 2200], [900, 1000]]),
           np.array([[300, 300], [420, 650], [700, 310]])]


def raster_kind_case(kind):
    """A raster of each index kind at 2 res, offset half a container pixel (container centres on
    raster pixel edges), larger than the shape (mask_i0, mask_j0 > 0) or smaller (nodata rule);
    each raster applied with a buffer (dilated scratch) and without (or_into)."""
    rng = np.random.default_rng(("uint8", "int16", "float32", "bool").index(kind))
    win = window_of([CONCAVE])
    if kind in ("uint8", "int16"):  # larger than the shape's box
        ny, nx = (8 * win.ny) // 16 + 20, (8 * win.nx) // 16 + 20
        ru0, rv0 = 8 * win.L + 4 - 16 * 10, 8 * win.T + 4 + 16 * 10
    else:  # smaller: covers the middle of the window only
        ny, nx = (8 * win.ny) // 16 - 40, (8 * win.nx) // 16 - 50
        ru0, rv0 = 8 * win.L + 4 + 16 * 30, 8 * win.T + 4 - 16 * 25
    if kind == "uint8":
        arr = rng.integers(0, 40, (ny, nx)).astype(np.uint8)
        arr[rng.random(arr.shape) < 0.05] = 255
        rs = [raster(arr, 16, ru0, rv0, codes=[7, 255], k=2),
              raster(arr, 16, ru0, rv0, codes=lambda v: v % 11 != 0, invert=True, nodata=0)]
    elif kind == "int16":
        arr = rng.integers(-32768, 32768, (ny, nx)).astype(np.int16)
        arr[::97, ::89] = np.int16(-32768)
        arr[5::101, 3::83] = np.int16(32767)
        rs = [raster(arr, 16, ru0, rv0, codes=lambda v: (v > 32700) | (v == -32768), k=9, nodata=-32768),
              raster(arr, 16, ru0, rv0, codes=lambda v: v < 31000, invert=True, nodata=32767)]
    elif kind == "float32":
        arr = rng.normal(-40, 30, (ny, nx)).astype(np.float32)
        arr[rng.random(arr.shape) < 0.03] = np.nan
        rs = [raster(arr, 16, ru0, rv0, codes=lambda d: d < -95, k=5, nodata=np.nan),
              raster(arr, 16, ru0, rv0, codes=lambda d: np.isnan(d) | (d > 40), nodata=np.nan)]
    else:
        arr = rng.random((ny, nx)) < 0.01
        rs = [raster(arr, 16, ru0, rv0, k=2), raster(~arr, 16, ru0, rv0, invert=True, nodata=0)]
    return case(f"raster_{kind}", F128, [CONCAVE], rasters=rs, branch="raster")


def tall_case():
    """70 x 68 750 pixels at 16 m: two launch slabs of raster sampling, 1075 dilation chunks."""
    nx, ny = 70, 68750
    rng = np.random.default_rng(11)
    shape = [[np.array([[2, 2], [8 * nx - 2, 2], [8 * nx - 2, 8 * ny - 2], [300, 8 * ny - 2], [2, 8 * ny - 600]])]]
    rny, rnx = ny // 2 - 3, nx // 2 + 2
    arr = (rng.random((rny, rnx)) < 0.002).astype(np.uint8)
    arr[-40:] = rng.integers(0, 3, (40, rnx))
    rs = [raster(arr, 16, -12, 8 * ny + 4, k=3, nodata=0), raster(arr, 16, -12, 8 * ny + 4, codes=[2], nodata=2)]
    return case("raster_tall", F16, shape, rasters=rs, branch="tall")


# ---------------------------------------------------------------- cases: geometry buffers
def coastline(n, box, seed):
    """A random walk of n segments (steps of 4 .. 24 units) inside ``box`` = (u0, v0, u1, v1)."""
    rng = np.random.default_rng(seed)
    u0, v0, u1, v1 = box
    p = np.empty((n + 1, 2), dtype=np.int64)
    p[0] = ((u0 + u1) // 2, (v0 + v1) // 2)
    h = 0.0
    for k in range(n):
        h += rng.normal(0, 0.5)
        s = rng.integers(4, 25)
        q = p[k] + np.rint([s * np.cos(h), s * np.sin(h)]).astype(np.int64)
        if not (u0 <= q[0] <= u1 and v0 <= q[1] <= v1):
            h += np.pi
            q = p[k] - (q - p[k])
        p[k + 1] = q
    return p


def polyline_case(buffer_m):
    nx, ny = 1003, 907
    line = coastline(20000, (8 * 300, 8 * 250, 8 * 700, 8 * 650), 3)
    g = geometry(lines=[line], buffer=buffer_m // 16)
    return case(f"geom_polyline_{buffer_m // 1000}km", F128, inset_box(nx, ny), geoms=[g], branch="polyline",
                buffer_m=buffer_m)


def negative_case():
    """A negative buffer on a generic polygon, and a line along a (3, 4) direction whose buffer
    (201 units) no centre's distance equals, where distances are 1.6 n units."""
    poly = [np.array([[40, 36], [1500, 100], [1300, 1203], [500, 900], [77, 1161]]),
            np.array([[300, 300], [700, 300], [700, 700], [300, 700]])]
    g1 = geometry(polys=[poly], buffer=-300)
    g2 = geometry(lines=[np.array([[100, 1300], [100 + 3 * 64, 1300 + 4 * 64]])], buffer=201)
    return case("geom_negative", F128, inset_box(203, 197), geoms=[g1, g2], branch="geometry")


def pinned_case(invert):
    """Ties where seg_dist2 is exact: points on centres with (3, 4) / (5, 0) offsets at b = 5
    pixels, zero-length segments, ends of axis-aligned segments (projection clamped), interiors of
    axis-aligned segments of power-of-two length, and a negative buffer on a square."""
    B = 40  # 5 pixels
    pts = np.array([[8 * 20 + 4, 8 * 20 + 4], [8 * 60 + 4, 8 * 30 + 4], [8 * 33 + 1, 8 * 70 + 3]])
    lines = [np.array([[8 * 100 + 4, 8 * 20 + 4], [8 * 100 + 4, 8 * 20 + 4]]),  # zero length
             np.array([[8 * 120 + 4, 8 * 60 + 4], [8 * 128 + 4, 8 * 60 + 4], [8 * 128 + 4, 8 * 76 + 4],
                       [8 * 128 + 4, 8 * 76 + 4]]),  # 8 and 16 pixels, then a repeated vertex
             np.array([[8 * 20 + 4, 8 * 100 + 4], [8 * 52 + 4, 8 * 100 + 4]])]
    square = [np.array([[8 * 150, 8 * 10], [8 * 150 + 256, 8 * 10], [8 * 150 + 256, 8 * 10 + 256],
                        [8 * 150, 8 * 10 + 256]])]
    g = geometry(lines=lines, points=pts, buffer=B, invert=invert)
    neg = geometry(polys=[square], buffer=-28)
    return case(f"geom_pinned_{'invert' if invert else 'plain'}", F128, inset_box(189, 121), geoms=[g, neg],
                branch="pinned")


# ---------------------------------------------------------------- cases: counts and bands
def count_case(frame, name, seed):
    """A 4326 container on a dyadic 0.25 degree cutout of 40 x 32 cells ([-4, 6] x [48, 56]); the
    shape reaches past the cutout's east and south edges."""
    per_deg = int(round(1 / frame.unit))
    c = lambda lon, lat: [int(round(lon * per_deg)), int(round(lat * per_deg))]  # noqa: E731
    if frame is F4:
        ext = [c(-3.5, 47.0), c(7.5, 47.5), c(6.5, 55.75), c(1.0, 53.0), c(-3.0, 55.5)]
        hole = [c(0.0, 50.0), c(2.0, 50.25), c(1.0, 52.0)]
    else:
        ext = [c(3.25, 47.75), c(6.25, 48.5), c(5.5, 50.75), c(4.0, 49.75), c(3.5, 50.5)]
        hole = [c(4.5, 49.0), c(5.0, 49.125), c(4.75, 49.5)]
    shape = [[np.array(ext), np.array(hole)]]
    win = window_of(shape)
    rng = np.random.default_rng(seed)
    arr = rng.integers(0, 9, (win.ny + 6, win.nx + 4)).astype(np.uint8)
    r = raster(arr, 8, 8 * win.L - 16, 8 * win.T + 24, codes=[0], nodata=1)
    grid = (-4 * per_deg, per_deg // 4, 48 * per_deg, per_deg // 4, 40, 32)
    return case(name, frame, shape, rasters=[r], branch="count", grid=grid)


def count_cases():
    return [count_case(F4, "count_global", 1), count_case(F7, "count_hist", 2)]


def band_case(rows):
    """Bands of ``rows`` rows with a raster buffer of k = 79 and a geometry buffer crossing band
    borders."""
    nx, ny = 240, 300
    rng = np.random.default_rng(rows)
    arr = np.zeros((ny, nx), dtype=np.uint8)
    arr[rng.integers(0, ny, 2), rng.integers(0, nx, 2)] = 1
    line = np.array([[8 * 10 + 3, 8 * 20 + 1], [8 * 200 + 5, 8 * 150 + 2], [8 * 60 + 1, 8 * 290 + 7]])
    g = geometry(lines=[line], points=[[8 * 230 + 4, 8 * 40 + 4]], buffer=8 * 12 + 3)
    shape = [[np.array([[2, 2], [8 * nx - 2, 2], [8 * nx - 2, 8 * ny - 2], [1000, 8 * ny - 2], [2, 900]])]]
    return case(f"bands_rows{rows}", F128, shape, rasters=[raster(arr, 8, 0, 8 * ny, k=79, nodata=0)], geoms=[g],
                branch="bands", rows=rows)


BAND_ROWS = (1, 40, 100)


def band_bytes(nx, rows, halo):
    """A device budget for which _Session._band_rows gives ``rows`` rows per band."""
    return availability._Session.PIXEL_BYTES * nx * (rows + 2 * halo)


# ---------------------------------------------------------------- CPU: references against the oracle
def _oracle_lattice(frame, win):
    return (float((frame.origin[0] + 8 * win.L) * frame.unit), frame.res,
            float((frame.origin[1] + 8 * win.T) * frame.unit), -frame.res)


@pytest.mark.parametrize("c", [mask_width_case(31), mask_width_case(1), ties_case(), winding_case(False)],
                         ids=lambda c: c.name)
def test_reference_mask_is_oracles(c):
    """Even-odd (shapes) and nonzero (geometry) masks equal the oracle's exact-orient2d masks."""
    polys = c.geoms[0]["polys"] if c.geoms else c.shape
    win = window_of(c.shape)
    nonzero = bool(c.geoms)
    e, w = edges_of(polys, orient=nonzero)
    want = mask_of(e, w, win.cu0, win.cv0, 8, win.nx, win.ny, nonzero=nonzero)
    left, a, top, ee = _oracle_lattice(c.frame, win)
    ef = np.c_[c.frame.xy(e[:, :2]), c.frame.xy(e[:, 2:])]
    got = AO.polygon_mask(ef, w, left, a, top, ee, win.nx, win.ny, nonzero=nonzero)
    assert np.array_equal(got, want)
    assert 0 < want.sum() < want.size


@pytest.mark.parametrize("k", [1, 9, 65])
def test_reference_dilation_is_oracles(k):
    m = np.zeros((150, 90), dtype=bool)
    m[[0, 64, 149, 77], [0, 45, 89, 3]] = True
    assert np.array_equal(dilate(m, k), AO.dilate(m, k))
    assert not dilate(np.zeros((5, 5), bool), k).any()


def test_reference_raster_is_oracles():
    c = raster_kind_case("uint8")
    win = window_of(c.shape)
    rings = [(c.frame.xy(r), k > 0) for k, r in enumerate(c.shape[0])]
    for r in c.rasters:
        o = dict(array=r["array"], transform=c.frame.transform(r["ra"], r["ru0"], r["rv0"]), epsg=3035)
        L = _oracle_lattice(c.frame, win)
        ex, tie = AO.raster_exclusion(rings, 3035, (L[0], L[2], win.nx, win.ny, c.frame.res), o, codes=r["codes"],
                                      buffer=(8 * (r["k"] - 1) + 4) * c.frame.unit if r["k"] else 0,
                                      invert=r["invert"], nodata=r["nodata"], res=c.frame.res)
        assert not tie.any()
        assert np.array_equal(ex, raster_excl(win, c.shape, r))


def test_reference_geometry_is_oracles():
    """Exact distances against the oracle's float ones, away from its ties."""
    c = negative_case()
    win = window_of(c.shape)
    L = _oracle_lattice(c.frame, win)
    for g in c.geoms:
        rings = [(c.frame.xy(r), k > 0) for p in g["polys"] for k, r in enumerate(p)]
        ex, tie = AO.geometry_exclusion((L[0], L[2], win.nx, win.ny, c.frame.res), rings,
                                        [c.frame.xy(a) for a in g["lines"]], [], buffer=g["buffer"] * c.frame.unit)
        want, _, _ = geometry_excl(win, g)
        assert not ((ex != want) & ~tie).any()


def test_same_crs_vertices_upload_unchanged():
    """Same-CRS projection is the identity: the edges and segments the kernels get are the input
    vertices, bit for bit."""
    for c in [ties_case(), negative_case(), pinned_case(False), count_cases()[0]]:
        p = availability._parts(shape_json(c.frame, c.shape), c.frame.crs, c.frame.crs, polygonal=True)
        e, _ = edges_of(c.shape)
        assert np.array_equal(p.edges()[0], np.c_[c.frame.xy(e[:, :2]), c.frame.xy(e[:, 2:])])
        for g in c.geoms:
            ex = container(NS(frame=c.frame, rasters=[], geoms=[g]))
            s = availability._parts(ex.geometries[0]["geometry"], c.frame.crs, c.frame.crs, polygonal=False)
            segs = segments_of(g)
            want = np.c_[c.frame.xy(segs[:, :2]), c.frame.xy(segs[:, 2:])]
            got = s.segments()
            assert len(got) == len(want)
            assert np.array_equal(got, want)


# ---------------------------------------------------------------- CPU: the branch table
def k_bin_counts(win, frame, segs, b):
    """Segments per 16 x 16 tile, by k_bin's float arithmetic (box range, then the tile centre
    within |b| + half the tile diagonal + one pixel)."""
    L = NS(c=float((frame.origin[0] + 8 * win.L) * frame.unit), a=frame.res,
           f=float((frame.origin[1] + 8 * win.T) * frame.unit), e=-frame.res)
    s = np.c_[frame.xy(segs[:, :2]), frame.xy(segs[:, 2:])]
    ntx, nty = -(-win.nx // TILE), -(-win.ny // TILE)
    u0 = (np.minimum(s[:, 0], s[:, 2]) - b - L.c) / L.a
    u1 = (np.maximum(s[:, 0], s[:, 2]) + b - L.c) / L.a
    v0 = (np.maximum(s[:, 1], s[:, 3]) + b - L.f) / L.e
    v1 = (np.minimum(s[:, 1], s[:, 3]) - b - L.f) / L.e
    ti0, ti1 = np.maximum(np.floor(u0 / TILE), 0).astype(int), np.minimum(np.floor(u1 / TILE), ntx - 1).astype(int)
    tj0, tj1 = np.maximum(np.floor(v0 / TILE), 0).astype(int), np.minimum(np.floor(v1 / TILE), nty - 1).astype(int)
    nx_, ny_ = np.maximum(ti1 - ti0 + 1, 0), np.maximum(tj1 - tj0 + 1, 0)
    half = 0.5 * TILE * L.a
    reach = b + half * 1.4142135623730951 + L.a
    out = np.zeros(ntx * nty, dtype=np.int64)
    for c0 in range(0, len(s), 1000):
        ids = np.arange(c0, min(c0 + 1000, len(s)))
        n = nx_[ids] * ny_[ids]
        sid = np.repeat(ids, n)
        k = np.arange(int(n.sum())) - np.repeat(np.cumsum(n) - n, n)
        ti, tj = ti0[sid] + k % nx_[sid], tj0[sid] + k // nx_[sid]
        cx, cy = L.c + (ti * TILE) * L.a + half, L.f + (tj * TILE) * L.e - half
        q = s[sid]
        dx, dy = q[:, 2] - q[:, 0], q[:, 3] - q[:, 1]
        l2 = dx * dx + dy * dy
        t = np.where(l2 > 0, ((cx - q[:, 0]) * dx + (cy - q[:, 1]) * dy) / np.where(l2 > 0, l2, 1), 0.0)
        t = np.clip(t, 0, 1)
        d2 = (cx - (q[:, 0] + t * dx)) ** 2 + (cy - (q[:, 1] + t * dy)) ** 2
        keep = d2 <= reach * reach
        out += np.bincount(tj[keep] * ntx + ti[keep], minlength=ntx * nty)
    return out


def k_count_global_share(c, eligible, win):
    """Share of the counted pixels that k_count sends to global atomics (hx or hy outside [0, 8) of
    the histogram around the tile centre's cell)."""
    gx0, gdx, gy0, gdy, gnx, gny = c.grid
    i, j = np.arange(win.nx), np.arange(win.ny)
    ix, iy = (win.cu0 + 8 * i - gx0) // gdx, (win.cv0 - 8 * j - gy0) // gdy
    ci = np.minimum((i // COUNT_TILE) * COUNT_TILE + COUNT_TILE // 2, win.nx - 1)
    cj = np.minimum((j // COUNT_TILE) * COUNT_TILE + COUNT_TILE // 2, win.ny - 1)
    hx = ix - ((win.cu0 + 8 * ci - gx0) // gdx - HIST // 2)
    hy = iy - ((win.cv0 - 8 * cj - gy0) // gdy - HIST // 2)
    ok = eligible & ((ix >= 0) & (ix < gnx))[None, :] & ((iy >= 0) & (iy < gny))[:, None]
    far = ((hx < 0) | (hx >= HIST))[None, :] | ((hy < 0) | (hy >= HIST))[:, None]
    return (ok & far).sum() / ok.sum(), ok.sum()


def tie_kinds(c):
    """Exact ties of the shape's mask: vertices on centres, horizontal edges on centre rows, crossings
    on a centre, crossings within 1 / D unit of one, centre columns on vertical edges."""
    win = window_of(c.shape)
    e, _ = edges_of(c.shape)
    v = np.concatenate([r for p in c.shape for r in p])
    on_centre = int((((v[:, 0] - 4) % 8 == 0) & ((v[:, 1] - 4) % 8 == 0)).sum())
    horiz = int(((e[:, 1] == e[:, 3]) & ((e[:, 1] - 4) % 8 == 0)).sum())
    _, _, _, K, D, _ = crossings(e, win.cu0, win.cv0, 8, win.nx, win.ny)
    r = K % (8 * D)  # orient2d at the centre left of the crossing, in units of D
    hit = int((r == 0).sum())
    near = int(((r == 1) | (r == 8 * D - 1)).sum())  # crossing 1 / D unit right or left of a centre
    vert = int(((e[:, 0] == e[:, 2]) & ((e[:, 0] - 4) % 8 == 0) & (e[:, 1] != e[:, 3])).sum())
    return dict(on_centre=on_centre, horizontal=horiz, hit=hit, near=near, vertical=vert)


def test_branch_table():
    rows = []
    # polygon mask: widths, ties, crossings per row
    for c in mask_cases():
        win = window_of(c.shape)
        e, _ = edges_of(c.shape)
        _, j, _, _, _, _ = crossings(e, win.cu0, win.cv0, 8, win.nx, win.ny)
        per_row = np.bincount(j, minlength=win.ny).max()
        tk = tie_kinds(c)
        rows.append((c.name, f"nx={win.nx} ny={win.ny} max crossings/row={per_row} {tk}"))
        if c.branch == "nx":
            assert win.nx == c.nx and tk["on_centre"] > 0 and tk["hit"] > 0
        elif c.branch == "ties":
            assert all(v > 0 for k, v in tk.items() if k != "near"), tk
        elif c.branch == "steep_flat":
            assert tk["hit"] >= 8 and tk["near"] >= 16, tk
        elif c.branch == "crossings":
            assert win.nx == 12000 and per_row > 1000 and -(-win.nx // 32) > 300
    for c in (winding_case(False),):
        win = window_of(c.shape)
        e, w = edges_of(c.geoms[0]["polys"], orient=True)
        assert sorted(set(w.tolist())) == [-1, 1]
        assert (e[:, [0, 2]].min(axis=1) >= 8 * (win.L + win.nx)).any()  # edges wholly right of the window
        m = mask_of(e, w, win.cu0, win.cv0, 8, win.nx, win.ny, nonzero=True)
        acc = np.zeros((win.ny, win.nx + 1), np.int64)
        idx, j, i, _, _, up = crossings(e, win.cu0, win.cv0, 8, win.nx, win.ny)
        np.add.at(acc, (j, i), np.where(up, w[idx], -w[idx]))
        wind = np.cumsum(acc[:, ::-1], axis=1)[:, ::-1][:, 1:]
        assert (wind == 2).any() and m.any()  # the opposite-orientation overlap winds twice
    # dilation: k against chunks, ny against the chunk size, k >= ny
    for c in [dilation_case(ny) for ny in (3007, 3008, 3009)] + [thin_case(5, (9, 79)), thin_case(1, (1, 64))]:
        win = window_of(c.shape)
        chunks = -(-win.ny // K_CHUNK)
        rows.append((c.name, f"{win.nx} x {win.ny}, {chunks} chunks, ny % 64 = {win.ny % K_CHUNK}, k = {c.ks}"))
        if c.branch == "dilate":
            assert win.nx * win.ny > 1e7 and win.ny % K_CHUNK in (K_CHUNK - 1, 0, 1)
            assert {-(-k // K_CHUNK) for k in c.ks} == {1, 2, 3}  # halos of one, two and three chunks
        else:
            assert max(c.ks) >= win.ny
    # raster sampling: launch slabs and chunks of the tall window; container centres on raster edges
    t = tall_case()
    win = window_of(t.shape)
    slabs = -(-win.ny // GRID_Y)
    rows.append((t.name, f"{win.nx} x {win.ny}, {slabs} slabs, {-(-win.ny // K_CHUNK)} chunks"))
    assert (win.nx, win.ny) == (70, 68750) and slabs == 2 and -(-win.ny // K_CHUNK) == 1075
    for kind in ("uint8", "int16", "float32", "bool"):
        c = raster_kind_case(kind)
        win = window_of(c.shape)
        r = c.rasters[0]
        u = win.cu0 + 8 * np.arange(win.nx) - r["ru0"]
        assert ((u % r["ra"]) == 0).any()  # centres exactly on raster pixel edges
        bu0, bv0, bu1, bv1 = bounds_of(c.shape)
        i0, j0 = (bu0 - r["ru0"]) // r["ra"], (r["rv0"] - bv1) // r["ra"]
        rny, rnx = r["array"].shape
        larger = i0 > 0 and j0 > 0
        smaller = r["ru0"] > 8 * win.L and r["ru0"] + rnx * r["ra"] < 8 * (win.L + win.nx)
        assert larger if kind in ("uint8", "int16") else smaller
        assert {bool(q["k"]) for q in c.rasters} == {True, False}  # dilated scratch and or_into
    # geometry buffers: segments per tile and reach in tiles
    for c in [polyline_case(2000), polyline_case(20000), negative_case(), pinned_case(False)]:
        win = window_of(c.shape)
        g = c.geoms[0]
        b = abs(g["buffer"]) * c.frame.unit
        per_tile = k_bin_counts(win, c.frame, segments_of(g), b)
        reach = b / (TILE * c.frame.res)
        rows.append((c.name, f"{win.nx} x {win.ny}, reach {reach:.2f} tiles, max {per_tile.max()} segments/tile"))
        assert win.nx % TILE and win.ny % TILE
        if c.branch == "polyline":
            assert len(segments_of(g)) == 20000
            assert (0.9 < reach < 1.1) if c.buffer_m == 2000 else (9 < reach < 11)
            assert per_tile.max() > (100 if c.buffer_m == 2000 else 3000)
    # counts: the share of pixels on the global path
    for c in count_cases():
        want, win, _, _ = reference(c)
        share, n = k_count_global_share(c, want, win)
        gx0, gdx, gy0, gdy, gnx, gny = c.grid
        cells = COUNT_TILE * 8 // gdx
        rows.append((c.name, f"{win.nx} x {win.ny}, a tile spans {cells} cells, {share:.3f} of {n} pixels global"))
        assert (share > 0.6) if c.name == "count_global" else (share == 0)
        bu0, bv0, bu1, bv1 = bounds_of(c.shape)
        assert bu1 > gx0 + gnx * gdx and bv0 < gy0  # partly off the cutout
    # bands: rows per band against the halo
    for rows_ in BAND_ROWS:
        c = band_case(rows_)
        win = window_of(c.shape)
        halo = max(r["k"] for r in c.rasters)
        budget = band_bytes(win.nx, rows_, halo)
        assert availability._Session.PIXEL_BYTES * win.nx * win.ny > budget
        got = budget // (availability._Session.PIXEL_BYTES * win.nx) - 2 * halo
        rows.append((c.name, f"{got} rows per band, halo {halo}, {-(-win.ny // got)} bands"))
        assert got == rows_ and (got < halo or rows_ == 100)
    print("\n".join(f"{n:24s} {s}" for n, s in rows))


# ---------------------------------------------------------------- GPU: polygon masks
@pytest.mark.gpu
@pytest.mark.parametrize("c", mask_cases(), ids=lambda c: c.name)
def test_mask(c):
    check_shape(c, pinned=True)


def _abi_mask(frame, edges, w, win, row0, mode):
    """atl_avail_mask on rows row0 .. row0 + ny - 1 of a window cut from larger polygons (every
    edge paired with every row, so the kernel alone decides which rows an edge crosses)."""
    import torch

    from atlite_b200.engine import _dptr, _stream_ptr

    lib = _lib.load()
    L = _lib.Lattice(float((frame.origin[0] + 8 * win.L) * frame.unit), frame.res,
                     float((frame.origin[1] + 8 * win.T) * frame.unit), -frame.res, win.nx, win.ny)
    ef = np.c_[frame.xy(edges[:, :2]), frame.xy(edges[:, 2:])]
    d = lambda a, t: torch.from_numpy(np.ascontiguousarray(a, dtype=t)).cuda()  # noqa: E731
    e_d, w_d = d(ef, np.float64), d(w, np.int32)
    p_d, r_d = d(np.arange(len(ef) + 1) * win.ny, np.int64), d(np.zeros(len(ef)), np.int32)
    cnt = torch.empty((win.ny, win.nx), dtype=torch.int32, device="cuda")
    out = torch.empty((win.ny, win.nx), dtype=torch.uint8, device="cuda")
    _lib.check(lib.atl_avail_mask(torch.cuda.current_device(), C.byref(L), row0, len(ef), _dptr(e_d), _dptr(w_d),
                                  _dptr(p_d), _dptr(r_d), _dptr(cnt), _dptr(out), mode, 0, _stream_ptr()))
    return out.cpu().numpy().astype(bool)


@pytest.mark.gpu
@pytest.mark.parametrize("nx", [1, 31, 32, 33])
@pytest.mark.parametrize("ny", [1, 7, 9, 33, 64])
def test_mask_window_cut_from_polygons(nx, ny):
    """Windows narrower and shorter than the polygons: edges wholly left, wholly right, above and
    below; banded rows (row0 > 0); even-odd and nonzero.  The row scan runs 8 rows per CTA: ny = 9
    and 33 end in a partial CTA, and the taller bands reach rows below every polygon."""
    polys = random_rings(np.random.default_rng(100 + nx), 60, 40, 8, 14)
    left = right = False
    for nonzero in (False, True):
        e, w = edges_of(polys, orient=nonzero)
        for L, T, row0 in ((11, 30, 0), (23, 38, 5), (0, 40, 31)):
            win = Win(L, T, nx, ny)
            got = _abi_mask(F128, e, w, win, row0, _lib.MASK_NONZERO if nonzero else _lib.MASK_EVEN_ODD)
            band = Win(L, T - row0, nx, ny)
            want = mask_of(e, w, band.cu0, band.cv0, 8, nx, ny, nonzero=nonzero)
            assert np.array_equal(got, want), (nonzero, L, T, row0)
            left |= bool((e[:, [0, 2]].max(axis=1) < 8 * L).any())
            right |= bool((e[:, [0, 2]].min(axis=1) >= 8 * (L + nx)).any())
    assert left and right


@pytest.mark.gpu
@pytest.mark.parametrize("invert", [False, True])
def test_geometry_winding(invert):
    check_shape(winding_case(invert), pinned=True)


# ---------------------------------------------------------------- GPU: dilation and raster sampling
@pytest.mark.gpu
@pytest.mark.parametrize("ny", [3007, 3008, 3009])
def test_dilation_production_window(ny):
    """3500 x ~3000 pixels, k from 1 to 157: halos of one to three 64-row chunks."""
    c = dilation_case(ny)
    win = window_of(c.shape)
    r = c.rasters[0]
    dist = ndi.distance_transform_cdt(r["array"] == 0, metric="taxicab")
    for k in c.ks:
        c.rasters[0] = dict(r, k=k)
        got, _ = run_shape(c)
        assert got.shape == (win.ny, win.nx)
        bad = got != (dist > k)
        assert not bad.any(), (k, int(bad.sum()), np.argwhere(bad)[0])


@pytest.mark.gpu
@pytest.mark.parametrize("ny,ks", [(5, (9, 79)), (1, (1, 64))])
def test_dilation_thin_window(ny, ks):
    """k at least the window's height, down to a window of one row."""
    c = thin_case(ny, ks)
    for k in ks:
        c.rasters[0] = dict(c.rasters[0], k=k)
        check_shape(c, pinned=True)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["uint8", "int16", "float32", "bool"])
def test_raster_kinds(kind):
    check_shape(raster_kind_case(kind), pinned=True)


@pytest.mark.gpu
def test_raster_tall_window():
    check_shape(tall_case(), pinned=True)


# ---------------------------------------------------------------- GPU: geometry buffers
@pytest.mark.gpu
@pytest.mark.parametrize("buffer_m", [2000, 20000])
def test_polyline_buffer(buffer_m):
    """A 20 000-segment coastline buffered by about one tile and about ten."""
    excused, ties, _, n = check_shape(polyline_case(buffer_m))
    print(f"{ties} pixels within 1e-12 b of b, {excused} of them decided the other way, of {n}")
    assert ties < 1e-4 * n


@pytest.mark.gpu
def test_negative_buffer():
    excused, ties, _, n = check_shape(negative_case())
    print(f"{ties} pixels within 1e-12 b of b, {excused} of them decided the other way, of {n}")
    assert ties < 1e-4 * n


@pytest.mark.gpu
@pytest.mark.parametrize("invert", [False, True])
def test_buffer_exact_ties(invert):
    """Where seg_dist2 is exact, a centre at distance b is within the buffer: nothing excused."""
    _, _, exact, _ = check_shape(pinned_case(invert), pinned=True)
    assert exact >= 24


# ---------------------------------------------------------------- GPU: counts and bands
def _cutout():
    return ab.Cutout(data=syn.make_dataset(40, 32, 2, x0=-3.875, y0=48.125, kinds=()))


def check_counts(c):
    cut = _cutout()
    assert (cut.dx, cut.dy) == (0.25, 0.25)
    A = np.asarray(cut.availabilitymatrix([shape_json(c.frame, c.shape)], container(c)).values)[0]
    want, win, _, _ = reference(c)
    cnt = counts_of(want, win, c.grid)
    assert cnt.sum() > 1000
    res = c.frame.res
    np.testing.assert_array_equal(A, cnt.astype(np.float64) * (res * res) / (0.25 * 0.25))


@pytest.mark.gpu
@pytest.mark.parametrize("c", count_cases(), ids=lambda c: c.name)
def test_counts(c):
    check_counts(c)


@pytest.mark.gpu
@pytest.mark.parametrize("rows", BAND_ROWS)
def test_bands(rows, monkeypatch):
    """Bands thinner than the raster's halo (k = 79), down to one row, against the exact reference."""
    c = band_case(rows)
    win = window_of(c.shape)
    monkeypatch.setattr(availability._Session, "BAND_BYTES", band_bytes(win.nx, rows, 79))
    excused, ties, _, n = check_shape(c)
    assert ties < 1e-4 * n


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [1, 20])
def test_banded_counts(rows, monkeypatch):
    """Counts of a shape processed in bands of 1 and 20 rows, with a raster buffer of k = 79."""
    c = count_cases()[1]
    sparse = np.zeros_like(c.rasters[0]["array"])
    sparse[[50, 51, 300], [20, 200, 333]] = 5
    c.rasters[0] = dict(c.rasters[0], array=sparse, codes=None, k=79, nodata=0)
    win = window_of(c.shape)
    monkeypatch.setattr(availability._Session, "BAND_BYTES", band_bytes(win.nx, rows, 79))
    check_counts(c)
