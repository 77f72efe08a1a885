"""The overlay form of the indicator matrix (csrc/overlay.cu) at production size, against exact areas.

tests/test_overlay.py checks the kernel on shapes of a few edges, so nearly every shape there has
one to three y-bands.  Here the shapes are as large as the workload of tools/prof_overlay.py
(Voronoi regions densified to about 10^6 vertices per side, 80-170 bands per shape), the borders
are digitised twice, partitions are nested with bitwise-shared borders, and the band cap
(kMaxBands) and the candidate-bin clamp and coarsening are reached.

CPU part: the sweep-line oracle (oracle/overlay_exact.py: intersection_area_sweep) against the
all-pairs definition, and the generators below checked in exact arithmetic on small instances.
GPU part: partition identities, densification invariance, transposition, nested partitions,
sampled pairs against the exact oracle, the band cap, the bin clamp, repeatability and order.

"1e-12" is an absolute error on a fraction, the bar of test_overlay.py.  Entries at most 1e-10
are not stored (kKeep), so a sum over a row or column may lack the true slivers below that:
their bound, 1e-10 per absent candidate pair, is added to the sums' tolerances.
"""

from fractions import Fraction as Fr

import numpy as np
import pytest

import overlay_exact as OX
from atlite_b200 import gis, synthetic as syn
from test_overlay import CASES, _jitter, _shift, box, gj, multi, poly

KEEP = 1e-10


# ---------------------------------------------------------------- generators

def densify(rings, vertices):
    """Every edge cut into k equal pieces in float64, k chosen so that the rings hold about
    ``vertices`` in all (tools/prof_overlay.py): each neighbour interpolates a shared edge from its
    own end, so the two copies of a border differ by a few ulps."""
    k = max(1, round(vertices / sum(len(r) for r in rings)))
    t = np.arange(k)[:, None] / k
    out = []
    for r in rings:
        a, b = r, np.roll(r, -1, axis=0)
        out.append(np.ascontiguousarray((a[:, None, :] + t[None] * (b - a)[:, None, :]).reshape(-1, 2)))
    return out


def snap(rings, bits=24):
    """Every vertex rounded to a multiple of 2^-bits (a vertex shared by neighbours stays shared)."""
    return [np.round(r * 2.0 ** bits) / 2.0 ** bits for r in rings]


def densify_dyadic(rings, pieces=256):
    """Every edge of snapped rings cut into ``pieces`` (a power of two) equal parts.  With vertices
    on multiples of 2^-24 below 2^7 in magnitude, a + (b - a) * k / pieces needs at most 39
    significant bits, so every new point is exact: on its edge (orient = 0) and bitwise the same
    point when a neighbour cuts the same edge from its other end."""
    t = np.arange(pieces)[:, None] / pieces
    return [np.ascontiguousarray((r[:, None, :] + t[None] * (np.roll(r, -1, axis=0) - r)[:, None, :]).reshape(-1, 2))
            for r in rings]


def nested_partition(n_cols, n_rows, per_row, block=(4, 5), enclaves=(), enclave_vertices=300, seed=0,
                     x0=-10.0, y0=35.0, w=0.5, h=0.8):
    """Fine and coarse regions of one rectangle, NUTS3 inside NUTS2.

    The rectangle is cut by ``n_cols - 1`` wavy "vertical" polylines (plus its two straight sides)
    sampled at the same ``n_rows * per_row + 1`` heights, and by ``n_rows - 1`` horizontal lines at
    every ``per_row``-th height, so each horizontal cut point is a vertex of every polyline.  Fine
    region (i, j) lies between polylines i, i + 1 and horizontal lines j, j + 1; coarse regions are
    ``block`` = (columns, rows) blocks of fine ones, built from the same vertex arrays, so every
    border is bitwise shared.  ``enclaves``: (i, j, owner) -- a ring of ``enclave_vertices``
    inside fine region (i, j), which becomes one more fine region and a hole of (i, j); it belongs
    to coarse region ``owner`` (a hole of the coarse region around it and a part of ``owner`` when
    these differ).  Returns (fine, coarse, coarse index of every fine region)."""
    rng = np.random.default_rng(seed)
    bx, by = block
    assert n_cols % bx == 0 and n_rows % by == 0
    ys = y0 + h * np.arange(n_rows * per_row + 1) / per_row
    xs = [np.full(len(ys), x0)]
    for i in range(1, n_cols):
        xs.append(x0 + i * w + 0.24 * w * np.sin(2 * np.pi * ys / 3.0 + i) + rng.uniform(-0.008, 0.008, len(ys)) * w)
    xs.append(np.full(len(ys), x0 + n_cols * w))
    P = lambda i, k: (xs[i][k], ys[k])  # noqa: E731

    def ring(i0, i1, k0, k1):
        """Polylines i0..i1 between heights k0..k1, counter-clockwise."""
        pts = [P(i, k0) for i in range(i0, i1 + 1)]
        pts += [P(i1, k) for k in range(k0 + 1, k1 + 1)]
        pts += [P(i, k1) for i in range(i1 - 1, i0 - 1, -1)]
        pts += [P(i0, k) for k in range(k1 - 1, k0, -1)]
        return np.array(pts)

    ncx = n_cols // bx
    fine = [[ring(i, i + 1, j * per_row, (j + 1) * per_row)] for j in range(n_rows) for i in range(n_cols)]
    of = [(j // by) * ncx + i // bx for j in range(n_rows) for i in range(n_cols)]
    coarse = [[ring(I * bx, (I + 1) * bx, J * by * per_row, (J + 1) * by * per_row)]
              for J in range(n_rows // by) for I in range(ncx)]
    coarse_parts = [[] for _ in coarse]  # extra exterior parts (enclaves of other regions)
    th = 2 * np.pi * np.arange(enclave_vertices) / enclave_vertices
    for i, j, owner in enclaves:
        kc = j * per_row + per_row // 2
        cx, cy = (xs[i][kc] + xs[i + 1][kc]) / 2, ys[kc]
        r = 0.1 * w * (1 + 0.2 * np.sin(5 * th))
        e = np.c_[cx + r * np.cos(th), cy + r * np.sin(th)]
        lo = (ys >= e[:, 1].min() - h / per_row) & (ys <= e[:, 1].max() + h / per_row)
        assert xs[i][lo].max() < e[:, 0].min() and e[:, 0].max() < xs[i + 1][lo].min()  # strictly inside (i, j)
        fine[j * n_cols + i].append(e)
        fine.append([e])
        of.append(owner)
        around = of[j * n_cols + i]
        if owner != around:
            coarse[around].append(e)
            coarse_parts[owner].append(e)

    def shape(rings, parts=()):
        close = lambda r: np.r_[r, r[:1]].tolist()  # noqa: E731
        poly_ = [close(r) for r in rings]
        if not parts:
            return {"type": "Polygon", "coordinates": poly_}
        return {"type": "MultiPolygon", "coordinates": [poly_] + [[close(p)] for p in parts]}

    return [shape(f) for f in fine], [shape(c, p) for c, p in zip(coarse, coarse_parts)], of


def star(n, cx=8.0, cy=46.0, r=4.0):
    """A star-shaped ring of ``n`` vertices (and edges), counter-clockwise."""
    th = 2 * np.pi * np.arange(n) / n
    rr = r * (1 + 0.25 * np.sin(7 * th) + 0.05 * np.sin(29 * th))
    return np.ascontiguousarray(np.c_[cx + rr * np.cos(th), cy + rr * np.sin(th)])


def cell_polygons(x, y):
    xlo, xhi = gis.cell_edges(x)
    ylo, yhi = gis.cell_edges(y)
    X0, Y0 = np.meshgrid(xlo, ylo)
    X1, Y1 = np.meshgrid(xhi, yhi)
    c = np.stack([X0.ravel(), Y0.ravel(), X1.ravel(), Y0.ravel(), X1.ravel(), Y1.ravel(), X0.ravel(), Y1.ravel()], 1)
    return list(c.reshape(-1, 4, 2))


# ---------------------------------------------------------------- helpers

def areas(shapes):
    """float64 shoelace areas of the packed rings (exteriors minus holes)."""
    return gis._ring_shape_areas(*gis.pack_shapes(shapes))


def boxes(shapes):
    out = np.empty((len(shapes), 4))
    for k, s in enumerate(shapes):
        pts = np.concatenate([r for r, _ in gis.geometry_rings(s)])
        out[k] = pts[:, 0].min(), pts[:, 1].min(), pts[:, 0].max(), pts[:, 1].max()
    return out


def candidates(orig, dest):
    """(dest, orig) index pairs whose bounding boxes' interiors overlap."""
    bo, bd = boxes(orig), boxes(dest)
    i, j = np.nonzero((bd[:, None, 0] < bo[None, :, 2]) & (bo[None, :, 0] < bd[:, None, 2])
                      & (bd[:, None, 1] < bo[None, :, 3]) & (bo[None, :, 1] < bd[:, None, 3]))
    return i, j


def entries(m):
    coo = m.tocoo()
    return {(int(i), int(j)): float(v) for i, j, v in zip(coo.row, coo.col, coo.data)}


def assert_same(a, b, atol=1e-12):
    """Pattern equal (entries within a factor 2 of the keep threshold may be in one only) and
    values within ``atol``."""
    ea, eb = entries(a), entries(b)
    assert a.shape == b.shape
    odd = {k: ea.get(k, eb.get(k)) for k in set(ea) ^ set(eb)}
    assert all(v <= 2 * KEEP for v in odd.values()), f"pattern differs: {sorted(odd.items())[:10]}"
    common = set(ea) & set(eb)
    err = max((abs(ea[k] - eb[k]) for k in common), default=0.0)
    assert err <= atol, f"max |diff| {err:.3e}"


def absent_candidates(m, orig, dest):
    """Number of box-overlapping pairs without an entry, per row and per column."""
    i, j = candidates(orig, dest)
    mask = np.asarray(m[i, j]).ravel() == 0
    return (np.bincount(i[mask], minlength=m.shape[0]), np.bincount(j[mask], minlength=m.shape[1]),
            i[mask], j[mask])


def assert_partition(m, orig, dest, cover_cols=True, cover_rows=True):
    """dest partitions a region that contains every orig shape: each column sums to 1; orig
    partitions a region containing every dest shape: sum_j I[i, j] area(orig_j) = area(dest_i).
    Each absent candidate pair may hide a true sliver of at most 1e-10 of its orig area."""
    ao, ad = areas(orig), areas(dest)
    n_row, n_col, ai, aj = absent_candidates(m, orig, dest)
    if cover_cols:
        col = np.asarray(m.sum(axis=0)).ravel()
        assert np.all(col <= 1 + 1e-11), f"column sum {col.max()!r}"
        assert np.all(col >= 1 - 1e-11 - KEEP * n_col), f"column sum {col.min()!r}"
    if cover_rows:
        row = m @ ao
        slack = np.bincount(ai, weights=KEEP * ao[aj], minlength=len(ad))
        err = np.abs(row - ad)
        assert np.all(err <= 1e-11 * ad + slack), f"row identity: worst relative {np.max(err / ad):.3e}"


def exact_fraction(o, d):
    """area(d ∩ o) / area(o) as a Fraction (the sweep oracle)."""
    ro, rd = gis.geometry_rings(o), gis.geometry_rings(d)
    return OX.intersection_area_sweep(rd, ro) / OX.shape_area(ro)


def orient(a, b, p):
    return (b[0] - a[0]) * (p[1] - a[1]) - (b[1] - a[1]) * (p[0] - a[0])


# ---------------------------------------------------------------- CPU: the sweep oracle

def _ring_list(s):
    return gis.geometry_rings(s)


@pytest.mark.parametrize("where", ["origin", "lon40"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_sweep_equals_definition_on_degenerate_cases(name, where):
    orig, dest = CASES[name]
    if where == "lon40":
        orig, dest = _shift(orig, 40.0, 50.0, 0.25), _shift(dest, 40.0, 50.0, 0.25)
    for d in dest:
        for o in orig:
            rd, ro = _ring_list(d), _ring_list(o)
            assert OX.intersection_area_sweep(rd, ro) == OX.intersection_area(rd, ro)
            assert OX.intersection_area_sweep(ro, rd) == OX.intersection_area(ro, rd)


def _random_ring(rng, n, cx, cy, r, grid=None):
    th = np.sort(rng.uniform(0, 2 * np.pi, n))
    rr = r * rng.uniform(0.4, 1.0, n)
    p = np.c_[cx + rr * np.cos(th), cy + rr * np.sin(th)]
    return np.round(p / grid) * grid if grid else p


def _random_pair(seed):
    """Small shape pairs of four kinds: holes, overlapping parts of one multipolygon, collinear
    shared edges (vertices on a coarse grid) and a border digitised twice with ulp jitter."""
    rng = np.random.default_rng(seed)
    kind = seed % 4
    if kind == 0:
        d = gj(_random_ring(rng, 9, 0, 0, 2), _random_ring(rng, 5, 0.2, 0.1, 0.6))
        o = gj(_random_ring(rng, 8, 0.5, 0.3, 2), _random_ring(rng, 6, 0.6, 0.2, 0.5))
    elif kind == 1:
        d = multi(gj(_random_ring(rng, 7, 0, 0, 1.5)), gj(_random_ring(rng, 6, 0.7, 0.4, 1.5)))
        o = multi(gj(_random_ring(rng, 6, 0.3, -0.2, 1.2)), gj(_random_ring(rng, 8, 0.1, 0.5, 1.4)))
    elif kind == 2:
        d = multi(gj(box(0, 0, 2, 1)), gj(_random_ring(rng, 7, 1, 1, 1.5, grid=0.25)))
        o = gj(_random_ring(rng, 9, 1, 0.5, 1.5, grid=0.25), box(0.5, 0.25, 1, 0.5))
    else:
        x0, y0 = rng.uniform(-5, 40), rng.uniform(30, 60)
        ys = y0 + np.linspace(0.0, 1.0, 12)
        border = np.c_[x0 + 0.5 + rng.uniform(-0.125, 0.125, 12), ys]
        left = np.r_[[[x0, y0]], border, [[x0, y0 + 1]]]
        moved = _jitter(border, rng)
        right = np.r_[moved[:1], [[x0 + 1, y0], [x0 + 1, y0 + 1]], moved[:0:-1]]
        d, o = (left, right) if seed % 8 == 3 else (right, left[::-1])
    return d, o


@pytest.mark.parametrize("seed", range(32))
def test_sweep_equals_definition_on_random_pairs(seed):
    d, o = _random_pair(seed)
    rd, ro = _ring_list(d), _ring_list(o)
    want = OX.intersection_area(rd, ro)
    assert OX.intersection_area_sweep(rd, ro) == want
    assert OX.intersection_area_sweep(ro, rd) == want  # the product w_D w_O is symmetric
    assert OX.intersection_area_sweep(rd, rd) == OX.intersection_area(rd, rd)


# ---------------------------------------------------------------- CPU: the generators

def test_nested_partition_tiles_exactly():
    fine, coarse, of = nested_partition(8, 10, 6, enclaves=((1, 2, 3), (5, 7, 3), (6, 1, 0)), enclave_vertices=24)
    assert len(fine) == 83 and len(coarse) == 4
    fine, coarse = [gis.geometry_rings(f) for f in fine], [gis.geometry_rings(c) for c in coarse]
    fa, ca = [OX.shape_area(f) for f in fine], [OX.shape_area(c) for c in coarse]
    for c in range(4):
        assert sum(a for a, k in zip(fa, of) if k == c) == ca[c]
    want = {(f, of[f]): fa[f] / ca[of[f]] for f in range(len(fine))}
    assert OX.overlay_fractions(coarse, fine) == want  # orig = coarse: each fine region in its own only
    assert OX.overlay_fractions(fine, coarse) == {(of[f], f): 1 for f in range(len(fine))}


def test_dyadic_densification_is_exact():
    x, y = syn.make_coords(20, 14, -12.0 + 0.125, 33.0 + 0.125)
    plain = snap(syn.make_voronoi_shapes(x, y, 12, seed=8))
    dense = densify_dyadic(plain, 16)
    vertex_sets = [set(map(tuple, r)) for r in dense]
    shared = 0
    for a, (p, q) in enumerate(zip(plain, dense)):
        fq = [(Fr(float(u)), Fr(float(v))) for u, v in q]
        for k in range(len(p)):
            e0, e1 = fq[16 * k], fq[(16 * (k + 1)) % len(fq)]
            assert all(orient(e0, e1, fq[16 * k + m]) == 0 for m in range(1, 16))
            # a neighbour holding the same edge cut it from its other end into the same points
            for b, other in enumerate(plain):
                if b == a:
                    continue
                ob = {tuple(v): n for n, v in enumerate(other)}
                u, v = tuple(p[k]), tuple(p[(k + 1) % len(p)])
                if u in ob and v in ob and (ob[u] - ob[v]) % len(other) == 1:
                    assert set(map(tuple, q[16 * k:16 * (k + 1)])) <= vertex_sets[b]
                    shared += 1
    assert shared > 20


# ---------------------------------------------------------------- GPU: production geometry

@pytest.fixture(scope="module")
def prod():
    """The geometry of tools/prof_overlay.py: a 216 x 156 grid of 0.25 degree cells over Europe,
    1 500 and 3 000 Voronoi regions (seeds 8, 9), each set densified to about 10^6 vertices."""
    x, y = syn.make_coords(216, 156, -12.0 + 0.125, 33.0 + 0.125)
    p1, p2 = syn.make_voronoi_shapes(x, y, 1500, seed=8), syn.make_voronoi_shapes(x, y, 3000, seed=9)
    return dict(x=x, y=y, cells=cell_polygons(x, y), plain1=p1, plain2=p2,
                dense1=densify(p1, 1_000_000), dense2=densify(p2, 1_000_000))


@pytest.fixture(scope="module")
def prod_mats(prod):
    """I(dense 1 500, dense 3 000) and the transposed call."""
    a, b = prod["dense1"], prod["dense2"]
    return {"AB": gis.compute_indicatormatrix(a, b), "BA": gis.compute_indicatormatrix(b, a)}


def test_production_shapes_have_many_bands(prod):
    n = np.array([len(r) for r in prod["dense1"]] + [len(r) for r in prod["dense2"]])
    assert 0.9e6 < n[:1500].sum() < 1.1e6 and 0.9e6 < n[1500:].sum() < 1.1e6
    assert np.median(n // 4) >= 80  # y-bands per shape (kBandEdges = 4)


@pytest.mark.gpu
def test_partition_identities_regions(prod, prod_mats):
    a, b = prod["dense1"], prod["dense2"]
    assert prod_mats["AB"].shape == (3000, 1500)
    assert_partition(prod_mats["AB"], a, b)
    assert_partition(prod_mats["BA"], b, a)


@pytest.mark.gpu
def test_partition_identities_and_grid_kernel_cells(prod):
    """Dense regions against cells both ways, and the overlay equal to the grid kernel
    (csrc/indicator.cu), an independent implementation, on shapes of about 670 vertices."""
    x, y, cells, regions = prod["x"], prod["y"], prod["cells"], prod["dense1"]
    rc = gis.compute_indicatormatrix(cells, regions)  # I[region, cell] = area / area(cell)
    cr = gis.compute_indicatormatrix(regions, cells)
    assert_partition(rc, cells, regions)
    assert_partition(cr, regions, cells)
    grid = gis.compute_indicatormatrix(x, y, regions).tocsr()
    grid.sort_indices()
    assert np.array_equal(rc.indptr, grid.indptr) and np.array_equal(rc.indices, grid.indices)
    assert np.abs(rc.data - grid.data).max() <= 1e-12


@pytest.mark.gpu
def test_densification_invariance_jittered(prod):
    """The plain regions and the same regions densified in float64 (borders digitised twice) give
    the same matrix; and each densified region covers exactly its plain self and nothing else."""
    plain = gis.compute_indicatormatrix(prod["plain1"], prod["plain2"])
    dense = gis.compute_indicatormatrix(prod["dense1"], prod["dense2"])
    assert_same(dense, plain)
    n = len(prod["plain1"])
    for orig, dest in ((prod["dense1"], prod["plain1"]), (prod["plain1"], prod["dense1"])):
        m = gis.compute_indicatormatrix(orig, dest)
        assert m.nnz == n and np.array_equal(m.indices, np.arange(n))
        assert np.abs(m.data - 1).max() <= 1e-12


@pytest.mark.gpu
def test_densification_invariance_exact(prod):
    """Snapped regions and the same cut into 2^8 exact pieces: every border identical on both sides
    and every new vertex exactly on the other shape's edge."""
    s1, s2 = snap(prod["plain1"]), snap(prod["plain2"])
    d1, d2 = densify_dyadic(s1), densify_dyadic(s2)
    assert_same(gis.compute_indicatormatrix(d1, d2), gis.compute_indicatormatrix(s1, s2))
    n = len(s1)
    for orig, dest in ((d1, s1), (s1, d1)):
        m = gis.compute_indicatormatrix(orig, dest)
        assert m.nnz == n and np.array_equal(m.indices, np.arange(n))
        assert np.abs(m.data - 1).max() <= 1e-12


@pytest.mark.gpu
def test_transposition(prod, prod_mats):
    """I(A, B)[i, j] area(A_j) = I(B, A)[j, i] area(B_i): the perturbation moves to the other side."""
    aa, ab = areas(prod["dense1"]), areas(prod["dense2"])
    AB, BA = entries(prod_mats["AB"]), entries(prod_mats["BA"])
    for (i, j), f in AB.items():  # f area(A_j) = area(B_i ∩ A_j)
        g = BA.get((j, i), 0.0)
        if f > 1e-9 and g > 1e-9:
            assert abs(f * aa[j] - g * ab[i]) <= 1e-12 * max(aa[j], ab[i]), (i, j, f, g)
        if f * aa[j] / ab[i] > 1e-9:  # what BA holds for it
            assert (j, i) in BA, (i, j, f)
    for (j, i), g in BA.items():
        if g * ab[i] / aa[j] > 1e-9:
            assert (i, j) in AB, (j, i, g)


@pytest.mark.gpu
def test_nested_partitions_shared_borders():
    enclaves = ((5, 2, 0), (22, 12, 31), (41, 20, 70))  # the last one belongs to the coarse region around it
    fine, coarse, of = nested_partition(60, 25, 80, enclaves=enclaves, seed=1)
    assert len(fine) == 1503 and len(coarse) == 75
    assert min(len(gis.geometry_rings(c)[0][0]) for c in coarse) > 800  # about 200 bands each
    fc = gis.compute_indicatormatrix(fine, coarse)  # (coarse, fine): one entry 1 per column
    assert fc.nnz == len(fine)
    coo = fc.tocoo()
    assert np.array_equal(np.sort(coo.col), np.arange(len(fine)))
    assert np.array_equal(coo.row[np.argsort(coo.col)], of)
    assert np.abs(coo.data - 1).max() <= 1e-12
    cf = gis.compute_indicatormatrix(coarse, fine)  # (fine, coarse): area(f) / area(c), nothing else
    want = areas(fine) / areas(coarse)[of]
    assert cf.nnz == len(fine)
    assert np.array_equal(cf.indptr, np.arange(len(fine) + 1)) and np.array_equal(cf.indices, of)
    assert np.abs(cf.data - want).max() <= 1e-12


@pytest.mark.gpu
def test_sampled_pairs_exact(prod, prod_mats):
    """Pairs of the 1 500 x 3 000 matrix at production vertex counts against the sweep oracle: the
    entries with the longest shared border (along the sides of the extent), random entries, and
    box-overlapping pairs with no entry."""
    A, B = prod["dense1"], prod["dense2"]
    got = entries(prod_mats["AB"])
    rng = np.random.default_rng(0)
    keys = sorted(got)

    def side_spans(rings):
        x, y = prod["x"], prod["y"]
        sides = ((0, x[0] - 0.125), (0, x[-1] + 0.125), (1, y[0] - 0.125), (1, y[-1] + 0.125))
        out = []
        for r in rings:
            sp = []
            for ax, v in sides:
                on = r[r[:, ax] == v, 1 - ax]
                sp.append((on.min(), on.max()) if len(on) > 1 else (0.0, 0.0))
            out.append(sp)
        return out

    sa, sb = side_spans(prod["plain1"]), side_spans(prod["plain2"])
    shared = {k: sum(max(0.0, min(p[1], q[1]) - max(p[0], q[0])) for p, q in zip(sb[k[0]], sa[k[1]])) for k in keys}
    border = sorted(keys, key=lambda k: -shared[k])[:15]
    assert shared[border[-1]] > 0
    rand = [keys[k] for k in rng.choice(len(keys), 25, replace=False)]
    _, _, ai, aj = absent_candidates(prod_mats["AB"], A, B)
    assert len(ai) > 0
    pick = rng.choice(len(ai), min(15, len(ai)), replace=False)
    for i, j in border + rand:
        want = float(exact_fraction(A[j], B[i]))
        assert abs(got[(i, j)] - want) <= 1e-12, ((i, j), got[(i, j)], want)
    for k in pick:
        i, j = int(ai[k]), int(aj[k])
        assert exact_fraction(A[j], B[i]) <= Fr(1, 10 ** 10), (i, j)


def _exact_cell_overlap(ring, cell):
    """Exact area(ring ∩ cell) from the ring's edges that meet the cell's y window only (the others
    add no slab boundary and span no slab); ``ring`` is counter-clockwise."""
    a, b = ring, np.roll(ring, -1, axis=0)
    ylo, yhi = cell[:, 1].min(), cell[:, 1].max()
    sel = np.nonzero((np.maximum(a[:, 1], b[:, 1]) >= ylo) & (np.minimum(a[:, 1], b[:, 1]) <= yhi))[0]
    f = lambda p: (Fr(float(p[0])), Fr(float(p[1])))  # noqa: E731
    eo = [(f(a[k]), f(b[k])) for k in sel]
    ed = OX._edges(OX._rings([(cell, False)]))
    return OX.edges_intersection_area(ed, eo)


@pytest.mark.gpu
@pytest.mark.parametrize("n_edges", [131072, 150000])
def test_band_cap(n_edges):
    """A ring with 131 072 edges has exactly kMaxBands = 2^15 bands; one with 150 000 edges is
    capped there, with about 4.6 edges per band.  On either side against cells."""
    x, y = syn.make_coords(64, 48, 0.125, 40.125)
    cells = cell_polygons(x, y)
    ring = star(n_edges)
    grid = gis.compute_indicatormatrix(x, y, [ring]).tocsr()
    grid.sort_indices()
    dest_side = gis.compute_indicatormatrix(cells, [ring])  # (1, cells): area / area(cell)
    orig_side = gis.compute_indicatormatrix([ring], cells)  # (cells, 1): area / area(ring)
    assert np.array_equal(dest_side.indices, grid.indices) and np.abs(dest_side.data - grid.data).max() <= 1e-12
    ca, ra = areas(cells), areas([ring])[0]
    want = grid.T.tocsr().multiply(ca[:, None] / ra).tocsr()
    want.data[want.data <= KEEP] = 0
    want.eliminate_zeros()
    assert_same(orig_side, want)
    assert_partition(dest_side, cells, [ring], cover_cols=False)
    assert_partition(orig_side, [ring], cells, cover_rows=False)
    g = entries(dest_side)
    edge_cells = sorted(c for (_, c), v in g.items() if 0.05 < v < 0.95)
    o = entries(orig_side)
    for c in np.random.default_rng(n_edges).choice(edge_cells, 6, replace=False):
        c = int(c)
        exact = _exact_cell_overlap(ring, cells[c])
        assert abs(g[(0, c)] - float(exact / OX.shape_area([(cells[c], False)]))) <= 1e-12, c
        assert abs(o[(c, 0)] - float(exact) / ra) <= 1e-12, c


@pytest.mark.gpu
def test_bin_clamp_and_coarsening():
    """10^4 cells of 2^-10 degree in one cluster, a triangle 50 degrees away and a continent over the
    cluster: the bins per axis hit kMaxBinsAxis, then the 4 n + 64 coarsening, and the continent
    is listed in many bins.

    The cluster lies near the origin.  The kernel rounds crossing points to float64 in absolute
    coordinates, so a fraction of a cell of side s at |x| ~ M is good to about ulp(M) / s per
    crossing: 7e-12 for these cells at latitude 50, above the 1e-12 bar; 1e-13 here."""
    s = 2.0 ** -10
    xc, yc = 0.5 + (np.arange(100) + 0.5) * s, 0.25 + (np.arange(100) + 0.5) * s
    cells = cell_polygons(xc, yc)
    tri = poly((35.0, 35.0), (36.0, 35.0), (35.5, 36.0))
    th = 2 * np.pi * np.arange(40) / 40
    continent = np.c_[0.5 + 12 * np.cos(th) * (1 + 0.1 * np.sin(3 * th)),
                      0.25 + 9 * np.sin(th) * (1 + 0.1 * np.cos(5 * th))]
    orig = cells + [tri, continent]
    ext = boxes(orig)
    span = ext[:, 2:].max(0) - ext[:, :2].min(0)
    assert (span / s > 2048).all() and 2048 ** 2 > 4 * len(orig) + 64  # clamped, then coarsened
    dest = syn.make_voronoi_shapes(xc, yc, 200, seed=3) + [box(34.5, 34.5, 36.5, 36.5)]
    m = gis.compute_indicatormatrix(orig, dest)
    _, n_col, ai, aj = absent_candidates(m, orig, dest)
    col = np.asarray(m.sum(axis=0)).ravel()
    n = len(cells)
    err = np.abs(col[:n] - 1) - KEEP * n_col[:n]
    assert err.max() <= 1e-12, f"cell {err.argmax()}: column sum {col[err.argmax()]!r}"
    assert abs(m[200, n] - 1) <= 1e-12 and m[:, n].nnz == 1
    assert abs(col[-1] - (100 * s) ** 2 / areas([continent])[0]) <= 1e-12
    got = entries(m)
    rng = np.random.default_rng(5)
    keys = sorted(got)
    pairs = [keys[k] for k in rng.choice(len(keys), 250, replace=False)]
    pairs += [(int(ai[k]), int(aj[k])) for k in rng.choice(len(ai), min(50, len(ai)), replace=False)]
    for i, j in pairs:
        want = exact_fraction(orig[j], dest[i])
        if (i, j) in got:
            assert abs(got[(i, j)] - float(want)) <= 1e-12, (i, j)
        else:
            assert want <= Fr(1, 10 ** 10), (i, j)


@pytest.mark.gpu
def test_repeatable_and_order_free(prod, prod_mats):
    """Each pair is summed by one warp over its own shapes' band lists, so repeating the call or
    permuting either side changes no bit."""
    a, b = prod["dense1"], prod["dense2"]
    ref = prod_mats["AB"]
    again = gis.compute_indicatormatrix(a, b)
    assert np.array_equal(again.indptr, ref.indptr) and np.array_equal(again.indices, ref.indices)
    assert again.data.tobytes() == ref.data.tobytes()
    rng = np.random.default_rng(2)
    po, pd_ = rng.permutation(len(a)), rng.permutation(len(b))
    m = gis.compute_indicatormatrix([a[k] for k in po], [b[k] for k in pd_]).tocsr()
    # row r of m is dest pd_[r], column c is orig po[c]: undo both permutations
    back = m[np.argsort(pd_)][:, np.argsort(po)].tocsr()
    back.sort_indices()
    assert np.array_equal(back.indptr, ref.indptr) and np.array_equal(back.indices, ref.indices)
    assert back.data.tobytes() == ref.data.tobytes()
