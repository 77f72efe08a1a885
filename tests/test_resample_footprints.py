"""The reproject and regrid kernels at production footprints, against exact sums.

Within one CRS the geometry can be made dyadic: source pixels of size 2, origins on multiples of
them, destination edges on multiples of 1/8 source pixel, values small integers (or NaN / nodata).
Then every overlap, every product wy * wx and every partial sum is exact in float64 whatever the
order of the sums, and the kernels' only rounding is the final S / W (and the cast to float32).
``exact_average`` forms S and W as exact integers (in units of 1/64 pixel), so the expected value
is S / W correctly rounded, float(Fraction(S, W)), and the tests ask for bitwise equality on every
tile, launch and batch walk:

* ``k_reproject_avg`` on the identity pair (``engine.ReprojectOp`` with one CRS twice): boxes of 31,
  32 and 33 pixels, widths of 1, 255, 256, 257 and 300+ pixels, tall boxes, a box of about 5e4
  pixels, boxes clipped at every source edge and one larger than the source, forced tiles, NaN and
  nodata inside boxes a whole CTA sums, and a batch long enough that every CTA walks 3 entries;
  ``k_reproject_nearest`` through the same batch walk;
* ``k_regrid`` (``gis.reproject`` within one CRS): a cell width that splits a row into more column
  tiles, strided source views at every 16-byte phase for int16, float32 and float64, 70 000 batch
  entries (more than the grid's 65535 y blocks), and an int16 terrain window streamed from a host
  reader in bands of rows;
* ``gis.reproject`` within one CRS for cells wider than ``k_regrid``'s shared memory holds, which
  runs ``k_reproject_avg`` on the identity pair instead (``RegridOp.ring_fits``).

Across CRSs nothing is dyadic: a float32 EPSG:3035 and a Mollweide source of 1500 x 2000 pixels go
onto 0.25 degree cells of about 1e4 pixels each, and sampled destination windows are compared with
``oracle/reproject_oracle.py`` to 1e-9.

The CPU tests check the exact reference against that oracle and recompute every GPU case's boxes
with the kernel's ``axis_span`` rule, so that each case provably reaches the code path it targets.
"""

import math
from fractions import Fraction
from types import SimpleNamespace

import numpy as np
import pytest

import reproject_oracle as RO
from atlite_b200 import _lib, engine, gis, proj

CRS = 3035  # the same-CRS cases run on the identity pair of any CRS
SRC_A, SRC_C, SRC_F = 2.0, 1024.0, 4096.0  # source transform (2, 0, 1024, 0, -2, 4096): north-up, dyadic
RP_THREADS, RP_SMALL, RP_EPS = 256, 32, 1e-10  # csrc/reproject.cu
RG_THREADS = 128  # csrc/regrid.cu: destination columns per column tile at most
MOLL = "ESRI:54009"


# ---------------------------------------------------------------- dyadic geometry and the exact reference

def dyadic(col0, cw, nx, row0, rh, ny, south_up=False):
    """(src_t, dst_t, dst_shape) of a destination whose column j spans source pixel columns
    [col0 + j cw, col0 + (j + 1) cw] and whose rows span [row0 + i rh, ...] (north-up rows; south-up
    destinations list the same rows bottom first).  Every argument is a multiple of 1/8."""
    for q in (col0, cw, row0, rh):
        assert q * 8 == int(q * 8), q
    st = (SRC_A, 0.0, SRC_C, 0.0, -SRC_A, SRC_F)
    if south_up:
        dt = (SRC_A * cw, 0.0, SRC_C + SRC_A * col0, 0.0, SRC_A * rh, SRC_F - SRC_A * (row0 + ny * rh))
    else:
        dt = (SRC_A * cw, 0.0, SRC_C + SRC_A * col0, 0.0, -SRC_A * rh, SRC_F - SRC_A * row0)
    return st, dt, (ny, nx)


def overlaps(s0, ss, n, d0, ds, m):
    """(m, n) int64: 8 x the overlap, in source pixels, of destination cell k (edges d0 + k ds and
    d0 + (k + 1) ds) with source pixel p (edges s0 + p ss and s0 + (p + 1) ss), in exact rationals.
    Dyadic geometry makes every overlap 0 or a multiple of 1/8 (so the 1e-10 sliver rule never
    applies); anything else fails here."""
    S0, SS, D0, DS = (Fraction(float(t)) for t in (s0, ss, d0, ds))
    out = np.zeros((m, n), dtype=np.int64)
    for k in range(m):
        t0, t1 = sorted(((D0 + k * DS - S0) / SS, (D0 + (k + 1) * DS - S0) / SS))
        for p in range(max(0, math.floor(t0)), min(n, math.ceil(t1))):
            o = 8 * (min(t1, p + 1) - max(t0, p))
            assert o.denominator == 1, "not a dyadic geometry"
            out[k, p] = max(int(o), 0)
    return out


def exact_sums(values, st, dt, dst_shape, nodata=None):
    """(S, W), float64 arrays (batch, *dst_shape) holding exact integers: 64 x the weighted sum of the
    valid pixels of each cell and 64 x their weight.  Valid: not NaN and not ``nodata``."""
    v = np.asarray(values, dtype=np.float64)
    v = v.reshape((-1,) + v.shape[-2:])
    ny, nx = v.shape[-2:]
    wy = overlaps(st[5], st[4], ny, dt[5], dt[4], dst_shape[0]).astype(np.float64)
    wx = overlaps(st[2], st[0], nx, dt[2], dt[0], dst_shape[1]).astype(np.float64)
    ok = ~np.isnan(v) if nodata is None else ~np.isnan(v) & (v != nodata)
    vals = np.where(ok, v, 0.0)
    assert (vals == np.round(vals)).all(), "values must be integers"
    # every product and partial sum is an integer below 2**53, so any summation order is exact
    assert 64 * (np.abs(vals).max(initial=0) + 1) * ny * nx < 2.0 ** 53
    return wy @ vals @ wx.T, wy @ ok.astype(np.float64) @ wx.T


def exact_average(values, st, dt, dst_shape, nodata=None, empty=np.nan, dtype=np.float64):
    """The average the kernels must give, bitwise: S / W of exact integers is correctly rounded
    (float(Fraction(S, W))); float32 output is that float64 cast, as in the kernels."""
    s, w = exact_sums(values, st, dt, dst_shape, nodata)
    with np.errstate(invalid="ignore", divide="ignore"):
        out = np.where(w > 0, s / np.where(w > 0, w, 1.0), empty)
    lead = np.shape(values)[:-2]
    return out.reshape(lead + tuple(dst_shape)).astype(dtype)


def exact_int16(values, st, dt, dst_shape, fill):
    """The int16 window average: S / W rounded half away from zero, exactly (from the integers);
    a cell without a valid value gets ``fill``."""
    s, w = exact_sums(values, st, dt, dst_shape, fill)
    si, wi = s.astype(np.int64), np.maximum(w.astype(np.int64), 1)
    r = np.sign(si) * ((2 * np.abs(si) + wi) // (2 * wi))
    return np.where(w > 0, r, fill).reshape(dst_shape).astype(np.int16)


def exact_nearest(values, st, dt, dst_shape, nodata=None, empty=np.nan):
    """The pixel under each destination centre, in exact rationals (``dst_nodata`` outside, and for
    NaN and nodata pixels)."""
    v = np.asarray(values, dtype=np.float64)
    ny, nx = v.shape[-2:]

    def pick(s0, ss, n, d0, ds, m):
        S0, SS, D0, DS = (Fraction(float(t)) for t in (s0, ss, d0, ds))
        p = np.array([math.floor((D0 + (k + Fraction(1, 2)) * DS - S0) / SS) for k in range(m)])
        return p, (p >= 0) & (p < n)

    r, rin = pick(st[5], st[4], ny, dt[5], dt[4], dst_shape[0])
    c, cin = pick(st[2], st[0], nx, dt[2], dt[0], dst_shape[1])
    got = v[..., np.clip(r, 0, ny - 1)[:, None], np.clip(c, 0, nx - 1)[None, :]]
    bad = np.isnan(got) | ((got == nodata) if nodata is not None else False) | ~(rin[:, None] & cin[None, :])
    return np.where(bad, empty, got)


def kernel_boxes(st, src_shape, dt, dst_shape, src_crs=CRS, dst_crs=CRS):
    """Every destination cell's box as k_reproject_avg computes it: the two corners taken to source
    pixel coordinates (rounded like the kernel's lattice), then reproject.cu's ``axis_span`` along
    each axis.  ``w`` / ``h`` / ``n``: columns, rows and pixels (0 when empty); ``u0 .. v1``: the
    unclipped box."""
    ny, nx = dst_shape
    jj, ii = np.meshgrid(np.arange(nx + 1.0), np.arange(ny + 1.0))
    x, y = dt[2] + jj * dt[0], dt[5] + ii * dt[4]
    if proj.epsg(src_crs) != proj.epsg(dst_crs):
        x, y = proj.transform(x, y, dst_crs, src_crs)
    u, v = (x - st[2]) / st[0], (y - st[5]) / st[4]
    u0, u1 = np.fmin(u[:-1, :-1], u[1:, 1:]), np.fmax(u[:-1, :-1], u[1:, 1:])
    v0, v1 = np.fmin(v[:-1, :-1], v[1:, 1:]), np.fmax(v[:-1, :-1], v[1:, 1:])

    def span(t0, t1, n):
        lo = np.clip(np.floor(t0 + RP_EPS), 0, n)
        hi = np.clip(np.ceil(t1 - RP_EPS), 0, n)
        return np.maximum(hi - lo, 0).astype(np.int64)

    w, h = span(u0, u1, src_shape[1]), span(v0, v1, src_shape[0])
    return SimpleNamespace(w=w, h=h, n=w * h, u0=u0, u1=u1, v0=v0, v1=v1, src_shape=src_shape)


# ---------------------------------------------------------------- the k_reproject_avg cases

# name: (source shape, dyadic(...) arguments); every destination edge is fractional at both ends
CASES = {
    "n31_32": ((15, 372), (0.125, 30.875, 12, 0.125, 0.875, 16)),  # 1 x 31, 1 x 32 (one thread), 2 x 31 ...
    "n32_33": ((16, 384), (0.375, 31.875, 12, 0.25, 0.875, 16)),  # ... 1 x 33 (the CTA), side by side
    "n32_33_south": ((16, 384), (0.375, 31.875, 12, 0.25, 0.875, 16, True)),
    "w255_256": ((16, 1021), (0.25, 254.875, 4, 0.625, 2.5, 6)),  # CTA walk with dr = 1, dc = 1 / 0
    "w256_257": ((10, 1024), (0.75, 255.5, 4, 0.125, 1.375, 6)),  # ... dr = 1, dc = 0 and dr = 0, dc = 256
    "w312": ((6, 936), (0.75, 311.625, 3, 0.375, 0.625, 8)),  # w > 256: dr = 0, dc = 256
    "tall": ((602, 16), (0.125, 0.625, 24, 0.5, 300.375, 2)),  # w in {1, 2}, h > 300: dc = 0
    "n5e4": ((751, 803), (0.875, 200.375, 4, 0.125, 250.25, 3)),  # about 201 x 251 pixels per box
    "clipped": ((40, 52), (-3.375, 9.625, 7, -2.625, 7.375, 7)),  # overhangs all four source edges
    "beyond": ((37, 45), (-2.5, 52.625, 1, -1.125, 41.5, 1)),  # one box larger than the whole source
}


def case(name):
    src_shape, args = CASES[name]
    st, dt, dshape = dyadic(*args)
    return src_shape, st, dt, dshape


def case_boxes(name):
    src_shape, st, dt, dshape = case(name)
    return kernel_boxes(st, src_shape, dt, dshape)


def default_tile(name):
    src_shape, st, dt, dshape = case(name)
    return engine.ReprojectOp._tile((st, src_shape, CRS), (dt, dshape, CRS))


def tile_mixes(b, tile):
    """Whether some CTA tile holds both a box its own thread sums and one the whole CTA sums."""
    ty, tx = tile
    ny, nx = b.n.shape
    for i0 in range(0, ny, ty):
        for j0 in range(0, nx, tx):
            n = b.n[i0:i0 + ty, j0:j0 + tx]
            if ((n > 0) & (n <= RP_SMALL)).any() and (n > RP_SMALL).any():
                return True
    return False


def _clipped(b):
    ny, nx = b.src_shape
    inside = b.n > 0
    return {"left": (inside & (b.u0 < 0)).any(), "right": (inside & (b.u1 > nx)).any(),
            "top": (inside & (b.v0 < 0)).any(), "bottom": (inside & (b.v1 > ny)).any(),
            "empty": (b.n == 0).any()}


CTA = lambda b: b.n > RP_SMALL  # noqa: E731

# (what the row proves, the case, the predicate on its boxes)
REACH = [
    ("a 31-pixel box (one thread)", "n31_32", lambda b: (b.n == 31).any()),
    ("a 32-pixel box (one thread, the threshold)", "n31_32", lambda b: (b.n == 32).any()),
    ("a 32-pixel box beside 33-pixel ones", "n32_33", lambda b: (b.n == 32).any()),
    ("a 33-pixel box (the CTA)", "n32_33", lambda b: (b.n == 33).any()),
    ("a 33-pixel box, south-up destination", "n32_33_south", lambda b: (b.n == 33).any()),
    ("boxes of more than 256 pixels", "w255_256", lambda b: (b.n > RP_THREADS).all()),
    ("boxes of about 5e4 pixels", "n5e4", lambda b: ((b.n > 4.5e4) & (b.n < 5.5e4)).all()),
    ("w == 1 in the CTA", "tall", lambda b: (CTA(b) & (b.w == 1)).any()),
    ("w == 255 in the CTA", "w255_256", lambda b: (CTA(b) & (b.w == 255)).any()),
    ("w == 256 in the CTA", "w255_256", lambda b: (CTA(b) & (b.w == 256)).any()),
    ("w == 256, a second case", "w256_257", lambda b: (CTA(b) & (b.w == 256)).any()),
    ("w == 257 in the CTA", "w256_257", lambda b: (CTA(b) & (b.w == 257)).any()),
    ("w >= 300 in the CTA", "w312", lambda b: (CTA(b) & (b.w >= 300)).all()),
    ("h > 256 with w < 8", "tall", lambda b: ((b.h > 256) & (b.w < 8)).all()),
    ("boxes clipped at every source edge, and cells outside", "clipped", lambda b: all(_clipped(b).values())),
    ("one box larger than the whole source", "beyond",
     lambda b: b.u0[0, 0] < 0 and b.v0[0, 0] < 0 and b.u1[0, 0] > b.src_shape[1] and b.v1[0, 0] > b.src_shape[0]
     and b.n[0, 0] == b.src_shape[0] * b.src_shape[1]),
    ("a default tile mixing one-thread and CTA boxes", "n32_33", lambda b: tile_mixes(b, default_tile("n32_33"))),
    ("an 8 x 32 tile mixing them", "n31_32", lambda b: tile_mixes(b, (8, 32))),
    ("a 256 x 1 tile mixing them", "n32_33", lambda b: tile_mixes(b, (256, 1))),
]


@pytest.mark.parametrize("what,name,pred", REACH, ids=[r[0] for r in REACH])
def test_cases_reach_their_paths(what, name, pred):
    assert pred(case_boxes(name)), what


def test_exact_boxes_are_the_kernel_boxes():
    """The exact reference's box sizes are the kernel's (the same pixels), and no case leaves the
    fractional edges: both ends of both axes fall between pixel edges for some cell."""
    for name in CASES:
        src_shape, st, dt, dshape = case(name)
        b = kernel_boxes(st, src_shape, dt, dshape)
        wy = overlaps(st[5], st[4], src_shape[0], dt[5], dt[4], dshape[0])
        wx = overlaps(st[2], st[0], src_shape[1], dt[2], dt[0], dshape[1])
        np.testing.assert_array_equal((wy > 0).sum(1)[:, None] * (wx > 0).sum(1)[None, :], b.n, err_msg=name)
        for t in (b.u0, b.u1, b.v0, b.v1):
            assert (t != np.round(t)).any(), name


def values_for(rng, shape, dtype=np.float64, lo=-40, hi=40, nan=0.0):
    v = rng.integers(lo, hi + 1, shape).astype(dtype)
    if nan:
        v[rng.random(shape) < nan] = np.nan
    return v


@pytest.mark.parametrize("south_up", [False, True])
@pytest.mark.parametrize("name", ["clipped", "beyond", "n31_32"])
def test_exact_reference_equals_oracle(name, south_up):
    """The exact reference is the oracle's semantics: to 1e-15 for the average, exactly for nearest."""
    src_shape, args = CASES[name]
    st, dt, dshape = dyadic(*args[:6], south_up)
    rng = np.random.default_rng(11)
    v = values_for(rng, (2,) + src_shape, nan=0.05)
    v[v == 7.0] = -9999.0
    for nodata, empty in ((None, np.nan), (-9999.0, -1.0)):
        want = RO.reproject(v, st, CRS, dt, CRS, dshape, 5, nodata, empty)
        got = exact_average(v, st, dt, dshape, nodata, empty)
        assert np.array_equal(np.isnan(got), np.isnan(want))
        np.testing.assert_allclose(got, want, rtol=1e-15, atol=0)
        got = exact_nearest(v, st, dt, dshape, nodata, empty)
        assert np.array_equal(got, RO.reproject(v, st, CRS, dt, CRS, dshape, 0, nodata, empty), equal_nan=True)


def test_exact_division_is_the_rational():
    """S / W of the float64 integers is float(Fraction(S, W)) (a correctly rounded division)."""
    src_shape, st, dt, dshape = case("clipped")
    v = values_for(np.random.default_rng(12), src_shape, nan=0.1)
    s, w = exact_sums(v, st, dt, dshape)
    got = exact_average(v, st, dt, dshape)
    for k in zip(*np.nonzero(w[0])):
        assert got[k] == float(Fraction(int(s[0][k]), int(w[0][k])))


# ---------------------------------------------------------------- launch shapes

def batch_grid_y(batch, n_ctas, sms):
    """gridDim.y of atl_reproject (reproject.cu's batch_chunks)."""
    want = (32 * sms + n_ctas - 1) // max(n_ctas, 1)
    return max(1, min(want, batch, 65535))


def walk_batch(n_ctas, sms):
    """A batch that makes every CTA of a launch over ``n_ctas`` blocks walk at least 3 entries."""
    return 3 * batch_grid_y(1 << 30, n_ctas, sms) + 1


def avg_ctas(dshape, tile):
    return -(-dshape[0] // tile[0]) * -(-dshape[1] // tile[1])


WALK = ((0.375, 31.875, 40, 0.25, 0.875, 24), (22, 1276))  # n32_33 geometry over 24 x 40 cells
NEAREST_WALK = ((0.125, 0.375, 512, 0.25, 0.375, 256), (97, 193))  # 131072 cells, 512 blocks


def walk_tiles():
    st, dt, dshape = dyadic(*WALK[0])
    return [(1, 1), engine.ReprojectOp._tile((st, WALK[1], CRS), (dt, dshape, CRS))]


@pytest.mark.parametrize("sms", [132, 114])
def test_walk_launches_walk_the_batch(sms):
    """The batch-walk cases launch fewer y blocks than entries, so each CTA takes 3 or more; the
    average case's default tile mixes one-thread and CTA boxes."""
    st, dt, dshape = dyadic(*WALK[0])
    b = kernel_boxes(st, WALK[1], dt, dshape)
    for tile in walk_tiles():
        n_ctas = avg_ctas(dshape, tile)
        batch = walk_batch(n_ctas, sms)
        gy = batch_grid_y(batch, n_ctas, sms)
        assert gy < batch and (batch - gy) // gy + 1 >= 3, (tile, gy, batch)
        assert (b.n > RP_SMALL).mean() > 0.5 and tile_mixes(b, tile) == (tile != (1, 1))
    st, dt, dshape = dyadic(*NEAREST_WALK[0])
    blocks = -(-dshape[0] * dshape[1] // RP_THREADS)
    batch = walk_batch(blocks, sms)
    gy = batch_grid_y(batch, blocks, sms)
    assert blocks > sms and (batch - gy) // gy + 1 >= 3


# ---------------------------------------------------------------- GPU: k_reproject_avg on the identity pair

def run_identity(v, st, dt, dshape, resampling=5, nodata=None, empty=np.nan, tile=None):
    import torch

    op = engine.ReprojectOp((st, v.shape[-2:], CRS), (dt, dshape, CRS), resampling, nodata, empty, tile=tile)
    t = torch.from_numpy(np.ascontiguousarray(v.reshape((-1,) + v.shape[-2:]))).cuda()
    return op(t).cpu().numpy().reshape(v.shape[:-2] + tuple(dshape))


def assert_bitwise(got, want, what=""):
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype, got.shape, want.shape)
    same = (got == want) | (np.isnan(got) & np.isnan(want))
    if not same.all():
        k = tuple(int(i) for i in np.argwhere(~same)[0])
        raise AssertionError(f"{what}: {int((~same).sum())} of {same.size} values differ; first at {k}: "
                             f"got {got[k]!r}, want {want[k]!r}")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", list(CASES))
def test_average_boxes_bitwise(name, dtype):
    src_shape, st, dt, dshape = case(name)
    v = values_for(np.random.default_rng(20), (2,) + src_shape, dtype, nan=0.01)
    want = exact_average(v, st, dt, dshape, dtype=dtype)
    assert (~np.isnan(want)).sum() >= min(want.size, 2)
    assert_bitwise(run_identity(v, st, dt, dshape), want, name)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", ["n5e4", "n32_33", "w312"])
def test_average_nodata_in_cta_boxes(name, dtype):
    """Sparse NaN and nodata inside boxes the CTA sums; nodata = 3 also occurs as an ordinary value
    (every 3 is skipped); one CTA box entirely invalid gives dst_nodata = 5, which is also the mean
    of a cell of fives."""
    src_shape, st, dt, dshape = case(name)
    rng = np.random.default_rng(21)
    v = values_for(rng, (2,) + src_shape, dtype, lo=0, hi=9, nan=0.01)
    assert (v == 3.0).mean() > 0.05
    b = kernel_boxes(st, src_shape, dt, dshape)
    big = np.argwhere(b.n > RP_SMALL)
    wy = overlaps(st[5], st[4], src_shape[0], dt[5], dt[4], dshape[0])
    wx = overlaps(st[2], st[0], src_shape[1], dt[2], dt[0], dshape[1])

    def footprint(i, j):
        rows, cols = np.flatnonzero(wy[i]), np.flatnonzero(wx[j])
        return slice(rows[0], rows[-1] + 1), slice(cols[0], cols[-1] + 1)

    (i0, j0), (i1, j1) = big[len(big) // 2], big[-1]
    ry, cx = footprint(i0, j0)
    v[0, ry, cx] = np.where(rng.random(v[0, ry, cx].shape) < 0.5, np.nan, 3.0)  # no valid pixel
    ry, cx = footprint(i1, j1)
    v[1, ry, cx] = 5.0
    want = exact_average(v, st, dt, dshape, nodata=3.0, empty=5.0, dtype=dtype)
    assert want[0, i0, j0] == 5.0 and want[1, i1, j1] == 5.0
    assert not np.isnan(want).any()
    assert_bitwise(run_identity(v, st, dt, dshape, nodata=3.0, empty=5.0), want, name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n32_33", "clipped", "beyond", "w256_257", "tall"])
def test_average_tiles_bitwise(name):
    """Forced tiles, (1, 256) and (256, 1) filling the 514-entry corner buffer: the same bits."""
    src_shape, st, dt, dshape = case(name)
    v = values_for(np.random.default_rng(22), (3,) + src_shape, nan=0.02)
    want = exact_average(v, st, dt, dshape)
    for tile in ((1, 1), (1, 256), (256, 1), (16, 16), (8, 32), None):
        assert_bitwise(run_identity(v, st, dt, dshape, tile=tile), want, f"{name} tile {tile}")


def device_sms():
    import torch

    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_average_batch_walk(dtype):
    """Every CTA walks at least 3 entries whose values differ, so anything carried over from one
    entry to the next (the boxes, the CTA list, the reduction buffer) would show."""
    st, dt, dshape = dyadic(*WALK[0])
    sms = device_sms()
    for tile in walk_tiles():
        batch = walk_batch(avg_ctas(dshape, tile), sms)
        v = values_for(np.random.default_rng(23), (batch,) + WALK[1], dtype, nan=0.01)
        v += np.arange(batch, dtype=dtype)[:, None, None] % 50
        want = exact_average(v, st, dt, dshape, dtype=dtype)
        assert_bitwise(run_identity(v, st, dt, dshape, tile=tile), want, f"tile {tile}, batch {batch}")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_nearest_batch_walk(dtype):
    st, dt, dshape = dyadic(*NEAREST_WALK[0])
    blocks = -(-dshape[0] * dshape[1] // RP_THREADS)
    batch = walk_batch(blocks, device_sms())
    rng = np.random.default_rng(24)
    v = values_for(rng, (batch,) + NEAREST_WALK[1], dtype, lo=0, hi=9, nan=0.01)
    v += np.arange(batch, dtype=dtype)[:, None, None] * 10
    want = exact_nearest(v, st, dt, dshape, nodata=4.0, empty=-1.0).astype(dtype)
    assert (want == -1.0).any()
    assert_bitwise(run_identity(v, st, dt, dshape, resampling=0, nodata=4.0, empty=-1.0), want, f"batch {batch}")


# ---------------------------------------------------------------- k_regrid within one CRS

SPLIT = ((0.625, 63.375, 200, 0.375, 1.625, 20), (34, 12700))  # kx 64 / 65 over 200 columns
PHASE = ((0.625, 5.375, 37, 0.25, 1.625, 18), (30, 203))
TINY = ((0.5, 2.375, 2, 0.125, 1.75, 2), (4, 6))
WIDE = ((0.25, 5000.375, 3, 0.5, 1.5, 3), (6, 15002))  # cells of about 5000 columns


def regrid_ctiles(xtab):
    """(column tiles, tile width) atl_regrid_create chooses for ``xtab`` (regrid.cu): as few tiles as
    RG_THREADS allows, more until the x weights and the row ring fit; None when no width fits."""
    first, count, w = xtab
    nx, kx = len(first), w.shape[1]
    for n_ct in range(max(1, -(-nx // RG_THREADS)), max(nx, 1) + 1):
        tj = -(-nx // n_ct)
        span = 1
        for t in range(n_ct):
            c = count[t * tj:(t + 1) * tj] > 0
            if c.any():
                f, n = first[t * tj:(t + 1) * tj][c], count[t * tj:(t + 1) * tj][c]
                span = max(span, int((f + n).max() - f.min()))
        if (kx * tj * 8 + 15) // 16 * 16 + 4 * ((span * 8 + 15) // 16 * 16 + 16) <= 160 << 10:
            return n_ct, tj
    return None


@pytest.mark.parametrize("geom", [SPLIT, PHASE, TINY, WIDE], ids=["split", "phase", "tiny", "wide"])
@pytest.mark.parametrize("south_up", [False, True])
def test_same_crs_tables_are_exact_overlaps(geom, south_up):
    """gis.reproject's same-CRS tables hold exactly the rational overlaps (multiples of 1/8)."""
    st, dt, dshape = dyadic(*geom[0], south_up)
    for tab, (s0, ss, n, d0, ds, m) in zip(gis._same_crs_tables(st, geom[1], dt, dshape, False),
                                           ((st[5], st[4], geom[1][0], dt[5], dt[4], dshape[0]),
                                            (st[2], st[0], geom[1][1], dt[2], dt[0], dshape[1]))):
        first, count, w = tab
        want = overlaps(s0, ss, n, d0, ds, m)
        got = np.zeros_like(want)
        for k in range(m):
            got[k, first[k]:first[k] + count[k]] = w[k, :count[k]] * 8
            assert (w[k, :count[k]] > 0).all() and (w[k, count[k]:] == 0).all()
        np.testing.assert_array_equal(got, want)


def test_split_and_ring_limits():
    """The split case needs more column tiles than RG_THREADS alone gives; the phase and tiny cases
    do not; the 5000-column cells fit no tile, and ring_fits says so."""
    for geom, split in ((SPLIT, True), (PHASE, False), (TINY, False)):
        st, dt, dshape = dyadic(*geom[0])
        _, xtab = gis._same_crs_tables(st, geom[1], dt, dshape, False)
        n_ct, _ = regrid_ctiles(xtab)
        assert (n_ct > -(-dshape[1] // RG_THREADS)) == split and engine.RegridOp.ring_fits(xtab)
    st, dt, dshape = dyadic(*SPLIT[0])
    assert gis._same_crs_tables(st, SPLIT[1], dt, dshape, False)[1][2].shape[1] in (64, 65)
    st, dt, dshape = dyadic(*WIDE[0])
    _, xtab = gis._same_crs_tables(st, WIDE[1], dt, dshape, False)
    assert regrid_ctiles(xtab) is None and not engine.RegridOp.ring_fits(xtab)


def _one_cell(span):
    return (np.zeros(1, np.int32), np.full(1, span, np.int32), np.ones((1, span)))


def test_ring_fits_is_atl_regrid_create():
    """The host rule and the plan agree at the boundary: 4094 columns fit, 4095 do not, and the plan
    refuses the latter before any device work."""
    assert engine.RegridOp.ring_fits(_one_cell(4094)) and regrid_ctiles(_one_cell(4094)) == (1, 1)
    assert not engine.RegridOp.ring_fits(_one_cell(4095)) and regrid_ctiles(_one_cell(4095)) is None
    n0 = _lib.launch_count()
    with pytest.raises(_lib.AtlError, match="a destination cell spans more source columns than shared memory holds"):
        engine.RegridOp((1, 4095), _one_cell(1), _one_cell(4095), device=0)
    assert _lib.launch_count() == n0


def test_wide_cells_take_the_identity_pair(monkeypatch):
    """Within one CRS, cells wider than k_regrid's ring go to atl_reproject's identity pair, decided
    before any device work; narrower cells keep k_regrid."""
    calls = []

    class Stop(Exception):
        pass

    def record(kind):
        def make(*a, **k):
            calls.append(kind)
            raise Stop

        return make

    monkeypatch.setattr(engine.RegridOp, "__init__", record("regrid"))
    monkeypatch.setattr(engine.ReprojectOp, "__init__", record("reproject"))
    for geom, resampling, kind in ((WIDE, 5, "reproject"), (SPLIT, 5, "regrid"), (WIDE, 0, "regrid")):
        st, dt, dshape = dyadic(*geom[0])  # nearest tables have one column per cell
        with pytest.raises(Stop):
            gis.reproject(np.zeros(geom[1]), dt, CRS, dshape, src_transform=st, src_crs=CRS, resampling=resampling)
        assert calls == [kind]
        calls.clear()


def test_regrid_keeps_its_limit():
    """gis.regrid has no fallback: cells spanning more columns than the ring holds raise the plan's
    error, before any launch."""
    import pandas as pd

    import atlite_b200 as ab

    xs, ys = np.arange(9000) + 0.5, np.arange(4) + 0.5
    da = ab.DataArray(np.ones((4, 9000)), {"y": ys, "x": xs}, ("y", "x"))
    n0 = _lib.launch_count()
    with pytest.raises(_lib.AtlError, match="a destination cell spans more source columns than shared memory holds"):
        gis.regrid(da, pd.Index([2500.0, 7500.0], name="x"), pd.Index([1.0, 3.0], name="y"), resampling=5)
    assert _lib.launch_count() == n0


@pytest.mark.gpu
def test_regrid_split_tiles_bitwise():
    import torch

    st, dt, dshape = dyadic(*SPLIT[0])
    tables = gis._same_crs_tables(st, SPLIT[1], dt, dshape, False)
    op = engine.RegridOp(SPLIT[1], *tables)
    assert (op.info["n_ctiles"], op.info["tile_cols"]) == regrid_ctiles(tables[1])
    assert op.info["n_ctiles"] > -(-dshape[1] // RG_THREADS)
    v = values_for(np.random.default_rng(30), (2,) + SPLIT[1], nan=0.01)
    want = exact_average(v, st, dt, dshape)
    got, _ = gis.reproject(torch.from_numpy(v).cuda(), dt, CRS, dshape, src_transform=st, src_crs=CRS, resampling=5)
    assert_bitwise(got.cpu().numpy(), want, "split")
    assert_bitwise(op(v), want, "split, RegridOp")


@pytest.mark.gpu
def test_ring_limit_on_the_device():
    engine.RegridOp((1, 4094), _one_cell(1), _one_cell(4094))
    with pytest.raises(_lib.AtlError, match="a destination cell spans more source columns than shared memory holds"):
        engine.RegridOp((1, 4095), _one_cell(1), _one_cell(4095))


def phase_view(base, off, nx):
    """``base[..., off:off + nx]`` and the 16-byte phase (in elements) of its first row."""
    view = base[..., off:off + nx]
    return view, (view.data_ptr() % 16) // view.element_size()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_regrid_strided_phases(dtype):
    """Strided source views at every 16-byte phase; the row stride is odd, so later rows take the
    other phases too."""
    import torch

    st, dt, dshape = dyadic(*PHASE[0])
    ny, nx = PHASE[1]
    per = 16 // np.dtype(dtype).itemsize
    v = values_for(np.random.default_rng(31), (2, ny, nx + per + 5), dtype, nan=0.02)
    base = torch.from_numpy(v).cuda()
    for off in range(per):
        view, phase = phase_view(base, off, nx)
        assert phase == off and view.stride(1) > nx
        want = exact_average(v[..., off:off + nx], st, dt, dshape, dtype=dtype)
        got, _ = gis.reproject(view, dt, CRS, dshape, src_transform=st, src_crs=CRS, resampling=5)
        assert_bitwise(got.cpu().numpy(), want, f"offset {off}")


@pytest.mark.gpu
def test_regrid_int16_window_phases():
    import torch

    st, dt, dshape = dyadic(*PHASE[0])
    ny, nx = PHASE[1]
    rng = np.random.default_rng(32)
    v = rng.integers(-20, 21, (ny, nx + 8 + 3)).astype(np.int16)
    v[rng.random(v.shape) < 0.03] = -32767
    op = engine.RegridOp(PHASE[1], *gis._same_crs_tables(st, PHASE[1], dt, dshape, False))
    base = torch.from_numpy(v).cuda()
    for off in range(8):
        view, phase = phase_view(base, off, nx)
        assert phase == off
        want = exact_int16(v[:, off:off + nx], st, dt, dshape, -32767)
        assert_bitwise(op.window(view, fill=-32767).cpu().numpy(), want, f"offset {off}")


@pytest.mark.gpu
def test_regrid_batch_beyond_grid_y():
    """70 000 entries: the grid has 65535 y blocks, so the first ones take a second entry.  Entry b
    holds b + a fixed pattern, so each mean carries its index."""
    import torch

    st, dt, dshape = dyadic(*TINY[0])
    batch = 70_000
    pattern = values_for(np.random.default_rng(33), TINY[1], lo=-3, hi=3)
    v = np.arange(batch, dtype=np.float64)[:, None, None] + pattern
    want = exact_average(v, st, dt, dshape)
    assert np.array_equal(np.floor(want[:, 0, 0] - want[0, 0, 0] + 0.5), np.arange(batch))
    got, _ = gis.reproject(torch.from_numpy(v).cuda(), dt, CRS, dshape, src_transform=st, src_crs=CRS, resampling=5)
    assert_bitwise(got.cpu().numpy(), want, "70000 entries")


class RowReader:
    """A host window read row band by row band, like ingest.GridWindow."""

    def __init__(self, values):
        self.values, self.shape, self.dtype, self.reads = values, values.shape, values.dtype, []

    def read(self, lo, hi, out):
        self.reads.append((lo, hi))
        out[...] = self.values[lo:hi]


@pytest.mark.gpu
def test_terrain_window_in_bands(monkeypatch):
    """A GEBCO-style int16 window at a split-tile width, streamed from a host reader in bands that
    start below row 0, with fill values, a cell of fill values only, and exact .5 ties both ways."""
    ny_dst = 40
    geom = SPLIT[0][:5] + (ny_dst,)
    src_shape = (68, SPLIT[1][1])
    st, dt, dshape = dyadic(*geom)
    rng = np.random.default_rng(34)
    v = rng.integers(-20, 21, src_shape).astype(np.int16)
    v[rng.random(src_shape) < 0.02] = -32767
    wy = overlaps(st[5], st[4], src_shape[0], dt[5], dt[4], dshape[0])
    wx = overlaps(st[2], st[0], src_shape[1], dt[2], dt[0], dshape[1])
    rows, cols = (lambda i, j: (np.flatnonzero(wy[i]), np.flatnonzero(wx[j])))(5, 7)
    v[rows[0]:rows[-1] + 1, cols[0]:cols[-1] + 1] = -32767  # a cell without a valid value
    for (i, j), pair in (((9, 11), (2, 3)), ((17, 40), (-2, -3)), ((30, 150), (6, 7))):  # means k + 1/2
        rows, cols = np.flatnonzero(wy[i]), np.flatnonzero(wx[j])
        v[rows[0]:rows[-1] + 1, cols[0]:cols[-1] + 1] = -32767
        v[rows[1], cols[1]:cols[3]] = pair  # two interior pixels of weight 1 x 1
    want = exact_int16(v, st, dt, dshape, -32767)
    s, w = exact_sums(v, st, dt, dshape, -32767)
    ties = (w > 0) & ((2 * s) % np.maximum(w, 1) == 0) & ((2 * s // np.maximum(w, 1)) % 2 == 1)
    assert (ties & (s > 0)).sum() >= 2 and (ties & (s < 0)).sum() >= 1 and (want == -32767).any()
    assert want[9, 11] == 3 and want[17, 40] == -3 and want[5, 7] == -32767

    op = engine.RegridOp(src_shape, *gis._same_crs_tables(st, src_shape, dt, dshape, False))
    assert op.info["n_ctiles"] > -(-dshape[1] // RG_THREADS)
    monkeypatch.setattr(engine.RegridOp, "WINDOW_SLAB_BYTES", 20 * src_shape[1] * 2)
    groups = op._window_bands(src_shape[1] * 2)
    assert len(groups) >= 3 and all(lo > 0 for _, _, lo, _ in groups[1:])
    reader = RowReader(v)
    got = op.window(reader, fill=-32767)
    assert [(lo, hi) for _, _, lo, hi in groups] == reader.reads
    assert_bitwise(got, want, "terrain window")


# ---------------------------------------------------------------- the same-CRS fallback

@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_wide_cells_bitwise(dtype):
    """Cells of about 5000 source columns, more than k_regrid's ring holds: gis.reproject gives the
    exact averages (it used to raise atl_regrid_create's error)."""
    import torch

    st, dt, dshape = dyadic(*WIDE[0])
    v = values_for(np.random.default_rng(40), (2,) + WIDE[1], dtype, nan=0.01)
    v[0, 2, 100:200] = -9999.0
    want = exact_average(v, st, dt, dshape, nodata=-9999.0, dtype=dtype)
    got, _ = gis.reproject(torch.from_numpy(v).cuda(), dt, CRS, dshape, src_transform=st, src_crs=CRS,
                           resampling=5, src_nodata=-9999.0, dst_nodata=np.nan)
    assert_bitwise(got.cpu().numpy(), want, "wide cells")
    host, _ = gis.reproject(v, dt, CRS, dshape, src_transform=st, src_crs=CRS, resampling=5, src_nodata=-9999.0,
                            dst_nodata=np.nan)
    assert_bitwise(host, want, "wide cells, host")


# ---------------------------------------------------------------- across CRSs at production scale

def production_case(src_crs):
    """A (3, 1500, 2000) float32 source of 250 m pixels about (10 E, 50 N) in ``src_crs``, and a
    0.25 degree EPSG:4326 grid that overhangs it."""
    x0, y0 = proj.transform(np.float64(10.0), np.float64(50.0), 4326, src_crs)
    st = (250.0, 0.0, float(x0) - 1000 * 250.0, 0.0, -250.0, float(y0) + 750 * 250.0)
    src_shape = (1500, 2000)
    lon, lat = proj.transform(st[2] + np.array([0, 2000, 0, 2000]) * 250.0,
                              st[5] - np.array([0, 0, 1500, 1500]) * 250.0, src_crs, 4326)
    w, e = math.floor(lon.min() * 4) / 4 - 0.25, math.ceil(lon.max() * 4) / 4 + 0.25
    s, n = math.floor(lat.min() * 4) / 4 - 0.25, math.ceil(lat.max() * 4) / 4 + 0.25
    dt = (0.25, 0.0, w, 0.0, -0.25, n)
    return st, src_shape, dt, (round((n - s) * 4), round((e - w) * 4))


def sample_windows(dshape, k=3):
    """k x k destination windows at the four corners, the middle of each edge and the centre."""
    ny, nx = dshape
    return [(i, j) for i in (0, (ny - k) // 2, ny - k) for j in (0, (nx - k) // 2, nx - k)]


@pytest.mark.parametrize("src_crs", [3035, MOLL])
def test_production_boxes(src_crs):
    st, src_shape, dt, dshape = production_case(src_crs)
    b = kernel_boxes(st, src_shape, dt, dshape, src_crs, 4326)
    n = b.n[b.n > 0]
    assert 5e3 < np.median(n) < 2e4 and (b.n == 0).any() and n.size > 100


@pytest.mark.gpu
@pytest.mark.parametrize("src_crs", [3035, MOLL])
def test_production_scale_against_oracle(src_crs):
    """float32 averages within 1e-9 of the float64 oracle before the cast: the result is the float32
    rounding of a value inside [want (1 - 1e-9), want (1 + 1e-9)]."""
    import torch

    st, src_shape, dt, dshape = production_case(src_crs)
    rng = np.random.default_rng(50)
    v = rng.uniform(0.5, 1.5, (3,) + src_shape).astype(np.float32)
    v[:, rng.random(src_shape) < 1e-3] = np.nan
    got, _ = gis.reproject(torch.from_numpy(v).cuda(), dt, 4326, dshape, src_transform=st, src_crs=src_crs,
                           resampling=5)
    got = got.cpu().numpy()
    assert got.dtype == np.float32
    k = 3
    n_valid = 0
    for i0, j0 in sample_windows(dshape, k):
        wt = (dt[0], 0.0, dt[2] + j0 * dt[0], 0.0, dt[4], dt[5] + i0 * dt[4])
        want = RO.reproject(v, st, src_crs, wt, 4326, (k, k), 5)
        g = got[:, i0:i0 + k, j0:j0 + k]
        assert np.array_equal(np.isnan(g), np.isnan(want)), (i0, j0)
        ok = ~np.isnan(want)
        lo = (want[ok] * (1 - 1e-9)).astype(np.float32)
        hi = (want[ok] * (1 + 1e-9)).astype(np.float32)
        assert ((g[ok] >= lo) & (g[ok] <= hi)).all(), (i0, j0)
        n_valid += ok.sum()
    assert n_valid >= 3 * 9 * 4
