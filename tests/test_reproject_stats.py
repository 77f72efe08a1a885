"""gis.reproject and gis.regrid statistics: sum, rms, min, max, med, q1, q3 and mode (rasterio's
Resampling 13, 14, 9, 8, 10, 11, 12, 6) over the average's boxes.

CPU: the oracle (oracle/reproject_stats_oracle.py) against the average oracle and hand-built cells,
and argument handling without a device, in Python and in the C entry.  GPU: every statistic on every
pair and regime of test_reproject.py against the oracle (min, max and the selections bitwise), the
dyadic sums of test_resample_footprints.py bit for bit, sum / count against the average on all three
paths, the one-thread and scratch tiers of the selections, scratch budgets, determinism, and a
production-sized footprint.
"""

import ctypes as C
import math

import numpy as np
import pandas as pd
import pytest

import reproject_oracle as RO
import reproject_stats_oracle as SO
from atlite_b200 import _lib, engine, gis
from atlite_b200.labelled import DataArray, LazyDataset
from test_reproject import MOLL, PAIRS, REGIMES, _case, _no_device
from test_resample_footprints import CASES, CRS, case, exact_sums, kernel_boxes, values_for

STATS = {"sum": 13, "rms": 14, "min": 9, "max": 8, "med": 10, "q1": 11, "q3": 12, "mode": 6}
EXACT = ("min", "max", "med", "q1", "q3", "mode")


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def assert_stat(got, want, name, dtype, wsum=None):
    """min, max and the selections bitwise (the sign of zero included); sum and rms to 1e-12 in float64
    and to one float32 rounding of the float64 value in float32.  ``wsum``: the cells' weights (sum
    over a field of ones) across CRSs, where the device's projection and NumPy's differ in the last
    bits of a corner's pixel coordinate, which moves a weight by up to about 1e-11 absolutely (the
    average's tests allow 1e-9 for the same reason); a cell of total weight W gets 2e-11 / W more
    relative tolerance."""
    got = _np(got)
    assert got.dtype == dtype and got.shape == want.shape
    assert np.array_equal(np.isnan(got), np.isnan(want)), name
    ok = ~np.isnan(got)
    if name in EXACT:
        w = want.astype(dtype)
        assert np.array_equal(got[ok].view(f"u{got.itemsize}"), w[ok].view(f"u{w.itemsize}")), name
        return
    if dtype == np.float64:
        ws = np.ones(got.shape) if wsum is None else np.broadcast_to(wsum, got.shape)
        rtol = 1e-12 + np.where(ws[ok] > 0, 2e-11 / np.where(ws[ok] > 0, ws[ok], 1.0), 0.0) * (wsum is not None)
        assert (np.abs(got[ok] - want[ok]) <= rtol * np.abs(want[ok])).all(), name
    else:
        w32 = want[ok].astype(np.float32)
        assert (np.abs(got[ok].astype(np.float64) - w32) <= np.spacing(np.abs(w32))).all(), name


def holes(v, nodata=-9999.0):
    """NaN and nodata holes, a block of cells without a valid pixel, and signed zeros."""
    v = v.copy()
    v[..., ::7, ::5] = np.nan
    v[..., 1::6, ::4] = nodata
    ny, nx = v.shape[-2:]
    v[..., ny // 3:ny // 2, nx // 3:nx // 2] = nodata
    v[..., ::11, 2::3] = -0.0
    v[..., 3::13, 1::3] = 0.0
    return v


def quantised(rng, shape):
    """Values on a grid of eighths, so equal values recur and the selections meet ties."""
    return np.round(rng.uniform(0.5, 1.5, shape) * 8.0) / 8.0


# ---------------------------------------------------------------- CPU: the oracle

def test_oracle_sum_over_count_is_the_average():
    rng = np.random.default_rng(1)
    for src, dst, regime in ((4326, 3035, "down"), (3035, 4326, "up"), (MOLL, 4326, "down")):
        v, st, dt, dshape = _case(src, dst, regime, False, lead=())
        v[::5, ::3] = np.nan
        v = v + rng.uniform(-0.1, 0.1, v.shape)
        ones = np.where(np.isnan(v), np.nan, 1.0)
        s = SO.reproject(v, st, src, dt, dst, dshape, SO.SUM)
        n = SO.reproject(ones, st, src, dt, dst, dshape, SO.SUM)
        want = RO.reproject(v, st, src, dt, dst, dshape, 5)
        assert np.array_equal(np.isnan(s), np.isnan(want))
        np.testing.assert_allclose(s / n, want, rtol=1e-12, atol=0)


def test_oracle_hand_built_cells():
    one = np.ones(4)
    v = np.array([1.0, 2.0, 3.0, 4.0])
    # equal weights: each quantile threshold is hit exactly at a value
    assert SO.cell_stat(v, one, SO.Q1) == 1.0 and SO.cell_stat(v, one, SO.MED) == 2.0
    assert SO.cell_stat(v, one, SO.Q3) == 3.0
    # a threshold met with equality by the heavier half
    assert SO.cell_stat(np.array([5.0, 1.0]), np.array([0.5, 0.5]), SO.MED) == 1.0
    assert SO.cell_stat(np.array([5.0, 1.0]), np.array([0.5, 0.5 + 2.0 ** -30]), SO.MED) == 1.0
    assert SO.cell_stat(np.array([5.0, 1.0]), np.array([0.5 + 2.0 ** -30, 0.5]), SO.MED) == 5.0
    # mode: ties go to the smaller value; weights count, not pixels
    assert SO.cell_stat(np.array([5.0, 3.0, 5.0, 3.0]), one, SO.MODE) == 3.0
    assert SO.cell_stat(np.array([5.0, 3.0, 5.0]), np.array([0.5, 0.75, 0.5]), SO.MODE) == 5.0
    # -0.0 counts as +0.0 in the selections; min and max keep the sign
    z = SO.cell_stat(np.array([-0.0, 0.0, 1.0]), np.array([1.0, 1.0, 1.5]), SO.MODE)
    assert z == 0.0 and math.copysign(1.0, z) == 1.0
    z = SO.cell_stat(np.array([-0.0, 1.0]), np.array([1.0, 0.5]), SO.MED)
    assert z == 0.0 and math.copysign(1.0, z) == 1.0
    assert math.copysign(1.0, SO.cell_stat(np.array([0.0, -0.0, 1.0]), np.ones(3), SO.MIN)) == -1.0
    assert math.copysign(1.0, SO.cell_stat(np.array([0.0, -0.0, -1.0]), np.ones(3), SO.MAX)) == 1.0
    # pixels with q = 0 take no part; a cell of them only gets dst_nodata
    tiny = 2.0 ** -42
    assert SO.weight_q([tiny, 2.0 ** -41, 1.0]) == [0, 1, 2 ** 40]
    assert SO.cell_stat(np.array([7.0]), np.array([tiny]), SO.MED) is None
    assert SO.cell_stat(np.array([7.0, 9.0]), np.array([tiny, 1.0]), SO.MODE) == 9.0
    assert SO.cell_stat(np.array([7.0]), np.array([tiny]), SO.SUM) == 7.0 * tiny  # sum keeps every weight
    # NaN and nodata are not valid; sum and rms
    assert SO.cell_stat(np.array([np.nan, -1.0]), np.ones(2), SO.MIN, src_nodata=-1.0) is None
    assert SO.cell_stat(np.array([3.0, 4.0]), np.array([0.5, 0.5]), SO.RMS) == math.sqrt(12.5)
    assert SO.cell_stat(np.array([3.0, 4.0]), np.array([0.5, 0.25]), SO.SUM) == 2.5


# ---------------------------------------------------------------- CPU: arguments

class _Boom:
    def __init__(self, *a, **k):
        raise AssertionError("reached the device")

    tables = classmethod(lambda cls, *a, **k: cls())
    ring_fits = staticmethod(lambda xtab: True)


def test_new_codes_pass_validation(monkeypatch):
    monkeypatch.setattr(engine, "ReprojectOp", _Boom)
    monkeypatch.setattr(engine, "RegridOp", _Boom)
    v = np.ones((4, 5))
    st, dt = (1.0, 0.0, 0.0, 0.0, -1.0, 4.0), (2.0, 0.0, 0.0, 0.0, -2.0, 4.0)
    da = DataArray(np.ones((4, 4)), {"y": np.arange(4.0), "x": np.arange(4.0)}, ("y", "x"), "v", {})
    cx, cy = pd.Index([0.5, 2.5], name="x"), pd.Index([0.5, 2.5], name="y")
    for code in STATS.values():
        for dst in (4326, 3035):
            with pytest.raises(AssertionError, match="reached the device"):
                gis.reproject(v, dt, dst, (2, 2), src_transform=st, src_crs=4326, resampling=code)
        with pytest.raises(AssertionError, match="reached the device"):
            gis.regrid(da, cx, cy, resampling=np.int64(code))


def test_refused_codes(monkeypatch):
    _no_device(monkeypatch)
    v = np.ones((4, 5))
    st, dt = (1.0, 0.0, 0.0, 0.0, -1.0, 4.0), (2.0, 0.0, 0.0, 0.0, -2.0, 4.0)
    da = DataArray(np.ones((4, 4)), {"y": np.arange(4.0), "x": np.arange(4.0)}, ("y", "x"), "v", {})
    cx, cy = pd.Index([0.5, 2.5], name="x"), pd.Index([0.5, 2.5], name="y")
    for code in (1, 2, 3, 4, 7, True, 15, -1, 13.0):
        with pytest.raises(NotImplementedError, match="resampling"):
            gis.reproject(v, dt, 4326, (2, 2), src_transform=st, src_crs=4326, resampling=code)
        with pytest.raises(NotImplementedError, match=r"0 \(nearest\) or 5 \(average\)"):
            gis.regrid(da, cx, cy, resampling=code)
    with pytest.raises(TypeError, match="float32 and float64"):
        gis.reproject(v.astype(np.int32), dt, 4326, (2, 2), src_transform=st, src_crs=4326, resampling=13)


def _err():
    return _lib.load().atl_last_error().decode()


def _c_call(resampling=13, spans=None, select_small=-1):
    lib = _lib.load()
    op = engine.ReprojectOp(((1.0, 0.0, 0.0, 0.0, -1.0, 4.0), (4, 5), 4326),
                            ((2.0, 0.0, 0.0, 0.0, -2.0, 4.0), (2, 2), 4326), resampling, tile=(8, 32))
    o = _lib.ReprojectOptions()
    o.select_small, keep = select_small, []
    if spans is not None:
        rows, cols = ((_lib.Span * 2)(*[_lib.Span(*s) for s in sp]) for sp in spans)
        keep += [rows, cols]
        o.row_spans, o.col_spans = C.addressof(rows), C.addressof(cols)
    # NULL source: the descriptor and the options are checked before the pointers and the device
    return lib.atl_reproject_ex(0, C.byref(op.desc), C.byref(o), 1, 1, None, 5, 20, None, None)


def test_c_entry_checks_its_arguments():
    good = ((0, 2, 1.0, 1.0), (2, 4, 1.0, 0.5))
    assert _c_call(13) == -1 and "NULL" in _err()  # every check above the pointers passed
    for code in (1, 2, 3, 4, 7, 15):
        assert _c_call(code) == -1 and "resampling" in _err()
    assert _c_call(10, select_small=33) == -1 and "select_small" in _err()
    assert _c_call(10, spans=(good, ((0, 2, 1.0, 1.0), (3, 6, 1.0, 1.0)))) == -1 and "spans" in _err()
    assert _c_call(10, spans=(good, ((0, 2, 1.0, 0.0), (2, 4, 1.0, 1.0)))) == -1 and "spans" in _err()
    assert _c_call(0, spans=(good, good)) == -1 and "nearest" in _err()
    assert _c_call(10, spans=(good, good)) == -1 and "NULL" in _err()


def test_regrid_tables_are_boxes():
    """regrid's padded average tables have weight 1 between their ends, so they are boxes."""
    for pad in (0, 3):
        first, count, w = gis.regrid_axis(0.125, 0.25, 40, 0.3, 1.1, 12, pad)
        for k in range(len(first)):
            assert (w[k, 1:max(count[k] - 1, 1)] == 1.0).all()
    spans = engine.ReprojectOp._spans(gis.regrid_axis(0.125, 0.25, 40, -0.5, 1.1, 12, 3))
    assert spans[0].lo == 0 and spans[0].w_lo > 1.0  # padded pixels fold into the border pixel


# ---------------------------------------------------------------- GPU

def _all_stats(v, st, src, dt, dst, dshape, src_nodata, dst_nodata):
    """Every statistic from the oracle, and the cells' weights."""
    boxes = SO.corner_boxes(st, src, v.shape[-2:], dt, dst, dshape)
    ones = np.where(RO._skip(v.astype(np.float64), src_nodata), np.nan, 1.0)
    want = {name: SO.resample(v, boxes, dshape, code, src_nodata, dst_nodata) for name, code in STATS.items()}
    return want, SO.resample(ones, boxes, dshape, SO.SUM)


@pytest.mark.gpu
@pytest.mark.parametrize("south_up", [False, True], ids=["north", "south"])
@pytest.mark.parametrize("regime", list(REGIMES))
@pytest.mark.parametrize("src,dst", PAIRS, ids=[f"{a}-{b}" for a, b in PAIRS])
def test_pairs_against_oracle(src, dst, regime, south_up):
    import torch

    _, st, dt, dshape = _case(src, dst, regime, south_up)
    rng = np.random.default_rng(10)
    v = holes(quantised(rng, (2,) + REGIMES[regime][0]))
    for dtype in (np.float64, np.float32):
        vd = v.astype(dtype)
        want, wsum = _all_stats(vd, st, src, dt, dst, dshape, -9999.0, -1.0)
        assert (want["sum"] == -1.0).any() and (want["sum"] != -1.0).sum() > 0.3 * want["sum"].size
        for name, code in STATS.items():
            got, _ = gis.reproject(torch.from_numpy(vd).cuda(), dt, dst, dshape, src_transform=st, src_crs=src,
                                   resampling=code, src_nodata=-9999.0, dst_nodata=-1.0)
            assert got.is_cuda
            assert_stat(got, want[name], name, dtype, wsum)


@pytest.mark.gpu
@pytest.mark.parametrize("dst,box", [(MOLL, (-2.0e7, -1.0e7, 2.0e7, 1.0e7)), (3857, (-2.2e7, -1.2e7, 2.2e7, 1.2e7))],
                         ids=["mollweide-ellipse", "mercator-map"])
def test_cells_without_an_image(dst, box):
    rng = np.random.default_rng(6)
    v = quantised(rng, (36, 72))
    st = (5.0, 0.0, -180.0, 0.0, -5.0, 90.0)
    left, bottom, right, top = box
    dshape = (12, 22)
    dt = ((right - left) / dshape[1], 0.0, left, 0.0, -(top - bottom) / dshape[0], top)
    want, wsum = _all_stats(v, st, 4326, dt, dst, dshape, None, np.nan)
    assert np.isnan(want["max"]).sum() >= 4
    for name, code in STATS.items():
        got, _ = gis.reproject(v, dt, dst, dshape, src_transform=st, src_crs=4326, resampling=code)
        assert_stat(got, want[name], name, np.float64, wsum)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n31_32", "n32_33", "n32_33_south", "w256_257", "tall", "n5e4", "clipped", "beyond"])
def test_dyadic_sum_is_exact(name):
    """On dyadic geometry every weight is a multiple of 1/8, so 64 x the sum is an exact integer S
    and the sum must be S / 64 (float64) and its rounding (float32), bit for bit."""
    src_shape, st, dt, dshape = case(name)
    v = values_for(np.random.default_rng(3), (2,) + src_shape, nan=0.05)
    s, w = exact_sums(v, st, dt, dshape)
    want = np.where(w > 0, s / 64.0, np.nan).reshape((2,) + dshape)
    for dtype in (np.float64, np.float32):
        got, _ = gis.reproject(v.astype(dtype), dt, CRS, dshape, src_transform=st, src_crs=CRS, resampling=13)
        assert np.array_equal(got, want.astype(dtype), equal_nan=True), (name, dtype)
        op = engine.ReprojectOp((st, src_shape, CRS), (dt, dshape, CRS), 13)  # the box walk on the identity pair
        assert np.array_equal(op(v.astype(dtype)), want.astype(dtype), equal_nan=True), (name, dtype)


def _sum_over_count(run, v):
    ones = np.where(np.isnan(v), np.nan, 1.0)
    return _np(run(v, 13)) / _np(run(ones, 13)), _np(run(v, 5))


@pytest.mark.gpu
def test_sum_over_count_is_the_average():
    rng = np.random.default_rng(4)
    # across CRSs
    v, st, dt, dshape = _case(4326, 3035, "down", True, lead=(2,), seed=4)
    v[:, ::5, ::3] = np.nan
    a, b = _sum_over_count(lambda x, c: gis.reproject(x, dt, 3035, dshape, src_transform=st, src_crs=4326,
                                                      resampling=c)[0], v)
    assert np.array_equal(np.isnan(a), np.isnan(b))
    np.testing.assert_allclose(a, b, rtol=1e-12)
    # within one CRS (regrid's tables, and the identity pair)
    v, st, dt, dshape = _case(3035, 3035, "down", False, lead=(2,), seed=5)
    v[:, ::5, ::3] = np.nan
    a, b = _sum_over_count(lambda x, c: gis.reproject(x, dt, 3035, dshape, src_transform=st, src_crs=3035,
                                                      resampling=c)[0], v)
    assert np.array_equal(np.isnan(a), np.isnan(b))
    np.testing.assert_allclose(a, b, rtol=1e-12)
    # regrid, with edge padding
    src = rng.uniform(0.5, 1.5, (3, 40, 48))
    src[:, ::6, ::5] = np.nan
    xs, ys = np.arange(48) * 0.25 + 0.125, np.arange(40) * 0.25 + 0.125
    cx, cy = pd.Index(np.arange(-0.5, 13.0, 1.1), name="x"), pd.Index(np.arange(10.5, -0.6, -0.9), name="y")

    def run(x, c):
        da = DataArray(x, {"time": np.arange(3), "y": ys, "x": xs}, ("time", "y", "x"), "v", {})
        return gis.regrid(da, cx, cy, resampling=c).values

    a, b = _sum_over_count(run, src)
    assert np.array_equal(np.isnan(a), np.isnan(b)) and not np.isnan(b).all()
    np.testing.assert_allclose(a, b, rtol=1e-12)


def _run_op(op, v, **attrs):
    saved = {k: getattr(engine.ReprojectOp, k) for k in attrs}
    try:
        for k, x in attrs.items():
            setattr(engine.ReprojectOp, k, x)
        return _np(op(v))
    finally:
        for k, x in saved.items():
            setattr(engine.ReprojectOp, k, x)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n31_32", "n32_33", "n32_33_south", "n5e4", "clipped", "beyond"])
def test_selection_tiers_agree(name):
    """Boxes of at most 32 pixels are selected by their own thread, larger ones in scratch: forcing
    every box through the scratch, or a budget of a few cells per band, gives the same bits, which
    are the oracle's."""
    src_shape, st, dt, dshape = case(name)
    b = kernel_boxes(st, src_shape, dt, dshape)
    rng = np.random.default_rng(7)
    v = holes(values_for(rng, (2,) + src_shape, lo=-6, hi=6).astype(np.float64) / 4.0)
    boxes = SO.corner_boxes(st, CRS, src_shape, dt, CRS, dshape)
    for code in (SO.MED, SO.Q1, SO.Q3, SO.MODE):
        op = engine.ReprojectOp((st, src_shape, CRS), (dt, dshape, CRS), code, -9999.0, np.nan)
        base = _run_op(op, v)
        if b.n.max() < 2e4:
            want = SO.resample(v, boxes, dshape, code, -9999.0, np.nan)
            assert np.array_equal(base.view(np.uint64), want.view(np.uint64)), (name, code)
        for attrs in (dict(SELECT_SMALL=0), dict(SELECT_SCRATCH_BYTES=1), dict(SELECT_SMALL=0,
                                                                                SELECT_SCRATCH_BYTES=4096)):
            assert np.array_equal(_run_op(op, v, **attrs).view(np.uint64), base.view(np.uint64)), (name, code, attrs)


@pytest.mark.gpu
def test_a_box_of_a_million_pixels():
    import torch

    rng = np.random.default_rng(8)
    ny, nx = 1100, 1000
    v = np.round(rng.normal(0.0, 3.0, (ny, nx))).astype(np.float32)
    v[::9, ::7] = np.nan
    st = (1.0, 0.0, 0.0, 0.0, -1.0, float(ny))
    dt = (nx / 1.5, 0.0, 0.25, 0.0, -ny / 1.25, ny - 0.375)  # cell (0, 0) spans about 667 x 880 pixels
    dshape = (2, 2)
    boxes = SO.corner_boxes(st, 3035, (ny, nx), dt, 3035, dshape)
    rows, wy, cols, wx = boxes[0, 0]
    assert len(rows) * len(cols) >= 5.8e5
    st2 = (0.5, 0.0, 0.0, 0.0, -0.5, float(ny))  # the same raster at half the pixel size: 2.3e6 pixels in cell (0, 0)
    v2 = np.repeat(np.repeat(v, 2, axis=0), 2, axis=1)
    t2 = torch.from_numpy(v2).cuda()
    for code in (SO.MED, SO.Q3, SO.MODE, SO.MAX):
        got = gis.reproject(torch.from_numpy(v).cuda(), dt, 3035, dshape, src_transform=st, src_crs=3035,
                            resampling=code)[0].cpu().numpy()
        want = SO.resample(v, {(0, 0): boxes[0, 0]}, (1, 1), code)
        assert got[0, 0].view(np.uint32) == want[0, 0].view(np.uint32), code
        big = gis.reproject(t2, dt, 3035, dshape, src_transform=st2, src_crs=3035, resampling=code)[0]
        assert (big.cpu().numpy().view(np.uint32) == got.view(np.uint32)).all(), code  # 4 x the same weights


@pytest.mark.gpu
def test_deterministic_and_slab_independent(monkeypatch):
    import torch

    v, st, dt, dshape = _case(3035, 4326, "down", True, lead=(5,), seed=8)
    v = holes(np.round(v * 8.0) / 8.0)
    for code in STATS.values():
        kw = dict(src_transform=st, src_crs=3035, resampling=code, src_nodata=-9999.0)
        dev = gis.reproject(torch.from_numpy(v).cuda(), dt, 4326, dshape, **kw)[0].cpu().numpy()
        host = gis.reproject(v, dt, 4326, dshape, **kw)[0]
        again = gis.reproject(v, dt, 4326, dshape, **kw)[0]
        assert np.array_equal(dev, host, equal_nan=True) and np.array_equal(host, again, equal_nan=True), code
        for b in range(5):
            assert np.array_equal(gis.reproject(v[b], dt, 4326, dshape, **kw)[0], host[b], equal_nan=True), code
        with monkeypatch.context() as m:
            m.setattr(engine.ReprojectOp, "HOST_SLAB_BYTES", 1)
            m.setattr(engine.ReprojectOp, "SELECT_SCRATCH_BYTES", 50000)  # batch slabs and bands of cells
            assert np.array_equal(gis.reproject(v, dt, 4326, dshape, **kw)[0], host, equal_nan=True), code
            assert np.array_equal(gis.reproject(v, dt, 4326, dshape, **kw)[0], host, equal_nan=True), code
        for tile in ((1, 1), (8, 32)):
            op = engine.ReprojectOp((st, v.shape[1:], 3035), (dt, dshape, 4326), code, -9999.0, -9999.0, tile=tile)
            assert np.array_equal(op(v), host, equal_nan=True), (code, tile)


@pytest.mark.gpu
def test_production_footprints():
    """A 3035 raster of 200 m pixels (about 1.2e4 per cell) onto 0.25 degree cells: sampled cells
    against the oracle, the mode on an integer class field."""
    import torch

    from test_reproject import _bounds

    left, bottom, right, top = _bounds(3035, 4.9, 6.6, 46.9, 48.1)
    res = 200.0
    x0, y0 = math.floor(left / res) * res, math.ceil(top / res) * res
    shape = (int(math.ceil((y0 - bottom) / res)), int(math.ceil((right - x0) / res)))
    st = (res, 0.0, x0, 0.0, -res, y0)
    dt, dshape = (0.25, 0.0, 5.0, 0.0, 0.25, 47.0), (4, 6)  # south-up like a cutout
    rng = np.random.default_rng(11)
    cont = (rng.normal(8.0, 2.0, shape) + np.linspace(0.0, 3.0, shape[1])[None, :]).astype(np.float32)
    cont[rng.random(shape) < 0.01] = np.nan
    classes = rng.integers(1, 45, shape).astype(np.float32)
    classes[: shape[0] // 2, : shape[1] // 3] = 12.0 + (rng.random((shape[0] // 2, shape[1] // 3)) < 0.6)
    boxes = SO.corner_boxes(st, 3035, shape, dt, 4326, dshape)
    n = [len(r) * len(c) for r, _, c, _ in boxes.values()]
    assert min(n) > 8e3 and len(boxes) == 24
    sample = [(0, 0), (1, 4), (3, 5), (2, 2)]
    for field, codes in ((cont, STATS.values()), (classes, (SO.MODE,))):
        t = torch.from_numpy(field).cuda()
        for code in codes:
            got = gis.reproject(t, dt, 4326, dshape, src_transform=st, src_crs=3035, resampling=code)[0].cpu().numpy()
            want = SO.resample(field, {c: boxes[c] for c in sample}, dshape, code)
            for c in sample:
                name = next(k for k, x in STATS.items() if x == code)
                assert_stat(got[c][None], want[c][None], name, np.float32)


@pytest.mark.gpu
def test_regrid_lazy_dataset_with_padding():
    """regrid on a LazyDataset, one time part at a time, with destination cells overhanging the
    source (padded pixels repeat the border pixel): every statistic against the oracle on
    regrid_axis tables."""
    rng = np.random.default_rng(12)
    nt, ny, nx = 5, 24, 32
    values = holes(quantised(rng, (nt, ny, nx)), nodata=np.nan)
    xs, ys = np.arange(nx) * 0.25 + 2.125, np.arange(ny) * 0.25 + 40.125
    cx = pd.Index(np.arange(1.75, 10.5, 0.75), name="x")  # overhangs both ends
    cy = pd.Index(np.arange(46.5, 39.4, -0.5), name="y")  # descending, overhangs both ends
    coords = {"time": pd.date_range("2020-01-01", periods=nt, freq="h"), "y": ys, "x": xs}
    lazy = LazyDataset({"v": lambda lo, hi: values[lo:hi]}, coords, attrs={}, time_chunk=2,
                       dtypes={"v": np.dtype(np.float64)})
    pad = int(0.75 // 0.25 * 1.1)
    ytab = gis.regrid_axis(ys[0], 0.25, ny, cy[0], -0.5, len(cy), pad)
    xtab = gis.regrid_axis(xs[0], 0.25, nx, cx[0], 0.75, len(cx), pad)
    assert (xtab[2][:, 0] > 1.0).any() and (ytab[2][:, 0] > 1.0).any()  # padding folded in
    boxes = SO.table_boxes(ytab, xtab)
    for name, code in STATS.items():
        got = gis.regrid(lazy, cx, cy, resampling=code)
        want = SO.resample(values, boxes, (len(cy), len(cx)), code)
        assert_stat(np.asarray(got.raw("v")), want, name, np.float64)
