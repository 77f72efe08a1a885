"""gis.regrid: resampling onto another regular grid of the same CRS (reference gis.py:765-871).

CPU: argument errors, the oracle (oracle/regrid_oracle.py) against the reference's known answers
(test_gis.py::test_regrid), the separable per-axis weights against exact rational overlaps, and
those weights applied on the host against the cell-by-cell oracle.  GPU: the public call against
the known answers and the oracle, on host and device data, Datasets, odd dim orders and lazy
cutouts.
"""

from fractions import Fraction as Fr

import numpy as np
import pandas as pd
import pytest

import atlite_b200 as ab
import regrid_oracle as RO
from atlite_b200 import gis
from atlite_b200.labelled import DataArray, Dataset, LazyDataset

A, B, C, D = 0.25, 0.5, 0.3, 0.1


def _blocks():
    ones = np.ones((4, 4))
    return np.block([[ones * A, ones * B], [ones * C, ones * D]]), np.arange(0.5, 8, 1)


KNOWN = [  # (z layers or None, destination centres, target)
    (None, np.arange(2, 8, 4), np.array([[A, B], [C, D]])),
    (10, np.arange(2, 8, 4), np.stack([np.array([[A, B], [C, D]])] * 10)),
    (None, np.arange(1, 6, 2), np.array([[A, A, B], [A, A, B], [C, C, D]])),
]


def _axis(first, step, n):
    return first + step * np.arange(n)


# (name, source step, destination step, source (x0, y0, nx, ny), destination (x0, y0, nx, ny))
CASES = [
    ("0.05->0.25", 0.05, 0.25, (5.025, 45.025, 60, 40), (5.1, 45.1, 11, 7)),
    ("0.1->0.25", 0.1, 0.25, (5.05, 45.05, 30, 20), (5.2, 45.2, 11, 7)),
    ("0.05->0.3", 0.05, 0.3, (5.025, 45.025, 60, 40), (5.15, 45.15, 9, 6)),
    ("0.25->0.1", 0.25, 0.1, (5.125, 45.125, 12, 8), (5.05, 45.05, 29, 19)),
    ("beyond padding", 0.1, 0.25, (5.05, 45.05, 30, 20), (4.0, 44.0, 22, 16)),
]


def _case(case, rng, nt=3, flip_src_y=False, flip_dst_y=False):
    """Source centres, positive values (well-conditioned means) and destination centres of a case."""
    _, ss, ds_, (sx0, sy0, snx, sny), (dx0, dy0, dnx, dny) = case
    xs, ys = _axis(sx0, ss, snx), _axis(sy0, ss, sny)
    v = rng.uniform(0.5, 1.5, (nt, sny, snx))
    if flip_src_y:
        ys, v = ys[::-1].copy(), v[:, ::-1].copy()
    dimx, dimy = pd.Index(_axis(dx0, ds_, dnx), name="x"), pd.Index(_axis(dy0, ds_, dny), name="y")
    if flip_dst_y:
        dimy = pd.Index(dimy[::-1], name="y")
    return xs, ys, v, dimx, dimy


def _host_tables(xs, ys, dimx, dimy, nearest):
    """The separable tables regrid hands the kernel, as dense (n_dst, n_src) matrices."""
    flipx, flipy = xs[-1] < xs[0], ys[-1] < ys[0]
    xa, ya = (xs[::-1] if flipx else xs), (ys[::-1] if flipy else ys)
    sx0, sdx = gis.regular_axis(xa, "x")
    sy0, sdy = gis.regular_axis(ya, "y")
    dx0, ddx = gis._transform_axis(dimx, "x")
    dy0, ddy = gis._transform_axis(dimy, "y")
    pad = int(abs(ddx) // min(sdx, sdy) * 1.1)
    out = []
    for s0, sd, n, d0, dd, nd, flip in ((sy0, sdy, len(ys), dy0, ddy, len(dimy), flipy),
                                          (sx0, sdx, len(xs), dx0, ddx, len(dimx), flipx)):
        tab = gis.regrid_axis(s0, sd, n, d0, dd, nd, pad, nearest)
        if flip:
            tab = gis._flip_axis_table(tab, n)
        first, count, w = tab
        M = np.zeros((nd, n))
        for j in range(nd):
            M[j, first[j]:first[j] + count[j]] = w[j, :count[j]]
        out.append(M)
    return out


def _apply_tables(v, My, Mx):
    ok = ~np.isnan(v)
    num = np.einsum("iy,jx,...yx->...ij", My, Mx, np.where(ok, v, 0.0))
    den = np.einsum("iy,jx,...yx->...ij", My, Mx, ok.astype(np.float64))
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(den > 0, num / den, np.nan)


def _f32_within_ulp(got, want64):
    got = np.asarray(got)
    want = want64.astype(np.float32)
    assert got.dtype == np.float32 and got.shape == want.shape
    assert np.array_equal(np.isnan(got), np.isnan(want)), "NaN positions differ"
    ok = ~np.isnan(want)
    err = np.abs(got[ok].astype(np.float64) - want[ok].astype(np.float64))
    assert (err <= np.spacing(np.abs(want[ok]))).all(), f"more than 1 ulp off: max {err.max()}"


# ---------------------------------------------------------------- CPU

def _fine_da():
    fine, c = _blocks()
    return DataArray(fine, {"y": c, "x": c}, ("y", "x"))


def test_argument_errors():
    da = _fine_da()
    cx, cy = pd.Index([2.0, 6.0], name="x"), pd.Index([2.0, 6.0], name="y")
    with pytest.raises(NotImplementedError, match="0 \\(nearest\\) or 5 \\(average\\)"):
        gis.regrid(da, cx, cy, resampling=1)
    with pytest.raises(NotImplementedError, match="0 \\(nearest\\) or 5 \\(average\\)"):
        gis.regrid(da, cx, cy, resampling="average")
    with pytest.raises(NotImplementedError, match="one CRS"):
        gis.regrid(da, cx, cy, resampling=5, src_crs=4326, dst_crs=3035)
    with pytest.raises(NotImplementedError, match="one CRS"):
        gis.regrid(da, cx, cy, dst_crs="EPSG:3035")
    with pytest.raises(TypeError, match="resampling, src_crs and dst_crs"):
        gis.regrid(da, cx, cy, resampling=5, num_threads=4)
    mixed = Dataset({"a": (("y", "x"), np.zeros((8, 8))), "b": (("y", "x"), np.zeros((8, 8), np.float32))},
                    coords={"y": da.coords["y"], "x": da.coords["x"]})
    with pytest.raises(AssertionError, match="regrid can only reproject datasets with homogeneous dtype"):
        gis.regrid(mixed, cx, cy)
    with pytest.raises(TypeError, match="float32 and float64"):
        gis.regrid(DataArray(np.zeros((8, 8), np.int32), da.coords, ("y", "x")), cx, cy)
    with pytest.raises(ValueError, match="names no coordinate"):
        gis.regrid(da, pd.Index([2.0, 6.0], name="lon"), cy)
    with pytest.raises(ValueError, match=".name"):
        gis.regrid(da, pd.Index([2.0, 6.0]), cy)
    lacking = Dataset({"a": (("y", "x"), np.zeros((8, 8))), "t": (("time",), np.zeros(3))},
                      coords={"y": da.coords["y"], "x": da.coords["x"], "time": np.arange(3)})
    with pytest.raises(ValueError, match="lacks the dim"):
        gis.regrid(lacking, cx, cy)
    uneven = DataArray(np.zeros((8, 8)), {"y": da.coords["y"], "x": np.r_[0.5, 1.5, 2.5, 3.5, 4.5, 5.5, 6.5, 7.9]},
                       ("y", "x"))
    with pytest.raises(ValueError, match="must be ascending and evenly spaced"):
        gis.regrid(uneven, cx, cy)
    with pytest.raises(ValueError, match="must be ascending and evenly spaced"):
        gis.regrid(da, pd.Index([1.0, 2.0, 4.0], name="x"), cy)
    with pytest.raises(ValueError, match="single value"):
        gis.regrid(da, pd.Index([2.0], name="x"), cy)


@pytest.mark.parametrize("k", range(len(KNOWN)))
def test_oracle_known_answers(k):
    z, coarse, target = KNOWN[k]
    fine, c = _blocks()
    v = fine if z is None else np.stack([fine] * z)
    got = RO.regrid(v, c, c, coarse, coarse, 5)
    np.testing.assert_array_equal(got, target)


def _exact_axis(src, dst, pad):
    """{(j, source index): overlap in source pixels} in rational arithmetic on the float64 values,
    padded pixels folded into the border pixel (flipped source axes not included)."""
    src = [Fr(float(s)) for s in src]
    dst = [Fr(float(d)) for d in dst]
    ss = (src[-1] - src[0]) / (len(src) - 1)
    ds_ = (dst[-1] - dst[0]) / (len(dst) - 1)
    so, do = src[0] - ss / 2, dst[0] - ds_ / 2
    out = {}
    for j in range(len(dst)):
        lo, hi = sorted((do + j * ds_, do + (j + 1) * ds_))
        u0, u1 = (lo - so) / ss, (hi - so) / ss
        for k in range(-pad, len(src) + pad):
            ov = min(k + 1, u1) - max(k, u0)
            if ov > 0:
                key = (j, min(max(k, 0), len(src) - 1))
                out[key] = out.get(key, 0) + ov
    return out


@pytest.mark.parametrize("case", CASES + [("blocks", 1.0, 4.0, (0.5, 0.5, 8, 8), (2.0, 2.0, 2, 2))],
                         ids=lambda c: c[0])
def test_axis_weights_against_fractions(case):
    _, ss, ds_, (sx0, _, snx, _), (dx0, _, dnx, _) = case
    xs, dst = _axis(sx0, ss, snx), _axis(dx0, ds_, dnx)
    for d in (dst, dst[::-1]):
        s0, sd = gis.regular_axis(xs, "x")
        d0, dd = gis._transform_axis(d, "x")
        pad = int(abs(dd) // sd * 1.1)
        first, count, w = gis.regrid_axis(s0, sd, len(xs), d0, dd, len(d), pad)
        want = _exact_axis(xs, d, pad)
        got = {(j, int(first[j]) + k): w[j, k] for j in range(len(d)) for k in range(count[j])}
        for key in set(got) | set(want):
            exact = want.get(key, Fr(0))
            if key not in got:
                assert exact <= Fr(gis.REGRID_EPS), (key, float(exact))
            else:
                assert abs(Fr(got[key]) - exact) <= Fr(1, 10 ** 12), (key, got[key], float(exact))


@pytest.mark.parametrize("nearest", [False, True], ids=["average", "nearest"])
@pytest.mark.parametrize("flip", [(False, False), (True, False), (False, True), (True, True)],
                         ids=["asc", "src-desc", "dst-desc", "both-desc"])
@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
def test_host_tables_against_oracle(case, flip, nearest):
    """The separable tables applied on the host equal the cell-by-cell oracle."""
    xs, ys, v, dimx, dimy = _case(case, np.random.default_rng(1), nt=2, flip_src_y=flip[0], flip_dst_y=flip[1])
    v[0, 3, 5] = v[1, 10:, :] = np.nan
    My, Mx = _host_tables(xs, ys, np.asarray(dimx), np.asarray(dimy), nearest)
    got = _apply_tables(v, My, Mx)
    want = RO.regrid(v, xs, ys, dimx, dimy, 0 if nearest else 5)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)


# ---------------------------------------------------------------- GPU

@pytest.mark.gpu
@pytest.mark.parametrize("k", range(len(KNOWN)))
def test_known_answers(k):
    z, coarse, target = KNOWN[k]
    fine, c = _blocks()
    if z is None:
        da = DataArray(fine, {"y": c, "x": c}, ("y", "x"))
    else:
        da = DataArray(np.stack([fine] * z), {"z": np.arange(z), "y": c, "x": c}, ("z", "y", "x"))
    cx, cy = pd.Index(coarse, name="x"), pd.Index(coarse, name="y")
    res = ab.regrid(da, cx, cy, resampling=5)
    np.testing.assert_array_equal(res.values, target)
    assert res.dims == (("y", "x") if z is None else ("z", "y", "x"))
    assert (res.coords["x"] == coarse).all() and (res.coords["y"] == coarse).all()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("resampling", [5, 0], ids=["average", "nearest"])
@pytest.mark.parametrize("flip", [(False, False), (True, False), (False, True)], ids=["asc", "src-desc", "dst-desc"])
@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
def test_random_fields_against_oracle(case, flip, resampling, dtype):
    xs, ys, v, dimx, dimy = _case(case, np.random.default_rng(7), flip_src_y=flip[0], flip_dst_y=flip[1])
    v[0, ::7, ::3] = np.nan  # scattered NaNs
    v[1, :12, :12] = np.nan  # an all-NaN window
    v = v.astype(dtype)
    da = DataArray(v, {"time": np.arange(len(v)), "y": ys, "x": xs}, ("time", "y", "x"), attrs={"units": "W m**-2"})
    res = ab.regrid(da, dimx, dimy, resampling=resampling)
    want = RO.regrid(v, xs, ys, dimx, dimy, resampling)
    assert res.dims == ("time", "y", "x") and res.attrs == {"units": "W m**-2"}
    assert (res.coords["y"] == np.asarray(dimy)).all() and (res.coords["x"] == np.asarray(dimx)).all()
    assert np.isnan(want[1]).any() and not np.isnan(want).all()
    if dtype == np.float32:
        _f32_within_ulp(res.values, want)
    else:
        assert res.values.dtype == np.float64
        np.testing.assert_array_equal(np.isnan(res.values), np.isnan(want))
        np.testing.assert_allclose(res.values, want, rtol=1e-12, atol=0)


@pytest.mark.gpu
def test_nearest_centres_on_borders():
    """Destination centres on source pixel borders take the pixel on the increasing side, in both
    axis orders; centres beyond the padded source give NaN."""
    xs = ys = np.arange(0.5, 8, 1.0)  # borders at the integers
    v = np.arange(64, dtype=np.float64).reshape(8, 8)
    da = DataArray(v, {"y": ys, "x": xs}, ("y", "x"))
    for dst in (np.arange(0.0, 9.0, 1.0), np.arange(9.0, -1.0, -1.0), np.arange(-12.0, 21.0, 3.0)):
        dimx, dimy = pd.Index(dst, name="x"), pd.Index(dst, name="y")
        got = ab.regrid(da, dimx, dimy, resampling=0).values
        np.testing.assert_array_equal(got, RO.regrid(v, xs, ys, dst, dst, 0))
    got = ab.regrid(da, pd.Index(np.arange(0.0, 9.0, 1.0), name="x"), pd.Index(np.arange(1.0, 8.0, 1.0), name="y"),
                    resampling=0).values
    np.testing.assert_array_equal(got[:, 1:8], v[1:8, 1:8])


def _cutout_like(rng, dtype, nt=5):
    xs, ys = _axis(5.025, 0.05, 60), _axis(45.025, 0.05, 40)
    a = rng.uniform(0.5, 1.5, (nt, 40, 60)).astype(dtype)
    h = rng.uniform(0.5, 1.5, (40, 60)).astype(dtype)
    return xs, ys, a, h


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_dataset_host_and_device(dtype):
    import torch

    rng = np.random.default_rng(3)
    xs, ys, a, h = _cutout_like(rng, dtype)
    coords = {"time": np.arange(len(a)), "y": ys, "x": xs, "lat": ys, "lon": xs}
    dimx, dimy = pd.Index(_axis(5.1, 0.25, 11), name="x"), pd.Index(_axis(45.1, 0.25, 7), name="y")
    host = Dataset({"a": (("time", "y", "x"), a), "h": (("y", "x"), h)}, coords=coords, attrs={"module": "era5"})
    res = ab.regrid(host, dimx, dimy, resampling=5)
    assert isinstance(res.raw("a"), np.ndarray) and res.attrs == {"module": "era5"}
    assert res.dims_of("a") == ("time", "y", "x") and res.dims_of("h") == ("y", "x")
    assert (res.coords["lon"] == np.asarray(dimx)).all() and (res.coords["lat"] == np.asarray(dimy)).all()
    want_a, want_h = RO.regrid(a, xs, ys, dimx, dimy), RO.regrid(h, xs, ys, dimx, dimy)
    check = _f32_within_ulp if dtype == np.float32 else (
        lambda g, w: np.testing.assert_allclose(g, w, rtol=1e-12, atol=0))
    check(res.raw("a"), want_a)
    check(res.raw("h"), want_h)
    # device-resident, with rows padded to a multiple of 4 as Cutout.to_device stores them
    dev = torch.device("cuda:0")
    pad_a = torch.nn.functional.pad(torch.from_numpy(a), (0, 4)).to(dev)
    d = Dataset({"a": (("time", "y", "x"), pad_a), "h": (("y", "x"), torch.from_numpy(h).to(dev))}, coords=coords)
    n0 = ab._lib.launch_count()
    dres = ab.regrid(d, dimx, dimy, resampling=5)
    assert ab._lib.launch_count() == n0 + 2
    for n in ("a", "h"):
        t = dres.raw(n)
        assert torch.is_tensor(t) and t.device == dev and t.dtype == pad_a.dtype
        np.testing.assert_array_equal(t.cpu().numpy(), res.raw(n))  # fixed order: host and device agree bitwise
    again = ab.regrid(d, dimx, dimy, resampling=5).raw("a")
    assert torch.equal(again, dres.raw("a"))


@pytest.mark.gpu
def test_time_last_and_leading_dims():
    rng = np.random.default_rng(4)
    xs, ys, a, _ = _cutout_like(rng, np.float32)
    ayxt = np.ascontiguousarray(np.moveaxis(a, 0, -1))  # (y, x, time)
    dimx, dimy = pd.Index(_axis(5.2, 0.25, 10), name="x"), pd.Index(_axis(45.2, 0.25, 6)[::-1], name="y")
    res = ab.regrid(DataArray(ayxt, {"y": ys, "x": xs, "time": np.arange(len(a))}, ("y", "x", "time")),
                    dimx, dimy, resampling=5)
    assert res.dims == ("time", "y", "x") and res.shape == (len(a), 6, 10)
    _f32_within_ulp(res.values, RO.regrid(a, xs, ys, dimx, dimy))
    four = rng.uniform(0.5, 1.5, (2, 40, 3, 60)).astype(np.float32)  # (level, y, member, x)
    res = ab.regrid(DataArray(four, {"y": ys, "x": xs}, ("level", "y", "member", "x")), dimx, dimy, resampling=5)
    assert res.dims == ("level", "member", "y", "x")
    _f32_within_ulp(res.values, RO.regrid(np.moveaxis(four, 2, 1), xs, ys, dimx, dimy))


@pytest.mark.gpu
def test_lazy_dataset_in_parts():
    rng = np.random.default_rng(5)
    xs, ys, a, h = _cutout_like(rng, np.float32, nt=23)
    coords = {"time": pd.date_range("2013-01-01", periods=len(a), freq="h"), "y": ys, "x": xs}
    lazy = LazyDataset({"a": lambda lo, hi: a[lo:hi]}, coords, static={"h": (("y", "x"), h)}, time_chunk=5)
    dimx, dimy = pd.Index(_axis(5.1, 0.25, 11), name="x"), pd.Index(_axis(45.1, 0.25, 7), name="y")
    res = ab.regrid(lazy, dimx, dimy, resampling=5)
    assert lazy.largest_read == 5 and lazy.loaded_steps == len(a)
    whole = ab.regrid(Dataset({"a": (("time", "y", "x"), a), "h": (("y", "x"), h)}, coords=coords), dimx, dimy,
                      resampling=5)
    assert list(res.keys()) == ["a", "h"]
    for n in ("a", "h"):
        np.testing.assert_array_equal(res.raw(n), whole.raw(n))
