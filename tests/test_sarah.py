"""sarah: SARAH irradiance for a cutout (reference datasets/sarah.py), and Cutout.merge (cutout.py:415-451).

Fixtures are synthetic SARAH-shaped NetCDF-3 day files (48 half-hours at 0.05 degrees, dawn and
dusk NaN runs, cells NaN for a whole day, one day without its SID file), as int16 with
scale_factor and _FillValue or as float32 with NaN.  CPU: file selection, the block rule, the
oracle (oracle/sarah_oracle.py) against hand-computed values, argument errors and Cutout.merge on
host and lazy Datasets.  GPU: the fill + pair-mean kernel bitwise against the oracle, get_data
against the oracle with and without regridding, the solar position, repeatability, and PV on a
SARAH + ERA5 merged cutout.
"""

import logging
import os

import numpy as np
import pandas as pd
import pytest
from scipy.io import netcdf_file

import atlite_b200 as ab
import sarah_oracle as SO
from atlite_b200 import era5, ingest, sarah
from atlite_b200 import synthetic as syn
from atlite_b200.engine import SarahOp
from atlite_b200.labelled import DataArray, Dataset, LazyDataset

LON = np.round(5.0 + 0.05 * np.arange(40), 4)
LAT = np.round(45.0 + 0.05 * np.arange(30), 4)
DAYS = pd.date_range("2013-01-01", periods=4, freq="D")
SCALE, FILL = 0.1, -999


def _raw_day(k):
    """int16 (48, lat, lon) values of day k, FILL where the value is missing."""
    rng = np.random.default_rng(100 + k)
    v = rng.integers(0, 9000, (48, len(LAT), len(LON))).astype(np.int16)
    dawn = rng.integers(4, 14, (len(LAT), len(LON)))
    dusk = rng.integers(34, 46, (len(LAT), len(LON)))
    t = np.arange(48)[:, None, None]
    v[(t < dawn) | (t >= dusk)] = FILL
    gaps = rng.random(v.shape) < 0.05
    v[gaps] = FILL
    v[:, 3, 5] = FILL  # NaN for the whole day
    v[:, 7, 2 + k] = FILL
    return v


def _decoded(raw):
    a = raw.astype(np.float32) * np.float32(SCALE)
    a[raw == FILL] = np.nan
    return a


def _write(path, var, day, raw, packed):
    f = netcdf_file(path, "w")
    f.createDimension("time", 48)
    f.createDimension("lat", len(LAT))
    f.createDimension("lon", len(LON))
    t = f.createVariable("time", "f8", ("time",))
    t[:] = np.arange(48) * 30.0
    t.units = f"minutes since {day:%Y-%m-%d} 00:00:00"
    for name, c in (("lat", LAT), ("lon", LON)):
        v = f.createVariable(name, "f8", (name,))
        v[:] = c
    if packed:
        v = f.createVariable(var, "i2", ("time", "lat", "lon"))
        v.scale_factor = SCALE
        v._FillValue = np.int16(FILL)
        v[:] = raw
    else:
        v = f.createVariable(var, "f4", ("time", "lat", "lon"))
        v[:] = _decoded(raw)
    f.close()


def _raws():
    return {(var, k): _raw_day(k + (0 if var == "SIS" else 10)) for var in ("SIS", "SID") for k in range(len(DAYS))}


@pytest.fixture(scope="module", params=["packed", "float"])
def sarah_dir(request, tmp_path_factory):
    d = tmp_path_factory.mktemp(f"sarah_{request.param}")
    raws = _raws()
    for (var, k), raw in raws.items():
        if var == "SID" and k == 3:
            continue  # the last SID day is missing
        sub = d / f"{DAYS[k]:%Y}" / var.lower()
        os.makedirs(sub, exist_ok=True)
        _write(sub / f"{var}in{DAYS[k]:%Y%m%d}00000042310001I1UD.nc", var, DAYS[k], raw, request.param == "packed")
    return str(d)


def _cutout(x, y, periods=72, freq="h", start="2013-01-01", chunk=None):
    time = pd.date_range(start, periods=periods, freq=freq)
    attrs = {"module": "era5"}
    if chunk:
        attrs["chunksize_time"] = chunk
    ds = Dataset({"temperature": (("time", "y", "x"), np.zeros((periods, len(y), len(x)), dtype=np.float32))},
                 coords=dict(time=time, x=x, y=y, lon=x, lat=y), attrs=attrs)
    return ab.Cutout(data=ds)


def _expected(cut, days=3, interpolate=True, hourly=True, chunk=None):
    """(direct, diffuse, lon, lat) from the oracle on the files get_data selects."""
    raws = _raws()
    sis = np.concatenate([_decoded(raws["SIS", k]) for k in range(days)])
    sid = np.concatenate([_decoded(raws["SID", k]) for k in range(days)])
    ext = cut.extent
    xs = (LON >= ext[0] - 0.01) & (LON <= ext[1] + 0.01)
    ys = (LAT >= ext[2] - 0.01) & (LAT <= ext[3] + 0.01)
    sis, sid = sis[:, ys][:, :, xs], sid[:, ys][:, :, xs]
    starts = sarah.block_starts([48] * days, chunk)
    regrid = cut.dx != 0.05 or cut.dy != 0.05
    kw = dict(lon=LON[xs], lat=LAT[ys], dst_lon=np.asarray(cut.coords["x"]), dst_lat=np.asarray(cut.coords["y"])) \
        if regrid else {}
    d, f = SO.influx(sis, sid, starts, interpolate, hourly, **kw)
    return d, f, (kw["dst_lon"] if regrid else LON[xs]), (kw["dst_lat"] if regrid else LAT[ys])


X25, Y25 = 5.25 + 0.25 * np.arange(6), 45.25 + 0.25 * np.arange(4)
X30, Y30 = 5.3 + 0.3 * np.arange(4), 45.3 + 0.3 * np.arange(3)
X05, Y05 = LON[4:20], LAT[3:15]


# ---------------------------------------------------------------- CPU


def test_module_constants():
    assert (sarah.crs, sarah.dx, sarah.dy, sarah.dt) == (4326, 0.05, 0.05, "30min")
    assert sarah.features == {"influx": ["influx_direct", "influx_diffuse", "solar_altitude", "solar_azimuth"]}
    assert sarah.static_features == {}
    assert ab.sarah is sarah


def test_get_filenames_joins_and_selects_days(sarah_dir):
    coords = {"time": pd.date_range("2013-01-02 06:00", "2013-01-03 18:00", freq="h")}
    files = sarah.get_filenames(sarah_dir, coords)
    assert list(files.columns) == ["sis", "sid"]
    assert list(files.index) == list(DAYS[1:3])
    assert all(os.path.basename(p).startswith("SIS") for p in files["sis"])
    assert all(os.path.basename(p).startswith("SID") for p in files["sid"])
    every = sarah.get_filenames(sarah_dir, {"time": pd.date_range("2013-01-01", "2013-01-03 23:00", freq="h")})
    assert list(every.index) == list(DAYS[:3])  # the fourth day has no SID file


def test_get_filenames_logs_uncovered_span(sarah_dir, caplog):
    with caplog.at_level(logging.ERROR, logger="atlite_b200.sarah"):
        files = sarah.get_filenames(sarah_dir, {"time": pd.date_range("2012-12-31", "2013-01-05", freq="h")})
    assert "do not cover the whole time span" in caplog.text
    assert list(files.index) == list(DAYS[:3])


def test_get_filenames_without_files(tmp_path):
    with pytest.raises(AssertionError, match="No files found"):
        sarah.get_filenames(str(tmp_path), {"time": DAYS})


def test_as_slice():
    s = sarah.as_slice(np.array([5.0, 6.0]))
    assert (s.start, s.stop) == pytest.approx((4.99, 6.01))
    keep = slice(1, 2)
    assert sarah.as_slice(keep) is keep


def test_block_rule():
    assert sarah.block_starts([48, 48, 48], 100) == [0, 48, 96]
    assert sarah.block_starts([48, 48, 48], None) == [0, 48, 96]
    assert sarah.block_starts([48, 48], 24) == [0, 24, 48, 72]
    assert sarah.block_starts([48, 30], 20) == [0, 20, 40, 48, 68]
    assert sarah.block_starts([], 24) == []


def test_launch_cuts_keep_blocks_and_pairs():
    op = SarahOp.__new__(SarahOp)
    assert op.launches([0, 48, 96], 144, True, 1) == [(0, 48, [0]), (48, 96, [0]), (96, 144, [0])]
    assert op.launches([0, 48, 96], 144, True, 2) == [(0, 96, [0, 48]), (96, 144, [0])]
    with pytest.raises(ValueError, match="no even block start"):
        op.launches([0, 3, 5], 9, True, 1)
    assert op.launches([0, 3, 5], 9, False, 1) == [(0, 3, [0]), (3, 5, [0]), (5, 9, [0])]
    with pytest.raises(ValueError, match="ascend"):
        op.launches([0, 5, 5], 9, False)
    with pytest.raises(ValueError, match="batch"):
        op.launches([0], 9, False, 0)


def test_oracle_known_values():
    nan = np.nan
    y = SO.fill_series([nan, nan, 2.0, nan, nan, 8.0, nan])
    np.testing.assert_array_equal(y, np.float32([2, 2, 2, 4, 6, 8, 8]))
    np.testing.assert_array_equal(SO.fill_series([nan, nan]), np.float32([nan, nan]))
    np.testing.assert_array_equal(SO.fill_series([nan, 1.0, nan], interpolate=False), np.float32([0, 1, 0]))
    third = SO.fill_series([0.0, nan, nan, 1.0])
    assert third[1] == np.float32(np.float64(1.0) / 3) and third[2] == np.float32(2.0 / 3)
    a = SO.fill(np.float32([[nan], [1.0], [nan], [3.0], [nan]]), [0, 2])
    np.testing.assert_array_equal(a[:, 0], np.float32([1, 1, 3, 3, 3]))  # blocks [0, 2) and [2, 5)
    np.testing.assert_array_equal(SO.hourly_mean(np.float32([1, 2, 3, nan, 5])), np.float32([1.5, nan]))


def test_get_data_argument_errors(sarah_dir):
    cut = _cutout(X25, Y25)
    with pytest.raises(KeyError):
        sarah.get_data(cut, "influx", None)
    with pytest.raises(ValueError, match="influx"):
        sarah.get_data(cut, "wind", None, sarah_dir=sarah_dir)
    with pytest.raises(AssertionError):
        sarah.get_data(_cutout(X25, Y25, periods=24, freq="3h"), "influx", None, sarah_dir=sarah_dir)


def _host_ds(names, x, y, nt=6, module="era5", seed=0):
    rng = np.random.default_rng(seed)
    time = pd.date_range("2013-01-01", periods=nt, freq="h")
    return Dataset({n: rng.random((nt, len(y), len(x))).astype(np.float32) for n in names},
                   coords=dict(time=time, x=x, y=y, lon=x, lat=y), attrs={"module": module})


def test_merge_host_datasets():
    x, y = np.arange(4.0), np.arange(3.0)
    a = ab.Cutout(data=_host_ds(["influx_direct", "albedo"], x, y, module="sarah", seed=1))
    b = ab.Cutout(data=_host_ds(["influx_direct", "temperature"], x, y, module="era5", seed=2))
    m = a.merge(b, compat="override")
    assert set(m.data.keys()) == {"influx_direct", "albedo", "temperature"}
    assert m.module == ["sarah", "era5"]
    assert m.data.raw("influx_direct") is a.data.raw("influx_direct")
    assert m.data.raw("temperature") is b.data.raw("temperature")
    with pytest.raises(ValueError, match="'influx_direct' differs"):
        a.merge(b)
    same = ab.Cutout(data=_host_ds(["influx_direct"], x, y, module=["era5", "sarah"], seed=1))
    same.data.raw("influx_direct")[0, 0, 0] = np.nan
    a.data.raw("influx_direct")[0, 0, 0] = np.nan
    assert sorted(a.merge(same).module) == ["era5", "sarah"]  # equal with NaN: no conflict
    with pytest.raises(TypeError, match="join"):
        a.merge(b, join="outer")
    with pytest.raises(TypeError, match="Cutout"):
        a.merge(b.data)


@pytest.mark.parametrize("coord", ["x", "y", "time"])
def test_merge_coordinate_mismatch(coord):
    x, y = np.arange(4.0), np.arange(3.0)
    a = ab.Cutout(data=_host_ds(["a"], x, y))
    if coord == "time":
        other = _host_ds(["b"], x, y, nt=5)
    else:
        other = _host_ds(["b"], x + (coord == "x"), y + (coord == "y"))
    with pytest.raises(ValueError, match=f"coordinate '{coord}'"):
        a.merge(ab.Cutout(data=other), compat="override")


def test_merge_with_lazy_stays_lazy(tmp_path):
    x, y = np.arange(5.0), np.arange(3.0)
    era = _host_ds(["influx_direct", "temperature"], x, y, nt=10, seed=3)
    path = ingest.write_chunked(str(tmp_path / "era.chunks"), {n: era.raw(n) for n in era.keys()},
                                {k: era.coords[k] for k in ("time", "x", "y")}, chunk=(4, None, None),
                                attrs={"module": "era5"})
    lazy = ab.Cutout(data=ingest.open_chunked(path))
    sar = ab.Cutout(data=_host_ds(["influx_direct", "influx_diffuse"], x, y, nt=10, module="sarah", seed=4))
    m = sar.merge(lazy, compat="override")
    assert isinstance(m.data, LazyDataset) and m.data.time_chunk == 4
    assert sorted(m.data.keys()) == ["influx_diffuse", "influx_direct", "temperature"]
    assert m.module == ["sarah", "era5"]
    part = m.data.isel_time(3, 9)
    np.testing.assert_array_equal(part.raw("influx_direct"), sar.data.raw("influx_direct")[3:9])
    np.testing.assert_array_equal(part.raw("influx_diffuse"), sar.data.raw("influx_diffuse")[3:9])
    np.testing.assert_array_equal(part.raw("temperature"), era.raw("temperature")[3:9])
    back = lazy.merge(sar, compat="override")  # the lazy side wins now
    np.testing.assert_array_equal(back.data.isel_time(0, 10).raw("influx_direct"), era.raw("influx_direct"))
    with pytest.raises(ValueError, match="differs"):
        lazy.merge(sar)


# ---------------------------------------------------------------- GPU


def _random_fields(rng, nt, ny, nx):
    a = rng.uniform(0, 900, (nt, ny, nx)).astype(np.float32)
    runs = rng.integers(0, nt, (nt // 3, 3))
    for t0, iy, ix in runs:
        a[t0:t0 + rng.integers(1, 12), iy % ny, ix % nx] = np.nan
    a[:, 0, 0] = np.nan
    a[: nt // 2, 1, 1] = np.nan
    a[rng.random(a.shape) < 0.1] = np.nan
    return a


def _bitwise(got, want):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape and got.dtype == want.dtype == np.float32
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    assert np.array_equal(got[ok].view(np.uint32), want[ok].view(np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("starts_kind", ["48", "100", "mixed"])
@pytest.mark.parametrize("hourly", [True, False])
@pytest.mark.parametrize("fill", [SarahOp.FILL_INTERP, SarahOp.FILL_ZERO])
def test_kernel_bitwise(starts_kind, hourly, fill):
    import torch

    rng = np.random.default_rng(7)
    nt = {"48": 192, "100": 300, "mixed": 155}[starts_kind]
    starts = {"48": list(range(0, nt, 48)), "100": [0, 100, 200],
              "mixed": [0, 7, 8, 30, 31, 100, 140]}[starts_kind]
    ny, nx = 9, 37
    sis, sid = _random_fields(rng, nt, ny, nx), _random_fields(rng, nt, ny, nx)
    want = []
    for a in (sis, sid):
        w = SO.fill(a, starts, fill == SarahOp.FILL_INTERP)
        want.append(SO.hourly_mean(w) if hourly else w)
    op = SarahOp(ny, nx)
    got = op(torch.from_numpy(sis).cuda(), torch.from_numpy(sid).cuda(), starts, fill=fill, hourly=hourly)
    for g, w in zip(got, want):
        _bitwise(g.cpu().numpy(), w)
    host = op(sis, sid, starts, fill=fill, hourly=hourly, batch=1 if not hourly else 2)
    for g, w in zip(host, want):
        _bitwise(g, w)


@pytest.mark.gpu
def test_kernel_does_not_depend_on_launch_size():
    rng = np.random.default_rng(8)
    sis, sid = _random_fields(rng, 240, 5, 33), _random_fields(rng, 240, 5, 33)
    starts = list(range(0, 240, 48))
    op = SarahOp(5, 33)
    ref = op(sis, sid, starts)
    for batch in (1, 2, 3):
        for g, r in zip(op(sis, sid, starts, batch=batch), ref):
            assert np.array_equal(g.view(np.uint32), r.view(np.uint32))


@pytest.mark.gpu
def test_interpolate_and_hourly_mean_public():
    rng = np.random.default_rng(9)
    a = _random_fields(rng, 48, 4, 6)
    time = pd.date_range("2013-01-01", periods=48, freq="30min")
    da = DataArray(a, {"time": time, "y": np.arange(4.0), "x": np.arange(6.0)}, ("time", "y", "x"), "SIS")
    _bitwise(sarah.interpolate(da).values, SO.fill(a, [0]))
    hm = sarah.hourly_mean(da)
    _bitwise(hm.values, SO.hourly_mean(a))
    assert list(hm.coords["time"]) == list(time[::2])
    ds = Dataset({"SIS": (("time", "y", "x"), a), "SID": (("time", "y", "x"), a[::-1].copy())},
                 coords={"time": time, "y": np.arange(4.0), "x": np.arange(6.0)})
    out = sarah.interpolate(ds)
    _bitwise(out.raw("SID"), SO.fill(a[::-1], [0]))
    tr = DataArray(np.ascontiguousarray(a.transpose(1, 2, 0)), {"time": time}, ("y", "x", "time"), "SIS")
    _bitwise(sarah.interpolate(tr).values, SO.fill(a, [0]).transpose(1, 2, 0))


@pytest.mark.gpu
@pytest.mark.parametrize("grid", ["0.05", "0.25", "0.3"])
def test_get_data_against_oracle(sarah_dir, grid):
    x, y = {"0.05": (X05, Y05), "0.25": (X25, Y25), "0.3": (X30, Y30)}[grid]
    cut = _cutout(x, y)
    ds = sarah.get_data(cut, "influx", None, sarah_dir=sarah_dir)
    d, f, lon, lat = _expected(cut)
    assert ds.attrs["module"] == "sarah"
    np.testing.assert_array_equal(ds.coords["x"], lon)
    np.testing.assert_array_equal(ds.coords["lat"], lat)
    assert list(ds.coords["time"]) == list(pd.date_range("2013-01-01", periods=72, freq="h"))
    got_d, got_f = ds.raw("influx_direct"), ds.raw("influx_diffuse")
    if grid == "0.05":
        _bitwise(got_d, d)
        _bitwise(got_f, f)
    else:
        assert np.array_equal(np.isnan(got_d), np.isnan(d))
        ok = ~np.isnan(d)
        assert (np.abs(got_d[ok] - d[ok]) <= np.spacing(np.abs(d[ok]))).all()
        sis = d + f  # the oracle's regridded SIS, to within its rounding
        tol = np.spacing(np.abs(sis[ok])) * 2 + np.spacing(np.abs(d[ok])) * 2
        assert (np.abs(got_f[ok] - f[ok]) <= tol).all()
    alt, az = era5.solar_position(ds.coords["time"], lon, lat, "0h")
    assert np.array_equal(ds.raw("solar_altitude"), alt.cpu().numpy())
    assert np.array_equal(ds.raw("solar_azimuth"), az.cpu().numpy())
    again = sarah.get_data(cut, "influx", None, sarah_dir=sarah_dir)
    for n in ds.keys():
        assert np.array_equal(again.raw(n), ds.raw(n), equal_nan=True)


@pytest.mark.gpu
def test_get_data_half_hourly_chunked_and_zero_filled(sarah_dir, monkeypatch):
    cut = _cutout(X05, Y05, periods=144, freq="30min", chunk=20)
    ds = sarah.get_data(cut, "influx", None, sarah_dir=sarah_dir, sarah_interpolate=False)
    d, f, _, _ = _expected(cut, interpolate=False, hourly=False, chunk=20)
    _bitwise(ds.raw("influx_direct"), d)
    _bitwise(ds.raw("influx_diffuse"), f)
    ds = sarah.get_data(cut, "influx", None, sarah_dir=sarah_dir)
    d, f, _, _ = _expected(cut, hourly=False, chunk=20)
    _bitwise(ds.raw("influx_direct"), d)
    monkeypatch.setattr(sarah, "_FILES_PER_LAUNCH", 1)
    one = sarah.get_data(cut, "influx", None, sarah_dir=sarah_dir)
    assert np.array_equal(one.raw("influx_direct"), ds.raw("influx_direct"), equal_nan=True)


@pytest.mark.gpu
def test_packed_equals_float(tmp_path_factory):
    dirs = {}
    raws = _raws()
    for kind in ("packed", "float"):
        d = tmp_path_factory.mktemp(f"cmp_{kind}")
        for (var, k), raw in raws.items():
            if k < 2:
                _write(d / f"{var}in{DAYS[k]:%Y%m%d}0000.nc", var, DAYS[k], raw, kind == "packed")
        dirs[kind] = str(d)
    cut = _cutout(X25, Y25, periods=48)
    a, b = (sarah.get_data(cut, "influx", None, sarah_dir=dirs[k]) for k in ("packed", "float"))
    for n in a.keys():
        assert np.array_equal(a.raw(n), b.raw(n), equal_nan=True)


@pytest.mark.gpu
def test_pv_on_merged_cutout(sarah_dir, tmp_path):
    era = syn.make_dataset(len(X25), len(Y25), 48, x0=X25[0], y0=Y25[0], dx=0.25, dy=0.25,
                           start="2013-01-02", kinds=("pv",))
    era_cut = ab.Cutout(data=era)
    full = ab.Cutout(data=sarah.get_data(_cutout(X25, Y25), "influx", None, sarah_dir=sarah_dir))
    sar = full.sel(time=slice(era.coords["time"][0], era.coords["time"][-1]))
    merged = sar.merge(era_cut, compat="override")
    assert sorted(merged.module) == ["era5", "sarah"]
    hand = Dataset(coords=dict(era.coords), attrs={"module": "era5"})
    for n in era.keys():
        hand[n] = (era.dims_of(n), era.raw(n))
    for n in sar.data.keys():
        hand[n] = (sar.data.dims_of(n), np.ascontiguousarray(sar.data.raw(n)))
    m = syn.make_shapes(len(X25), len(Y25), 3)
    prev = ab.set_deterministic(True)
    try:
        def pv(c):
            return np.asarray(c.pv("CSi", "latitude_optimal", matrix=m, aggregate_time=None).values)

        want = pv(ab.Cutout(data=hand))
        assert np.isfinite(want).all() and want.max() > 0
        assert np.array_equal(pv(merged), want)
        assert np.array_equal(pv(merged.to_device()), pv(ab.Cutout(data=hand).to_device()))
        path = ingest.write_chunked(str(tmp_path / "era.chunks"), {n: era.raw(n) for n in era.keys()},
                                    {k: era.coords[k] for k in ("time", "x", "y")}, chunk=(16, None, None),
                                    attrs={"module": "era5"})
        lazy = sar.merge(ab.Cutout(data=ingest.open_chunked(path)), compat="override")
        assert getattr(lazy.data, "lazy", False)
        hand_lazy = LazyDataset({n: (lambda lo, hi, a=hand.raw(n): a[lo:hi]) for n in hand.keys()},
                                dict(hand.coords), time_chunk=16, dtypes={n: hand.raw(n).dtype for n in hand.keys()})
        assert np.array_equal(pv(lazy), pv(ab.Cutout(data=hand_lazy)))
    finally:
        ab.set_deterministic(prev)
