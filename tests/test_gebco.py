"""gebco: GEBCO terrain height averaged onto a cutout (reference datasets/gebco.py), the windowed grid
reader (ingest.open_grid), gebco.raster, and integer heights in runoff and line_rating.

Fixtures are GEBCO-like NetCDF-3 files written with scipy: ascending ``lat`` / ``lon`` centres and an
int16 ``elevation``, with and without ``_FillValue``, or a float32 one.  CPU: the window against
rasterio's from_bounds arithmetic (oracle/gebco_oracle.py), the reader, the argument errors and the
raster.  GPU: the average against the float64 oracle (oracle/gebco_oracle.py), several host bands
and device input bitwise against one band, and runoff / line_rating on a merged cutout.
"""

import numpy as np
import pandas as pd
import pytest
from scipy.io import netcdf_file

import atlite_b200 as ab
import gebco_oracle as GO
from atlite_b200 import gebco, ingest
from atlite_b200 import synthetic as syn
from atlite_b200.engine import RegridOp
from atlite_b200.labelled import Dataset

FILL = -32767
RES = 1 / 240  # 15 arc-seconds


def _axes(lon0, lon1, lat0, lat1, res=RES):
    n_lon, n_lat = round((lon1 - lon0) / res), round((lat1 - lat0) / res)
    return lon0 + (np.arange(n_lon) + 0.5) * res, lat0 + (np.arange(n_lat) + 0.5) * res


def _elevation(lon, lat, seed=0):
    """int16 (lat, lon): smooth terrain and sea floor plus noise."""
    rng = np.random.default_rng(seed)
    g = 3000 * np.sin(np.radians(lat * 40))[:, None] * np.cos(np.radians(lon * 30))[None, :]
    return (g + rng.integers(-400, 400, (len(lat), len(lon)))).astype(np.int16)


def _write(path, lon, lat, elev, fill=None, name="elevation"):
    f = netcdf_file(str(path), "w")
    f.createDimension("lat", len(lat))
    f.createDimension("lon", len(lon))
    for n, c in (("lat", lat), ("lon", lon)):
        v = f.createVariable(n, "f8", (n,))
        v[:] = c
    v = f.createVariable(name, "i2" if elev.dtype == np.int16 else "f4", ("lat", "lon"))
    v[:] = elev
    v.units = "m"
    v.long_name = "Elevation relative to sea level"
    if fill is not None:
        v._FillValue = np.asarray(fill, dtype=elev.dtype)
    f.close()
    return str(path)


@pytest.fixture(scope="module")
def grid(tmp_path_factory):
    """(path, lon, lat, elevation): lon 5..9, lat 44..47 at 15'', no fill value."""
    lon, lat = _axes(5.0, 9.0, 44.0, 47.0)
    elev = _elevation(lon, lat)
    return _write(tmp_path_factory.mktemp("gebco") / "gebco.nc", lon, lat, elev), lon, lat, elev


def _cutout(x, y, nt=2):
    time = pd.date_range("2013-01-01", periods=nt, freq="h")
    ds = Dataset({"temperature": (("time", "y", "x"), np.zeros((nt, len(y), len(x)), dtype=np.float32))},
                 coords=dict(time=time, x=x, y=y, lon=x, lat=y), attrs={"module": "era5"})
    return ab.Cutout(data=ds)


X25, Y25 = 5.125 + 0.25 * np.arange(14), 44.375 + 0.25 * np.arange(9)  # 0.25 deg on 15'': 60 x 60 pixels
X07, Y07 = 5.3 + 0.07 * np.arange(41), 44.23 + 0.07 * np.arange(33)  # fractional ratio and offsets


# ---------------------------------------------------------------------------------------- CPU


@pytest.mark.parametrize("xy", [(X25, Y25), (X07, Y07), (np.array([6.0, 6.5]), np.array([45.0, 45.1]))])
def test_window_is_from_bounds(grid, xy):
    _, lon, lat, _ = grid
    t = gebco.grid_transform(lon, lat)
    assert t == tuple(GO.transform(lon, lat))
    want = GO.cutout_window(lon, lat, *xy)
    assert gebco._cutout_window(*xy, t, (len(lat), len(lon))) == tuple(want)
    assert gebco.window(t, 5.3, 44.7, 8.1, 46.9) == tuple(GO.from_bounds(t, 5.3, 44.7, 8.1, 46.9))


def test_integer_ratio_window_and_tables(grid):
    _, lon, lat, _ = grid
    win = gebco._cutout_window(X25, Y25, gebco.grid_transform(lon, lat), (len(lat), len(lon)))
    np.testing.assert_allclose(win, (0.0, 120.0, 14 * 60, 9 * 60), atol=1e-9)
    (r0, r1), (c0, c1), ytab, xtab = gebco._tables(win, len(X25), len(Y25), (len(lat), len(lon)), True)
    assert (c0, c1) == (0, 14 * 60) and (r0, r1) == (60, 600)  # north-up rows 120 .. 659, ascending in the file
    assert (xtab[1] == 60).all() and (ytab[1] == 60).all()
    np.testing.assert_allclose(xtab[2], 1.0, atol=1e-9)
    assert (np.diff(ytab[0]) == 60).all() and ytab[0][0] == 0  # ascending y reads ascending file rows


def test_reader_slices_without_loading(grid):
    path, lon, lat, elev = grid
    lo, la, var = ingest.open_grid(path)
    assert np.array_equal(lo, lon) and np.array_equal(la, lat)
    assert var.shape == elev.shape and var.dtype == np.dtype(np.int16) and var.fill is None
    assert var.attrs["units"] == "m"
    assert not var._var.flags["OWNDATA"] and var._var.dtype == np.dtype(">i2")  # the file's memory map
    part = var[17:61, 100:333]
    assert part.dtype == np.dtype(np.int16) and part.flags["OWNDATA"]
    assert np.array_equal(part, elev[17:61, 100:333])
    w = var.window(17, 61, 100, 333)
    assert w.shape == (44, 233)
    out = np.empty((5, 233), dtype=np.int16)
    w.read(3, 8, out)
    assert np.array_equal(out, elev[20:25, 100:333])
    assert np.array_equal(np.asarray(w), elev[17:61, 100:333])


def test_reader_picks_the_variable_and_fill(tmp_path):
    lon, lat = _axes(0.0, 0.5, 0.0, 0.25, 1 / 24)
    elev = _elevation(lon, lat)
    p = _write(tmp_path / "z.nc", lon, lat, elev, fill=FILL, name="z")
    _, _, var = ingest.open_grid(p)
    assert var.fill == FILL and np.array_equal(var[0:2, 0:3], elev[0:2, 0:3])
    f = netcdf_file(str(tmp_path / "two.nc"), "w")
    for n, c in (("lat", lat), ("lon", lon)):
        f.createDimension(n, len(c))
        f.createVariable(n, "f8", (n,))[:] = c
    for n in ("a", "b"):
        f.createVariable(n, "i2", ("lat", "lon"))[:] = elev
    f.close()
    with pytest.raises(ValueError, match="elevation"):
        ingest.open_grid(str(tmp_path / "two.nc"))


def test_argument_errors(grid):
    path = grid[0]
    cut = _cutout(X25, Y25)
    with pytest.raises(ValueError, match="height"):
        gebco.get_data(cut, "influx", None, gebco_path=path)
    with pytest.raises(KeyError, match="gebco_path"):
        gebco.get_data(cut, "height", None)
    with pytest.raises(ValueError, match="at least 2 cells"):
        gebco.get_data(_cutout(X25[:1], Y25), "height", None, gebco_path=path)
    with pytest.raises(ValueError, match="at least 2 cells"):
        gebco.get_data(_cutout(X25, Y25[:1]), "height", None, gebco_path=path)
    with pytest.raises(ValueError, match="ascend"):
        gebco.get_data(_cutout(X25, Y25[::-1]), "height", None, gebco_path=path)
    for x, y in ((X25 - 0.25, Y25), (X25 + 0.75, Y25), (X25, Y25 - 0.5), (X25, Y25 + 0.75)):
        with pytest.raises(ValueError, match="not inside"):
            gebco.get_data(_cutout(x, y), "height", None, gebco_path=path)
    assert gebco.crs == 4326 and gebco.features == {"height": ["height"]}


def test_raster_is_a_flipped_slice(grid):
    path, lon, lat, elev = grid
    r = gebco.raster(path, (6.1012, 45.2031, 7.3007, 46.0491))  # edges inside pixels
    c0, c1 = int(np.floor((6.1012 - 5.0) * 240)), int(np.ceil((7.3007 - 5.0) * 240))
    r0, r1 = int(np.floor((45.2031 - 44.0) * 240)), int(np.ceil((46.0491 - 44.0) * 240))
    assert r.array.dtype == np.int16 and r.array.flags["C_CONTIGUOUS"]
    assert np.array_equal(r.array, elev[r0:r1, c0:c1][::-1])
    np.testing.assert_allclose(r.transform, (RES, 0, 5.0 + c0 * RES, 0, -RES, 44.0 + r1 * RES), rtol=0, atol=1e-12)
    whole = gebco.raster(path)
    assert np.array_equal(whole.array, elev[::-1])
    np.testing.assert_allclose(whole.bounds, (5.0, 44.0, 9.0, 47.0), atol=1e-12)
    with pytest.raises(ValueError, match="overlap"):
        gebco.raster(path, (20.0, 10.0, 21.0, 11.0))


def test_height_consumers_cast_integer_heights():
    from atlite_b200 import convert

    ds = Dataset({"height": (("y", "x"), np.array([[1, -2]], dtype=np.int16))},
                 coords=dict(x=np.array([0.0, 1.0]), y=np.array([0.0])))
    h = convert._height(ds)
    assert h.dtype == np.float32 and np.array_equal(h, [[1.0, -2.0]])
    f = np.array([[1.5, 2.5]], dtype=np.float64)
    ds["height"] = (("y", "x"), f)
    h = convert._height(ds)
    assert h.dtype == np.float64 and np.array_equal(h, f)


# ---------------------------------------------------------------------------------------- GPU


def _check(got, mean, fill=None):
    """int16 ``got`` is the oracle's mean rounded half away from zero, except within 1e-9 of a .5."""
    want = GO.round_half_away(mean)
    tie = np.abs(np.abs(mean - np.trunc(mean)) - 0.5) <= 1e-9
    assert got.dtype == np.int16
    bad = (got != want) & ~tie
    assert not bad.any(), f"{bad.sum()} cells differ, e.g. got {got[bad][:5]} want {mean[bad][:5]}"


@pytest.fixture
def small_slab(monkeypatch):
    monkeypatch.setattr(RegridOp, "WINDOW_SLAB_BYTES", 97 * 1024)
    return 97 * 1024


@pytest.mark.gpu
@pytest.mark.parametrize("xy", ["0.25", "0.07"])
def test_height_against_oracle(grid, xy):
    path, lon, lat, elev = grid
    x, y = {"0.25": (X25, Y25), "0.07": (X07, Y07)}[xy]
    ds = gebco.get_data(_cutout(x, y), "height", None, gebco_path=path)
    got = ds.raw("height")
    mean = GO.height(elev, lon, lat, x, y)
    _check(got, mean)
    if xy == "0.25":  # 60 x 60 whole pixels: the exact mean
        blocks = elev[60:600, :840].reshape(9, 60, 14, 60).astype(np.float64).mean(axis=(1, 3))
        np.testing.assert_array_equal(mean, blocks)
    assert ds.attrs["module"] == "gebco" and ds.dims_of("height") == ("y", "x")
    for c in ("x", "y", "time", "lon", "lat"):
        assert np.array_equal(np.asarray(ds.coords[c]), np.asarray(_cutout(x, y).coords[c]))
    da = gebco.get_data_gebco_height(x, y, path)
    assert np.array_equal(da.values, got) and da.attrs["units"] == "m"


@pytest.mark.gpu
def test_fill_values_are_skipped(tmp_path):
    lon, lat = _axes(5.0, 9.0, 44.0, 47.0)
    elev = _elevation(lon, lat, seed=3)
    rng = np.random.default_rng(4)
    elev[rng.random(elev.shape) < 0.2] = FILL
    elev[60 + 60:60 + 120, 120:180] = FILL  # cell (y 1, x 2) of the 0.25 deg cutout: only fill pixels
    path = _write(tmp_path / "fill.nc", lon, lat, elev, fill=FILL)
    for x, y in ((X25, Y25), (X07, Y07)):
        got = gebco.get_data(_cutout(x, y), "height", None, gebco_path=path).raw("height")
        _check(got, GO.height(elev, lon, lat, x, y, fill=FILL))
    got = gebco.get_data(_cutout(X25, Y25), "height", None, gebco_path=path).raw("height")
    assert got[1, 2] == FILL and (np.delete(got.ravel(), 1 * 14 + 2) != FILL).all()


@pytest.mark.gpu
def test_float32_elevation(tmp_path):
    lon, lat = _axes(5.0, 9.0, 44.0, 47.0)
    elev = _elevation(lon, lat, seed=5).astype(np.float32) + np.float32(0.25)
    elev[10:200, 300:310] = np.nan
    path = _write(tmp_path / "f32.nc", lon, lat, elev)
    got = gebco.get_data(_cutout(X07, Y07), "height", None, gebco_path=path).raw("height")
    mean = GO.height(elev, lon, lat, X07, Y07)
    assert got.dtype == np.float32
    np.testing.assert_allclose(got, mean, rtol=2 ** -23, atol=0)


@pytest.mark.gpu
def test_bands_and_device_input_bitwise(grid, small_slab):
    import torch

    path, lon, lat, elev = grid
    for x, y in ((X25, Y25), (X07, Y07)):
        _, _, var = ingest.open_grid(path)
        win = gebco._cutout_window(x, y, gebco.grid_transform(lon, lat), var.shape)
        (r0, r1), (c0, c1), ytab, xtab = gebco._tables(win, len(x), len(y), var.shape, True)
        op = RegridOp((r1 - r0, c1 - c0), ytab, xtab)
        groups = op._window_bands((c1 - c0) * 2)
        assert len(groups) >= 2
        assert [g[0] for g in groups] == list(np.cumsum([0] + [g[1] for g in groups[:-1]]))
        banded = op.window(var.window(r0, r1, c0, c1))
        RegridOp.WINDOW_SLAB_BYTES = 1 << 40  # one band (the fixture restores it)
        assert len(op._window_bands((c1 - c0) * 2)) == 1
        one = op.window(var.window(r0, r1, c0, c1))
        RegridOp.WINDOW_SLAB_BYTES = small_slab
        assert np.array_equal(banded, one)
        host = np.ascontiguousarray(elev[r0:r1, c0:c1])
        assert np.array_equal(op.window(host), one)
        dev = torch.from_numpy(elev).cuda()[r0:r1, c0:c1]  # row-strided
        assert np.array_equal(op.window(dev).cpu().numpy(), one)
        _check(one, GO.height(elev, lon, lat, x, y))
        again = gebco.get_data(_cutout(x, y), "height", None, gebco_path=path).raw("height")
        assert np.array_equal(again, one)


def _raw_era5(x, y, nt, seed=0):
    rng = np.random.default_rng(seed)
    sh = (nt, len(y), len(x))
    f = dict(t2m=rng.uniform(255.0, 305.0, sh), u100=rng.uniform(-15, 15, sh), v100=rng.uniform(-15, 15, sh),
             fdir=rng.uniform(0.0, 3e6, sh), ro=rng.uniform(-1e-5, 4e-4, sh))
    time = pd.date_range("2013-06-01", periods=nt, freq="h")
    return Dataset({k: (("time", "y", "x"), v.astype(np.float32)) for k, v in f.items()},
                   coords=dict(time=time, x=x, y=y, lon=x, lat=y), attrs={"module": "era5"})


@pytest.mark.gpu
def test_runoff_and_line_rating_on_merged_cutout(tmp_path):
    lon, lat = _axes(5.0, 9.0, 44.0, 47.0, 1 / 60)
    elev = (_elevation(lon, lat, seed=9) // 2 + 1500).astype(np.int16)
    path = _write(tmp_path / "gebco.nc", lon, lat, elev)
    era = _raw_era5(X07, Y07, 30)
    era_cut = ab.Cutout(data=era)
    geb = gebco.get_data(era_cut, "height", None, gebco_path=path)
    merged = era_cut.merge(ab.Cutout(data=geb), compat="override")
    assert sorted(merged.module) == ["era5", "gebco"]
    assert merged.data.raw("height").dtype == np.int16
    hand = Dataset(coords=dict(era.coords), attrs={"module": "era5"})
    for n in era.keys():
        hand[n] = (era.dims_of(n), era.raw(n))
    hand["height"] = (("y", "x"), geb.raw("height").astype(np.float32))
    m = syn.make_shapes(len(X07), len(Y07), 4)
    lines = syn.make_line_network(X07, Y07, 6)
    prev = ab.set_deterministic(True)
    try:
        for a, b in ((merged, ab.Cutout(data=hand)), (merged.to_device(), ab.Cutout(data=hand).to_device())):
            ra = np.asarray(a.runoff(weight_with_height=True, matrix=m).values)
            rb = np.asarray(b.runoff(weight_with_height=True, matrix=m).values)
            assert np.isfinite(rb).all() and np.abs(rb).max() > 0
            assert np.array_equal(ra, rb)
            la = np.asarray(a.line_rating(lines, 1e-4).values)
            lb = np.asarray(b.line_rating(lines, 1e-4).values)
            assert np.isfinite(lb).any()
            assert np.array_equal(la, lb, equal_nan=True)
    finally:
        ab.set_deterministic(prev)
