"""Dynamic line rating (convert.py:1152-1367): the float64 oracle against the reference's own
source (golden vectors) and the reference's known answers, the host logic of ``line_rating``,
and on the GPU the flat evaluator and the fused per-line min-reduce against the oracle."""

import os

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

import intersection_exact as IX
import line_rating_oracle as LO
import atlite_b200 as ab
from atlite_b200 import _lib, convert, engine, gis, synthetic as syn
from conftest import assert_parity

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_line_rating.npz")

# the reference's test/test_dynamic_line_rating.py conductor and weather, restated
IEEE = dict(temperature=313.0, wnd100m=0.61, height=0.0, wnd_azimuth=0.0, influx_direct=1027.0,
            solar_altitude=np.pi / 2, solar_azimuth=np.pi)
IEEE_LINE = dict(R=9.39e-5, D=0.02814, Ts=373.0, epsilon=0.8, alpha=0.8)
CALM = dict(IEEE, wnd100m=0.0, influx_direct=0.0)


def _golden():
    g = np.load(GOLDEN, allow_pickle=False)
    return {k: g[k] for k in g.files}


def _golden_case(g, name):
    """(oracle ds, R, params) of a golden case."""
    index = list(g["index"])
    ds = {k[3:]: g[k] for k in g if k.startswith("in_")}
    ds.update(time=pd.DatetimeIndex(g["time_ns"]), lon=g["x"], lat=g["y"])
    if name in ("stored_f64", "series"):
        ds.update(solar_altitude=g["stored_alt"], solar_azimuth=g["stored_az"])
    elif name == "stored_f32":
        ds.update(solar_altitude=g["stored_alt"].astype(np.float32), solar_azimuth=g["stored_az"].astype(np.float32))
    R, params = 9.39e-5, {}
    if name == "series":
        R = pd.Series(g["R_series_values"], index=list(g["R_series_index"]))
        params = {"D": pd.Series(g["D_series_values"], index=index), "Ts": 363.0, "epsilon": 0.8}
    elif name == "negative":
        params = {"D": 0.028, "Ts": 373.0, "epsilon": 0.6, "alpha": pd.Series(g["alpha_big_values"], index=index)}
    return ds, R, params


def _golden_matrix(g):
    n, s = (int(v) for v in g["I_shape"])
    return sp.csr_matrix((np.ones(len(g["I_indices"])), g["I_indices"], g["I_indptr"]), shape=(n, s))


def _rel_close(got, want, rtol):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    np.testing.assert_allclose(got[ok], want[ok], rtol=rtol, atol=0)


# ---------------------------------------------------------------- oracle vs the reference
@pytest.mark.parametrize("name", ["computed", "stored_f64", "stored_f32", "series", "negative"])
def test_oracle_matches_reference_line_rating(name):
    g = _golden()
    ds, R, params = _golden_case(g, name)
    az = pd.Series(g["azimuth_raw"], index=list(g["index"]))
    got = LO.line_rating(ds, _golden_matrix(g), az, R, **params)
    _rel_close(got, g[f"out_{name}"], 1e-9)
    want = g[f"out_{name}"]
    assert np.isnan(want[len(want) - 2]).all()  # the line outside the grid: the NaN dummy row
    assert np.isfinite(want[len(want) - 1]).all()  # the one-cell line
    if name == "negative":
        assert np.isnan(want[1]).any() and np.isfinite(want[1]).any()  # qs > qc + qr by day only


def test_oracle_matches_reference_flat():
    g = _golden()
    d = {k[5:]: g[k] for k in g if k.startswith("flat_") and k != "flat_psi"}
    got = LO.convert_line_rating(d, g["flat_psi"], 1e-4, D=0.03, Ts=368.0, epsilon=0.7, alpha=0.5)
    _rel_close(got, g["out_flat"], 1e-9)


def test_oracle_known_answers():
    assert np.isclose(LO.convert_line_rating(IEEE, 90, **IEEE_LINE), 1025, rtol=0.005)  # IEEE 738 sample
    al = dict(R=0.1188e-3, D=0.0218, Ts=353.0, epsilon=0.8, alpha=0.8)  # Oeding / Oswald Al 240/40
    assert np.isclose(LO.convert_line_rating(dict(CALM, temperature=303.0), 90, **al), 645, rtol=0.015)
    i = LO.convert_line_rating(dict(CALM, temperature=293.0), 0, 0.0136e-3, Ts=363)  # Suedkabel
    assert np.isclose(i, 2460, rtol=0.02)
    assert np.isclose(np.sqrt(3) * i * 380000 / 1e6, 1619, rtol=0.02)


def _symmetry_cases():
    """(ds, psi) pairs that the reference's right-angle test expects to equal (IEEE, 90)."""
    return [(IEEE, 270), (dict(IEEE, wnd_azimuth=np.pi / 2), 0), (dict(IEEE, wnd_azimuth=np.pi / 2), 180),
            (dict(IEEE, wnd_azimuth=np.pi), 90), (dict(IEEE, wnd_azimuth=np.pi), 270)]


def test_oracle_symmetries():
    f = lambda ds, psi: LO.convert_line_rating(ds, psi, **IEEE_LINE)  # noqa: E731
    expected = f(IEEE, 90)
    for ds, psi in _symmetry_cases():
        assert np.isclose(f(ds, psi), expected, rtol=1e-12, atol=0)
    res = pd.Series([f(IEEE, psi) for psi in np.arange(0, 370, 10)])
    assert (res.iloc[:10].diff().dropna() >= 0).all()  # rising capacity up to 90 deg
    assert (res.iloc[9:19].diff().dropna() <= 0).all()
    assert np.allclose(res.iloc[:19].values, res.iloc[:17:-1].values, rtol=1e-10, atol=1e-10)  # point symmetry
    assert np.allclose(res.iloc[:19].values, res.iloc[18:].values, rtol=1e-10, atol=1e-10)


# ---------------------------------------------------------------- host logic
def _line(xy):
    return {"type": "LineString", "coordinates": np.asarray(xy, dtype=np.float64)}


def test_line_azimuth_and_wrap():
    assert gis.line_azimuth(_line([[0, 0], [0, -1]])) == pytest.approx(0.0)  # start north of the end
    assert gis.line_azimuth(_line([[1, 0], [0, 0]])) == pytest.approx(np.pi / 2)
    assert gis.line_azimuth(_line([[0, 0], [1, 0]])) == pytest.approx(-np.pi / 2)
    ring = {"type": "LinearRing", "coordinates": np.array([[0.0, 0.0], [1.0, 1.0], [0.0, 0.0]])}
    assert gis.line_azimuth(ring) == 0.0
    _, _, df = convert._line_parameters([_line([[0, 0], [1, 0]]), _line([[0, 0], [-1, -1]])], 1e-4, {})
    # negative azimuths get + pi (convert.py:1340); the value stays in radians and goes in as psi
    np.testing.assert_allclose(df["psi"].values, [np.pi / 2, np.arctan2(1, 1)])


def test_psi_quirk_is_reproduced():
    """line_rating hands its azimuth (radians) to convert_line_rating as psi (degrees): a line
    at 90 deg rates as a line at psi = pi / 2 degrees."""
    _, _, df = convert._line_parameters([_line([[1, 0], [0, 0]])], IEEE_LINE["R"], {})
    assert df["psi"].iloc[0] == pytest.approx(np.pi / 2)
    assert not np.isclose(LO.convert_line_rating(IEEE, np.pi / 2, **IEEE_LINE),
                          LO.convert_line_rating(IEEE, 90, **IEEE_LINE))


def test_parameters_align_by_index_and_assert():
    lines = {"a": _line([[0, 0], [1, 1]]), "b": _line([[0, 0], [2, 1]]), "c": _line([[0, 0], [1, 3]])}
    R = pd.Series([3.0, 1.0, 2.0], index=["c", "a", "b"])
    _, dim, df = convert._line_parameters(lines, R, {"D": pd.Series({"b": 0.02, "a": 0.01, "c": 0.03})})
    assert dim == "concat_dim" and list(df.index) == ["a", "b", "c"]  # R's unnamed index drops "dim_0"
    np.testing.assert_array_equal(df["R"].values, [1.0, 2.0, 3.0])
    np.testing.assert_array_equal(df["D"].values, [0.01, 0.02, 0.03])
    assert list(df.columns) == ["psi", "R", "D", "Ts", "epsilon", "alpha"]
    with pytest.raises(AssertionError, match="Nan values encountered."):
        convert._line_parameters(lines, pd.Series([1.0, 2.0], index=["a", "b"]), {})
    with pytest.raises(AssertionError):  # params in another order than the reference's columns
        convert._line_parameters(lines, 1e-4, {"alpha": 0.5, "D": 0.03})
    with pytest.raises(AssertionError):
        convert._line_parameters(lines, 1e-4, {"unknown": 1.0})


class GeoSeries(pd.Series):
    """Stands in for geopandas.GeoSeries (matched by class name, as without geopandas)."""


def test_line_dimension_naming():
    """xr.concat(..., dim=df.index) names the line dimension after the parameter table's index."""
    ln = [_line([[0, 0], [1, 1]]), _line([[0, 0], [2, 1]])]
    s, dim, _ = convert._line_parameters(ln, 1e-4, {})
    assert dim == "dim_0" and list(s.index) == [0, 1] and s.index.name == "dim_0"
    s, dim, _ = convert._line_parameters({"x": ln[0], "y": ln[1]}, 1e-4, {})
    assert dim == "dim_0" and list(s.index) == ["x", "y"]
    s, dim, _ = convert._line_parameters(pd.Series(ln, index=pd.Index([7, 9], name="Line")), 1e-4, {})
    assert dim == "dim_0" and list(s.index) == [7, 9]  # GeoSeries(shapes).rename_axis("dim_0")
    s, dim, _ = convert._line_parameters(GeoSeries(ln, index=pd.Index(["l1", "l2"], name="Line")), 1e-4, {})
    assert dim == "Line" and list(s.index) == ["l1", "l2"]
    _, dim, _ = convert._line_parameters(GeoSeries(ln), 1e-4, {})
    assert dim == "concat_dim"
    # a Series parameter whose index name differs: pandas drops the name of the union
    _, dim, df = convert._line_parameters({"x": ln[0], "y": ln[1]}, pd.Series([1e-4, 2e-4], index=["y", "x"]), {})
    assert dim == "concat_dim" and df.index.name is None
    R = pd.Series([1e-4, 2e-4], index=pd.Index(["x", "y"], name="dim_0"))
    _, dim, _ = convert._line_parameters({"x": ln[0], "y": ln[1]}, R, {})
    assert dim == "dim_0"


class _FakeCutout:
    def __init__(self, data, time_shard=None):
        self.data, self.time_shard, self.devices = data, time_shard, None

    def intersectionmatrix(self, shapes):  # never reached by the error paths below
        raise AssertionError("not expected")


def test_errors_for_shapes_variables_and_time_shards():
    ds = syn.make_line_rating_dataset(8, 6, 4)
    poly = {"type": "Polygon", "coordinates": [[[0, 0], [1, 0], [1, 1], [0, 0]]]}
    with pytest.raises(TypeError, match="LineString or LinearRing, not Polygon"):
        convert._line_parameters([poly], 1e-4, {})
    with pytest.raises(TypeError, match="not MultiLineString"):
        convert._line_parameters([{"type": "MultiLineString", "coordinates": [[[0, 0], [1, 1]]]}], 1e-4, {})
    x, y = ds.coords["x"], ds.coords["y"]
    lines = [_line([[x[0], y[0]], [x[3], y[2]]])]
    d2 = ab.Dataset({k: ds.raw(k) for k in ds.keys() if k != "wnd_azimuth"},
                    coords=dict(ds.coords))
    with pytest.raises(KeyError, match="wnd_azimuth"):
        ab.line_rating(_FakeCutout(d2), lines, 1e-4)
    with pytest.raises(NotImplementedError, match="time-sharded"):
        ab.line_rating(_FakeCutout(ds, time_shard=object()), lines, 1e-4)
    with pytest.raises(TypeError, match="dict"):
        ab.convert_line_rating(ds, 90, 1e-4)


# ---------------------------------------------------------------- GPU
def _flat(ds, psi, R, **kw):
    return ab.convert_line_rating(ds, psi, R, **kw)


@pytest.mark.gpu
def test_flat_known_answers_and_symmetries():
    want = LO.convert_line_rating(IEEE, 90, **IEEE_LINE)
    assert_parity(_flat(IEEE, 90, **IEEE_LINE), want, what="dlr flat ieee")
    for ds, psi in _symmetry_cases():
        _rel_close(_flat(ds, psi, **IEEE_LINE), want, 1e-6)
    psis = np.arange(0, 370, 10.0)
    assert_parity(_flat(IEEE, psis, **IEEE_LINE), LO.convert_line_rating(IEEE, psis, **IEEE_LINE), what="dlr flat psi")
    i = _flat(dict(CALM, temperature=293.0), 0, 0.0136e-3, Ts=363)  # Suedkabel
    assert np.isclose(i, 2460, rtol=0.02)
    al = dict(R=0.1188e-3, D=0.0218, Ts=353.0, epsilon=0.8, alpha=0.8)  # Oeding / Oswald Al 240/40
    i = _flat(dict(CALM, temperature=303.0), 90, **al)
    assert np.isclose(i, 645, rtol=0.015)
    assert_parity(i, LO.convert_line_rating(dict(CALM, temperature=303.0), 90, **al), what="dlr flat al240")
    g = _golden()
    d = {k[5:]: g[k] for k in g if k.startswith("flat_") and k != "flat_psi"}
    got = _flat(d, g["flat_psi"], 1e-4, D=0.03, Ts=368.0, epsilon=0.7, alpha=0.5)
    assert_parity(got, LO.convert_line_rating(d, g["flat_psi"], 1e-4, D=0.03, Ts=368.0, epsilon=0.7, alpha=0.5),
                  what="dlr flat golden")


def _planted_dataset(nx, ny, nt, solar=None, **kw):
    """make_line_rating_dataset with a NaN cell, a NaN step and a cell hotter than Ts; ``solar``:
    None (computed in-kernel), np.float64 / np.float32 (stored, from the oracle's almanac)."""
    ds = syn.make_line_rating_dataset(nx, ny, nt, **kw)
    t = np.array(ds.raw("temperature"))
    t[:, 3, 5] = np.nan  # every step: a cell no line may take
    t[2:5, 6, 2] = np.nan
    t[4:9, 1, 7] = 380.0  # Ta > Ts: NaN, skipped
    ds["temperature"] = t
    if solar is not None:
        import atlite_oracle as O

        p = O.solar_position({"time": ds.coords["time"], "lon": ds.coords["lon"], "lat": ds.coords["lat"]},
                             time_shift="-30min")
        ds["solar_altitude"] = np.ascontiguousarray(np.broadcast_to(p["altitude"], t.shape), dtype=solar)
        ds["solar_azimuth"] = np.ascontiguousarray(np.broadcast_to(p["azimuth"], t.shape), dtype=solar)
    return ds


def _network(x, y, n_sites=12):
    """make_line_network plus two multi-cell lines through the planted cells (along row 3 across
    the all-NaN cell (3, 5), along row 1 across the Ta > Ts cell (1, 7)), then a line outside the
    grid, a one-cell line and a line through the all-NaN cell (3, 5) only."""
    lines = syn.make_line_network(x, y, n_sites)
    dx = x[1] - x[0]
    lines.append(_line([[x[4], y[3]], [x[6], y[3]]]))
    lines.append(_line([[x[6], y[1]], [x[8], y[1]]]))
    lines.append(_line([[x[-1] + 5 * dx, y[0]], [x[-1] + 9 * dx, y[-1]]]))
    lines.append(_line([[x[4] - 0.2 * dx, y[2] + 0.1 * dx], [x[4] + 0.3 * dx, y[2] - 0.2 * dx]]))
    lines.append(_line([[x[5] - 0.2 * dx, y[3] + 0.1 * dx], [x[5] + 0.2 * dx, y[3] - 0.1 * dx]]))
    return lines


def _oracle(cut_ds, lines, R=1e-4, **params):
    """The oracle on ``lines`` (a list, or a dict whose keys label the lines)."""
    ds = {k: np.asarray(cut_ds.raw(k)) for k in cut_ds.keys()}
    ds.update(time=cut_ds.coords["time"], lon=np.asarray(cut_ds.coords["lon"]), lat=np.asarray(cut_ds.coords["lat"]))
    x, y = np.asarray(cut_ds.coords["x"]), np.asarray(cut_ds.coords["y"])
    s = convert._line_shapes(lines)
    I = sp.csr_matrix(IX.intersectionmatrix(x, y, [gis.geometry_parts(g) for g in s.values]))
    az = pd.Series([LO.line_azimuth(g["coordinates"]) for g in s.values], index=s.index)
    return LO.line_rating(ds, I, az, R, **params)


@pytest.mark.gpu
@pytest.mark.parametrize("solar", [None, np.float64, np.float32])
@pytest.mark.parametrize("layout", ["device_vec", "device_padded", "device_scalar", "host"])
def test_fused_line_rating_matches_oracle(solar, layout):
    nx = 36 if layout == "device_vec" else 35
    ds = _planted_dataset(nx, 14, 29, solar=solar, x0=6.0, y0=47.0)
    x, y = np.asarray(ds.coords["x"]), np.asarray(ds.coords["y"])
    lines = _network(x, y)
    cut = ab.Cutout(data=ds)
    if layout.startswith("device"):
        cut = cut.to_device(pad=layout != "device_scalar")
    import warnings

    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        res = cut.line_rating(lines, 1e-4)
    assert any(issubclass(k.category, DeprecationWarning) for k in w) == (solar is None)
    assert res.dims == ("dim_0", "time") and res.attrs["units"] == "A"
    want = _oracle(ds, lines)
    got = np.asarray(res.values)
    assert np.isnan(want[-3]).all() and np.isnan(want[-1]).all()  # outside the grid; only a NaN cell
    assert np.isfinite(want[-2]).all()
    # the planted cells lie on multi-cell lines: the NaN cell is skipped, the Ta > Ts cell too
    I = IX.intersectionmatrix(x, y, [gis.geometry_parts(g) for g in lines])
    row_nan, row_hot = len(lines) - 5, len(lines) - 4
    assert I[row_nan, 3 * nx + 5] == 1 and I[row_nan].sum() > 1
    assert I[row_hot, 1 * nx + 7] == 1 and I[row_hot].sum() > 1
    assert np.isfinite(want[row_nan]).all() and np.isfinite(want[row_hot]).all()
    assert_parity(got, want, what="dlr fused")


@pytest.mark.gpu
def test_series_parameters():
    ds = _planted_dataset(33, 10, 13)
    x, y = np.asarray(ds.coords["x"]), np.asarray(ds.coords["y"])
    lines = {f"L{i}": s for i, s in enumerate(_network(x, y, 8))}
    idx = list(lines)
    rng = np.random.default_rng(3)
    R = pd.Series(rng.uniform(5e-5, 2e-4, len(idx)), index=idx[::-1])
    params = {"D": pd.Series(rng.uniform(0.02, 0.04, len(idx)), index=idx), "Ts": 363.0,
              "epsilon": pd.Series(rng.uniform(0.5, 0.9, len(idx)), index=idx)}
    res = ab.Cutout(data=ds).to_device().line_rating(lines, R, **params)
    # pandas sorts the union of the shapes' and R's index, and row i of that table meets row i of
    # the intersection matrix (shapes order) as in the reference (convert.py:1347, 1354-1358)
    # (R's unnamed index drops the shapes' "dim_0" from the union: xr.concat names it "concat_dim")
    _, dim, df = convert._line_parameters(lines, R, params)
    assert res.dims == ("concat_dim", "time") and dim == "concat_dim"
    assert list(np.asarray(res.coords["concat_dim"])) == list(df.index) == sorted(idx)
    assert_parity(np.asarray(res.values), _oracle(ds, lines, R, **params), what="dlr series")


@pytest.mark.gpu
def test_host_float64_fields():
    """A host-resident cutout whose weather fields and height are float64 (CF-decoded packed ERA5,
    NumPy-built datasets) is cast on the host like every other converter's input: the result equals
    the float32 cutout's bit for bit and the oracle on the float64 fields at the parity bar."""
    ds32 = _planted_dataset(35, 12, 30, solar=np.float64)
    x, y = np.asarray(ds32.coords["x"]), np.asarray(ds32.coords["y"])
    lines = _network(x, y)
    ds64 = ab.Dataset({k: np.asarray(ds32.raw(k), dtype=np.float64) for k in ds32.keys()},
                      coords=dict(ds32.coords))
    assert all(np.asarray(ds64.raw(k)).dtype == np.float64 for k in ds64.keys())
    got = np.asarray(ab.Cutout(data=ds64).line_rating(lines, 1e-4).values)
    assert np.array_equal(got, np.asarray(ab.Cutout(data=ds32).line_rating(lines, 1e-4).values), equal_nan=True)
    assert_parity(got, _oracle(ds64, lines), what="dlr host float64")


@pytest.mark.gpu
def test_dense_network_on_a_coarse_grid():
    """More than 24 slots and 256 entries per tile: the plan does not tile (fused = 0) and the
    kernel walks its entry lists from global memory."""
    ds = syn.make_line_rating_dataset(40, 8, 11, dx=1.0, dy=1.0, x0=0.0, y0=40.0)
    x, y = np.asarray(ds.coords["x"]), np.asarray(ds.coords["y"])
    lines = syn.make_line_network(x, y, 220)
    I = gis.compute_intersectionmatrix(x, y, lines)
    info = engine.Plan(I, 8, 40, entries=True).info
    assert info["slots_per_active_tile"] > 24 and info["n_pairs"] / info["n_active_tiles"] > 256
    assert not info["fused"]
    res = ab.Cutout(data=ds).to_device().line_rating(lines, 1e-4)
    assert_parity(np.asarray(res.values), _oracle(ds, lines), what="dlr dense")


@pytest.mark.gpu
def test_residency_and_repeatability(tmp_path):
    ds = _planted_dataset(37, 12, 250)
    x, y = np.asarray(ds.coords["x"]), np.asarray(ds.coords["y"])
    lines = _network(x, y)
    cut = ab.Cutout(data=ds)
    dev = np.asarray(cut.to_device().line_rating(lines, 1e-4).values)
    host = np.asarray(cut.line_rating(lines, 1e-4).values)
    pinned = np.asarray(cut.pin_host().line_rating(lines, 1e-4).values)
    path = str(tmp_path / "lr.atl")
    cut.to_file(path)
    lazy = ab.Cutout(path)
    assert getattr(lazy.data, "lazy", False)
    lz = np.asarray(lazy.line_rating(lines, 1e-4).values)
    for other in (host, pinned, lz):
        assert np.array_equal(dev, other, equal_nan=True)
    assert np.array_equal(dev, np.asarray(cut.to_device().line_rating(lines, 1e-4).values), equal_nan=True)
    prev = _lib.set_deterministic(True)
    try:
        det = np.asarray(cut.to_device().line_rating(lines, 1e-4).values)
    finally:
        _lib.set_deterministic(prev)
    assert np.array_equal(dev, det, equal_nan=True)
    assert_parity(dev, _oracle(ds, lines), what="dlr residency")


@pytest.mark.gpu
def test_multi_device_equals_single():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ds = _planted_dataset(33, 10, 40)
    lines = _network(np.asarray(ds.coords["x"]), np.asarray(ds.coords["y"]))
    one = np.asarray(ab.Cutout(data=ds).line_rating(lines, 1e-4).values)
    many = np.asarray(ab.Cutout(data=ds, devices="all").line_rating(lines, 1e-4).values)
    assert np.array_equal(one, many, equal_nan=True)


@pytest.mark.gpu
def test_europe_sized_window():
    """One 48-step window of the 220 x 160 grid at 0.25 deg with the ~6000-line network."""
    ds = syn.make_line_rating_dataset(220, 160, 48, x0=-10.0, y0=35.0)
    x, y = np.asarray(ds.coords["x"]), np.asarray(ds.coords["y"])
    lines = syn.make_line_network(x, y, 2000)
    res = ab.Cutout(data=ds).to_device().line_rating(lines, 1e-4)
    I = gis.compute_intersectionmatrix(x, y, lines)
    d = {k: np.asarray(ds.raw(k)) for k in ds.keys()}
    d.update(time=ds.coords["time"], lon=x, lat=y)
    az = pd.Series([LO.line_azimuth(l["coordinates"]) for l in lines])
    assert_parity(np.asarray(res.values), LO.line_rating(d, I, az, 1e-4), what="dlr europe window")
