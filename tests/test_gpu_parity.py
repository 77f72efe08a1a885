"""GPU parity tests: the CUDA path (through the C ABI / public API) against the
float64 oracle on the same seeded synthetic inputs.

Tolerance (stated once, see conftest.assert_parity; SURVEY.md section 8c): fp32
kernels vs float64 oracle, |gpu - oracle| <= 1e-4 * max(|oracle|, 1e-6 * capacity_bus).
"""

import warnings

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp
from conftest import assert_parity, oracle_ds

import atlite_oracle as O
import atlite_b200 as ab
from atlite_b200 import _lib, engine, synthetic as syn

pytestmark = pytest.mark.gpu

warnings.filterwarnings("ignore", category=DeprecationWarning)


def cap_of(m):
    return np.asarray(sp.csr_matrix(m).sum(-1)).flatten()


def bt(res):
    """public API result (bus, time) -> oracle layout (time, bus)"""
    assert res.dims[1] == "time"
    return np.asarray(res.values).T


@pytest.fixture(scope="module")
def ds_full():
    # 70 x 45 cells (neither a multiple of 32 nor of 4), 3 days, both hemispheres
    return syn.make_dataset(70, 45, 72, x0=-10.0, y0=-20.0, dx=0.5, dy=1.0,
                            extra=("wnd_shear_exp", "humidity"))


@pytest.fixture(scope="module")
def shapes(ds_full):
    return syn.make_shapes(70, 45, 23)


# ------------------------------------------------------------------ wind


@pytest.mark.parametrize("turbine", ["Vestas_V112_3MW", "Enercon_E126_7500kW", "NREL_ReferenceTurbine_5MW_offshore"])
@pytest.mark.parametrize("method", ["logarithmic", "power"])
def test_wind_reduce(ds_full, shapes, turbine, method):
    c = ab.Cutout(data=ds_full)
    res = c.wind(turbine, matrix=shapes, interpolation_method=method, aggregate_time=None)
    t = ab.get_windturbineconfig(turbine)
    want = O.convert_and_aggregate(oracle_ds(ds_full), O.convert_wind, matrix=shapes,
                                   aggregate_time=None, turbine=t, interpolation_method=method)
    assert_parity(bt(res), want, cap_of(shapes), what=f"wind {turbine} {method}")
    assert res.attrs["units"] == "MW"


def test_wind_smooth_and_fast_lane(ds_full, shapes):
    c = ab.Cutout(data=ds_full)
    t = O.windturbine_smooth(ab.get_windturbineconfig("Vestas_V112_3MW"))
    res = c.wind("Vestas_V112_3MW", smooth=True, matrix=shapes, aggregate_time=None)
    want = O.convert_and_aggregate(oracle_ds(ds_full), O.convert_wind, matrix=shapes,
                                   aggregate_time=None, turbine=t)
    assert_parity(bt(res), want, cap_of(shapes), what="wind smooth")
    # hub height == available height: wind.py:75-78
    t100 = dict(ab.get_windturbineconfig("Vestas_V112_3MW"), hub_height=100)
    res = c.wind(t100, matrix=shapes, aggregate_time=None)
    want = O.convert_and_aggregate(oracle_ds(ds_full), O.convert_wind, matrix=shapes,
                                   aggregate_time=None, turbine=t100)
    assert_parity(bt(res), want, cap_of(shapes), what="wind fast lane")


def test_wind_interp_edges():
    """np.interp semantics at and around the knots: duplicate cut-out knot, values
    below the first / above the last knot, NaN, zero/negative roughness."""
    nx, ny, nt = 33, 5, 2
    ds = syn.make_dataset(nx, ny, nt, kinds=("wind",))
    t = dict(ab.get_windturbineconfig("Vestas_V112_3MW"), hub_height=100)  # no extrapolation
    w = ds.raw("wnd100m")
    specials = np.array([0.0, 2.0, np.nextafter(np.float32(2.0), np.float32(3)), 3.0, 12.999999, 13.0, 24.999998,
                         25.0, np.nextafter(np.float32(25.0), np.float32(26)), 30.0, 1e6, -1.0, 1e-30],
                        dtype=np.float32)
    w[0, 0, : len(specials)] = specials
    c = ab.Cutout(data=ds).to_device()
    got = np.asarray(c.wind(t, aggregate_time=None).values)
    want = O.convert_wind(oracle_ds(ds), t)
    assert_parity(got, want, what="interp edges")
    assert got[0, 0, 7] == 0.0 and got[0, 0, 6] == 1.0  # exactly at / just below cut-out
    # NaN propagates to exactly the buses that contain the cell
    w[1, 2, 3] = np.nan
    r = ds.raw("roughness")
    r[1, 1, 1] = 0.0
    r[1, 1, 2] = -1.0
    m = sp.csr_matrix(np.kron(np.eye(ny), np.ones((1, nx))))  # one bus per row of cells
    t80 = ab.get_windturbineconfig("Vestas_V112_3MW")
    got = bt(ab.Cutout(data=ds).wind(t80, matrix=m, aggregate_time=None))
    want = O.convert_and_aggregate(oracle_ds(ds), O.convert_wind, matrix=m, aggregate_time=None, turbine=t80)
    assert np.isnan(want[1, 2]) and np.isnan(want[1, 1]) and not np.isnan(want[1, 0])
    assert_parity(got, want, cap_of(m), what="NaN routing")


def test_result_tail_on_the_device_equals_the_numpy_statement():
    """convert._finish_results on a CUDA tensor (float64, per-unit with a zero-capacity bus, NaN -> 0,
    inf kept, NaN-skipping aggregation, (bus, time) layout) against the NumPy statement of
    convert.py:259-271; and through the public call: per_unit + return_capacity + aggregate_time on a
    device-resident cutout equal the host-resident cutout's results."""
    import torch

    from atlite_b200 import convert

    rng = np.random.default_rng(0)
    res = rng.uniform(0, 5, (53, 17)).astype(np.float32)
    res[3, 2], res[5, 4] = np.nan, np.inf
    res[:, 7] = np.nan
    caps = rng.uniform(1, 3, 17)
    caps[1] = 0.0
    for c in (None, caps):
        for agg in (None, "sum", "mean"):
            for bus_major in (False, True):
                want = convert._finish_results(res, c, agg, bus_major)
                got = convert._finish_results(torch.from_numpy(res).cuda(), c, agg, bus_major)
                assert got.dtype == np.float64 and got.shape == want.shape
                np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
                np.testing.assert_allclose(got, want, rtol=1e-14, atol=0)
    ds = syn.make_dataset(40, 24, 30, x0=0.0, y0=30.0)
    m = syn.make_shapes(40, 24, 6).tolil()
    m[2, :] = 0  # a bus without cells: capacity 0 -> per-unit 0
    m = m.tocsr()
    for kw in (dict(aggregate_time=None), dict(aggregate_time="mean"), dict(aggregate_time="sum")):
        host, cap_h = ab.Cutout(data=ds).wind("Vestas_V112_3MW", matrix=m, per_unit=True, return_capacity=True, **kw)
        dev, cap_d = ab.Cutout(data=ds).to_device().wind("Vestas_V112_3MW", matrix=m, per_unit=True,
                                                         return_capacity=True, **kw)
        assert host.dims == dev.dims and host.attrs["units"] == dev.attrs["units"] == "p.u."
        np.testing.assert_allclose(np.asarray(dev.values), np.asarray(host.values), rtol=1e-4, atol=1e-6)
        np.testing.assert_array_equal(np.asarray(cap_d.values), np.asarray(cap_h.values))
        assert np.all(np.asarray(dev.values)[2] == 0.0) if kw["aggregate_time"] is None else np.asarray(dev.values)[2] == 0.0


@pytest.mark.parametrize("table", [0, 1, 2, 3])
def test_wind_every_table_form(monkeypatch, table):
    """ATL_WIND_TABLE forces the power-curve table form (binary search, general LUT, lattice LUT with
    compares, saturating lattice LUT): each one is np.interp -- at the knots, one float either side, beyond
    the ends, for +-inf (the saturating table serves those through the cold exact path) and NaN -- in the
    per-cell kernel and in the fused reduce (resident weights, several slot groups per tile)."""
    monkeypatch.setenv("ATL_WIND_TABLE", str(table))
    nx, ny, nt = 132, 6, 5
    ds = syn.make_dataset(nx, ny, nt, kinds=("wind",))
    t = dict(ab.get_windturbineconfig("Vestas_V112_3MW"), hub_height=100)  # no extrapolation
    w = ds.raw("wnd100m")
    f32 = np.float32
    specials = np.array([0.0, 2.0, np.nextafter(f32(3.0), f32(0)), 3.0, np.nextafter(f32(3.0), f32(9)), 12.999999, 13.0,
                         np.nextafter(f32(25.0), f32(0)), 25.0, np.nextafter(f32(25.0), f32(26)), 30.0, 1e6, 1e30,
                         np.inf, -np.inf, -1.0, -1e30, 1e-30], dtype=np.float32)
    w[0, 0, : len(specials)] = specials
    w[2, 3, 40: 40 + len(specials)] = specials
    c = ab.Cutout(data=ds).to_device()
    with np.errstate(invalid="ignore"):
        got = np.asarray(c.wind(t, aggregate_time=None).values)
        want = O.convert_wind(oracle_ds(ds), t)
    assert_parity(got, want, what=f"table {table}: per-cell")
    assert got[0, 0, 8] == 0.0 and got[0, 0, 7] == 1.0 and got[0, 0, 13] == 0.0 and got[0, 0, 14] == 0.0
    w[1, 2, 3] = np.nan
    m = syn.make_shapes(nx, ny, 40)  # many small shapes: tiles with more than one slot group
    for hub in (100, 80):
        tt = dict(t, hub_height=hub)
        with np.errstate(invalid="ignore", divide="ignore"):
            got = bt(ab.Cutout(data=ds).wind(tt, matrix=m, aggregate_time=None))
            want = O.convert_and_aggregate(oracle_ds(ds), O.convert_wind, matrix=m, aggregate_time=None, turbine=tt)
        assert np.isnan(want[1]).any() and not np.isnan(want[0]).any()
        assert_parity(got, want, cap_of(m), what=f"table {table}: reduce, hub {hub}")


def test_wind_interp_binary_search_fallback():
    """Knots too close for the uniform-bucket LUT -> branch-free binary search path."""
    ds = syn.make_dataset(40, 8, 6, kinds=("wind",))
    curve = dict(V=[0.0, 1.0, 1.0001, 3.0, 3.0, 7.5, 12.0, 25.0, 25.0],
                 POW=[0.0, 0.0, 0.1, 0.4, 0.5, 1.5, 2.0, 2.0, 0.0], P=2.0, hub_height=100)
    got = np.asarray(ab.Cutout(data=ds).to_device().wind(dict(curve), aggregate_time=None).values)
    want = O.convert_wind(oracle_ds(ds), ab.get_windturbineconfig(dict(curve)))
    assert_parity(got, want, what="binary search fallback")
    m = syn.make_shapes(40, 8, 3)
    got = bt(ab.Cutout(data=ds).wind(dict(curve, hub_height=80), matrix=m, aggregate_time=None))
    want = O.convert_and_aggregate(oracle_ds(ds), O.convert_wind, matrix=m, aggregate_time=None,
                                   turbine=ab.get_windturbineconfig(dict(curve, hub_height=80)))
    assert_parity(got, want, cap_of(m), what="binary search fallback, reduce")


# ------------------------------------------------------------------ pv


PV_CASES = [
    dict(panel="CSi", orientation="latitude_optimal"),
    dict(panel="CdTe", orientation={"slope": 0.0, "azimuth": 0.0}),
    dict(panel="KANENA", orientation="latitude_optimal"),
    dict(panel="CSi", orientation="latitude", trigon_model="other"),
    dict(panel="CSi", orientation={"slope": 35.0, "azimuth": 160.0}, trigon_model="other"),
    dict(panel="CSi", orientation={"slope": 0.0, "azimuth": 180.0}, tracking="horizontal"),
    dict(panel="CSi", orientation={"slope": 30.0, "azimuth": 170.0}, tracking="tilted_horizontal"),
    dict(panel="CSi", orientation={"slope": 30.0, "azimuth": 180.0}, tracking="vertical"),
    dict(panel="CdTe", orientation={"slope": 30.0, "azimuth": 180.0}, tracking="dual"),
    dict(panel="CSi", orientation={"slope": 25.0, "azimuth": 200.0}, tracking="horizontal", trigon_model="other"),
    dict(panel="CSi", orientation={"slope": 25.0, "azimuth": 200.0}, tracking="tilted_horizontal", trigon_model="other"),
    dict(panel="CSi", orientation={"slope": 25.0, "azimuth": 200.0}, tracking="dual", trigon_model="other"),
]


def _oracle_pv(ds, matrix, case, **kw):
    case = dict(case)
    panel = ab.get_solarpanelconfig(case.pop("panel"))
    orientation = O.get_orientation(case.pop("orientation"))
    return O.convert_and_aggregate(oracle_ds(ds) if not isinstance(ds, dict) else ds, O.convert_pv,
                                   matrix=matrix, aggregate_time=None, panel=panel,
                                   orientation=orientation, **case, **kw)


@pytest.mark.parametrize("case", PV_CASES, ids=lambda c: "-".join(str(v) for v in c.values())[:60])
def test_pv_reduce(ds_full, shapes, case):
    c = ab.Cutout(data=ds_full)
    res = c.pv(matrix=shapes, aggregate_time=None, **case)
    want = _oracle_pv(ds_full, shapes, case)
    assert_parity(bt(res), want, cap_of(shapes), what=f"pv {case}")
    assert want.sum() > 0


def test_pv_night_is_exactly_zero_and_capacity(ds_full, shapes):
    c = ab.Cutout(data=ds_full)
    lay = syn.make_layout(70, 45)
    layout = ab.DataArray(lay, {"y": ds_full.coords["y"], "x": ds_full.coords["x"]}, ("y", "x"))
    res, cap = c.pv("CdTe", {"slope": 0.0, "azimuth": 0.0}, matrix=shapes, layout=layout,
                    return_capacity=True, aggregate_time=None)
    want, wcap = O.convert_and_aggregate(
        oracle_ds(ds_full), O.convert_pv, matrix=shapes, layout=lay, return_capacity=True,
        aggregate_time=None, panel=ab.get_solarpanelconfig("CdTe"),
        orientation=O.get_orientation({"slope": 0.0, "azimuth": 0.0}))
    assert_parity(bt(res), want, wcap, what="pv layout")
    np.testing.assert_allclose(cap.values, wcap, rtol=1e-12)
    assert (bt(res)[want == 0] == 0).all(), "oracle-zero entries (night) must be exactly zero"
    assert (want == 0).any()
    assert cap.attrs["units"] == "MW"


@pytest.mark.parametrize("variant", ["influx_simple", "influx_enhanced", "outflux", "stored_f32", "stored_f64"])
def test_pv_input_variants(variant):
    extra = {"influx_simple": ("influx",), "influx_enhanced": ("influx", "humidity"),
             "outflux": ("outflux",), "stored_f32": (), "stored_f64": ()}[variant]
    ds = syn.make_dataset(40, 21, 48, x0=5.0, y0=35.0, kinds=("pv",), extra=extra)
    kw = {}
    if variant.startswith("stored"):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            sp_ = O.solar_position(oracle_ds(ds))
        dt = np.float32 if variant.endswith("f32") else np.float64
        ds["solar_altitude"] = sp_["altitude"].astype(dt)
        ds["solar_azimuth"] = sp_["azimuth"].astype(dt)
    if variant == "influx_simple":
        kw["clearsky_model"] = "simple"
    m = syn.make_shapes(40, 21, 9)
    case = dict(panel="CSi", orientation="latitude_optimal")
    res = ab.Cutout(data=ds).pv(matrix=m, aggregate_time=None, **case, **kw)
    # pv() passes clearsky_model=None by default (auto: enhanced iff humidity present)
    want = _oracle_pv(ds, m, case, clearsky_model=kw.get("clearsky_model"))
    assert_parity(bt(res), want, cap_of(m), what=variant)
    assert want.sum() > 0


def test_pv_missing_variables_raise():
    ds = syn.make_dataset(8, 6, 4, kinds=("pv",))
    d = {k: ds.raw(k) for k in ds.keys() if k != "albedo"}
    d.update(time=ds.coords["time"], x=ds.coords["x"], y=ds.coords["y"])
    with pytest.raises(AssertionError, match="albedo or outflux"):
        ab.Cutout(data=d).pv("CSi", "latitude_optimal", aggregate_time="sum")
    d.pop("influx_direct")
    with pytest.raises(AssertionError, match="influx_direct and influx_diffuse"):
        ab.Cutout(data=d).pv("CSi", "latitude_optimal", aggregate_time="sum")


# ------------------------------------------------------------------ heat demand


@pytest.mark.parametrize("hour_shift", [0.0, 4.0, -5.0])
def test_heat_demand(ds_full, shapes, hour_shift):
    c = ab.Cutout(data=ds_full)
    res = c.heat_demand(threshold=17.0, a=1.3, constant=0.2, hour_shift=hour_shift,
                        matrix=shapes, aggregate_time=None)
    want = O.convert_and_aggregate(oracle_ds(ds_full), O.convert_heat_demand, matrix=shapes,
                                   aggregate_time=None, threshold=17.0, a=1.3, constant=0.2,
                                   hour_shift=hour_shift)
    assert_parity(bt(res), want, cap_of(shapes) * 50.0, what=f"heat {hour_shift}")
    labels, _ = O.day_bins(ds_full.coords["time"], hour_shift)
    assert list(pd.DatetimeIndex(res.coords["time"])) == list(labels)


# ------------------------------------------------------------------ further converters (SURVEY 8 f3)


@pytest.fixture(scope="module")
def ds_more():
    return syn.make_dataset(44, 26, 60, x0=-6.0, y0=-15.0, dx=0.75, dy=2.0,
                            extra=("soil temperature", "dewpoint temperature", "runoff"))


@pytest.fixture(scope="module")
def shapes_more():
    return syn.make_shapes(44, 26, 11)


@pytest.mark.parametrize("kind,kw", [
    ("total", {}), ("direct", {}), ("diffuse", {}), ("ground", {}),
    ("total", dict(trigon_model="other")), ("diffuse", dict(trigon_model="other")),
    ("total", dict(tracking="horizontal")), ("direct", dict(tracking="tilted_horizontal")),
    ("total", dict(tracking="dual")),
])
def test_irradiation(ds_more, shapes_more, kind, kw):
    o = {"slope": 30.0, "azimuth": 170.0}
    res = ab.Cutout(data=ds_more).irradiation(o, irradiation=kind, matrix=shapes_more, aggregate_time=None, **kw)
    want = O.convert_and_aggregate(oracle_ds(ds_more), O.convert_irradiation, matrix=shapes_more,
                                   aggregate_time=None, orientation=O.get_orientation(o), irradiation=kind,
                                   clearsky_model=None, **kw)
    assert_parity(bt(res), want, cap_of(shapes_more) * 1000.0, what=f"irradiation {kind} {kw}")
    assert want.sum() > 0


def test_solar_thermal(ds_more, shapes_more):
    c = ab.Cutout(data=ds_more)
    res = c.solar_thermal(matrix=shapes_more, aggregate_time=None)
    want = O.convert_and_aggregate(
        oracle_ds(ds_more), O.convert_solar_thermal, matrix=shapes_more, aggregate_time=None,
        orientation=O.get_orientation({"slope": 45.0, "azimuth": 180.0}), trigon_model="simple",
        clearsky_model="simple", c0=0.8, c1=3.0, t_store=80.0)
    assert_parity(bt(res), want, cap_of(shapes_more) * 1000.0, what="solar thermal")
    assert want.sum() > 0
    res = c.solar_thermal("latitude_optimal", c0=0.7, c1=2.0, t_store=40.0, aggregate_time="sum")
    want = O.convert_solar_thermal(oracle_ds(ds_more), O.get_orientation("latitude_optimal"), "simple", "simple",
                                   0.7, 2.0, 40.0).sum(0)
    assert_parity(res.values, want, 60 * 1000.0, what="solar thermal cells sum")


def test_temperature_family_and_cop(ds_more, shapes_more):
    c = ab.Cutout(data=ds_more)
    od = oracle_ds(ds_more)
    capk = cap_of(shapes_more) * 300.0
    for meth, fn in (("temperature", O.convert_temperature), ("soil_temperature", O.convert_soil_temperature),
                     ("dewpoint_temperature", O.convert_dewpoint_temperature)):
        res = getattr(c, meth)(matrix=shapes_more, aggregate_time=None)
        want = O.convert_and_aggregate(od, fn, matrix=shapes_more, aggregate_time=None)
        assert not np.isnan(want).any() or meth != "soil_temperature"
        assert_parity(bt(res), want, capk, what=meth, additive=True)  # signed deg C values: bus sums cancel
    assert_parity(c.temperature(aggregate_time="mean").values, O.convert_temperature(od).mean(0), 300.0,
                  what="temperature mean", additive=True)
    assert_parity(c.to_device().soil_temperature(aggregate_time=None).values, O.convert_soil_temperature(od),
                  300.0, what="soil cells", additive=True)
    for args in (dict(), dict(source="soil", sink_T=45.0), dict(sink_T=35.0, c0=7.0, c1=-0.1, c2=0.0005)):
        res = c.coefficient_of_performance(matrix=shapes_more, aggregate_time=None, **args)
        full = dict(dict(source="air", sink_T=55.0, c0=None, c1=None, c2=None), **args)
        want = O.convert_and_aggregate(od, O.convert_coefficient_of_performance, matrix=shapes_more,
                                       aggregate_time=None, **full)
        assert_parity(bt(res), want, cap_of(shapes_more) * 10.0, what=f"cop {args}")
    with pytest.raises(AssertionError):
        c.coefficient_of_performance(source="water", aggregate_time="sum")


@pytest.mark.parametrize("hour_shift", [0.0, 3.0])
def test_cooling_demand(ds_more, shapes_more, hour_shift):
    res = ab.Cutout(data=ds_more).cooling_demand(threshold=5.0, a=1.7, constant=0.3, hour_shift=hour_shift,
                                                 matrix=shapes_more, aggregate_time=None)
    want = O.convert_and_aggregate(oracle_ds(ds_more), O.convert_cooling_demand, matrix=shapes_more,
                                   aggregate_time=None, threshold=5.0, a=1.7, constant=0.3,
                                   hour_shift=hour_shift)
    assert_parity(bt(res), want, cap_of(shapes_more) * 50.0, what="cooling")
    assert want.sum() > 0


@pytest.mark.parametrize("inst,tech", [("SAM_solar_tower", None), ("SAM_parabolic_trough", None),
                                       ("SAM_parabolic_trough", "solar tower"), ("lossless_installation", "solar tower")])
def test_csp(ds_full, shapes, inst, tech):
    c = ab.Cutout(data=ds_full)
    res = c.csp(inst, technology=tech, matrix=shapes, aggregate_time=None)
    cfg = ab.get_cspinstallationconfig(inst)
    if tech is not None:
        cfg = dict(cfg, technology=tech)
    want = O.convert_and_aggregate(oracle_ds(ds_full), O.convert_csp, matrix=shapes, aggregate_time=None,
                                   installation=cfg)
    assert_parity(bt(res), want, cap_of(shapes), what=f"csp {inst} {tech}")
    assert want.sum() > 0 and res.attrs["units"] == "MW"
    with pytest.raises(ValueError, match="Unknown CSP technology"):
        c.csp("lossless_installation", aggregate_time="sum")


def test_csp_cells_and_stored_solar():
    ds = syn.make_dataset(36, 22, 48, x0=5.0, y0=-10.0, dx=1.0, dy=2.0, kinds=("pv",))
    cfg = ab.get_cspinstallationconfig("SAM_solar_tower")
    got = ab.Cutout(data=ds).to_device().csp(cfg, aggregate_time=None)
    want = O.convert_csp(oracle_ds(ds), cfg)
    assert_parity(got.values, want, what="csp cells")
    assert got.attrs["units"] == "kWh/kW_ref"
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sp_ = O.solar_position(oracle_ds(ds))
    ds["solar_altitude"], ds["solar_azimuth"] = sp_["altitude"], sp_["azimuth"]  # float64, as ERA5 cutouts store them
    m = syn.make_shapes(36, 22, 7)
    got = ab.Cutout(data=ds).csp(cfg, matrix=m, aggregate_time=None)
    want = O.convert_and_aggregate(oracle_ds(ds), O.convert_csp, matrix=m, aggregate_time=None, installation=cfg)
    assert_parity(bt(got), want, cap_of(m), what="csp stored solar")


def test_runoff(ds_more, shapes_more):
    c = ab.Cutout(data=ds_more)
    od = oracle_ds(ds_more)
    idx = pd.Index([f"c{i}" for i in range(11)], name="countries")
    for wh in (True, False):
        res = c.runoff(matrix=shapes_more, index=idx, aggregate_time=None, weight_with_height=wh)
        want = O.convert_and_aggregate(od, O.convert_runoff, matrix=shapes_more, aggregate_time=None,
                                       weight_with_height=wh)
        scale = np.abs(want).max(0)
        assert_parity(bt(res), want, scale * 10, what=f"runoff height={wh}")
    # post-processing of convert.py:1044-1058: rolling mean (min_periods=1) and lower-quantile cut
    sm = c.runoff(matrix=shapes_more, index=idx, aggregate_time=None, smooth=5, lower_threshold_quantile=0.1)
    base = O.convert_and_aggregate(od, O.convert_runoff, matrix=shapes_more, aggregate_time=None)
    roll = pd.DataFrame(base).rolling(5, min_periods=1).mean().values
    thr = pd.Series(roll.T.ravel()).quantile(0.1)
    want = np.where(roll >= thr, roll, 0.0)
    np.testing.assert_allclose(bt(sm), want, rtol=2e-4, atol=np.abs(want).max() * 1e-5)


# ------------------------------------------------------------------ orchestration semantics


def test_no_matrix_modes(ds_full):
    c = ab.Cutout(data=ds_full)
    od = oracle_ds(ds_full)
    t = ab.get_windturbineconfig("Vestas_V112_3MW")
    cube = c.wind("Vestas_V112_3MW", aggregate_time=None)
    assert cube.dims == ("time", "y", "x")
    want = O.convert_wind(od, t)
    assert_parity(cube.values, want, what="wind cells")
    assert_parity(c.wind("Vestas_V112_3MW", aggregate_time="mean").values, want.mean(0), what="wind mean")
    assert_parity(c.wind("Vestas_V112_3MW", aggregate_time="sum").values, want.sum(0), 72.0, what="wind sum")
    with pytest.warns(FutureWarning, match="legacy"):
        leg = c.pv("CSi", "latitude_optimal")
    pvw = O.convert_pv(od, ab.get_solarpanelconfig("CSi"), O.get_orientation("latitude_optimal"))
    assert leg.dims == ("y", "x")
    assert_parity(leg.values, pvw.sum(0), 72.0, what="pv legacy sum")
    hd = c.heat_demand(aggregate_time=None)
    hw, labels = O.convert_heat_demand(od, 15.0, 1.0, 0.0, 0.0)
    assert_parity(hd.values, hw, 50.0, what="heat cells", unit=300.0)  # differences of ~288 K float32 values
    assert_parity(c.heat_demand(aggregate_time="sum").values, hw.sum(0), 150.0, what="heat sum")


def test_per_unit_and_time_aggregation(ds_full, shapes):
    c = ab.Cutout(data=ds_full)
    od = oracle_ds(ds_full)
    t = ab.get_windturbineconfig("Vestas_V112_3MW")
    for agg in ("mean", "sum", None):
        res = c.wind("Vestas_V112_3MW", matrix=shapes, per_unit=True, aggregate_time=agg)
        want = O.convert_and_aggregate(od, O.convert_wind, matrix=shapes, per_unit=True,
                                       aggregate_time=agg, turbine=t)
        got = bt(res) if agg is None else res.values
        assert_parity(got, want, 72.0 if agg == "sum" else 1.0, what=f"per_unit {agg}")
        assert res.attrs["units"] == "p.u."
    # empty bus -> capacity 0 -> per-unit 0 (convert.py:264-266)
    m = sp.vstack([shapes, sp.csr_matrix((1, shapes.shape[1]))]).tocsr()
    res = c.wind("Vestas_V112_3MW", matrix=m, per_unit=True, aggregate_time=None)
    assert (bt(res)[:, -1] == 0).all()
    with pytest.warns(FutureWarning, match="legacy"):
        leg = c.wind("Vestas_V112_3MW", matrix=shapes)
    assert "time" in leg.dims
    idx = pd.Index([f"bus{i}" for i in range(23)], name="bus")
    res = c.wind("Vestas_V112_3MW", matrix=shapes, index=idx, aggregate_time="mean")
    assert res.dims == ("bus",) and list(res.coords["bus"]) == list(idx)
    with pytest.raises(ValueError, match="single dimension|pandas index"):
        c.wind("Vestas_V112_3MW", matrix=shapes, index=[1, 2, 3], aggregate_time=None)


def test_reference_aggregate_time_suite_on_gpu():
    """test/test_aggregate_time.py ported: MockCutout + identity_convert, layout path."""
    rng = np.random.RandomState(42)
    times = pd.date_range("2020-01-01", periods=24, freq="h")
    var = rng.rand(24, 3, 4)
    ds = ab.Dataset({"var": var}, coords=dict(time=times, y=[50.0, 51.0, 52.0], x=[5.0, 6.0, 7.0, 8.0]))
    cutout = ab.Cutout(data=ds)

    def identity_convert(d, **kwargs):
        return d["var"]

    layout = ab.DataArray(np.ones((3, 4)), {"y": ds.coords["y"], "x": ds.coords["x"]}, ("y", "x"))
    ts = ab.convert_and_aggregate(cutout, identity_convert, layout=layout, aggregate_time=None)
    assert "time" in ts.dims
    np.testing.assert_allclose(ts.values[0], var.reshape(24, -1).sum(1), rtol=1e-6)
    mean = ab.convert_and_aggregate(cutout, identity_convert, layout=layout, aggregate_time="mean")
    assert "time" not in mean.dims
    np.testing.assert_allclose(mean.values, ts.mean("time").values, rtol=1e-6)
    tot = ab.convert_and_aggregate(cutout, identity_convert, layout=layout, aggregate_time="sum")
    np.testing.assert_allclose(tot.values, ts.sum("time").values, rtol=1e-6)
    with pytest.warns(FutureWarning, match="aggregate_time='legacy'"):
        r = ab.convert_and_aggregate(cutout, identity_convert, layout=layout)
    assert "time" in r.dims
    lay2 = layout * 2.0
    pu = ab.convert_and_aggregate(cutout, identity_convert, layout=lay2, per_unit=True, aggregate_time="mean")
    pu_ts = ab.convert_and_aggregate(cutout, identity_convert, layout=lay2, per_unit=True, aggregate_time=None)
    np.testing.assert_allclose(pu.values, pu_ts.mean("time").values, rtol=1e-6)
    np.testing.assert_allclose(pu_ts.values[0], var.reshape(24, -1).mean(1), rtol=1e-6)
    with pytest.warns(FutureWarning, match="capacity_factor_timeseries is deprecated"):
        r = ab.convert_and_aggregate(cutout, identity_convert, layout=layout, capacity_factor_timeseries=True)
    assert "time" in r.dims


# ------------------------------------------------------------------ plans / matrices / paths


def test_plan_edge_cases(ds_full):
    c = ab.Cutout(data=ds_full)
    od = oracle_ds(ds_full)
    t = ab.get_windturbineconfig("Vestas_V112_3MW")
    S = 70 * 45
    rng = np.random.default_rng(0)
    mats = {
        "one_bus_all_cells": sp.csr_matrix(np.ones((1, S))),
        "identity_one_bus_per_cell": sp.identity(S, format="csr"),  # two-pass fallback
        "random_sparse": sp.random(11, S, density=0.02, random_state=3, format="csr"),
        "dense_rows": sp.csr_matrix(rng.uniform(0, 1, size=(5, S))),
        "empty": sp.csr_matrix((4, S)),
        "duplicates": sp.csr_matrix((np.ones(6), ([0, 0, 1, 1, 1, 2], [5, 5, 7, 7, 7, S - 1])), shape=(3, S)),
        "negative_and_zero_weights": sp.csr_matrix(
            (np.array([-1.5, 0.0, 2.0]), ([0, 0, 1], [0, 1, 2])), shape=(2, S)),
    }
    infos = {}
    for name, m in mats.items():
        res = c.wind("Vestas_V112_3MW", matrix=m, aggregate_time=None)
        want = O.convert_and_aggregate(od, O.convert_wind, matrix=m, aggregate_time=None, turbine=t)
        cap = np.asarray(abs(sp.csr_matrix(m)).sum(-1)).flatten()
        assert_parity(bt(res), want, cap, what=name)
        infos[name] = engine.get_plan(m, 45, 70).info
    assert infos["identity_one_bus_per_cell"]["fused"] == 0
    assert infos["one_bus_all_cells"]["fused"] == 1
    assert infos["empty"]["n_active_tiles"] == 0
    with pytest.raises(ValueError, match="columns"):
        c.wind("Vestas_V112_3MW", matrix=np.ones((2, 10)), aggregate_time=None)


def test_generic_convert_func_uses_gpu_spmm(ds_full, shapes):
    c = ab.Cutout(data=ds_full)

    def convert_custom(ds, scale):
        return ds["temperature"] * scale

    n0 = _lib.launch_count()
    res = c.convert_and_aggregate(convert_custom, matrix=shapes, aggregate_time=None, scale=0.5)
    assert _lib.launch_count() > n0
    want = (shapes @ (0.5 * ds_full.raw("temperature").astype(np.float64)).reshape(72, -1).T).T
    assert_parity(bt(res), want, cap_of(shapes) * 300, what="generic spmm")  # Kelvin values, all positive


def test_device_resident_matches_host_streaming(ds_full, shapes):
    """Same result through atl_*_reduce (device tensors) and atl_*_reduce_host
    (pinned/pageable host streaming with small slabs)."""
    host = ab.Cutout(data=ds_full)
    dev = host.to_device()
    a = host.pv("CSi", "latitude_optimal", matrix=shapes, aggregate_time=None).values
    b = dev.pv("CSi", "latitude_optimal", matrix=shapes, aggregate_time=None).values
    np.testing.assert_allclose(a, b, rtol=2e-5, atol=1e-6)
    plan = engine.get_plan(shapes, 45, 70)
    spec_fields = {k: ds_full.raw(k) for k in ("influx_toa", "influx_direct", "influx_diffuse", "albedo", "temperature")}
    from atlite_b200.convert import _PvSpec

    spec = _PvSpec(ds_full, ab.get_solarpanelconfig("CSi"), ab.get_orientation("latitude_optimal"))
    whole = spec.op.reduce(plan, spec_fields)
    chunked = spec.op.reduce(plan, spec_fields, chunk_steps=7)  # ragged slabs through the ring
    np.testing.assert_allclose(whole, chunked, rtol=2e-5, atol=1e-6)
    hh = host.heat_demand(matrix=shapes, aggregate_time=None, hour_shift=3.0).values
    hd = dev.heat_demand(matrix=shapes, aggregate_time=None, hour_shift=3.0).values
    np.testing.assert_allclose(hh, hd, rtol=2e-5, atol=1e-4)


def test_pinned_and_pageable_host_paths_agree(ds_full, shapes):
    """Pageable NumPy inputs are staged through the library's pinned ring (kept across
    calls, multi-threaded copy); pin_host() inputs are DMA'd directly: same numbers."""
    page = ab.Cutout(data=ds_full)
    pinned = page.pin_host()
    for name, kw in (("pv", dict(panel="CSi", orientation="latitude_optimal")), ("wind", dict(turbine="Vestas_V112_3MW")),
                     ("heat_demand", {})):
        a = getattr(page, name)(matrix=shapes, aggregate_time=None, **kw).values
        b = getattr(pinned, name)(matrix=shapes, aggregate_time=None, **kw).values
        c = getattr(page, name)(matrix=shapes, aggregate_time=None, **kw).values  # staging buffers reused
        np.testing.assert_allclose(a, b, rtol=2e-5, atol=1e-4)
        np.testing.assert_allclose(a, c, rtol=2e-5, atol=1e-4)
    ab.release_host_staging()
    d = page.pv("CSi", "latitude_optimal", matrix=shapes, aggregate_time=None).values  # pool refills
    assert d.shape == (23, 72)


def test_time_slab_offsets(ds_full, shapes):
    """A slab [t0, t0+nt) of the operator's time axis equals the same rows of the whole."""
    from atlite_b200.convert import _PvSpec

    dev = ab.Cutout(data=ds_full).to_device()
    spec = _PvSpec(dev.data, ab.get_solarpanelconfig("CSi"), ab.get_orientation("latitude_optimal"))
    assert spec.pitch == 72  # to_device() pads 70-wide rows to the next multiple of 4
    plan = engine.get_plan(shapes, 45, 70, pitch=spec.pitch)
    whole = spec.op.reduce(plan, spec.fields).cpu().numpy()
    part = spec.op.reduce(plan, {k: v[30:61] for k, v in spec.fields.items()}, t0=30, nt=31).cpu().numpy()
    np.testing.assert_allclose(part, whole[30:61], rtol=2e-5, atol=1e-6)


def test_padded_rows_equal_unpadded_and_padding_is_never_read_into_results(ds_full, shapes):
    """Device layout with a row pitch (to_device pads 70 -> 72 so the 128-bit lane
    layout applies) against the unpadded layout (scalar lane layout): same values
    for bus reductions, per-cell cubes and time sums, for every operator family;
    NaN written into the padding columns must not reach any result."""
    import torch

    host = ab.Cutout(data=ds_full)
    flat, padded = host.to_device(pad=False), host.to_device()
    assert flat.data.raw("temperature").shape[-1] == 70 and padded.data.raw("temperature").shape[-1] == 72
    for n in padded.data.data_vars:
        padded.data.raw(n)[..., 70:] = float("nan")
    calls = [
        ("pv", dict(panel="CSi", orientation="latitude_optimal")),
        ("pv", dict(panel="CdTe", orientation={"slope": 30.0, "azimuth": 180.0}, tracking="vertical")),
        ("wind", dict(turbine="Vestas_V112_3MW")),
        ("heat_demand", dict(hour_shift=2.0)),
        ("temperature", {}),
        ("irradiation", dict(orientation="latitude_optimal")),
        ("csp", dict(installation="SAM_solar_tower")),
    ]
    for name, kw in calls:
        for extra in (dict(matrix=shapes, aggregate_time=None), dict(aggregate_time=None), dict(aggregate_time="sum")):
            a = np.asarray(getattr(flat, name)(**kw, **extra).values)
            b = np.asarray(getattr(padded, name)(**kw, **extra).values)
            assert a.shape == b.shape and not np.isnan(b).any(), (name, extra)
            np.testing.assert_allclose(a, b, rtol=2e-5, atol=1e-5 * max(1.0, np.abs(a).max()), err_msg=name)
    # the tiling really differs: vec plan for the padded layout, scalar for the flat one
    assert engine.get_plan(shapes, 45, 70, pitch=72).info["vec"] == 1
    assert engine.get_plan(shapes, 45, 70).info["vec"] == 0
    torch.cuda.synchronize()


def test_field_shape_and_dtype_are_checked_before_the_raw_pointer_call(ds_full, shapes):
    import torch
    from atlite_b200.convert import _WindSpec

    dev = ab.Cutout(data=ds_full).to_device()
    spec = _WindSpec(dev.data, ab.get_windturbineconfig("Vestas_V112_3MW"))
    plan = engine.get_plan(shapes, 45, 70, pitch=spec.pitch)
    with pytest.raises(ValueError, match="expected"):
        spec.op.reduce(plan, spec.wnd[:, :, :70], spec.aux[:, :, :70] if spec.aux is not None else None)
    with pytest.raises(TypeError, match="float32"):
        spec.op.reduce(plan, spec.wnd.double(), spec.aux.double() if spec.aux is not None else None)
    with pytest.raises(RuntimeError):  # plan built for another pitch
        spec.op.reduce(engine.get_plan(shapes, 45, 70), spec.wnd, spec.aux)
    # generic SpMM: the dense field must have the plan's layout
    flat_plan = engine.get_plan(shapes, 45, 70)
    with pytest.raises(ValueError, match="expects"):
        flat_plan.spmm(torch.zeros(3, 45, 72, device="cuda"))
    with pytest.raises(ValueError, match="expects"):
        plan.spmm(torch.zeros(3, 45 * 70, device="cuda"))
    ones = plan.spmm(torch.ones(2, 45, 72, device="cuda")).cpu().numpy()
    np.testing.assert_allclose(ones, np.tile(cap_of(shapes), (2, 1)), rtol=1e-6)


# ------------------------------------------------------------------ size-independent properties


def test_properties_at_scale():
    """Bigger than the oracle is comfortable with: check structure instead.
    (a) linearity in the weights; (b) a partition of the grid sums to the
    all-cells bus; (c) per-cell cube reduced on the host == fused result."""
    nx, ny, nt = 256, 160, 240
    ds = syn.make_dataset(nx, ny, nt, kinds=("pv",))
    c = ab.Cutout(data=ds).to_device()
    m = syn.make_shapes(nx, ny, 150)
    kw = dict(panel="CSi", orientation="latitude_optimal", aggregate_time=None)
    r1 = bt(c.pv(matrix=m, **kw))
    r3 = bt(c.pv(matrix=m * 3.0, **kw))
    np.testing.assert_allclose(r3, 3.0 * r1, rtol=1e-5, atol=1e-5)
    allc = bt(c.pv(matrix=sp.csr_matrix(np.ones((1, nx * ny))), **kw))[:, 0]
    np.testing.assert_allclose(r1.sum(1), allc, rtol=5e-5, atol=1e-3)  # border weights sum to 1 per cell
    cube = c.pv("CSi", "latitude_optimal", aggregate_time=None).values.reshape(nt, -1).astype(np.float64)
    np.testing.assert_allclose(r1, (m @ cube.T).T, rtol=5e-5, atol=1e-4)
    assert (cube >= 0).all() and not np.isnan(cube).any() and cube.max() < 1.2


# ------------------------------------------------------------------ NaN / Inf inputs, per-cell orientation


def test_pv_nan_inputs_match_the_reference_golden_vectors():
    """A NaN (and an Inf) planted in every PV input in turn: the per-cell results must equal
    what the reference's own source produced (tests/golden/reference_nan.npz: NaN-preserving
    clip, per-term fillna(0) for the simple trigon model, mask, panel models), and the fused
    reduce must poison exactly the buses that contain a NaN cell."""
    import os

    G = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_nan.npz"), allow_pickle=False)
    time = pd.DatetimeIndex(G["time_ns"].astype("datetime64[ns]"))
    x, y = G["x"], G["y"]
    names = ("influx_toa", "influx_direct", "influx_diffuse", "albedo", "temperature")
    m = syn.make_shapes(len(x), len(y), 4)
    for case in [str(c) for c in G["cases"]]:
        name, trigon = case.split("|")
        f = {n: np.array(G[f"base|{n}"]) for n in names}
        f[name] = np.array(G[f"in|{name}"])
        for dev in (False, True):
            c = ab.Cutout(data=ab.Dataset(f, coords=dict(time=time, x=x, y=y, lon=x, lat=y)))
            c = c.to_device() if dev else c
            for key, panel in (("pv", "CSi"), ("pvbof", "KANENA")):
                got = np.asarray(c.pv(panel, "latitude_optimal", trigon_model=trigon, aggregate_time=None).values)
                assert_parity(got, G[f"{key}|{case}"], what=f"pv-nan cells {key} {case}")
            for kind in ("total", "ground"):
                got = np.asarray(c.irradiation("latitude_optimal", irradiation=kind, trigon_model=trigon,
                                               aggregate_time=None).values)
                assert_parity(got, G[f"irr_{kind}|{case}"], 1000.0, what=f"irradiation-nan {kind} {case}")
            want = (m @ G[f"pv|{case}"].reshape(len(time), -1).T).T  # scipy: NaN only where a stored entry meets it
            got = bt(c.pv("CSi", "latitude_optimal", trigon_model=trigon, matrix=m, aggregate_time=None))
            assert_parity(got, want, cap_of(m), what=f"pv-nan reduce {case}")
    # Reindl branch (total influx)
    for name in ("influx", "humidity", "influx_toa"):
        f = {"influx_toa": np.array(G["base|influx_toa"]), "influx": np.array(G["in_influx_total"]),
             "albedo": np.array(G["base|albedo"]), "temperature": np.array(G["base|temperature"]),
             "humidity": np.array(G["in_humidity"])}
        f[name] = np.array(G[f"in_reindl|{name}"])
        c = ab.Cutout(data=ab.Dataset(f, coords=dict(time=time, x=x, y=y, lon=x, lat=y))).to_device()
        got = np.asarray(c.pv("CSi", "latitude_optimal", aggregate_time=None).values)
        assert_parity(got, G[f"pv_reindl|{name}"], what=f"pv-nan reindl {name}")


def test_per_cell_mean_skips_nan_steps_like_the_reference():
    """aggregate_time='mean' without a matrix is da.mean('time') (convert.py:51-56): NaN steps
    are skipped per cell, an all-NaN cell gives NaN; 'sum' gives 0 there."""
    ds = syn.make_dataset(37, 9, 30, kinds=("wind",))
    w = ds.raw("wnd100m")
    w[3:9, 2, 5] = np.nan
    w[:, 4, 7] = np.nan
    want = O.convert_wind(oracle_ds(ds), ab.get_windturbineconfig("Vestas_V112_3MW"))
    for c in (ab.Cutout(data=ds), ab.Cutout(data=ds).to_device()):
        mean = np.asarray(c.wind("Vestas_V112_3MW", aggregate_time="mean").values)
        tot = np.asarray(c.wind("Vestas_V112_3MW", aggregate_time="sum").values)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            assert_parity(mean, np.nanmean(want, axis=0), what="wind nanmean")
        assert_parity(tot, np.nansum(want, axis=0), 30.0, what="wind nansum")
        assert np.isnan(mean[4, 7]) and tot[4, 7] == 0.0 and not np.isnan(mean[2, 5])
    # heat demand: a day whose temperatures are all NaN is skipped by the mean over days
    dt = syn.make_dataset(20, 6, 96, kinds=("temperature",))
    dt.raw("temperature")[24:48, 1, 2] = np.nan
    hw, _ = O.convert_heat_demand(oracle_ds(dt), 15.0, 1.0, 0.0, 0.0)
    got = np.asarray(ab.Cutout(data=dt).heat_demand(aggregate_time="mean").values)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        assert_parity(got, np.nanmean(hw, axis=0), 50.0, what="heat nanmean", unit=300.0)


def test_orientation_callback_returning_yx_arrays(ds_full, shapes):
    """pv/orientation.py:107 accepts any f(lon, lat, solar_position); one that returns
    (y, x)-dependent slope / azimuth runs through the per-cell orientation table."""
    ny, nx = 45, 70
    rng = np.random.default_rng(5)
    slope2d = np.radians(rng.uniform(5.0, 50.0, (ny, nx)))
    az2d = np.radians(rng.uniform(90.0, 270.0, (ny, nx)))

    def orient_gpu(lon, lat, solar_position):
        return dict(slope=ab.DataArray(slope2d, {"y": lat.coords["y"], "x": lon.coords["x"]}, ("y", "x")),
                    azimuth=ab.DataArray(az2d, {"y": lat.coords["y"], "x": lon.coords["x"]}, ("y", "x")))

    def orient_oracle(lon, lat, solar_position):
        return dict(slope=slope2d, azimuth=az2d)

    od = oracle_ds(ds_full)
    for kw in (dict(), dict(trigon_model="other"), dict(tracking="tilted_horizontal"), dict(tracking="vertical")):
        for c in (ab.Cutout(data=ds_full), ab.Cutout(data=ds_full).to_device()):
            res = c.pv("CSi", orient_gpu, matrix=shapes, aggregate_time=None, **kw)
            want = O.convert_and_aggregate(od, O.convert_pv, matrix=shapes, aggregate_time=None,
                                           panel=ab.get_solarpanelconfig("CSi"), orientation=orient_oracle, **kw)
            assert_parity(bt(res), want, cap_of(shapes), what=f"pv orientation2d {kw}")
    # slope per cell, azimuth per latitude (mixed ranks broadcast)
    def orient_mixed(lon, lat, solar_position):
        return dict(slope=ab.DataArray(slope2d, {"y": lat.coords["y"], "x": lon.coords["x"]}, ("y", "x")),
                    azimuth=np.where(np.asarray(lat.values) < 0, 0.0, np.pi))

    res = ab.Cutout(data=ds_full).to_device().pv("CSi", orient_mixed, aggregate_time=None)
    want = O.convert_pv(od, ab.get_solarpanelconfig("CSi"),
                        lambda lon, lat, sp_: dict(slope=slope2d, azimuth=np.where(lat < 0, 0.0, np.pi)[:, None] * np.ones((1, nx))))
    assert_parity(np.asarray(res.values), want, what="pv orientation2d mixed cells")


def test_lazily_loaded_cutout_is_converted_part_by_part(shapes, monkeypatch):
    """A LazyDataset (reader callbacks; the role a dask-backed xarray dataset plays for the
    reference, cutout.py:142-154) is never materialised whole: the conversion pulls one time
    part after the other, and the result equals the in-memory one."""
    from atlite_b200 import convert as cv

    ds = syn.make_dataset(70, 45, 24 * 9, x0=-10.0, y0=-20.0, dx=0.5, dy=1.0)
    arrs = {k: np.asarray(ds.raw(k)) for k in ds.keys()}
    lz = ab.LazyDataset({k: (lambda lo, hi, a=a: a[lo:hi]) for k, a in arrs.items()}, coords=dict(ds.coords),
                        time_chunk=24)
    monkeypatch.setattr(cv, "PART_BYTES", 48 * cv._bytes_per_step(lz))  # 48-step parts
    ref, lazy = ab.Cutout(data=ds), ab.Cutout(data=lz)
    calls = (lambda c: c.pv("CSi", "latitude_optimal", matrix=shapes, aggregate_time=None),
             lambda c: c.wind("Vestas_V112_3MW", matrix=shapes, aggregate_time=None),
             lambda c: c.heat_demand(matrix=shapes, aggregate_time=None, hour_shift=3.0),
             lambda c: c.wind("Vestas_V112_3MW", aggregate_time="mean"),
             lambda c: c.pv("CSi", "latitude_optimal", matrix=shapes, aggregate_time="sum", per_unit=True))
    for call in calls:
        lz.largest_read = 0
        a, b = call(ref), call(lazy)
        av, bv = np.asarray(a.values), np.asarray(b.values)
        if a.dims != b.dims:  # lazily loaded cutouts return (time, bus) like the reference's dask branch
            bv = bv.T
        np.testing.assert_allclose(bv, av, rtol=2e-5, atol=1e-6)
        assert 0 < lz.largest_read <= 72, lz.largest_read  # parts, never the whole axis (216 steps)
    with pytest.raises(RuntimeError):
        lz.raw("wnd100m")


def test_era5_height_and_runoff_on_a_prepared_cutout():
    """datasets/era5.py:65-81: height = z / g0 (first step of a time-dependent z)."""
    from atlite_b200 import era5

    nx, ny, nt = 24, 10, 6
    rng = np.random.default_rng(3)
    z = rng.uniform(-50.0, 30000.0, (nt, ny, nx)).astype(np.float32)
    x, y = syn.make_coords(nx, ny)
    raw = ab.Dataset({"z": z, "ro": rng.exponential(2e-4, (nt, ny, nx)).astype(np.float32)},
                     coords=dict(time=syn.make_time(nt), x=x, y=y, lon=x, lat=y))
    prepared = era5.prepare(raw, features=("runoff",))
    h = prepared.raw("height").cpu().numpy()
    np.testing.assert_allclose(h, z[0] / np.float32(9.80665), rtol=1e-6)
    m = syn.make_shapes(nx, ny, 3)
    got = bt(ab.Cutout(data=prepared).runoff(matrix=m, aggregate_time=None))
    want = (m @ (np.maximum(raw.raw("ro"), 0) * (z[0] / 9.80665)[None]).reshape(nt, -1).astype(np.float64).T).T
    np.testing.assert_allclose(got, want, rtol=2e-5)
    with pytest.raises(KeyError, match="height"):
        ab.Cutout(data=era5.prepare(ab.Dataset({"ro": raw.raw("ro")}, coords=raw.coords), features=("runoff",))).runoff(matrix=m)


# ------------------------------------------------------------------ BASELINE.json configs


def test_config0_wind_50x50x24_one_shape_full_parity():
    """BASELINE configs[0]: 50x50x24 cutout, convert_wind with 1 shape (the reference's
    own CPU-runnable plumbing case) -- full parity against the oracle."""
    ds = syn.make_dataset(50, 50, 24, kinds=("wind",))
    m = syn.make_shapes(50, 50, 1)
    res = ab.Cutout(data=ds).wind("Vestas_V112_3MW", matrix=m, aggregate_time=None)
    want = O.convert_and_aggregate(oracle_ds(ds), O.convert_wind, matrix=m, aggregate_time=None,
                                   turbine=ab.get_windturbineconfig("Vestas_V112_3MW"))
    assert_parity(bt(res), want, cap_of(m), what="config 0")


def _device_cutout(nx, ny, nt, x0, y0, t_skip=0, dx=0.25, dy=0.25):
    import torch

    dev = torch.device("cuda", 0)
    x, y = syn.make_coords(nx, ny, x0, y0, dx, dy)
    tm = syn.make_time(nt + t_skip)[t_skip:]
    f = syn.make_pv_fields_device(tm, x, y, dev, seed=3)
    f["wnd100m"] = (f["temperature"] - 255.0) * 0.5
    f["roughness"] = f["albedo"] * 0.5 + 1e-3
    ds = ab.Dataset(f, coords=dict(time=tm, x=x, y=y, lon=x, lat=y))
    return ab.Cutout(data=ds), f


def _bus_windows(m, nx, buses):
    """For each bus: its index, the bounding (y, x) window of its cells and the dense
    weight window -- the oracle then only has to evaluate that window."""
    m = sp.csr_matrix(m)
    for b in buses:
        cols = m.indices[m.indptr[b]:m.indptr[b + 1]]
        w = m.data[m.indptr[b]:m.indptr[b + 1]]
        iy, ix = cols // nx, cols % nx
        ys, xs = slice(int(iy.min()), int(iy.max()) + 1), slice(int(ix.min()), int(ix.max()) + 1)
        W = np.zeros((ys.stop - ys.start, xs.stop - xs.start))
        np.add.at(W, (iy - ys.start, ix - xs.start), w)
        yield int(b), ys, xs, W


def _window_ds(c, f, names, ts, ys, xs):
    od = {k: f[k][ts, ys, xs].cpu().numpy() for k in names}
    od.update(time=c.data.coords["time"][ts], lon=c.data.coords["x"][xs], lat=c.data.coords["y"][ys])
    return od


PV_NAMES = ("influx_toa", "influx_direct", "influx_diffuse", "albedo", "temperature")


def test_config1_pv_200x200x8760_full_size_properties():
    """BASELINE configs[1] at FULL size (3.5e8 cell-timesteps): size-independent
    properties plus the oracle on 48 time steps spread over the year."""
    import torch

    nx, ny, nt, nbus = 200, 200, 8760, 100
    c, f = _device_cutout(nx, ny, nt, 0.0, 30.0)
    m = syn.make_shapes(nx, ny, nbus)
    kw = dict(panel="CSi", orientation="latitude_optimal", aggregate_time=None)
    r = bt(c.pv(matrix=m, **kw))
    assert r.shape == (nt, nbus) and not np.isnan(r).any() and (r >= 0).all()
    # (a) border weights sum to 1 per cell -> buses partition the all-cells bus
    allc = bt(c.pv(matrix=sp.csr_matrix(np.ones((1, nx * ny))), **kw))[:, 0]
    np.testing.assert_allclose(r.sum(1), allc, rtol=1e-4, atol=1e-2)
    # (b) linearity in the weights
    np.testing.assert_allclose(bt(c.pv(matrix=m * 0.25, **kw)), 0.25 * r, rtol=1e-5, atol=1e-6)
    # (c) any time slab equals the same rows of the whole (slab offsets into the almanac)
    sub = ab.Cutout(data=ab.Dataset({k: v[4000:4500] for k, v in f.items()},
                                    coords=dict(time=c.data.coords["time"][4000:4500], x=c.data.coords["x"],
                                                y=c.data.coords["y"], lon=c.data.coords["x"], lat=c.data.coords["y"])))
    np.testing.assert_allclose(bt(sub.pv(matrix=m, **kw)), r[4000:4500], rtol=2e-5, atol=1e-6)
    # (d) fused == per-cell cube reduced on the host
    cube = sub.pv("CSi", "latitude_optimal", aggregate_time=None).values.reshape(500, -1).astype(np.float64)
    np.testing.assert_allclose(r[4000:4500], (m @ cube.T).T, rtol=5e-5, atol=1e-4)
    # (e) the oracle on 48 steps spread over the year (every 182nd hour + a phase, so all hours of
    # the day and all seasons occur)
    tsel = (np.arange(48) * 182 + 7) % nt
    idx = torch.as_tensor(tsel, device=f["albedo"].device)
    od = {k: f[k][idx].cpu().numpy() for k in PV_NAMES}
    od.update(time=c.data.coords["time"][tsel], lon=c.data.coords["x"], lat=c.data.coords["y"])
    want = O.convert_and_aggregate(od, O.convert_pv, matrix=m, aggregate_time=None,
                                   panel=ab.get_solarpanelconfig("CSi"), orientation=O.get_orientation("latitude_optimal"))
    assert (want > 0).any(axis=1).sum() >= 12, "the sample must contain daytime steps"
    assert_parity(r[tsel], want, cap_of(m), what="pv config1 48-step sample vs oracle")
    # night rows are exactly zero somewhere in the year
    assert (r == 0).any() and r.max() > 0


def test_north_star_1440x720_3000_shapes_vs_oracle_windows():
    """The graded configuration (BASELINE north star / configs[2] / configs[3]): 1440 x 720
    -> 3000 shapes, PV, wind and heat demand, 48 steps.  The oracle cannot run on 1e6 cells
    in test time, but both the per-cell physics and a bus sum only depend on the cells
    involved: (a) three cell windows x 48 steps of the per-cell results, (b) five whole
    buses x 48 steps (3 days for heat) of the fused results, against the oracle evaluated
    on exactly those cells."""
    nx, ny, nt, nbus = 1440, 720, 48, 3000
    c, f = _device_cutout(nx, ny, nt, -180.0, -90.0, t_skip=24 * 171)
    m = syn.make_shapes(nx, ny, nbus)
    panel, orient = ab.get_solarpanelconfig("CSi"), O.get_orientation("latitude_optimal")
    turb = ab.get_windturbineconfig("Vestas_V112_3MW")
    ts = slice(0, nt)
    # ---- (a) per-cell cubes on windows: tropics, mid latitudes (both hemispheres), near the pole / date line
    pv_cube = np.asarray(c.pv("CSi", "latitude_optimal", aggregate_time=None).values)
    w_cube = np.asarray(c.wind("Vestas_V112_3MW", aggregate_time=None).values)
    h_cube = np.asarray(c.heat_demand(aggregate_time=None).values)
    assert pv_cube.shape == w_cube.shape == (nt, ny, nx) and h_cube.shape == (2, ny, nx)
    for ys, xs in ((slice(352, 360), slice(700, 716)), (slice(560, 566), slice(40, 64)),
                   (slice(100, 108), slice(1424, 1440)), (slice(712, 720), slice(0, 12))):
        od = _window_ds(c, f, PV_NAMES + ("wnd100m", "roughness"), ts, ys, xs)
        assert_parity(pv_cube[:, ys, xs], O.convert_pv(od, panel, orient), what="pv north-star window")
        assert_parity(w_cube[:, ys, xs], O.convert_wind(od, turb), what="wind north-star window")
        assert_parity(h_cube[:, ys, xs], O.convert_heat_demand(od, 15.0, 1.0, 0.0, 0.0)[0], 50.0,
                      what="heat north-star window", unit=300.0)
    assert (pv_cube > 0).any() and (pv_cube == 0).any()
    del pv_cube, w_cube, h_cube
    # ---- (b) whole buses of the fused (physics + shape reduce) results
    pv = bt(c.pv("CSi", "latitude_optimal", matrix=m, aggregate_time=None))
    w = bt(c.wind("Vestas_V112_3MW", matrix=m, aggregate_time=None))
    h = bt(c.heat_demand(matrix=m, aggregate_time=None))
    assert pv.shape == w.shape == (nt, nbus) and h.shape == (2, nbus)
    cap = cap_of(m)
    sizes = np.diff(sp.csr_matrix(m).indptr)
    buses = [int(np.argmax(sizes)), int(np.argmin(sizes)), 0, 1234, nbus - 1]
    for b, ys, xs, W in _bus_windows(m, nx, buses):
        od = _window_ds(c, f, PV_NAMES + ("wnd100m", "roughness"), ts, ys, xs)
        assert_parity(pv[:, b], (O.convert_pv(od, panel, orient) * W).sum((1, 2)), cap[b], what="pv north-star bus")
        assert_parity(w[:, b], (O.convert_wind(od, turb) * W).sum((1, 2)), cap[b], what="wind north-star bus")
        assert_parity(h[:, b], (O.convert_heat_demand(od, 15.0, 1.0, 0.0, 0.0)[0] * W).sum((1, 2)), cap[b] * 50.0,
                      what="heat north-star bus")
    # partition of unity across all 3000 buses (every cell's weights sum to 1)
    ones = sp.csr_matrix(np.ones((1, nx * ny)))
    np.testing.assert_allclose(pv.sum(1), bt(c.pv("CSi", "latitude_optimal", matrix=ones, aggregate_time=None))[:, 0],
                               rtol=1e-4, atol=1e-2)


def test_config2_3_wind_heat_1440x720_3000_shapes_properties():
    """BASELINE configs[2,3] at full spatial size (1440x720 -> 3000 shapes), 240 steps."""
    nx, ny, nt, nbus = 1440, 720, 240, 3000
    c, f = _device_cutout(nx, ny, nt, -180.0, -90.0, t_skip=24 * 100)
    m = syn.make_shapes(nx, ny, nbus)
    ones = sp.csr_matrix(np.ones((1, nx * ny)))
    w = bt(c.wind("Vestas_V112_3MW", matrix=m, aggregate_time=None))
    assert w.shape == (nt, nbus) and not np.isnan(w).any()
    np.testing.assert_allclose(w.sum(1), bt(c.wind("Vestas_V112_3MW", matrix=ones, aggregate_time=None))[:, 0],
                               rtol=1e-4)
    cap = cap_of(m)
    assert (w <= cap[None, :] * (1 + 1e-5)).all() and (w >= 0).all()  # capacity factor in [0, 1]
    h = bt(c.heat_demand(matrix=m, aggregate_time=None))
    assert h.shape == (10, nbus)
    np.testing.assert_allclose(h.sum(1), bt(c.heat_demand(matrix=ones, aggregate_time=None))[:, 0], rtol=1e-4)
    # oracle on one day for 5 buses' worth of cells is too slow at this size: check the
    # daily-mean identity instead: a=1, constant=0, huge threshold => thr+273.15 - mean(T)
    hh = bt(c.heat_demand(threshold=1000.0, matrix=ones, aggregate_time=None))[:, 0]
    tmean = f["temperature"].reshape(10, 24, -1).double().mean(1).sum(1).cpu().numpy()
    np.testing.assert_allclose(hh, (1273.15 * nx * ny - tmean), rtol=1e-5)


def test_config4_percell_capacity_factors_1000x800_properties():
    """BASELINE configs[4]: Europe-scale 1000 x 800 grid, pv + wind capacity factors per
    cell with per-cell layout weights, no shapes reduction (the no-matrix branch,
    convert.py:200-211, twice).  96 steps; checked through (a) the oracle on a window
    of cells (per-cell physics is independent of the neighbours), (b) mean == mean of
    the per-cell cube, (c) layout-weighted sum == the layout= (one bus) matrix path."""
    nx, ny, nt = 1000, 800, 96
    c, f = _device_cutout(nx, ny, nt, -12.0, 33.0, t_skip=24 * 150, dx=0.05, dy=0.05)
    cf_pv = c.pv("CSi", "latitude_optimal", aggregate_time="mean")
    cf_w = c.wind("Vestas_V112_3MW", aggregate_time="mean")
    assert cf_pv.dims == ("y", "x") and cf_pv.shape == cf_w.shape == (ny, nx)
    pv, w = np.asarray(cf_pv.values), np.asarray(cf_w.values)
    assert not np.isnan(pv).any() and (pv >= 0).all() and (pv < 1.2).all() and (w >= 0).all() and (w <= 1 + 1e-6).all()
    # (a) oracle on a window
    ys, xs = slice(397, 403), slice(500, 512)
    od = {k: v[:, ys, xs].cpu().numpy() for k, v in f.items()}
    od.update(time=c.data.coords["time"], lon=c.data.coords["x"][xs], lat=c.data.coords["y"][ys])
    want_pv = O.convert_pv(od, ab.get_solarpanelconfig("CSi"), O.get_orientation("latitude_optimal")).mean(0)
    want_w = O.convert_wind(od, ab.get_windturbineconfig("Vestas_V112_3MW")).mean(0)
    assert_parity(pv[ys, xs], want_pv, what="config4 pv window")
    assert_parity(w[ys, xs], want_w, what="config4 wind window")
    # (b) the same through the per-cell cube of the first day
    day = ab.Cutout(data=ab.Dataset({k: v[:24] for k, v in f.items()},
                                    coords=dict(time=c.data.coords["time"][:24], x=c.data.coords["x"], y=c.data.coords["y"],
                                                lon=c.data.coords["x"], lat=c.data.coords["y"])))
    cube = np.asarray(day.wind("Vestas_V112_3MW", aggregate_time=None).values)
    assert cube.shape == (24, ny, nx)
    np.testing.assert_allclose(cube.mean(0, dtype=np.float64), day.wind("Vestas_V112_3MW", aggregate_time="mean").values,
                               rtol=2e-5, atol=1e-6)
    # (c) per-cell layout weights: sum(layout * cf) == the one-bus layout= path
    lay = syn.make_layout(nx, ny)
    layout = ab.DataArray(lay, {"y": c.data.coords["y"], "x": c.data.coords["x"]}, ("y", "x"))
    bus = c.pv("CSi", "latitude_optimal", layout=layout, aggregate_time="mean")
    np.testing.assert_allclose(float(np.asarray(bus.values).ravel()[0]), float((lay * pv.astype(np.float64)).sum()), rtol=2e-5)
    combined = float((lay * (pv.astype(np.float64) + w)).sum())
    busw = c.wind("Vestas_V112_3MW", layout=layout, aggregate_time="mean")
    np.testing.assert_allclose(combined, float(np.asarray(bus.values).ravel()[0] + np.asarray(busw.values).ravel()[0]), rtol=2e-5)


def test_fused_kernel_meets_the_parity_bar(ds_full, shapes):
    """The fused reduce kernel meets the bar for PV (default and general path) and wind, device-
    and host-resident, including NaN routing and the tail of a time block that is not a multiple
    of the batch."""
    od = oracle_ds(ds_full)
    for c in (ab.Cutout(data=ds_full).to_device(), ab.Cutout(data=ds_full)):
        res = c.pv("CSi", "latitude_optimal", matrix=shapes, aggregate_time=None)
        assert_parity(bt(res), _oracle_pv(ds_full, shapes, dict(panel="CSi", orientation="latitude_optimal")),
                      cap_of(shapes), what="fused pv")
        res = c.pv("CSi", {"slope": 30.0, "azimuth": 170.0}, tracking="tilted_horizontal", trigon_model="other",
                   matrix=shapes, aggregate_time=None)
        want = _oracle_pv(ds_full, shapes, dict(panel="CSi", orientation={"slope": 30.0, "azimuth": 170.0},
                                                tracking="tilted_horizontal", trigon_model="other"))
        assert_parity(bt(res), want, cap_of(shapes), what="fused pv-general")
        res = c.wind("Vestas_V112_3MW", matrix=shapes, aggregate_time=None)
        want = O.convert_and_aggregate(od, O.convert_wind, matrix=shapes, aggregate_time=None,
                                       turbine=ab.get_windturbineconfig("Vestas_V112_3MW"))
        assert_parity(bt(res), want, cap_of(shapes), what="fused wind")
    # NaN routing + a time axis (13 steps) that is no multiple of any batch length
    ds = syn.make_dataset(70, 45, 13, x0=-10.0, y0=-20.0, dx=0.5, dy=1.0)
    ds.raw("wnd100m")[5, 20, 33] = np.nan
    ds.raw("albedo")[7, 11, 40] = np.nan
    od2 = oracle_ds(ds)
    c = ab.Cutout(data=ds).to_device()
    want = O.convert_and_aggregate(od2, O.convert_wind, matrix=shapes, aggregate_time=None,
                                   turbine=ab.get_windturbineconfig("Vestas_V112_3MW"))
    assert np.isnan(want).sum() == 1
    assert_parity(bt(c.wind("Vestas_V112_3MW", matrix=shapes, aggregate_time=None)), want, cap_of(shapes),
                  what="fused wind-nan")
    want = _oracle_pv(ds, shapes, dict(panel="CSi", orientation="latitude_optimal"))
    assert not np.isnan(want).any()  # simple trigon model: a NaN albedo only zeroes the ground term
    assert_parity(bt(c.pv("CSi", "latitude_optimal", matrix=shapes, aggregate_time=None)), want, cap_of(shapes),
                  what="fused pv-nan")


def test_deterministic_mode_is_bitwise_repeatable(ds_full, shapes):
    """atl_set_deterministic: fixed summation order -> identical bits run to run, same parity."""
    c = ab.Cutout(data=ds_full).to_device()
    od = oracle_ds(ds_full)
    prev = ab.set_deterministic(True)
    try:
        runs = [c.pv("CSi", "latitude_optimal", matrix=shapes, aggregate_time=None).values for _ in range(3)]
        assert all(np.array_equal(runs[0], r) for r in runs[1:])
        want = _oracle_pv(ds_full, shapes, dict(panel="CSi", orientation="latitude_optimal"))
        assert_parity(runs[0].T, want, cap_of(shapes), what="deterministic pv")
        w1 = c.wind("Vestas_V112_3MW", matrix=shapes, aggregate_time=None).values
        w2 = c.wind("Vestas_V112_3MW", matrix=shapes, aggregate_time=None).values
        assert np.array_equal(w1, w2)
        h1 = c.heat_demand(matrix=shapes, aggregate_time=None).values
        h2 = c.heat_demand(matrix=shapes, aggregate_time=None).values
        assert np.array_equal(h1, h2)
        want = O.convert_and_aggregate(od, O.convert_heat_demand, matrix=shapes, aggregate_time=None,
                                       threshold=15.0, a=1.0, constant=0.0, hour_shift=0.0)
        assert_parity(h1.T, want, cap_of(shapes) * 50.0, what="deterministic heat")
        s1 = c.pv("CSi", "latitude_optimal", aggregate_time="sum").values
        s2 = c.pv("CSi", "latitude_optimal", aggregate_time="sum").values
        assert np.array_equal(s1, s2)
        # empty plan and host-streamed path
        e = c.wind("Vestas_V112_3MW", matrix=sp.csr_matrix((2, 70 * 45)), aggregate_time=None).values
        assert (e == 0).all()
        # the summation order is fixed per lane layout: host streaming uses the unpadded
        # (scalar-lane) layout, so it is bit-identical to an unpadded device cutout and
        # equal within rounding to the padded (128-bit lane) one
        hs = ab.Cutout(data=ds_full).pv("CSi", "latitude_optimal", matrix=shapes, aggregate_time=None).values
        flat = ab.Cutout(data=ds_full).to_device(pad=False)
        assert np.array_equal(hs, flat.pv("CSi", "latitude_optimal", matrix=shapes, aggregate_time=None).values)
        np.testing.assert_allclose(hs, runs[0], rtol=2e-5, atol=1e-6)
    finally:
        ab.set_deterministic(prev)
    nd = c.pv("CSi", "latitude_optimal", matrix=shapes, aggregate_time=None).values
    np.testing.assert_allclose(nd, runs[0], rtol=2e-5, atol=1e-6)


def test_empty_time_axis_returns_empty_results(shapes):
    """A rank whose time shard is empty (e.g. 7 day blocks on 8 GPUs) must not fail."""
    ds = syn.make_dataset(70, 45, 0, x0=-10.0, y0=-20.0, dx=0.5, dy=1.0, t_offset=72)
    for c in (ab.Cutout(data=ds), ab.Cutout(data=ds).to_device()):
        assert c.pv("CSi", "latitude_optimal", matrix=shapes, aggregate_time=None).shape == (23, 0)
        assert c.wind("Vestas_V112_3MW", matrix=shapes, aggregate_time=None).shape == (23, 0)
        assert c.heat_demand(matrix=shapes, aggregate_time=None).shape == (23, 0)
        assert c.temperature(matrix=shapes, aggregate_time=None).shape == (23, 0)
        assert c.csp("SAM_solar_tower", matrix=shapes, aggregate_time=None).shape == (23, 0)
        assert (c.wind("Vestas_V112_3MW", aggregate_time="sum").values == 0).all()
