"""Cutouts that carry raw ERA5 variables (CDS short names: ssrd, ssr, tisr, fdir, t2m, u100, v100,
u10, v10, fsr, stl4, d2m) are converted directly: the PV and wind kernels derive influx, albedo,
wind speed, roughness and shear exponent in registers with the arithmetic of csrc/era5.cu, and
the temperature family reads t2m / stl4 / d2m in place of the names era5.prepare gives them.

GPU tests hold every route to the parity bar against the float64 oracle fed with the oracle's
ERA5 derivations and the solar position at -30 min (what era5.prepare stores); CPU tests check
which fields and which kernel branch each converter picks."""

import warnings

import numpy as np
import pytest
import scipy.sparse as sp

import atlite_oracle as O
import era5_oracle as EO
import atlite_b200 as ab
from atlite_b200 import _lib, convert, engine, synthetic as syn
from conftest import assert_parity

RAW_PV = ("ssrd", "ssr", "tisr", "fdir")
PREPARED_PV = ("influx_toa", "influx_direct", "influx_diffuse", "albedo")


def _raw_arrays(nx, ny, nt, seed=0):
    """Seeded raw ERA5 fields with the edge cells of tests/test_era5.py's raw dataset, plus
    negative accumulations (ERA5's post-processing leaves small negative values)."""
    rng = np.random.default_rng(seed)
    shp = (nt, ny, nx)
    f = lambda lo, hi: rng.uniform(lo, hi, shp).astype(np.float32)  # noqa: E731
    d = dict(u100=f(-15, 15), v100=f(-15, 15), u10=f(-8, 8), v10=f(-8, 8), fsr=f(-0.05, 2.0),
             ssrd=f(0, 3.0e6), tisr=f(0, 4.5e6), t2m=f(250, 305), stl4=f(270, 290), d2m=f(250, 295))
    d["ssr"] = (d["ssrd"] * rng.uniform(0.6, 1.0, shp)).astype(np.float32)
    d["fdir"] = (d["ssrd"] * rng.uniform(0.0, 1.1, shp)).astype(np.float32)  # sometimes > ssrd: negative diffuse
    d["ssrd"][:, 0, :5] = 0.0        # albedo must be 0, not NaN
    d["ssr"][:, 1, 2] = np.nan       # NaN albedo -> 0
    d["fsr"][:, 2, 2] = np.nan       # NaN roughness -> 2e-4
    d["fsr"][:, 3, 1] = -0.3         # negative roughness -> 2e-4
    d["ssrd"][:, 2, 4] = -40.0       # negative accumulations
    d["fdir"][:, 3, 3] = -25.0
    d["tisr"][:, 1, 6] = -3.6
    d["stl4"][:, 0, 0] = np.nan      # sea: soil temperature NaN -> 0
    return d


def _coords(nx, ny, nt, x0=-10.0, y0=35.0):
    x, y = syn.make_coords(nx, ny, x0, y0, 0.5, 0.5)
    t = syn.make_time(nt + 24 * 40)[24 * 40:]  # February: day, night and the terminator
    return dict(time=t, x=x, y=y, lon=x, lat=y)


def _dataset(d, co, names=None):
    names = list(d) if names is None else names
    return ab.Dataset({k: (("time", "y", "x"), d[k]) for k in names}, coords=dict(co))


def _oracle(d, co):
    ow = EO.get_data_wind(d["u100"], d["v100"], d["u10"], d["v10"], d["fsr"])
    oi = EO.get_data_influx(d["ssrd"], d["ssr"], d["tisr"], d["fdir"])
    c = dict(time=co["time"], lon=co["x"], lat=co["y"])
    sol = O.solar_position(c, time_shift="-30min")
    od = dict(c, solar_altitude=sol["altitude"], solar_azimuth=sol["azimuth"],
              temperature=d["t2m"].astype(np.float64), **{"soil temperature": d["stl4"].astype(np.float64),
                                                         "dewpoint temperature": d["d2m"].astype(np.float64)})
    od.update({k: ow[k] for k in ("wnd100m", "roughness", "wnd_shear_exp")})
    od.update({k: oi[k] for k in PREPARED_PV})
    return od


NX, NY, NT = 37, 14, 60  # odd width: to_device pads the rows to 40


@pytest.fixture(scope="module")
def case():
    co = _coords(NX, NY, NT)
    d = _raw_arrays(NX, NY, NT, seed=3)
    m = syn.make_shapes(NX, NY, 7)
    return dict(d=d, co=co, m=m, cap=np.asarray(sp.csr_matrix(m).sum(-1)).ravel(), od=_oracle(d, co))


def _cutout(case, residency, tmp_path=None, names=None):
    ds = _dataset(case["d"], case["co"], names)
    if residency == "host":
        return ab.Cutout(data=ds)
    if residency == "device":
        return ab.Cutout(data=ds).to_device()
    from atlite_b200 import ingest

    names = list(case["d"]) if names is None else names
    p = ingest.write_chunked(tmp_path / "raw.bin", {k: case["d"][k] for k in names}, dict(case["co"]),
                             chunk=(16, None, None))
    return ab.Cutout(data=ingest.open_cutout(p))


def _time_bus(res):
    """(time, bus) values of a reduced result, whichever dim order it has."""
    v = np.asarray(res.values)
    return v if res.dims[0] == "time" else v.T


def _no_deprecation(fn):
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        out = fn()
    assert not [x for x in w if issubclass(x.category, DeprecationWarning)], [str(x.message) for x in w]
    return out


# --------------------------------------------------------------------------------------------
# GPU: every converter, output form and residency against the oracle
# --------------------------------------------------------------------------------------------

PV_CASES = [
    ("CSi", "latitude_optimal", {}),                       # ERA5 default: the compiled raw mode
    ("CdTe", {"slope": 30.0, "azimuth": 170.0}, {}),
    ("KANENA", "latitude_optimal", {}),                    # Bofinger
    ("CSi", "latitude_optimal", dict(tracking="horizontal")),
    ("CSi", "latitude_optimal", dict(tracking="tilted_horizontal")),
    ("CSi", "latitude_optimal", dict(tracking="vertical")),
    ("CSi", "latitude_optimal", dict(tracking="dual")),
    ("CSi", "latitude_optimal", dict(trigon_model="hay_davies")),
]


@pytest.mark.gpu
@pytest.mark.parametrize("panel,orientation,kw", PV_CASES)
def test_gpu_raw_pv_matches_the_oracle(case, panel, orientation, kw):
    c = _cutout(case, "device")
    res = _no_deprecation(lambda: c.pv(panel, orientation, matrix=case["m"], aggregate_time=None, **kw))
    want = O.convert_and_aggregate(case["od"], O.convert_pv, matrix=case["m"], aggregate_time=None,
                                   panel=ab.get_solarpanelconfig(panel), orientation=O.get_orientation(orientation),
                                   **kw)
    assert want.sum() > 0
    assert_parity(_time_bus(res), want, case["cap"], what=f"raw-era5 pv {panel} {kw}")


@pytest.mark.gpu
@pytest.mark.parametrize("kind,kw", [("total", {}), ("direct", {}), ("diffuse", {}), ("ground", {}),
                                     ("total", dict(tracking="dual"))])
def test_gpu_raw_irradiation_matches_the_oracle(case, kind, kw):
    o = {"slope": 30.0, "azimuth": 170.0}
    res = _cutout(case, "device").irradiation(o, irradiation=kind, matrix=case["m"], aggregate_time=None, **kw)
    want = O.convert_and_aggregate(case["od"], O.convert_irradiation, matrix=case["m"], aggregate_time=None,
                                   orientation=O.get_orientation(o), irradiation=kind, clearsky_model=None, **kw)
    assert want.sum() > 0
    assert_parity(_time_bus(res), want, case["cap"] * 1000.0, what=f"raw-era5 irradiation {kind} {kw}")


@pytest.mark.gpu
def test_gpu_raw_solar_thermal_matches_the_oracle(case):
    res = _cutout(case, "host").solar_thermal(matrix=case["m"], aggregate_time=None)
    want = O.convert_and_aggregate(case["od"], O.convert_solar_thermal, matrix=case["m"], aggregate_time=None,
                                   orientation=O.get_orientation({"slope": 45.0, "azimuth": 180.0}),
                                   trigon_model="simple", clearsky_model="simple", c0=0.8, c1=3.0, t_store=80.0)
    assert want.sum() > 0
    assert_parity(_time_bus(res), want, case["cap"] * 1000.0, what="raw-era5 solar thermal")


def _wind_turbine(hub):
    t = ab.get_windturbineconfig("Vestas_V112_3MW")
    return dict(t, hub_height=hub)


@pytest.mark.gpu
@pytest.mark.parametrize("residency", ["device", "host", "lazy"])
@pytest.mark.parametrize("hub,method", [(80, "logarithmic"), (120, "power"), (100, "logarithmic")])
def test_gpu_raw_wind_matches_the_oracle(case, tmp_path, residency, hub, method):
    turb = _wind_turbine(hub)
    res = _cutout(case, residency, tmp_path).wind(turb, interpolation_method=method, matrix=case["m"],
                                                  aggregate_time=None)
    want = O.convert_and_aggregate(case["od"], O.convert_wind, matrix=case["m"], aggregate_time=None, turbine=turb,
                                   interpolation_method=method)
    assert not np.isnan(want).any()
    assert_parity(_time_bus(res), want, case["cap"], what=f"raw-era5 wind {hub} {method} {residency}")


@pytest.mark.gpu
@pytest.mark.parametrize("residency", ["device", "host", "lazy"])
@pytest.mark.parametrize("kw", [{}, dict(tracking="horizontal", trigon_model="hay_davies")])
def test_gpu_raw_pv_every_residency(case, tmp_path, residency, kw):
    res = _no_deprecation(lambda: _cutout(case, residency, tmp_path).pv("CSi", "latitude_optimal", matrix=case["m"],
                                                                      aggregate_time=None, **kw))
    want = O.convert_and_aggregate(case["od"], O.convert_pv, matrix=case["m"], aggregate_time=None,
                                   panel=ab.get_solarpanelconfig("CSi"),
                                   orientation=O.get_orientation("latitude_optimal"), **kw)
    assert_parity(_time_bus(res), want, case["cap"], what=f"raw-era5 pv {residency} {kw}")


@pytest.mark.gpu
@pytest.mark.parametrize("residency", ["device", "host"])
def test_gpu_raw_output_forms(case, residency):
    """Two-pass plan (one bus per cell), the per-cell cube, the time sum and mean."""
    c = _cutout(case, residency)
    od, S = case["od"], NX * NY
    eye = sp.identity(S, format="csr")
    assert engine.get_plan(eye, NY, NX).info["fused"] == 0
    turb = _wind_turbine(80)
    for name, call, fn, kw, scale in (
            ("pv", lambda **a: c.pv("CSi", "latitude_optimal", **a), O.convert_pv,
             dict(panel=ab.get_solarpanelconfig("CSi"), orientation=O.get_orientation("latitude_optimal")), 1.0),
            ("wind", lambda **a: c.wind(turb, **a), O.convert_wind, dict(turbine=turb), 1.0)):
        cube = fn(od, **kw)
        want = O.convert_and_aggregate(od, fn, matrix=eye, aggregate_time=None, **kw)
        assert_parity(_time_bus(call(matrix=eye, aggregate_time=None)), want, np.ones(S),
                      what=f"raw-era5 {name} two-pass")
        assert_parity(call(aggregate_time=None).values, cube, what=f"raw-era5 {name} cells")
        assert_parity(call(aggregate_time="sum").values, cube.sum(0), NT * scale, what=f"raw-era5 {name} sum")
        assert_parity(call(aggregate_time="mean").values, cube.mean(0), scale, what=f"raw-era5 {name} mean")


@pytest.mark.gpu
def test_gpu_raw_temperature_family(case):
    c = _cutout(case, "host")
    od, m = case["od"], case["m"]
    capk = case["cap"] * 300.0
    for meth, fn in (("temperature", O.convert_temperature), ("soil_temperature", O.convert_soil_temperature),
                     ("dewpoint_temperature", O.convert_dewpoint_temperature)):
        want = O.convert_and_aggregate(od, fn, matrix=m, aggregate_time=None)
        assert_parity(_time_bus(getattr(c, meth)(matrix=m, aggregate_time=None)), want, capk,
                      what=f"raw-era5 {meth}", additive=True)
    for args in (dict(), dict(source="soil", sink_T=45.0)):
        full = dict(dict(source="air", sink_T=55.0, c0=None, c1=None, c2=None), **args)
        want = O.convert_and_aggregate(od, O.convert_coefficient_of_performance, matrix=m, aggregate_time=None, **full)
        assert_parity(_time_bus(c.coefficient_of_performance(matrix=m, aggregate_time=None, **args)), want,
                      case["cap"] * 10.0, what=f"raw-era5 cop {args}")
    for meth, fn, kw in (("heat_demand", O.convert_heat_demand, dict(threshold=15.0, a=1.0, constant=0.0)),
                         ("cooling_demand", O.convert_cooling_demand, dict(threshold=5.0, a=1.7, constant=0.3))):
        want = O.convert_and_aggregate(od, fn, matrix=m, aggregate_time=None, hour_shift=0.0, **kw)
        assert_parity(_time_bus(getattr(c.to_device(), meth)(matrix=m, aggregate_time=None, **kw)), want,
                      case["cap"] * 50.0, what=f"raw-era5 {meth}")


@pytest.mark.gpu
def test_gpu_raw_with_stored_solar_position_reads_it(case):
    """A raw dataset that also stores the solar position: the general raw kernel reads it, as the
    getter in pv/solar_position.py:54-60 would."""
    d = dict(case["d"], solar_altitude=case["od"]["solar_altitude"], solar_azimuth=case["od"]["solar_azimuth"])
    c = ab.Cutout(data=_dataset(d, case["co"])).to_device()
    res = c.pv("CSi", "latitude_optimal", matrix=case["m"], aggregate_time=None)
    want = O.convert_and_aggregate(case["od"], O.convert_pv, matrix=case["m"], aggregate_time=None,
                                   panel=ab.get_solarpanelconfig("CSi"), orientation=O.get_orientation("latitude_optimal"))
    assert_parity(_time_bus(res), want, case["cap"], what="raw-era5 pv stored solar position")


@pytest.mark.gpu
def test_gpu_prepared_variables_take_precedence_bitwise(case):
    """A dataset with raw AND prepared variables converts exactly as the prepared-only dataset."""
    from atlite_b200 import era5

    raw = _dataset(case["d"], case["co"])
    prep = era5.prepare(raw, features=("wind", "influx", "temperature"))
    both = era5.prepare(raw, features=("wind", "influx", "temperature"))
    for k in case["d"]:
        both[k] = (("time", "y", "x"), raw.raw(k))
    m, turb = case["m"], _wind_turbine(80)
    prev = _lib.set_deterministic(True)  # a fixed summation order: bitwise comparable
    try:
        for call in (lambda c: c.pv("CSi", "latitude_optimal", matrix=m, aggregate_time=None),
                     lambda c: c.pv("CSi", "latitude_optimal", matrix=m, aggregate_time=None, tracking="dual"),
                     lambda c: c.wind(turb, matrix=m, aggregate_time=None),
                     lambda c: c.wind(turb, interpolation_method="power", matrix=m, aggregate_time=None),
                     lambda c: c.temperature(matrix=m, aggregate_time=None)):
            a = np.asarray(call(ab.Cutout(data=prep)).values)
            b = np.asarray(call(ab.Cutout(data=both)).values)
            assert np.array_equal(a, b, equal_nan=True)
    finally:
        _lib.set_deterministic(prev)


@pytest.mark.gpu
@pytest.mark.parametrize("width", [NX, 40])  # scalar and 128-bit lanes
def test_gpu_raw_derivation_is_k_era5_influx_bitwise(case, width):
    """Per-cell values from raw inputs equal, bit for bit, those from era5.get_data_influx's fields:
    the in-kernel derivation is the same arithmetic as k_era5_influx."""
    import torch

    from atlite_b200 import era5

    d = case["d"]

    def dev(a):
        return torch.from_numpy(np.ascontiguousarray(np.pad(a, ((0, 0), (0, 0), (0, width - NX))))).cuda()

    prev = _lib.set_deterministic(True)
    try:
        prep = era5.get_data_influx(_dataset(d, case["co"]), solar_position_vars=False)
        raw_f = dict(influx=dev(d["ssrd"]), outflux=dev(d["ssr"]), influx_toa=dev(d["tisr"]),
                     influx_direct=dev(d["fdir"]), temperature=dev(d["t2m"]))
        prep_f = {k: dev(prep.raw(k).cpu().numpy()) for k in PREPARED_PV}
        prep_f["temperature"] = raw_f["temperature"]
        op_raw = _pitched(case, _lib.IRR_ERA5_RAW, width)
        a = torch.nan_to_num(op_raw.cells(raw_f), 7.0)
        b = torch.nan_to_num(_pitched(case, _lib.IRR_DIRECT_DIFFUSE, width).cells(prep_f), 7.0)
        assert a.abs().sum() > 0
        assert torch.equal(a, b)
        assert torch.equal(a, torch.nan_to_num(op_raw.cells(raw_f), 7.0))
    finally:
        _lib.set_deterministic(prev)


def _pitched(case, irr_branch, pitch):
    co = case["co"]
    return engine.PvOp(ny=NY, nx=NX, time=co["time"], lon=co["x"], lat=co["y"],
                       slope=np.full(NY, np.radians(30.0)), azimuth=np.full(NY, np.radians(180.0)), tracking=None,
                       trigon_model=_lib.TRIGON_SIMPLE, clearsky_model=0, irr_branch=irr_branch,
                       albedo_src=_lib.ALBEDO_VAR, solar_src=_lib.SOLAR_COMPUTED, panel=ab.get_solarpanelconfig("CSi"),
                       time_shift="-30min", pitch=pitch)


@pytest.mark.gpu
def test_gpu_raw_deterministic_runs_are_bitwise_repeatable(case):
    prev = _lib.set_deterministic(True)
    try:
        c = _cutout(case, "device")
        m, turb = case["m"], _wind_turbine(80)
        for call in (lambda: c.pv("CSi", "latitude_optimal", matrix=m, aggregate_time=None),
                     lambda: c.pv("CSi", "latitude_optimal", matrix=m, aggregate_time=None, tracking="vertical"),
                     lambda: c.wind(turb, matrix=m, aggregate_time=None),
                     lambda: c.wind(turb, interpolation_method="power", matrix=m, aggregate_time="sum")):
            a, b = np.asarray(call().values), np.asarray(call().values)
            assert np.array_equal(a, b, equal_nan=True)
    finally:
        _lib.set_deterministic(prev)


def _n_gpus():
    try:
        import torch

        return torch.cuda.device_count()
    except Exception:  # noqa: BLE001
        return 0


@pytest.mark.gpu
@pytest.mark.skipif(_n_gpus() < 2, reason="needs 2 GPUs")
def test_gpu_raw_several_devices(case):
    many = ab.Cutout(data=_dataset(case["d"], case["co"]), devices="all")
    one = _cutout(case, "host")
    m = case["m"]
    for call in (lambda c: c.pv("CSi", "latitude_optimal", matrix=m, aggregate_time=None),
                 lambda c: c.wind(_wind_turbine(80), matrix=m, aggregate_time=None)):
        assert_parity(_time_bus(call(many)), _time_bus(call(one)), case["cap"], what="raw-era5 multi-gpu")


# --------------------------------------------------------------------------------------------
# CPU: detection, field choice, kernel branch, errors, warnings
# --------------------------------------------------------------------------------------------


class _Recorder:
    """Stands in for an engine operator: records what the spec asks for."""

    def __init__(self, **kw):
        self.kw = kw


def _small(names, nt=3, nx=6, ny=4):
    d = {k: np.full((nt, ny, nx), i + 1.0, dtype=np.float32) for i, k in enumerate(names)}
    return ab.Dataset({k: (("time", "y", "x"), v) for k, v in d.items()}, coords=dict(_coords(nx, ny, nt))), d


@pytest.fixture
def record_ops(monkeypatch):
    for name in ("PvOp", "WindOp", "PointwiseOp", "HeatOp"):
        monkeypatch.setattr(convert.engine, name, _Recorder)


def test_raw_pv_spec_reads_raw_fields_into_the_raw_branch(record_ops):
    ds, d = _small(list(RAW_PV) + ["t2m"])
    spec = _no_deprecation(lambda: convert._PvSpec(ds, ab.get_solarpanelconfig("CSi"),
                                                   ab.get_orientation("latitude_optimal")))
    kw = spec.op.kw
    assert kw["irr_branch"] == _lib.IRR_ERA5_RAW and kw["solar_src"] == _lib.SOLAR_COMPUTED
    assert kw["time_shift"] == "-30min"
    want = dict(influx="ssrd", outflux="ssr", influx_toa="tisr", influx_direct="fdir", temperature="t2m")
    assert set(spec.fields) == set(want)
    for slot, var in want.items():
        assert spec.fields[slot] is ds.raw(var), slot


def test_raw_pv_spec_reads_a_stored_solar_position(record_ops):
    ds, _ = _small(list(RAW_PV) + ["temperature"])
    ds["solar_altitude"] = (("time", "y", "x"), np.zeros((3, 4, 6)))
    ds["solar_azimuth"] = (("time", "y", "x"), np.zeros((3, 4, 6)))
    spec = _no_deprecation(lambda: convert._IrradiationSpec(ds, ab.get_orientation("latitude_optimal")))
    assert spec.op.kw["irr_branch"] == _lib.IRR_ERA5_RAW
    assert spec.op.kw["solar_src"] == _lib.SOLAR_STORED_F64
    assert spec.fields["temperature"] is ds.raw("temperature")  # the prepared name wins
    assert {"solar_altitude", "solar_azimuth"} <= set(spec.fields)


@pytest.mark.parametrize("extra", list(PREPARED_PV) + ["influx", "outflux"])
def test_any_prepared_pv_variable_keeps_the_prepared_path(record_ops, extra):
    """One prepared irradiation variable next to a complete raw set: the prepared path is taken, and
    its inputs being incomplete fails as it did before."""
    ds, _ = _small(list(RAW_PV) + ["t2m", "temperature", extra])
    assert not convert._pv_raw(ds)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        with pytest.raises(AssertionError, match="Need either"):
            convert._PvSpec(ds, ab.get_solarpanelconfig("CSi"), ab.get_orientation("latitude_optimal"))
    full, _ = _small(list(RAW_PV) + ["t2m", "temperature"] + list(PREPARED_PV))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        spec = convert._PvSpec(full, ab.get_solarpanelconfig("CSi"), ab.get_orientation("latitude_optimal"))
    assert spec.op.kw["irr_branch"] == _lib.IRR_DIRECT_DIFFUSE and spec.op.kw["time_shift"] == "0h"
    assert spec.fields["influx_toa"] is full.raw("influx_toa")


@pytest.mark.parametrize("missing", RAW_PV)
def test_incomplete_raw_pv_raises_todays_error(record_ops, missing):
    ds, _ = _small([n for n in RAW_PV if n != missing] + ["t2m"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        with pytest.raises(AssertionError, match="Need either influx or influx_direct and influx_diffuse"):
            convert._PvSpec(ds, ab.get_solarpanelconfig("CSi"), ab.get_orientation("latitude_optimal"))


@pytest.mark.parametrize("hub,method,want_method,fields", [
    (100, "logarithmic", _lib.WIND_NONE, {"u100", "v100"}),
    (100, "power", _lib.WIND_NONE, {"u100", "v100"}),
    (80, "logarithmic", _lib.WIND_LOG, {"u100", "v100", "fsr"}),
    (120, "power", _lib.WIND_POWER, {"u100", "v100", "u10", "v10"}),
])
def test_raw_wind_spec_picks_method_and_fields(record_ops, hub, method, want_method, fields):
    ds, _ = _small(["u100", "v100", "u10", "v10", "fsr"])
    turb = dict(ab.get_windturbineconfig("Vestas_V112_3MW"), hub_height=hub)
    spec = convert._WindSpec(ds, turb, method)
    assert spec.op.kw["method"] == want_method and spec.op.kw["from_height"] == 100
    assert set(spec.raw) == fields
    for n in fields:
        assert spec.raw[n] is ds.raw(n)


def test_prepared_wind_speed_keeps_the_prepared_path(record_ops):
    ds, _ = _small(["u100", "v100", "u10", "v10", "fsr", "wnd100m", "roughness"])
    spec = convert._WindSpec(ds, ab.get_windturbineconfig("Vestas_V112_3MW"), "logarithmic")
    assert spec.raw is None and spec.wnd is ds.raw("wnd100m") and spec.aux is ds.raw("roughness")


@pytest.mark.parametrize("names,method", [(["u100", "u10", "v10", "fsr"], "logarithmic"),
                                          (["u100", "v100", "u10", "v10"], "logarithmic"),
                                          (["u100", "v100", "fsr"], "power"),
                                          (["u100", "v100", "fsr", "u10", "v10"], "cubic")])
def test_incomplete_raw_wind_raises_todays_error(record_ops, names, method):
    ds, _ = _small(names)
    with pytest.raises(AssertionError, match="Wind speed is not in dataset"):
        convert._WindSpec(ds, ab.get_windturbineconfig("Vestas_V112_3MW"), method)


def test_temperature_family_aliases_the_raw_names(record_ops):
    ds, _ = _small(["t2m", "stl4", "d2m"])
    assert convert._temperature_spec(ds).field is ds.raw("t2m")
    assert convert._soil_temperature_spec(ds).field is ds.raw("stl4")
    assert convert._dewpoint_temperature_spec(ds).field is ds.raw("d2m")
    assert convert._cop_spec(ds, "soil", 55.0, None, None, None).field is ds.raw("stl4")
    assert convert._HeatSpec(ds, 15.0, 1.0, 0.0, 0.0).temp is ds.raw("t2m")
    both, _ = _small(["t2m", "temperature"])
    assert convert._temperature_spec(both).field is both.raw("temperature")
    none, _ = _small(["stl4"])
    with pytest.raises(KeyError, match="temperature"):
        convert._temperature_spec(none)
