"""Raw ERA5 variables in line_rating, csp and runoff: a cutout that holds the download (t2m, u100,
v100, fdir, ro, z, ...) converts directly, with the result era5.prepare's cutout would give.

line_rating derives wind speed, wind azimuth and direct influx in its kernel (atl_line_rating_raw_reduce),
csp derives the direct influx (atl_csp_raw_create), runoff clips ro at 0 (atl_pointwise_create_ex), and
both weight with the height of z's first step over the WHOLE cutout.  GPU tests hold every route to the
parity bar against the float64 oracles fed with the ERA5 oracle's derivations and the solar position at
-30 min; CPU tests check the detection rules, the fields each converter hands to its operator and the
runoff / height oracle (oracle/era5_runoff_height_oracle.py) against
tests/golden/reference_era5_runoff_height.npz (tests/golden/make_golden_era5_runoff_height.py)."""

import os
import types
import warnings

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

import atlite_oracle as O
import era5_oracle as EO
import era5_runoff_height_oracle as ERH
import intersection_exact as IX
import line_rating_oracle as LO
import atlite_b200 as ab
from atlite_b200 import _lib, convert, engine, gis, synthetic as syn
from conftest import assert_parity

HERE = os.path.dirname(os.path.abspath(__file__))
G0 = 9.80665
NY, NT = 14, 29
CSP_INST = ("SAM_solar_tower", "SAM_parabolic_trough")


def _raw_arrays(nx, ny, nt, seed=0):
    """Seeded raw ERA5 fields (every variable era5.prepare reads) with planted cells: calm winds, a
    signed-zero wind, negative fdir and ro, NaN u100 and t2m, a t2m above the conductor's Ts, and a
    geopotential that changes from step to step (the height is its FIRST step's)."""
    rng = np.random.default_rng(seed)
    shp = (nt, ny, nx)
    f = lambda lo, hi: rng.uniform(lo, hi, shp).astype(np.float32)  # noqa: E731
    d = dict(u100=f(-15, 15), v100=f(-15, 15), u10=f(-8, 8), v10=f(-8, 8), fsr=f(0.0, 2.0),
             ssrd=f(0, 3.0e6), tisr=f(0, 4.5e6), t2m=f(255, 305), stl4=f(270, 290), d2m=f(250, 295),
             ro=f(-1e-4, 2e-3))
    d["ssr"] = (d["ssrd"] * rng.uniform(0.6, 1.0, shp)).astype(np.float32)
    d["fdir"] = (d["ssrd"] * rng.uniform(0.0, 0.95, shp)).astype(np.float32)
    base = rng.uniform(0.0, 1500.0 * G0, (ny, nx)).astype(np.float32)
    d["z"] = (base[None] + (np.arange(nt, dtype=np.float32) * 40.0 * G0)[:, None, None]).astype(np.float32)
    d["u100"][:, 0, 0], d["v100"][:, 0, 0] = 0.0, 0.0     # calm
    d["u100"][:, 0, 1], d["v100"][:, 0, 1] = 0.0, -0.0    # u = +0, v = -0
    d["u100"][:, 0, 2], d["v100"][:, 0, 2] = -0.0, -0.0   # u = -0, v = -0
    d["fdir"][:, 2, 3] = -25.0
    d["fdir"][:, 4, 9] = -3.6e3
    d["ro"][:, 1, 4] = -3e-5
    d["u100"][:, 3, 5] = np.nan   # every step: a cell no line may take
    d["t2m"][2:5, 6, 2] = np.nan
    d["t2m"][4:9, 1, 7] = 380.0   # Ta > Ts: NaN, skipped
    return d


def _coords(nx, ny, nt, x0=6.0, y0=47.0, dx=0.25):
    x, y = syn.make_coords(nx, ny, x0, y0, dx, dx)
    t = syn.make_time(nt + 24 * 150)[24 * 150:]  # May: day, night and the terminator
    return dict(time=t, x=x, y=y, lon=x, lat=y)


def _dataset(d, co, names=None):
    names = list(d) if names is None else names
    return ab.Dataset({k: ((("time", "y", "x")[-d[k].ndim:]), d[k]) for k in names}, coords=dict(co))


def _line(xy):
    return {"type": "LineString", "coordinates": np.asarray(xy, dtype=np.float64)}


def _network(x, y):
    """make_line_network plus two multi-cell lines through the planted cells (row 3 across the NaN-wind
    cell (3, 5), row 1 across the hot cell (1, 7)), a line across the calm and signed-zero cells and a
    one-cell line on the negative-fdir cell."""
    lines = syn.make_line_network(x, y, 10)
    dx = x[1] - x[0]
    lines.append(_line([[x[4], y[3]], [x[6], y[3]]]))
    lines.append(_line([[x[6], y[1]], [x[8], y[1]]]))
    lines.append(_line([[x[0], y[0]], [x[2], y[0]]]))
    lines.append(_line([[x[3] - 0.2 * dx, y[2] + 0.1 * dx], [x[3] + 0.3 * dx, y[2] - 0.2 * dx]]))
    return lines


def _oracle_ds(d, co):
    """What era5.prepare stores, from the ERA5 oracle, plus the solar position at -30 min."""
    ow = EO.get_data_wind(d["u100"], d["v100"], d["u10"], d["v10"], d["fsr"])
    oi = EO.get_data_influx(d["ssrd"], d["ssr"], d["tisr"], d["fdir"])
    c = dict(time=co["time"], lon=co["x"], lat=co["y"])
    sol = O.solar_position(c, time_shift="-30min")
    od = dict(c, solar_altitude=sol["altitude"], solar_azimuth=sol["azimuth"], temperature=d["t2m"],
              wnd100m=ow["wnd100m"], wnd_azimuth=ow["wnd_azimuth"], influx_direct=oi["influx_direct"],
              runoff=ERH.get_data_runoff(d["ro"])["runoff"], height=ERH.get_data_height(d["z"])["height"])
    return od


def _lr_oracle(od, co, lines, R=1e-4):
    x, y = np.asarray(co["x"]), np.asarray(co["y"])
    s = convert._line_shapes(lines)
    I = sp.csr_matrix(IX.intersectionmatrix(x, y, [gis.geometry_parts(g) for g in s.values]))
    az = pd.Series([LO.line_azimuth(g["coordinates"]) for g in s.values], index=s.index)
    return LO.line_rating(od, I, az, R), I


_CASES = {}


def _case(nx):
    """One raw case per width (36: 128-bit lanes, 37: padded to 40 or scalar)."""
    if nx not in _CASES:
        co = _coords(nx, NY, NT)
        d = _raw_arrays(nx, NY, NT, seed=11)
        m = syn.make_shapes(nx, NY, 6)
        _CASES[nx] = dict(nx=nx, d=d, co=co, m=m, cap=np.asarray(sp.csr_matrix(m).sum(-1)).ravel(),
                          od=_oracle_ds(d, co), lines=_network(co["x"], co["y"]))
    return _CASES[nx]


def _cutout(c, residency, tmp_path=None, names=None):
    ds = _dataset(c["d"], c["co"], names)
    cut = ab.Cutout(data=ds)
    if residency == "host":
        return cut
    if residency == "pinned":
        return cut.pin_host()
    if residency.startswith("device"):
        return cut.to_device(pad=residency != "device_scalar")
    from atlite_b200 import ingest

    names = list(c["d"]) if names is None else names
    p = ingest.write_chunked(tmp_path / "raw.bin", {k: c["d"][k] for k in names}, dict(c["co"]), chunk=(8, None, None))
    return ab.Cutout(data=ingest.open_cutout(p))


def _no_deprecation(fn):
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        out = fn()
    assert not [x for x in w if issubclass(x.category, DeprecationWarning)], [str(x.message) for x in w]
    return out


def _time_bus(res):
    v = np.asarray(res.values)
    return v if res.dims[0] == "time" else v.T


@pytest.fixture
def count_parts(monkeypatch):
    """Records the time parts every partitioned conversion is cut into."""
    seen = []
    orig = convert._partition

    def rec(*a, **k):
        parts = orig(*a, **k)
        seen.append(parts)
        return parts

    monkeypatch.setattr(convert, "_partition", rec)
    return seen


LR_NAMES = ["t2m", "u100", "v100", "fdir", "z"]


# --------------------------------------------------------------------------------------------
# GPU: line_rating
# --------------------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("residency", ["device_vec", "device_padded", "device_scalar", "host", "pinned", "lazy",
                                       "lazy_parts"])
def test_gpu_raw_line_rating_matches_oracle(tmp_path, monkeypatch, count_parts, residency):
    c = _case(36 if residency == "device_vec" else 37)
    if residency == "lazy_parts":
        monkeypatch.setattr(convert, "PART_BYTES", 1)  # one dataset time chunk (8 steps) per part
    cut = _cutout(c, residency.replace("_vec", "").replace("_parts", ""), tmp_path, LR_NAMES)
    res = _no_deprecation(lambda: cut.line_rating(c["lines"], 1e-4))
    if residency == "lazy_parts":
        assert len(count_parts[-1]) > 2
    want, I = _lr_oracle(c["od"], c["co"], c["lines"])
    nx, n = c["nx"], len(c["lines"])
    row_nan, row_hot = n - 4, n - 3
    assert I[row_nan, 3 * nx + 5] == 1 and I[row_nan].sum() > 1
    assert I[row_hot, 1 * nx + 7] == 1 and I[row_hot].sum() > 1
    assert np.isfinite(want[row_nan]).all() and np.isfinite(want[row_hot]).all()
    assert np.isfinite(want[n - 2]).all()  # calm and signed-zero winds
    assert res.dims == ("dim_0", "time") and res.attrs["units"] == "A"
    assert_parity(np.asarray(res.values), want, what=f"raw dlr {residency}")


@pytest.mark.gpu
@pytest.mark.parametrize("width", [37, 40])  # scalar and 128-bit lanes
def test_gpu_raw_line_rating_op_is_prepared_op_bitwise(width):
    """reduce_raw on t2m / u100 / v100 / fdir equals reduce on era5.get_data_wind / get_data_influx /
    get_data_height's fields bit for bit: the same derivations, in registers."""
    import torch

    from atlite_b200 import era5

    c = _case(37)
    d, co, nx = c["d"], c["co"], c["nx"]
    raw_ds = _dataset(d, co)

    def dev(a):
        a = a.cpu().numpy() if engine._is_torch(a) else a
        pad = ((0, 0),) * (a.ndim - 1) + ((0, width - nx),)
        return torch.from_numpy(np.ascontiguousarray(np.pad(a, pad))).cuda()

    wind = era5.get_data_wind(raw_ds)
    infl = era5.get_data_influx(raw_ds, solar_position_vars=False)
    height = dev(era5.get_data_height(raw_ds).raw("height"))
    _, _, df = convert._line_parameters(c["lines"], 1e-4, {})
    I = gis.compute_intersectionmatrix(co["x"], co["y"], c["lines"])
    plan = engine.get_plan(I, NY, nx, pitch=width, entries=True)
    op = engine.LineRatingOp(ny=NY, nx=nx, time=co["time"], lon=co["x"], lat=co["y"], solar_src=_lib.SOLAR_COMPUTED,
                             params={k: df[k].to_numpy(np.float64) for k in _lib.LINE_PARAMS}, time_shift="-30min",
                             pitch=width)
    a = op.reduce_raw(plan, dict(t2m=dev(d["t2m"]), u100=dev(d["u100"]), v100=dev(d["v100"]), fdir=dev(d["fdir"]),
                                 height=height))
    b = op.reduce(plan, dict(temperature=dev(d["t2m"]), wnd100m=dev(wind.raw("wnd100m")),
                             wnd_azimuth=dev(wind.raw("wnd_azimuth")), influx_direct=dev(infl.raw("influx_direct")),
                             height=height))
    assert torch.isfinite(a).sum() > 0
    assert torch.equal(torch.nan_to_num(a, 7.0), torch.nan_to_num(b, 7.0))


# --------------------------------------------------------------------------------------------
# GPU: csp
# --------------------------------------------------------------------------------------------


def _csp_cfg(inst):
    return ab.get_cspinstallationconfig(inst)


@pytest.mark.gpu
@pytest.mark.parametrize("residency", ["device", "host", "lazy"])
@pytest.mark.parametrize("inst", CSP_INST)
def test_gpu_raw_csp_matches_oracle(tmp_path, residency, inst):
    c = _case(37)
    cut = _cutout(c, residency, tmp_path, ["fdir"])
    cfg, od, m = _csp_cfg(inst), c["od"], c["m"]
    res = _no_deprecation(lambda: cut.csp(cfg, matrix=m, aggregate_time=None))
    want = O.convert_and_aggregate(od, O.convert_csp, matrix=m, aggregate_time=None, installation=cfg)
    assert want.sum() > 0
    assert_parity(_time_bus(res), want, c["cap"], what=f"raw csp {inst} {residency}")
    cube = O.convert_csp(od, cfg)
    assert_parity(cut.csp(cfg, aggregate_time=None).values, cube, what=f"raw csp cells {inst} {residency}")
    assert_parity(cut.csp(cfg, aggregate_time="sum").values, cube.sum(0), NT, what=f"raw csp sum {inst} {residency}")
    assert_parity(cut.csp(cfg, aggregate_time="mean").values, cube.mean(0), what=f"raw csp mean {inst} {residency}")


@pytest.mark.gpu
def test_gpu_raw_csp_reads_a_stored_solar_position():
    c = _case(37)
    d = dict(fdir=c["d"]["fdir"], solar_altitude=c["od"]["solar_altitude"].astype(np.float64),
             solar_azimuth=c["od"]["solar_azimuth"].astype(np.float64))
    d = {k: np.ascontiguousarray(np.broadcast_to(v, c["d"]["fdir"].shape)) for k, v in d.items()}
    cfg = _csp_cfg("SAM_solar_tower")
    res = _no_deprecation(lambda: ab.Cutout(data=_dataset(d, c["co"])).to_device().csp(cfg, matrix=c["m"],
                                                                                      aggregate_time=None))
    want = O.convert_and_aggregate(c["od"], O.convert_csp, matrix=c["m"], aggregate_time=None, installation=cfg)
    assert_parity(_time_bus(res), want, c["cap"], what="raw csp stored solar position")


@pytest.mark.gpu
@pytest.mark.parametrize("width", [37, 40])
@pytest.mark.parametrize("inst", CSP_INST)
def test_gpu_raw_csp_op_is_prepared_op_bitwise(width, inst):
    import torch

    from atlite_b200 import era5
    from atlite_b200.resource import EfficiencyTable

    c = _case(37)
    d, co, nx = c["d"], c["co"], c["nx"]
    infl = era5.get_data_influx(_dataset(d, co), solar_position_vars=False)

    def dev(a):
        a = a.cpu().numpy() if engine._is_torch(a) else a
        return torch.from_numpy(np.ascontiguousarray(np.pad(a, ((0, 0), (0, 0), (0, width - nx))))).cuda()

    cfg = _csp_cfg(inst)
    eff = EfficiencyTable.from_any(cfg["efficiency"])

    def op(raw):
        return engine.CspOp(ny=NY, nx=nx, time=co["time"], lon=co["x"], lat=co["y"], solar_src=_lib.SOLAR_COMPUTED,
                            technology=_lib.CSP_TECH[cfg["technology"]], r_irradiance=cfg["r_irradiance"],
                            altitude=eff.altitude, azimuth=eff.azimuth, efficiency=eff.values, time_shift="-30min",
                            raw=raw, pitch=width)

    a = op(True).cells({"influx_direct": dev(d["fdir"])})
    b = op(False).cells({"influx_direct": dev(infl.raw("influx_direct"))})
    assert a.abs().sum() > 0
    assert torch.equal(torch.nan_to_num(a, 7.0), torch.nan_to_num(b, 7.0))


# --------------------------------------------------------------------------------------------
# GPU: runoff
# --------------------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("residency", ["device", "host", "lazy"])
def test_gpu_raw_runoff_matches_oracle(tmp_path, monkeypatch, count_parts, residency):
    c = _case(37)
    if residency == "lazy":
        monkeypatch.setattr(convert, "PART_BYTES", 1)
    cut = _cutout(c, residency, tmp_path, ["ro", "z"])
    od, m = c["od"], c["m"]
    for wh in (True, False):
        res = cut.runoff(matrix=m, aggregate_time=None, weight_with_height=wh)
        want = O.convert_and_aggregate(od, O.convert_runoff, matrix=m, aggregate_time=None, weight_with_height=wh)
        assert_parity(_time_bus(res), want, np.abs(want).max(0) * 10, what=f"raw runoff height={wh} {residency}")
    if residency == "lazy":
        assert len(count_parts[-1]) > 2
    sm = cut.runoff(matrix=m, aggregate_time=None, smooth=5, lower_threshold_quantile=0.1)
    base = O.convert_and_aggregate(od, O.convert_runoff, matrix=m, aggregate_time=None)
    roll = pd.DataFrame(base).rolling(5, min_periods=1).mean().values
    thr = pd.Series(roll.T.ravel()).quantile(0.1)
    want = np.where(roll >= thr, roll, 0.0)
    np.testing.assert_allclose(_time_bus(sm), want, rtol=2e-4, atol=np.abs(want).max() * 1e-5)
    cube = O.convert_runoff(od)
    assert_parity(cut.runoff(aggregate_time=None).values, cube, unit=np.abs(cube).max(), what="raw runoff cells")


# --------------------------------------------------------------------------------------------
# GPU: precedence, every converter, several devices
# --------------------------------------------------------------------------------------------


@pytest.mark.gpu
def test_gpu_prepared_variables_take_precedence_bitwise():
    """A dataset with raw AND prepared variables converts exactly as the prepared-only dataset."""
    from atlite_b200 import era5

    c = _case(37)
    raw = _dataset(c["d"], c["co"])
    feats = ("wind", "influx", "temperature", "runoff")
    prep, both = era5.prepare(raw, features=feats), era5.prepare(raw, features=feats)
    for k in c["d"]:
        both[k] = (raw.dims_of(k), raw.raw(k))
    m, cfg = c["m"], _csp_cfg("SAM_solar_tower")
    prev = _lib.set_deterministic(True)
    try:
        for call in (lambda cut: cut.line_rating(c["lines"], 1e-4),
                     lambda cut: cut.csp(cfg, matrix=m, aggregate_time=None),
                     lambda cut: cut.csp(cfg, aggregate_time="sum"),
                     lambda cut: cut.runoff(matrix=m, aggregate_time=None)):
            a = np.asarray(call(ab.Cutout(data=prep)).values)
            b = np.asarray(call(ab.Cutout(data=both)).values)
            assert np.array_equal(a, b, equal_nan=True)
    finally:
        _lib.set_deterministic(prev)


@pytest.mark.gpu
@pytest.mark.parametrize("residency", ["device", "host"])
def test_gpu_one_raw_dataset_through_every_converter(residency):
    c = _case(37)
    cut = _cutout(c, residency)
    m = c["m"]
    turb = dict(ab.get_windturbineconfig("Vestas_V112_3MW"), hub_height=80)
    calls = {
        "pv": lambda: cut.pv("CSi", "latitude_optimal", matrix=m, aggregate_time=None),
        "wind": lambda: cut.wind(turb, matrix=m, aggregate_time=None),
        "wind_power": lambda: cut.wind(turb, interpolation_method="power", matrix=m, aggregate_time=None),
        "irradiation": lambda: cut.irradiation({"slope": 30.0, "azimuth": 180.0}, matrix=m, aggregate_time=None),
        "solar_thermal": lambda: cut.solar_thermal(matrix=m, aggregate_time=None),
        "temperature": lambda: cut.temperature(matrix=m, aggregate_time=None),
        "soil_temperature": lambda: cut.soil_temperature(matrix=m, aggregate_time=None),
        "dewpoint_temperature": lambda: cut.dewpoint_temperature(matrix=m, aggregate_time=None),
        "cop": lambda: cut.coefficient_of_performance(matrix=m, aggregate_time=None),
        "heat_demand": lambda: cut.heat_demand(matrix=m, aggregate_time=None),
        "cooling_demand": lambda: cut.cooling_demand(matrix=m, aggregate_time=None),
        "csp": lambda: cut.csp("SAM_parabolic_trough", matrix=m, aggregate_time=None),
        "runoff": lambda: cut.runoff(matrix=m, aggregate_time=None),
        "line_rating": lambda: cut.line_rating(c["lines"], 1e-4),
    }
    for name, call in calls.items():
        res = _no_deprecation(call)
        assert np.isfinite(np.asarray(res.values)).any(), name


def _n_gpus():
    try:
        import torch

        return torch.cuda.device_count()
    except Exception:  # noqa: BLE001
        return 0


@pytest.mark.gpu
@pytest.mark.skipif(_n_gpus() < 2, reason="needs 2 GPUs")
def test_gpu_raw_several_devices():
    c = _case(37)
    many = ab.Cutout(data=_dataset(c["d"], c["co"]), devices="all")
    one = _cutout(c, "host")
    m, cfg = c["m"], _csp_cfg("SAM_solar_tower")
    for call in (lambda cut: cut.line_rating(c["lines"], 1e-4),
                 lambda cut: cut.csp(cfg, matrix=m, aggregate_time=None),
                 lambda cut: cut.runoff(matrix=m, aggregate_time=None)):
        assert np.array_equal(np.asarray(call(many).values), np.asarray(call(one).values), equal_nan=True)


# --------------------------------------------------------------------------------------------
# CPU: detection, field choice, height, errors, oracle pinning
# --------------------------------------------------------------------------------------------


class _Recorder:
    """Stands in for an engine operator: records what the spec asks for."""

    def __init__(self, **kw):
        self.kw = kw


def _small(names, nt=6, nx=6, ny=4, z_time=True):
    d = {k: np.full((nt, ny, nx), i + 1.0, dtype=np.float32) for i, k in enumerate(names)}
    if "z" in d:
        d["z"] = (np.arange(nt * ny * nx, dtype=np.float32).reshape(nt, ny, nx) * G0 if z_time
                  else np.arange(ny * nx, dtype=np.float32).reshape(ny, nx) * G0)
    return _dataset(d, _coords(nx, ny, nt)), d


@pytest.fixture
def record_ops(monkeypatch):
    for name in ("LineRatingOp", "CspOp", "PointwiseOp"):
        monkeypatch.setattr(convert.engine, name, _Recorder)
    from atlite_b200 import era5

    # z / g0 without a GPU: the CPU stand-in of era5.height_from_z
    monkeypatch.setattr(era5, "height_from_z", lambda z, device=None: np.asarray(z[0] if z.ndim == 3 else z) / G0)


LP = {k: np.ones(2) for k in _lib.LINE_PARAMS}


def test_raw_line_rating_spec_reads_raw_fields(record_ops):
    ds, d = _small(LR_NAMES)
    spec = _no_deprecation(lambda: convert._LineRatingSpec(ds, LP))
    assert spec.raw and spec.op.kw["solar_src"] == _lib.SOLAR_COMPUTED and spec.op.kw["time_shift"] == "-30min"
    assert set(spec.fields) == {"t2m", "u100", "v100", "fdir", "height"}
    for n in ("t2m", "u100", "v100", "fdir"):
        assert spec.fields[n] is ds.raw(n)
    np.testing.assert_array_equal(spec.fields["height"], d["z"][0] / G0)
    both, _ = _small(LR_NAMES + ["temperature", "height"])
    spec = convert._LineRatingSpec(both, LP)
    assert spec.fields["t2m"] is both.raw("temperature") and spec.fields["height"] is both.raw("height")


def test_raw_line_rating_spec_reads_a_stored_solar_position(record_ops):
    ds, _ = _small(LR_NAMES)
    ds["solar_altitude"] = (("time", "y", "x"), np.zeros((6, 4, 6), dtype=np.float32))
    ds["solar_azimuth"] = (("time", "y", "x"), np.zeros((6, 4, 6), dtype=np.float32))
    spec = _no_deprecation(lambda: convert._LineRatingSpec(ds, LP))
    assert spec.op.kw["solar_src"] == _lib.SOLAR_STORED_F32 and spec.op.kw["time_shift"] == "0h"


@pytest.mark.parametrize("extra", ["wnd100m", "wnd_azimuth", "influx_direct"])
def test_any_prepared_line_rating_variable_keeps_the_prepared_path(record_ops, extra):
    ds, _ = _small(LR_NAMES + ["temperature", "height", extra])
    assert not convert._line_rating_raw(ds)
    with pytest.raises(KeyError):  # the prepared path's own inputs are incomplete
        convert._LineRatingSpec(ds, LP)
    full, _ = _small(LR_NAMES + ["temperature", "height", "wnd100m", "wnd_azimuth", "influx_direct"])
    with pytest.warns(DeprecationWarning):
        spec = convert._LineRatingSpec(full, LP)
    assert not spec.raw and spec.op.kw["time_shift"] == "0h"
    assert spec.fields["wnd100m"] is full.raw("wnd100m") and spec.fields["height"] is full.raw("height")


class _FakeCutout:
    def __init__(self, data, devices=None):
        self.data, self.time_shard, self._devices = data, None, devices

    devices = property(lambda s: s._devices)

    def intersectionmatrix(self, shapes):
        return sp.csr_matrix(np.ones((len(shapes), 24)))


_LINES = [_line([[6.0, 47.0], [6.5, 47.5]]), _line([[6.2, 47.0], [6.7, 47.2]])]


@pytest.mark.parametrize("names,missing", [(["t2m", "u100", "v100", "z"], "temperature"),
                                           (["u100", "v100", "fdir", "z"], "temperature"),
                                           (["t2m", "u100", "v100", "fdir"], "height"),
                                           (["temperature", "u100", "fdir", "height"], "wnd100m")])
def test_incomplete_raw_line_rating_raises_todays_error(names, missing):
    ds, _ = _small(names)
    with pytest.raises(KeyError, match=missing):
        ab.line_rating(_FakeCutout(ds), _LINES, 1e-4)


def _record_parts(monkeypatch):
    """_run_partitioned stand-in: builds every part's spec as the real one does and records it."""
    specs, kwds = [], []

    def run_partitioned(ds, spec_cls, convert_kwds, parts, run, wpd):
        kwds.append(convert_kwds)
        out = []
        for lo, hi, _ in parts:
            spec = spec_cls(convert._time_slice(ds, lo, hi), **convert_kwds)
            specs.append(spec)
            out.append((np.zeros((hi - lo, 4, 6) if spec.name == "runoff" else (hi - lo, 2), np.float32),
                        types.SimpleNamespace(units=None, name=spec.name, time_labels=spec.time_labels)))
        return out

    monkeypatch.setattr(convert, "_run_partitioned", run_partitioned)
    return specs, kwds


def test_raw_line_rating_height_comes_from_the_whole_cutouts_first_step(record_ops, monkeypatch):
    ds, d = _small(LR_NAMES)
    specs, kwds = _record_parts(monkeypatch)
    _no_deprecation(lambda: ab.line_rating(_FakeCutout(ds, devices=[0, 1, 2]), _LINES, 1e-4))
    assert len(specs) == 3 and kwds[0]["height"] is not None
    want = d["z"][0] / G0
    for s in specs:
        assert s.raw and s.fields["height"] is kwds[0]["height"]
    np.testing.assert_array_equal(kwds[0]["height"], want)
    assert not np.array_equal(d["z"][2], d["z"][0])


def test_raw_runoff_height_comes_from_the_whole_cutouts_first_step(record_ops, monkeypatch):
    ds, d = _small(["ro", "z"])
    specs, kwds = _record_parts(monkeypatch)
    convert.convert_and_aggregate(_FakeCutout(ds, devices=[0, 1, 2]), convert.convert_runoff, aggregate_time=None)
    assert len(specs) == 3
    for s in specs:
        assert s.op.kw["clip_min_zero"] and s.field.shape[0] == 2
        np.testing.assert_array_equal(s.op.kw["cell_scale"], d["z"][0] / G0)


def test_raw_runoff_spec(record_ops):
    ds, d = _small(["ro", "z"], z_time=False)
    spec = convert._runoff_spec(ds)
    assert spec.field is ds.raw("ro") and spec.op.kw["clip_min_zero"]
    np.testing.assert_array_equal(spec.op.kw["cell_scale"], d["z"] / G0)
    spec = convert._runoff_spec(ds, weight_with_height=False)
    assert spec.op.kw["cell_scale"] is None and spec.op.kw["clip_min_zero"]
    prep, _ = _small(["ro", "z", "runoff", "height"])
    spec = convert._runoff_spec(prep)
    assert spec.field is prep.raw("runoff") and "clip_min_zero" not in spec.op.kw
    no_h, _ = _small(["ro"])
    with pytest.raises(KeyError, match="height"):
        convert._runoff_spec(no_h)
    assert convert._runoff_spec(no_h, weight_with_height=False).field is no_h.raw("ro")
    prep_z, _ = _small(["runoff", "z"])  # the prepared path weights with `height` only, as before
    with pytest.raises(KeyError, match="height"):
        convert._runoff_spec(prep_z)


def test_raw_csp_spec(record_ops):
    cfg = _csp_cfg("SAM_solar_tower")
    ds, _ = _small(["fdir"])
    spec = _no_deprecation(lambda: convert._CspSpec(ds, cfg))
    assert spec.op.kw["raw"] and spec.op.kw["time_shift"] == "-30min" and spec.op.kw["solar_src"] == _lib.SOLAR_COMPUTED
    assert set(spec.fields) == {"influx_direct"} and spec.fields["influx_direct"] is ds.raw("fdir")
    ds["solar_altitude"] = (("time", "y", "x"), np.zeros((6, 4, 6)))
    ds["solar_azimuth"] = (("time", "y", "x"), np.zeros((6, 4, 6)))
    spec = _no_deprecation(lambda: convert._CspSpec(ds, cfg))
    assert spec.op.kw["raw"] and spec.op.kw["time_shift"] == "0h" and spec.op.kw["solar_src"] == _lib.SOLAR_STORED_F64
    both, _ = _small(["fdir", "influx_direct"])
    with pytest.warns(DeprecationWarning):
        spec = convert._CspSpec(both, cfg)
    assert not spec.op.kw["raw"] and spec.op.kw["time_shift"] == "0h"
    assert spec.fields["influx_direct"] is both.raw("influx_direct")
    none, _ = _small(["ssrd"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        with pytest.raises(KeyError, match="influx_direct"):
            convert._CspSpec(none, cfg)


def test_oracle_runoff_and_height_match_the_reference():
    g = np.load(os.path.join(HERE, "golden", "reference_era5_runoff_height.npz"))
    r = ERH.get_data_runoff(g["raw|ro"], sanitize=False)["runoff"]
    assert r.dtype == np.float32 and np.array_equal(r, g["runoff|runoff"], equal_nan=True)
    r = ERH.get_data_runoff(g["raw|ro"])["runoff"]
    assert r.dtype == np.float32 and np.array_equal(r, g["runoff_sanitized|runoff"], equal_nan=True)
    for tag, z in (("time", g["raw|z"]), ("static", g["raw|z_static"])):
        h = ERH.get_data_height(z)["height"]
        assert h.shape == g[f"height|{tag}"].shape and h.dtype == np.float32
        assert np.array_equal(h, g[f"height|{tag}"], equal_nan=True), tag
    assert not np.array_equal(g["raw|z"][1], g["raw|z"][0], equal_nan=True)
