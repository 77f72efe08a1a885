"""Raw ERA5 variables at their edges: NaN, +-inf, 0, -0 and negative values in every raw variable
in turn (at a lit and at a dark step), calm winds at 10 m and 100 m, wind components whose float32
square overflows, zero / negative / NaN roughness and the accumulation corner cases of the albedo
and the diffuse influx.  These are the inputs where a kernel's fast path and its cold exact path,
and the sun gate, decide the answer.

tests/golden/reference_era5_edges.npz holds the reference's own derivations (datasets/era5.py)
and per-cell conversions of them (make_golden.py::era5_edge_cases).  On the CPU the oracle is
pinned to it; on the GPU the ERA5 kernels and every converter that reads raw variables directly
(PV MODE 5 and 6, irradiation, solar thermal, wind for every power-curve table form) are held to
the reference's per-cell values in every output form and lane layout."""

import os
import warnings

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

import atlite_oracle as O
import era5_oracle as EO
import atlite_b200 as ab
from atlite_b200 import synthetic as syn
from conftest import assert_parity

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_era5_edges.npz"))
RAW = {k.split("|")[1]: G[k] for k in G.files if k.startswith("raw|")}
TIME = pd.DatetimeIndex(G["time_ns"].astype("datetime64[ns]"))
X, Y = G["x"], G["y"]
NT, NY, NX = RAW["ssrd"].shape
T_LIT, T_DARK = int(G["t_lit"]), int(G["t_dark"])


def _class(a):
    """0 finite, 1 NaN, 2 +inf, 3 -inf"""
    a = np.asarray(a, dtype=np.float64)
    return np.select([np.isnan(a), np.isposinf(a), np.isneginf(a)], [1, 2, 3], 0)


def _close(got, want, what, tol):
    """Identical NaN / +inf / -inf positions, finite values to `tol` (relative and absolute)."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    cg, cw = _class(got), _class(want)
    assert np.array_equal(cg, cw), f"{what}: value classes differ at {np.argwhere(cg != cw)[:5].tolist()}"
    fin = cw == 0
    np.testing.assert_allclose(got[fin], want[fin], rtol=tol, atol=tol, err_msg=what)


def _oracle_fields():
    """The oracle's ERA5 derivations of the raw fields (sanitized) and the solar position at -30 min."""
    ow = EO.get_data_wind(RAW["u100"], RAW["v100"], RAW["u10"], RAW["v10"], RAW["fsr"])
    oi = EO.get_data_influx(RAW["ssrd"], RAW["ssr"], RAW["tisr"], RAW["fdir"])
    co = dict(time=TIME, lon=X, lat=Y)
    sol = O.solar_position(co, time_shift="-30min")
    od = dict(co, solar_altitude=np.broadcast_to(sol["altitude"], (NT, NY, NX)),
              solar_azimuth=np.broadcast_to(sol["azimuth"], (NT, NY, NX)), temperature=RAW["t2m"])
    od.update({k: ow[k] for k in ("wnd100m", "roughness", "wnd_shear_exp")})
    od.update({k: oi[k] for k in ("influx_toa", "influx_direct", "influx_diffuse", "albedo")})
    return od


# name -> (golden key, Cutout call, (oracle function, keywords), value scale, unit).  `unit` (conftest.
# assert_parity): solar thermal's value is irr * c0 - c1 * (t_store - T), a difference of O(1e3) W m-2
# float32 quantities
_LATOPT = "latitude_optimal"
SOLAR = {
    "pv-mode5": ("pv|CSi|latitude_optimal", lambda c, **kw: c.pv("CSi", _LATOPT, **kw),
                 (O.convert_pv, dict(panel=ab.get_solarpanelconfig("CSi"), orientation=O.get_orientation(_LATOPT))),
                 1.0, 1.0),
    "pv-mode6-bofinger": ("pv|KANENA|latitude_optimal", lambda c, **kw: c.pv("KANENA", _LATOPT, **kw),
                          (O.convert_pv, dict(panel=ab.get_solarpanelconfig("KANENA"),
                                              orientation=O.get_orientation(_LATOPT))), 1.0, 1.0),
    "pv-mode6-dual-hay-davies": ("pv|CSi|dual|other",
                                 lambda c, **kw: c.pv("CSi", _LATOPT, tracking="dual", trigon_model="other", **kw),
                                 (O.convert_pv, dict(panel=ab.get_solarpanelconfig("CSi"),
                                                     orientation=O.get_orientation(_LATOPT), tracking="dual",
                                                     trigon_model="other")), 1.0, 1.0),
    "irradiation-direct": ("irradiation|direct", lambda c, **kw: c.irradiation(_LATOPT, irradiation="direct", **kw),
                           (O.convert_irradiation, dict(orientation=O.get_orientation(_LATOPT), irradiation="direct",
                                                        clearsky_model=None)), 1000.0, 1.0),
    "irradiation-total": ("irradiation|total", lambda c, **kw: c.irradiation(_LATOPT, irradiation="total", **kw),
                          (O.convert_irradiation, dict(orientation=O.get_orientation(_LATOPT), irradiation="total",
                                                       clearsky_model=None)), 1000.0, 1.0),
    "solar-thermal": ("solar_thermal", lambda c, **kw: c.solar_thermal(**kw),
                      (O.convert_solar_thermal, dict(orientation=O.get_orientation({"slope": 45.0, "azimuth": 180.0}),
                                                     trigon_model="simple", clearsky_model="simple", c0=0.8, c1=3.0,
                                                     t_store=80.0)), 1000.0, 1000.0),
}
# hub tag -> (hub height, interpolation method); hub 100 reads the wind speed at 100 m as it is
HUBS = {"hub100": (100, "logarithmic"), "log80": (80, "logarithmic"), "power80": (80, "power"),
        "power120": (120, "power")}
CURVES = ("Vestas_V112_3MW", "lattice0", "lattice1", "lattice2")


def _turbine(name, hub):
    if name == "Vestas_V112_3MW":
        return dict(ab.get_windturbineconfig(name), hub_height=hub)
    return dict(V=G[f"curve|{name}|V"], POW=G[f"curve|{name}|POW"], P=2.0, hub_height=hub)


def _curve_info(name, table):
    from test_wind_curve import curve_info

    t = _turbine(name, 100)
    return curve_info(np.asarray(t["V"], float), np.asarray(t["POW"], float) / t["P"], table)


def _lmode(info):
    """The kernels' compile-time table form (wind.cu lut_mode): 0 binary search or general LUT,
    1 + n lattice LUT with n compares, 4 saturating lattice LUT."""
    return {0: 0, 1: 0, 2: 1 + info["compares"], 3: 4}[info["table"]]


# (curve, ATL_WIND_TABLE) -> the table form the raw wind kernels must run; -1 = not forced
WIND_TABLES = {("Vestas_V112_3MW", -1): 1, ("Vestas_V112_3MW", 0): 0, ("Vestas_V112_3MW", 1): 0,
               ("Vestas_V112_3MW", 2): 2, ("Vestas_V112_3MW", 3): 4,
               ("lattice0", 2): 1, ("lattice1", 2): 2, ("lattice2", -1): 3}


# --------------------------------------------------------------------------------------------
# CPU: the oracle pinned to the reference's edge values
# --------------------------------------------------------------------------------------------


def test_golden_plants_every_edge_value():
    """Each raw variable carries NaN, +inf, -inf, 0, -0 and a negative value at the lit and the
    dark step; the sun is up at the lit step and down at the dark one everywhere."""
    for name, a in RAW.items():
        for t in (T_LIT, T_DARK):
            v = a[t]
            assert np.isnan(v).any() and np.isposinf(v).any() and np.isneginf(v).any(), name
            assert (v == 0).any() and (np.signbit(v) & (v == 0)).any() and (v < 0).any(), name
    alt = G["influx|solar_altitude"]
    assert (alt[T_LIT] > np.radians(30)).all() and (alt[T_DARK] < 0).all()
    assert min(np.abs(alt - np.radians(t)).min() for t in (0.0, 1.0, 3.75)) > 5e-4
    # a float32 square overflows where float64 would not
    assert np.isposinf(G["wind|wnd100m"][np.isfinite(RAW["u100"]) & np.isfinite(RAW["v100"])]).any()


def test_oracle_derivations_match_the_reference_edges():
    for sanitize, tag in ((False, ""), (True, "_sanitized")):
        w = EO.get_data_wind(RAW["u100"], RAW["v100"], RAW["u10"], RAW["v10"], RAW["fsr"], sanitize=sanitize)
        for k in ("wnd100m", "wnd_shear_exp", "wnd_azimuth"):
            _close(w[k], G[f"wind|{k}"], k, 6e-7)
        _close(w["roughness"], G[f"wind{tag}|roughness"], "roughness" + tag, 6e-7)
        i = EO.get_data_influx(RAW["ssrd"], RAW["ssr"], RAW["tisr"], RAW["fdir"], sanitize=sanitize)
        _close(i["albedo"], G["influx|albedo"], "albedo", 6e-7)
        for k in ("influx_toa", "influx_direct", "influx_diffuse"):
            _close(i[k], G[f"influx{tag}|{k}"], k + tag, 6e-7)
    sol = O.solar_position(dict(time=TIME, lon=X, lat=Y), time_shift="-30min")
    np.testing.assert_allclose(np.broadcast_to(sol["altitude"], (NT, NY, NX)), G["influx|solar_altitude"], rtol=0,
                               atol=1e-12)


def test_oracle_edge_values_take_the_float32_class():
    """Where float32 and float64 arithmetic disagree on the class of a value the oracle follows the
    reference (float32): a 2e19 m/s component gives an infinite speed and shear exponent
    ln(0) / ln(0.1) = +inf."""
    w = EO.get_data_wind(np.float32([2e19, 3.0]), np.float32([0.0, 4.0]), np.float32([1.0, 1.0]),
                         np.float32([0.0, 0.0]), np.float32([0.1, 0.1]))
    assert np.isposinf(w["wnd100m"][0]) and np.isposinf(w["wnd_shear_exp"][0]) and w["wnd100m"][1] == 5.0
    w64 = EO.get_data_wind([2e19], [0.0], [1.0], [0.0], [0.1])
    assert np.isfinite(w64["wnd100m"][0])


@pytest.mark.parametrize("name", list(SOLAR))
def test_oracle_solar_conversions_match_the_reference_edges(name):
    key, _, (fn, kw), _, _ = SOLAR[name]
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore")
        got = fn(_oracle_fields(), **kw)
    _close(got, G[key], name, 1e-9)


@pytest.mark.parametrize("curve", CURVES)
def test_oracle_wind_conversions_match_the_reference_edges(curve):
    od = _oracle_fields()
    for tag, (hub, method) in HUBS.items():
        with np.errstate(all="ignore"):
            got = O.convert_wind(od, _turbine(curve, hub), interpolation_method=method)
        _close(got, G[f"wind|{curve}|{tag}"], f"{curve} {tag}", 1e-9)


def test_raw_wind_cases_reach_every_table_form():
    """The (curve, ATL_WIND_TABLE) cases of the GPU test reach all five table forms of the raw wind
    kernels, each for the log law and the power law."""
    reached = {}
    for (curve, table), want in WIND_TABLES.items():
        assert _lmode(_curve_info(curve, table)) == want, (curve, table)
        reached.setdefault(want, []).append((curve, table))
    assert sorted(reached) == [0, 1, 2, 3, 4], reached
    assert {_curve_info("Vestas_V112_3MW", t)["table"] for t in (0, 1)} == {0, 1}  # search and general LUT


# --------------------------------------------------------------------------------------------
# GPU: the ERA5 kernels and every raw converter on the edge dataset
# --------------------------------------------------------------------------------------------

RESIDENCIES = ["device-vec", "device-scalar", "host"]
FORMS = ["cells", "sum", "mean", "reduce", "two-pass"]


def _dataset():
    return ab.Dataset({k: (("time", "y", "x"), v) for k, v in RAW.items()},
                      coords=dict(time=TIME, x=X, y=Y, lon=X, lat=Y))


@pytest.fixture(scope="module")
def cutouts():
    host = ab.Cutout(data=_dataset())
    vec = host.to_device()
    assert vec.data.raw("ssrd").shape[-1] == 24
    for n in vec.data.data_vars:  # padding must not leak into any result
        vec.data.raw(n)[..., NX:] = float("nan")
    scalar = host.to_device(pad=False)
    assert scalar.data.raw("ssrd").shape[-1] == NX
    return {"device-vec": vec, "device-scalar": scalar, "host": host}


@pytest.fixture(scope="module")
def shapes():
    from atlite_b200 import engine

    m = syn.make_shapes(NX, NY, 9)
    assert engine.get_plan(m, NY, NX).info["fused"]
    eye = sp.identity(NX * NY, format="csr")
    assert not engine.get_plan(eye, NY, NX).info["fused"]
    return m, eye


def _time_bus(res):
    v = np.asarray(res.values)
    return v if res.dims[0] == "time" else v.T


def _check_forms(call, cube, scale, cutout, shapes, what, unit=1.0):
    """Every output form of one converter on one cutout against the reference's per-cell cube:
    the parity bar, identical NaN, +inf and -inf positions, and exactly 0 wherever the reference is
    exactly 0."""
    m, eye = shapes
    flat = cube.reshape(NT, -1)
    with np.errstate(all="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want = {"cells": (cube, scale), "sum": (np.nansum(cube, 0), NT * scale), "mean": (np.nanmean(cube, 0), scale),
                "reduce": (np.asarray((m @ flat.T).T), np.asarray(m.sum(-1)).ravel() * scale),
                "two-pass": (flat, scale)}
    for form in FORMS:
        kw = dict(aggregate_time={"sum": "sum", "mean": "mean"}.get(form))
        if form in ("reduce", "two-pass"):
            kw["matrix"] = m if form == "reduce" else eye
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            res = call(cutout, **kw)
        got = _time_bus(res) if "matrix" in kw else np.asarray(res.values)
        w, cap = want[form]
        label = f"{what} {form}"
        assert_parity(got, w, cap, what=label, unit=unit)
        # the parity bar cannot see an infinite reference value (its tolerance is infinite there)
        cg, cw = _class(got), _class(w)
        assert np.array_equal(cg, cw), f"{label}: value classes differ at {np.argwhere(cg != cw)[:5].tolist()}"
        z = w == 0
        assert (got[z] == 0).all(), f"{label}: {int((got[z] != 0).sum())} reference zeros are not exactly 0"


@pytest.mark.gpu
def test_gpu_era5_kernels_match_the_reference_edges():
    from atlite_b200 import era5

    ds = _dataset()
    for sanitize, tag in ((False, ""), (True, "_sanitized")):
        w = era5.get_data_wind(ds, sanitize=sanitize)
        for k in ("wnd100m", "wnd_shear_exp", "wnd_azimuth"):
            _close(w.raw(k).cpu().numpy(), G[f"wind|{k}"], k, 4e-6)
        _close(w.raw("roughness").cpu().numpy(), G[f"wind{tag}|roughness"], "roughness" + tag, 4e-6)
        i = era5.get_data_influx(ds, sanitize=sanitize, solar_position_vars=False)
        _close(i.raw("albedo").cpu().numpy(), G["influx|albedo"], "albedo", 4e-6)
        for k in ("influx_toa", "influx_direct", "influx_diffuse"):
            _close(i.raw(k).cpu().numpy(), G[f"influx{tag}|{k}"], k + tag, 4e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("residency", RESIDENCIES)
@pytest.mark.parametrize("name", list(SOLAR))
def test_gpu_raw_solar_matches_the_reference_edges(cutouts, shapes, name, residency):
    key, call, _, scale, unit = SOLAR[name]
    cube = G[key]
    assert (cube[T_LIT] > 0).any() and (cube[T_DARK] == 0).sum() > NX * NY // 2
    _check_forms(call, cube, scale, cutouts[residency], shapes, f"raw-edges-{name} {residency}", unit)


@pytest.mark.gpu
@pytest.mark.parametrize("residency", RESIDENCIES)
@pytest.mark.parametrize("curve,table", list(WIND_TABLES), ids=[f"{c}-table{t}" for c, t in WIND_TABLES])
def test_gpu_raw_wind_matches_the_reference_edges(monkeypatch, cutouts, shapes, curve, table, residency):
    """Each table form of the raw wind kernels, with the speed alone (hub 100), the log law and the
    power law: none of LMODE 0..3 has a cold exact path, so every +-inf and 0 * inf of the
    derivation must come out right from the fast code."""
    lmode = WIND_TABLES[(curve, table)]
    assert _lmode(_curve_info(curve, table)) == lmode
    if table >= 0:
        monkeypatch.setenv("ATL_WIND_TABLE", str(table))
    else:
        monkeypatch.delenv("ATL_WIND_TABLE", raising=False)
    for tag, (hub, method) in HUBS.items():
        turb = _turbine(curve, hub)
        call = lambda c, turb=turb, method=method, **kw: c.wind(turb, interpolation_method=method, **kw)  # noqa: E731
        law = "speed" if hub == 100 else method[:3]
        _check_forms(call, G[f"wind|{curve}|{tag}"], 1.0, cutouts[residency], shapes,
                     f"raw-edges-wind-{law}-lmode{lmode} {curve} table={table} {tag} {residency}")
