#!/usr/bin/env python
"""Generate the golden vectors that pin the oracle:  run the REFERENCE'S OWN
source (atlite/convert.py, aggregate.py, wind.py, pv/*.py, resource.py) from
/root/reference on small seeded synthetic cutouts and store inputs + outputs.

The reference cannot be imported as a package in the build container
(xarray / dask / geopandas are not installed and there is no network), so its
hot-path modules are loaded from their files under the container stand-ins of
``xr_shim.py``; every formula that executes is the reference's own line.

    python tests/golden/make_golden.py        # needs /root/reference; writes tests/golden/*.npz
    python tests/golden/make_golden.py era5_edges   # only reference_era5_edges.npz

The outputs are committed; tests/test_oracle_vs_reference.py (CPU) checks the
oracle against them, so nothing reads /root/reference at test time.
"""

import os
import sys
import warnings

import numpy as np
import pandas as pd
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import xr_shim  # noqa: E402

from atlite_b200 import synthetic as syn  # noqa: E402  (input generator only)

warnings.simplefilter("ignore")
conv = xr_shim.install()
import atlite.resource as ref_resource  # noqa: E402  (the reference's module, loaded by the shim)
from atlite.pv.orientation import get_orientation as ref_get_orientation  # noqa: E402
from atlite.pv.solar_position import SolarPosition as RefSolarPosition  # noqa: E402


class MockCutout:  # reference test/test_aggregate_time.py:13-18
    def __init__(self, data):
        self.data = data
        grid = np.array([(x, y) for y in np.asarray(data.coords["y"].values) for x in np.asarray(data.coords["x"].values)])
        self.grid = pd.DataFrame(grid, columns=["x", "y"])


MockCutout.convert_and_aggregate = conv.convert_and_aggregate  # bound as in cutout.py:659


def ref_dataset(fields, time, x, y):
    return xr_shim.Dataset({k: ((("time", "y", "x") if v.ndim == 3 else ("y", "x")), v) for k, v in fields.items()},
                           coords=dict(time=time, x=x, y=y, lon=x, lat=y), attrs={"module": "era5"})


def values_tb(res):
    """Values in the oracle's layout, transposed BY DIM NAME: (time, bus) (the reference's
    NumPy branch returns (bus, time), aggregate.py:34-35) and (time, y, x) (the reference's
    per-cell PV cube comes out as (y, time, x): xarray orders dims by first appearance and
    sin(slope[y]) leads the product in pv/orientation.py:115)."""
    if res.ndim == 2 and "time" in res.dims:
        other = [d for d in res.dims if d != "time"][0]
        return np.asarray(res.transpose("time", other).values)
    if res.ndim == 3:
        return np.asarray(res.transpose("time", "y", "x").values)
    return np.asarray(res.values)


def main():
    nx, ny, nt, nbus = 14, 9, 54, 5
    base = syn.make_dataset(nx, ny, nt, x0=-8.0, y0=-30.0, dx=1.5, dy=7.5, start="2013-03-09 05:00",
                            extra=("wnd_shear_exp", "humidity", "soil temperature", "dewpoint temperature", "runoff"))
    x, y, time = base.coords["x"], base.coords["y"], base.coords["time"]
    F = {k: np.asarray(base.raw(k)) for k in base.keys()}
    m = syn.make_shapes(nx, ny, nbus)
    lay = syn.make_layout(nx, ny)
    out = {"x": x, "y": y, "time_ns": pd.DatetimeIndex(time).as_unit("ns").asi8,
           "matrix_data": m.data, "matrix_indices": m.indices, "matrix_indptr": m.indptr,
           "matrix_shape": np.array(m.shape), "layout": lay}
    for k, v in F.items():
        out["in_" + k] = v
    cases = []

    def run(name, func, ds, **kw):
        res = func(MockCutout(ds), **kw)
        if isinstance(res, tuple):
            out[f"out_{name}"] = values_tb(res[0])
            out[f"out_{name}__capacity"] = np.asarray(res[1].values)
        else:
            out[f"out_{name}"] = values_tb(res)
        r0 = res[0] if isinstance(res, tuple) else res
        out[f"dims_{name}"] = np.array(list(r0.dims))
        cases.append(name)

    pv_names = ["influx_toa", "influx_direct", "influx_diffuse", "albedo", "temperature"]
    ds_pv = ref_dataset({k: F[k] for k in pv_names}, time, x, y)
    ds_wind = ref_dataset({k: F[k] for k in ("wnd100m", "roughness", "wnd_shear_exp")}, time, x, y)
    ds_t = ref_dataset({"temperature": F["temperature"]}, time, x, y)

    # ---- wind (convert.py:634-744, wind.py:24-128, resource.py)
    for turb in ("Vestas_V112_3MW", "Enercon_E126_7500kW"):
        for method in ("logarithmic", "power"):
            run(f"wind|{turb}|{method}", conv.wind, ds_wind, turbine=turb, matrix=m,
                interpolation_method=method, aggregate_time=None)
    run("wind|Vestas_V112_3MW|smooth", conv.wind, ds_wind, turbine="Vestas_V112_3MW", smooth=True,
        matrix=m, aggregate_time=None)
    t100 = dict(ref_resource.get_windturbineconfig("Vestas_V112_3MW"), hub_height=100)
    run("wind|hub100|fastlane", conv.wind, ds_wind, turbine=t100, matrix=m, aggregate_time=None)
    run("wind|cells", conv.wind, ds_wind, turbine="Vestas_V112_3MW", aggregate_time=None)
    run("wind|cells_mean", conv.wind, ds_wind, turbine="Vestas_V112_3MW", aggregate_time="mean")
    xl = xr_shim.DataArray(lay, {"y": y, "x": x}, ("y", "x"))
    run("wind|layout_capacity", conv.wind, ds_wind, turbine="Vestas_V112_3MW", matrix=m, layout=xl,
        return_capacity=True, aggregate_time=None)
    run("wind|per_unit_mean", conv.wind, ds_wind, turbine="Vestas_V112_3MW", matrix=m, per_unit=True,
        aggregate_time="mean")
    run("wind|layout_only_sum", conv.wind, ds_wind, turbine="Vestas_V112_3MW", layout=xl, aggregate_time="sum")
    sm = ref_resource.windturbine_smooth(ref_resource.get_windturbineconfig("Vestas_V112_3MW"))
    out["smooth_V"], out["smooth_POW"] = sm["V"], sm["POW"]

    # ---- pv (convert.py:840-936, pv/*.py)
    pv_cases = {
        "CSi|latitude_optimal|None|simple": dict(panel="CSi", orientation="latitude_optimal"),
        "CdTe|flat|None|simple": dict(panel="CdTe", orientation={"slope": 0.0, "azimuth": 0.0}),
        "KANENA|latitude_optimal|None|simple": dict(panel="KANENA", orientation="latitude_optimal"),
        "CSi|latitude|None|other": dict(panel="CSi", orientation="latitude", trigon_model="other"),
        "CSi|s35a160|None|other": dict(panel="CSi", orientation={"slope": 35.0, "azimuth": 160.0}, trigon_model="other"),
        "CSi|s0a180|horizontal|simple": dict(panel="CSi", orientation={"slope": 0.0, "azimuth": 180.0}, tracking="horizontal"),
        "CSi|s30a170|tilted_horizontal|simple": dict(panel="CSi", orientation={"slope": 30.0, "azimuth": 170.0}, tracking="tilted_horizontal"),
        "CSi|s30a180|vertical|simple": dict(panel="CSi", orientation={"slope": 30.0, "azimuth": 180.0}, tracking="vertical"),
        "CdTe|s30a180|dual|simple": dict(panel="CdTe", orientation={"slope": 30.0, "azimuth": 180.0}, tracking="dual"),
        "CSi|s25a200|horizontal|other": dict(panel="CSi", orientation={"slope": 25.0, "azimuth": 200.0}, tracking="horizontal", trigon_model="other"),
        "CSi|s25a200|tilted_horizontal|other": dict(panel="CSi", orientation={"slope": 25.0, "azimuth": 200.0}, tracking="tilted_horizontal", trigon_model="other"),
        "CSi|s25a200|dual|other": dict(panel="CSi", orientation={"slope": 25.0, "azimuth": 200.0}, tracking="dual", trigon_model="other"),
    }
    for name, kw in pv_cases.items():
        run(f"pv|{name}", conv.pv, ds_pv, matrix=m, aggregate_time=None, **kw)
    run("pv|cells", conv.pv, ds_pv, panel="CSi", orientation="latitude_optimal", aggregate_time=None)
    # input variants: total influx + Reindl split, outflux albedo, stored solar position
    infl = F["influx_direct"] + F["influx_diffuse"]
    ds_inf = ref_dataset({"influx_toa": F["influx_toa"], "influx": infl, "albedo": F["albedo"],
                          "temperature": F["temperature"]}, time, x, y)
    run("pv|influx_simple", conv.pv, ds_inf, panel="CSi", orientation="latitude_optimal", matrix=m,
        aggregate_time=None)
    ds_enh = ref_dataset({"influx_toa": F["influx_toa"], "influx": infl, "albedo": F["albedo"],
                          "temperature": F["temperature"], "humidity": F["humidity"]}, time, x, y)
    run("pv|influx_enhanced", conv.pv, ds_enh, panel="CSi", orientation="latitude_optimal", matrix=m,
        aggregate_time=None)
    outflux = infl * F["albedo"]
    out["in_outflux"] = outflux
    ds_out = ref_dataset({"influx_toa": F["influx_toa"], "influx_direct": F["influx_direct"],
                          "influx_diffuse": F["influx_diffuse"], "outflux": outflux,
                          "temperature": F["temperature"]}, time, x, y)
    run("pv|outflux", conv.pv, ds_out, panel="CSi", orientation="latitude_optimal", matrix=m,
        aggregate_time=None)
    sp_ = RefSolarPosition(ds_pv)
    out["solar_altitude"], out["solar_azimuth"] = sp_["altitude"].values, sp_["azimuth"].values
    ds_st = ref_dataset({**{k: F[k] for k in pv_names}, "solar_altitude": sp_["altitude"].values,
                         "solar_azimuth": sp_["azimuth"].values}, time, x, y)
    run("pv|stored_solar", conv.pv, ds_st, panel="CSi", orientation="latitude_optimal", matrix=m,
        aggregate_time=None)

    # ---- heat demand (convert.py:405-471)
    for hs in (0.0, 4.0, -5.0):
        run(f"heat|{hs}", conv.heat_demand, ds_t, threshold=17.0, a=1.3, constant=0.2, hour_shift=hs,
            matrix=m, aggregate_time=None)
    run("heat|cells", conv.heat_demand, ds_t, aggregate_time=None)

    # ---- next-row converters on the same path (SURVEY section 8 f3)
    for kind in ("total", "direct", "diffuse", "ground"):
        run(f"irradiation|{kind}|simple", conv.irradiation, ds_pv, orientation="latitude_optimal",
            irradiation=kind, matrix=m, aggregate_time=None)
    run("irradiation|total|other", conv.irradiation, ds_pv, orientation={"slope": 35.0, "azimuth": 160.0},
        irradiation="total", trigon_model="other", matrix=m, aggregate_time=None)
    run("irradiation|diffuse|other", conv.irradiation, ds_pv, orientation={"slope": 35.0, "azimuth": 160.0},
        irradiation="diffuse", trigon_model="other", matrix=m, aggregate_time=None)
    run("irradiation|total|horizontal", conv.irradiation, ds_pv, orientation={"slope": 0.0, "azimuth": 180.0},
        irradiation="total", tracking="horizontal", matrix=m, aggregate_time=None)
    run("irradiation|cells", conv.irradiation, ds_pv, orientation="latitude_optimal", aggregate_time=None)
    run("solar_thermal|default", conv.solar_thermal, ds_pv, matrix=m, aggregate_time=None)
    run("solar_thermal|latopt_c", conv.solar_thermal, ds_pv, orientation="latitude_optimal", c0=0.7, c1=2.5,
        t_store=60.0, matrix=m, aggregate_time=None)
    ds_tmp = ref_dataset({k: F[k] for k in ("temperature", "soil temperature", "dewpoint temperature")}, time, x, y)
    run("temperature", conv.temperature, ds_tmp, matrix=m, aggregate_time=None)
    run("soil_temperature", conv.soil_temperature, ds_tmp, matrix=m, aggregate_time=None)
    run("dewpoint_temperature", conv.dewpoint_temperature, ds_tmp, matrix=m, aggregate_time=None)
    run("temperature|cells_mean", conv.temperature, ds_tmp, aggregate_time="mean")
    run("cop|air", conv.coefficient_of_performance, ds_tmp, matrix=m, aggregate_time=None)
    run("cop|soil", conv.coefficient_of_performance, ds_tmp, source="soil", sink_T=45.0, matrix=m,
        aggregate_time=None)
    run("cop|air_custom", conv.coefficient_of_performance, ds_tmp, sink_T=35.0, c0=7.0, c1=-0.1, c2=0.0005,
        matrix=m, aggregate_time=None)
    for hs in (0.0, 3.0):
        run(f"cooling|{hs}", conv.cooling_demand, ds_t, threshold=5.0, a=1.7, constant=0.3, hour_shift=hs,
            matrix=m, aggregate_time=None)
    ds_ro = ref_dataset({"runoff": F["runoff"], "height": F["height"]}, time, x, y)
    run("runoff|height", conv.runoff, ds_ro, matrix=m, aggregate_time=None)
    run("runoff|plain", conv.runoff, ds_ro, weight_with_height=False, matrix=m, aggregate_time=None)

    # ---- CSP (convert.py:940-1024, csp.py:18-58).  The efficiency DataArray is built as
    # resource.py:190-220 does (deg -> rad, % -> p.u.) from the reference's own YAML.
    import yaml

    for inst_name in ("SAM_solar_tower", "SAM_parabolic_trough"):
        cfg = yaml.safe_load(open(f"/root/reference/atlite/resources/cspinstallation/{inst_name}.yaml"))
        df = pd.DataFrame(cfg["efficiency"]).set_index(["altitude", "azimuth"])["value"].unstack("azimuth")
        eff = xr_shim.DataArray(df.values / 1.0e2,
                                {"altitude": np.radians(df.index.values.astype(float)),
                                 "azimuth": np.radians(df.columns.values.astype(float))},
                                ("altitude", "azimuth"))
        inst = {"technology": cfg["technology"], "r_irradiance": cfg["r_irradiance"], "efficiency": eff}
        run(f"csp|{inst_name}", conv.csp, ds_pv, installation=dict(inst), matrix=m, aggregate_time=None)
    run("csp|tower_as_trough", conv.csp, ds_pv, installation=dict(inst, technology="solar tower"), matrix=m,
        aggregate_time=None)
    run("csp|cells", conv.csp, ds_pv, installation=dict(inst), aggregate_time=None)
    run("csp|stored_solar", conv.csp, ds_st, installation=dict(inst, technology="solar tower"), matrix=m,
        aggregate_time=None)

    out["cases"] = np.array(cases)
    path = os.path.join(HERE, "reference_outputs.npz")
    np.savez_compressed(path, **out)
    print(f"{len(cases)} cases -> {path} ({os.path.getsize(path) / 1e3:.0f} kB)")


def nan_cases():
    """NaN handling of the PV chain, from the reference's own source: per-cell convert_pv /
    convert_irradiation outputs with a NaN planted in every input field in turn, at a daytime
    and at a night-time cell (pv/irradiation.py:198-200 NaN-preserving clip, :226 per-term
    fillna(0), :252 mask; pv/solar_panel_model.py:23-36).  -> tests/golden/reference_nan.npz"""
    nx, ny, nt = 9, 6, 30
    base = syn.make_dataset(nx, ny, nt, x0=2.0, y0=35.0, dx=1.0, dy=2.0, start="2013-06-21 00:00",
                            extra=("humidity",))
    x, y, time = base.coords["x"], base.coords["y"], base.coords["time"]
    F = {k: np.array(base.raw(k)) for k in base.keys()}
    pv_names = ["influx_toa", "influx_direct", "influx_diffuse", "albedo", "temperature"]
    day = int(np.argmax(F["influx_toa"][:, 2, 3]))
    night = int(np.argmin(F["influx_toa"][:, 2, 3]))
    assert F["influx_toa"][day, 2, 3] > 500 and F["influx_toa"][night, 2, 3] == 0
    out = {"x": x, "y": y, "time_ns": pd.DatetimeIndex(time).as_unit("ns").asi8, "day": day, "night": night}
    cases = []
    for k, name in enumerate(pv_names):
        f = {n: F[n].copy() for n in pv_names}
        f[name][day, 2, 3] = np.nan        # daytime cell
        f[name][night, 1, 4] = np.nan      # night-time cell (masked: alt < 1 deg)
        f[name][day, 4, k] = np.inf if name != "temperature" else -np.inf
        out[f"in|{name}"] = f[name]
        ds = ref_dataset(f, time, x, y)
        for trigon in ("simple", "other"):
            tag = f"{name}|{trigon}"
            out[f"pv|{tag}"] = values_tb(conv.pv(MockCutout(ds), panel="CSi", orientation="latitude_optimal",
                                                 trigon_model=trigon, aggregate_time=None))
            out[f"pvbof|{tag}"] = values_tb(conv.pv(MockCutout(ds), panel="KANENA", orientation="latitude_optimal",
                                                    trigon_model=trigon, aggregate_time=None))
            for kind in ("total", "direct", "diffuse", "ground"):
                out[f"irr_{kind}|{tag}"] = values_tb(conv.irradiation(
                    MockCutout(ds), orientation="latitude_optimal", irradiation=kind, trigon_model=trigon,
                    aggregate_time=None))
            cases.append(tag)
    # total influx (Reindl split) with NaN influx / humidity
    infl = F["influx_direct"] + F["influx_diffuse"]
    for name in ("influx", "humidity", "influx_toa"):
        f = {"influx_toa": F["influx_toa"].copy(), "influx": infl.copy(), "albedo": F["albedo"].copy(),
             "temperature": F["temperature"].copy(), "humidity": F["humidity"].copy()}
        f[name][day, 2, 3] = np.nan
        f[name][night, 1, 4] = np.nan
        out[f"in_reindl|{name}"] = f[name]
        ds = ref_dataset(f, time, x, y)
        out[f"pv_reindl|{name}"] = values_tb(conv.pv(MockCutout(ds), panel="CSi", orientation="latitude_optimal",
                                                     aggregate_time=None))
    out["in_influx_total"] = infl
    out["in_humidity"] = F["humidity"]
    for n in pv_names:
        out[f"base|{n}"] = F[n]
    out["cases"] = np.array(cases)
    path = os.path.join(HERE, "reference_nan.npz")
    np.savez_compressed(path, **out)
    print(f"{len(cases)} NaN cases -> {path} ({os.path.getsize(path) / 1e3:.0f} kB)")


def era5_cases():
    """The arithmetic of datasets/era5.py AFTER the download (get_data_wind :120-135,
    sanitize_wind :141-146, get_data_influx :163-188, sanitize_influx :195-201) executed from
    the reference's own source: ``retrieve_data`` (the CDS request) and
    ``_rename_and_clean_coords`` (longitude/latitude renaming) are replaced by a stand-in that
    hands over seeded raw fields.  -> tests/golden/reference_era5.npz"""
    era5 = xr_shim.load_reference_era5()
    nx, ny, nt = 11, 7, 30
    rng = np.random.default_rng(21)
    x, y = np.arange(nx) * 1.5 - 9.0, np.arange(ny) * 6.0 - 20.0
    t = pd.date_range("2013-09-21 18:00", periods=nt, freq="h")
    co = dict(time=t, x=x, y=y, lon=x, lat=y)

    def f(lo, hi):
        return rng.uniform(lo, hi, (nt, ny, nx)).astype(np.float32)

    raw = dict(u100=f(-15, 15), v100=f(-15, 15), u10=f(-8, 8), v10=f(-8, 8), fsr=f(-0.05, 2.0),
               ssrd=f(0, 3.0e6), tisr=f(-50, 4.5e6))
    raw["ssr"] = (raw["ssrd"] * rng.uniform(0.6, 1.0, (nt, ny, nx))).astype(np.float32)
    raw["fdir"] = (raw["ssrd"] * rng.uniform(0.0, 1.1, (nt, ny, nx))).astype(np.float32)
    raw["ssrd"][0, 0, :4] = 0.0
    raw["ssr"][0, 1, 2] = np.nan
    raw["fsr"][0, 2, 2] = np.nan
    raw["u100"][0, 0, 0], raw["v100"][0, 0, 0] = 0.0, -3.0
    raw["u100"][0, 0, 1], raw["v100"][0, 0, 1] = -2.0, 0.0
    units = dict(u100="m s**-1", v100="m s**-1", u10="m s**-1", v10="m s**-1", fsr="m",
                 ssrd="J m**-2", ssr="J m**-2", tisr="J m**-2", fdir="J m**-2")
    ds_raw = xr_shim.Dataset({k: xr_shim.DataArray(v, co, ("time", "y", "x"), attrs={"units": units[k]})
                              for k, v in raw.items()}, coords=co)
    era5.retrieve_data = lambda **kw: ds_raw  # noqa: E731  (every get_data_* picks its variables by name)
    era5._rename_and_clean_coords = lambda ds, add_lon_lat=True: ds  # noqa: E731
    out = {"x": x, "y": y, "time_ns": pd.DatetimeIndex(t).as_unit("ns").asi8}
    out.update({f"raw|{k}": v for k, v in raw.items()})
    wind = era5.get_data_wind({})
    for k in ("wnd100m", "wnd_shear_exp", "wnd_azimuth", "roughness"):
        out[f"wind|{k}"] = np.asarray(wind[k].values)
    wind_s = era5.sanitize_wind(wind)
    out["wind_sanitized|roughness"] = np.asarray(wind_s["roughness"].values)
    infl = era5.get_data_influx({})
    for k in ("influx_toa", "influx_direct", "influx_diffuse", "albedo", "solar_altitude", "solar_azimuth"):
        out[f"influx|{k}"] = np.asarray(infl[k].values)
    infl_s = era5.sanitize_influx(infl)
    for k in ("influx_toa", "influx_direct", "influx_diffuse"):
        out[f"influx_sanitized|{k}"] = np.asarray(infl_s[k].values)
    path = os.path.join(HERE, "reference_era5.npz")
    np.savez_compressed(path, **out)
    print(f"era5 derivations -> {path} ({os.path.getsize(path) / 1e3:.0f} kB)")


# Raw ERA5 variables of the edge-value dataset, and the special values planted in each in turn
EDGE_VARS = ("ssrd", "ssr", "tisr", "fdir", "t2m", "u100", "v100", "u10", "v10", "fsr")
EDGE_NEGATIVE = dict(ssrd=-40.0, ssr=-40.0, tisr=-100.0, fdir=-25.0, t2m=-5.0, u100=-7.5, v100=-7.5, u10=-3.0,
                     v10=-3.0, fsr=-0.3)
# power curves that reach the lattice table with 0, 1 and 2 per-cell compares (the cut-out step at
# the last knot, and a cut-in step at the first knot that cannot fold)
EDGE_CURVES = {"lattice0": dict(V=[0.0, 3.0, 5.0, 12.0, 25.0], POW=[0.0, 0.0, 0.6, 2.0, 2.0], P=2.0),
               "lattice1": dict(V=[0.0, 3.0, 5.0, 12.0, 25.0, 25.0], POW=[0.0, 0.0, 0.6, 2.0, 2.0, 0.0], P=2.0),
               "lattice2": dict(V=[3.0, 3.0, 5.0, 12.0, 25.0, 25.0], POW=[0.0, 0.2, 0.6, 2.0, 2.0, 0.0], P=2.0)}
EDGE_WIND = (("hub100", 100, "logarithmic"), ("log80", 80, "logarithmic"), ("power80", 80, "power"),
             ("power120", 120, "power"))


def _savez_reproducible(path, arrays):
    """np.savez_compressed without the wall-clock time stamps of the zip members: the same
    arrays give the same bytes."""
    import zipfile

    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for k, v in arrays.items():
            zi = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            zi.compress_type = zipfile.ZIP_DEFLATED
            with zf.open(zi, "w", force_zip64=True) as fh:
                np.lib.format.write_array(fh, np.asanyarray(v), allow_pickle=False)


def era5_edge_cases():
    """datasets/era5.py's derivations and the conversions that consume them, at the edges of the
    raw inputs, from the reference's own source (as era5_cases): NaN, +inf, -inf, 0, -0 and a
    negative value planted in every raw variable in turn, at a lit and at a dark step, plus calm
    winds, float32-overflowing wind components, zero / negative / NaN roughness and the
    accumulation corner cases of the albedo and the diffuse influx.  The conversions run per cell
    on the sanitized fields and the stored solar position, as a cutout that era5.prepare made
    would convert.  -> tests/golden/reference_era5_edges.npz"""
    era5 = xr_shim.load_reference_era5()
    nx, ny, nt = 21, 5, 16  # odd width: a device cutout pads the rows to 24 or keeps the scalar lanes
    rng = np.random.default_rng(38)
    # no cell's sun altitude within 7e-4 rad of the 0, 1 and 3.75 degree thresholds
    x, y = np.arange(nx) * 0.75 - 6.5, np.arange(ny) * 2.5 + 38.0
    t = pd.date_range("2013-06-21 00:00", periods=nt, freq="h")
    t_lit, t_dark = 12, 1  # sun at 11:30 / 00:30 (the -30 min shift) over 6.5 W .. 8.5 E, 38 .. 48 N
    co = dict(time=t, x=x, y=y, lon=x, lat=y)

    def f(lo, hi):
        return rng.uniform(lo, hi, (nt, ny, nx)).astype(np.float32)

    raw = dict(u100=f(-15, 15), v100=f(-15, 15), u10=f(-8, 8), v10=f(-8, 8), fsr=f(0.0, 1.5),
               ssrd=f(0, 3.0e6), tisr=f(3.2e6, 4.5e6), t2m=f(275, 305))
    raw["ssr"] = (raw["ssrd"] * rng.uniform(0.6, 1.0, (nt, ny, nx))).astype(np.float32)
    raw["fdir"] = (raw["ssrd"] * rng.uniform(0.0, 0.9, (nt, ny, nx))).astype(np.float32)
    raw = {k: raw[k] for k in EDGE_VARS}
    # every raw variable in turn: cell vi * 6 + si of rows 0..2 at the lit and the dark step
    specials = []
    for vi, name in enumerate(EDGE_VARS):
        for si, val in enumerate((np.nan, np.inf, -np.inf, 0.0, -0.0, EDGE_NEGATIVE[name])):
            cy, cx = divmod(vi * 6 + si, nx)
            raw[name][[t_lit, t_dark], cy, cx] = val
            specials.append((name, val, cy, cx))
    # combined cells: row 3 onwards
    combos = [dict(u100=0.0, v100=0.0),                        # calm at 100 m: shear exponent +-inf
              dict(u10=0.0, v10=0.0),                          # calm at 10 m under a moving 100 m wind
              dict(u100=0.0, v100=0.0, u10=0.0, v10=0.0),      # both: log(0 / 0) = NaN
              dict(u100=2.0e19), dict(v100=-3.0e19),           # float32 u**2 overflows
              dict(u100=2.0e19, v100=2.0e19), dict(u10=2.5e19), dict(u100=1.0e19, v100=1.5e19),
              dict(fsr=0.0), dict(fsr=-0.3), dict(fsr=np.nan),
              dict(ssrd=0.0, ssr=5.0e5),                       # albedo: ssrd = 0 with ssr != 0
              dict(ssrd=2.0e6, ssr=2.0e6),                     # albedo exactly 0
              dict(tisr=-3.6e3), dict(fdir=-3.6e3),
              dict(ssrd=1.0e6, fdir=1.5e6),                    # fdir > ssrd: negative diffuse
              dict(ssrd=2.0e6, fdir=2.0e6, tisr=1.0e6)]        # direct above the top of atmosphere
    for k, c in enumerate(combos):
        cy, cx = divmod(3 * nx + k, nx)
        for name, val in c.items():
            raw[name][[t_lit, t_dark], cy, cx] = val
    units = dict(u100="m s**-1", v100="m s**-1", u10="m s**-1", v10="m s**-1", fsr="m", t2m="K",
                 ssrd="J m**-2", ssr="J m**-2", tisr="J m**-2", fdir="J m**-2")
    ds_raw = xr_shim.Dataset({k: xr_shim.DataArray(v, co, ("time", "y", "x"), attrs={"units": units[k]})
                              for k, v in raw.items()}, coords=co)
    era5.retrieve_data = lambda **kw: ds_raw  # noqa: E731
    era5._rename_and_clean_coords = lambda ds, add_lon_lat=True: ds  # noqa: E731
    out = {"x": x, "y": y, "time_ns": pd.DatetimeIndex(t).as_unit("ns").asi8, "t_lit": t_lit, "t_dark": t_dark}
    out.update({f"raw|{k}": v for k, v in raw.items()})
    wind = era5.get_data_wind({})
    for k in ("wnd100m", "wnd_shear_exp", "wnd_azimuth", "roughness"):
        out[f"wind|{k}"] = np.asarray(wind[k].values)
    wind_s = era5.sanitize_wind(wind)
    out["wind_sanitized|roughness"] = np.asarray(wind_s["roughness"].values)
    infl = era5.get_data_influx({})
    for k in ("influx_toa", "influx_direct", "influx_diffuse", "albedo", "solar_altitude", "solar_azimuth"):
        out[f"influx|{k}"] = np.asarray(infl[k].values)
    infl_s = era5.sanitize_influx(infl)
    for k in ("influx_toa", "influx_direct", "influx_diffuse"):
        out[f"influx_sanitized|{k}"] = np.asarray(infl_s[k].values)

    # per-cell conversions of the sanitized fields (what a prepared cutout stores)
    pv_f = {k: out[f"influx_sanitized|{k}"] for k in ("influx_toa", "influx_direct", "influx_diffuse")}
    pv_f.update(albedo=out["influx|albedo"], solar_altitude=out["influx|solar_altitude"],
                solar_azimuth=out["influx|solar_azimuth"], temperature=raw["t2m"])
    ds_pv = ref_dataset(pv_f, t, x, y)
    cut = MockCutout(ds_pv)
    out["pv|CSi|latitude_optimal"] = values_tb(conv.pv(cut, panel="CSi", orientation="latitude_optimal",
                                                      aggregate_time=None))
    out["pv|KANENA|latitude_optimal"] = values_tb(conv.pv(cut, panel="KANENA", orientation="latitude_optimal",
                                                         aggregate_time=None))
    out["pv|CSi|dual|other"] = values_tb(conv.pv(cut, panel="CSi", orientation="latitude_optimal", tracking="dual",
                                                 trigon_model="other", aggregate_time=None))
    for kind in ("direct", "total"):
        out[f"irradiation|{kind}"] = values_tb(conv.irradiation(cut, orientation="latitude_optimal", irradiation=kind,
                                                               aggregate_time=None))
    out["solar_thermal"] = values_tb(conv.solar_thermal(cut, aggregate_time=None))
    ds_wind = ref_dataset({"wnd100m": out["wind|wnd100m"], "wnd_shear_exp": out["wind|wnd_shear_exp"],
                           "roughness": out["wind_sanitized|roughness"]}, t, x, y)
    turbines = {"Vestas_V112_3MW": "Vestas_V112_3MW"}
    for name, c in EDGE_CURVES.items():
        turbines[name] = dict(c, V=np.array(c["V"]), POW=np.array(c["POW"]), hub_height=100)
        out[f"curve|{name}|V"], out[f"curve|{name}|POW"] = turbines[name]["V"], turbines[name]["POW"]
    for tname, turb in turbines.items():
        for tag, hub, method in EDGE_WIND:
            tt = (dict(ref_resource.get_windturbineconfig(turb), hub_height=hub) if isinstance(turb, str)
                  else dict(turb, hub_height=hub))
            out[f"wind|{tname}|{tag}"] = values_tb(conv.wind(MockCutout(ds_wind), turbine=tt,
                                                             interpolation_method=method, aggregate_time=None))
    out["specials"] = np.array([f"{n}|{v!r}|{cy}|{cx}" for n, v, cy, cx in specials])
    path = os.path.join(HERE, "reference_era5_edges.npz")
    _savez_reproducible(path, out)
    print(f"era5 edge values -> {path} ({os.path.getsize(path) / 1e3:.0f} kB)")


if __name__ == "__main__":
    # `make_golden.py era5_edges` writes only reference_era5_edges.npz
    if sys.argv[1:] == ["era5_edges"]:
        era5_edge_cases()
    else:
        main()
        era5_cases()
        nan_cases()
        era5_edge_cases()
