"""
CPU ORACLE for the atlite convert+aggregate hot path  --  TEST INFRASTRUCTURE ONLY.

This module is a line-by-line NumPy restatement of the reference's algorithm
for ``Cutout.convert_and_aggregate`` and the pv / wind / heat_demand physics
it calls.  It is *not* part of the product: only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl
reference`` leg may import it, and only as the checker / CPU baseline.  The
product path (``atlite_b200``) never imports it and fails loudly if the CUDA
library is missing.

Pinning status: PINNED against the reference's own source executed in the build
container.  The reference's tests hold no numeric golden vectors for this path
(SURVEY.md section 8c) and ``import atlite`` is impossible here (xarray / dask /
geopandas are not installed, no network), so ``tests/golden/make_golden.py``
loads the reference's hot-path modules from their files under a minimal
xarray/dask container stand-in (``tests/golden/xr_shim.py``), runs 32 cases and
stores inputs + outputs in ``tests/golden/reference_outputs.npz``;
``tests/test_oracle_vs_reference.py`` holds this oracle to them at 1e-9
relative.  Not pinned against genuine xarray/dask objects (see DESIGN.md section 4).

Conventions (same as the reference):
  * ``ds`` is a mapping name -> ndarray.  Fields are ``(time, y, x)``
    (usually float32), plus ``ds["time"]`` (pandas.DatetimeIndex),
    ``ds["lon"]`` (nx,) and ``ds["lat"]`` (ny,) in degrees.
  * dtype promotion is left to NumPy exactly as xarray would leave it
    (python scalars are weak, float32 fields stay float32 until they meet a
    float64 array), so float32 roundings happen where the reference has them.
  * xarray idioms are emulated explicitly: ``.where(c)`` -> NaN fill,
    ``.fillna(v)``, ``.clip``; comparisons with NaN are False.

Every function cites the reference file:line it follows
(paths relative to atlite/).
"""

from __future__ import annotations

import numpy as np
import pandas as pd
import scipy.sparse as sp

pi = np.pi

# --------------------------------------------------------------------------
# xarray-semantics helpers
# --------------------------------------------------------------------------


def _where(a, cond, other=np.nan):
    """xarray ``a.where(cond, other)``: keep ``a`` where cond else ``other``."""
    return np.where(cond, a, other)


def _fillna(a, value):
    a = np.asarray(a)
    return np.where(np.isnan(a), value, a)


def _T(v):
    """(time,) -> (time,1,1)"""
    return np.asarray(v)[:, None, None]


def _Y(v):
    """(y,) -> (1,y,1); scalars pass through."""
    v = np.asarray(v)
    return v[None, :, None] if v.ndim == 1 else v


def _X(v):
    v = np.asarray(v)
    return v[None, None, :] if v.ndim == 1 else v


# --------------------------------------------------------------------------
# pv/solar_position.py
# --------------------------------------------------------------------------


def solar_position(ds, time_shift="0h"):
    """pv/solar_position.py:13-121.  Returns dict(altitude, azimuth) (T,ny,nx) f64,
    or the stored variables in getter mode (54-60)."""
    if "solar_azimuth" in ds and "solar_altitude" in ds:  # :54-60
        return {"altitude": ds["solar_altitude"], "azimuth": ds["solar_azimuth"]}

    time_shift = pd.to_timedelta(time_shift)  # :71
    t = pd.DatetimeIndex(ds["time"]) + time_shift  # :73
    n = np.asarray(t.to_julian_date(), dtype=np.float64) - 2451545.0  # :74
    hour = np.asarray(t.hour)  # :75
    minute = np.asarray(t.minute)  # :76

    L = 280.460 + 0.9856474 * n  # :86
    g = np.radians(357.528 + 0.9856003 * n)  # :87
    l = np.radians(L + 1.915 * np.sin(g) + 0.020 * np.sin(2 * g))  # :88
    ep = np.radians(23.439 - 4e-7 * n)  # :89

    ra = np.arctan2(np.cos(ep) * np.sin(l), np.cos(l))  # :91
    lmst = _T((6.697375 + (hour + minute / 60.0) + 0.0657098242 * n) * 15.0) + _X(
        np.asarray(ds["lon"], dtype=np.float64)
    )  # :92-94
    h = (np.radians(lmst) - _T(ra) + pi) % (2 * pi) - pi  # :95

    dec = _T(np.arcsin(np.sin(ep) * np.sin(l)))  # :97

    lat = _Y(np.radians(np.asarray(ds["lat"], dtype=np.float64)))  # :100
    alt = np.arcsin(
        np.clip(
            np.sin(dec) * np.sin(lat) + np.cos(dec) * np.cos(lat) * np.cos(h),
            -1.0,
            1.0,
        )
    )  # :103-105
    with np.errstate(divide="ignore", invalid="ignore"):
        az = np.arccos(
            np.clip(
                (np.sin(dec) * np.cos(lat) - np.cos(dec) * np.sin(lat) * np.cos(h))
                / np.cos(alt),
                -1.0,
                1.0,
            )
        )  # :109-113
    az = np.where(h <= 0, az, 2 * pi - az)  # :114
    return {"altitude": alt, "azimuth": az}


# --------------------------------------------------------------------------
# pv/orientation.py
# --------------------------------------------------------------------------


def make_latitude_optimal():
    """pv/orientation.py:26-69 (note ``+ radians(0.31)``, sic)."""

    def latitude_optimal(lon, lat, solar_position):
        lat = np.asarray(lat, dtype=np.float64)
        slope = np.empty_like(lat)
        below_25 = np.abs(lat) <= np.radians(25)
        below_50 = np.abs(lat) <= np.radians(50)
        slope[below_25] = 0.87 * np.abs(lat[below_25])
        slope[~below_25 & below_50] = 0.76 * np.abs(
            lat[~below_25 & below_50]
        ) + np.radians(0.31)
        slope[~below_50] = np.radians(40.0)
        azimuth = np.where(lat < 0, 0, pi)
        return dict(slope=slope, azimuth=azimuth)

    return latitude_optimal


def make_constant(slope, azimuth):
    """pv/orientation.py:72-79"""
    slope = np.radians(slope)
    azimuth = np.radians(azimuth)

    def constant(lon, lat, solar_position):
        return dict(slope=slope, azimuth=azimuth)

    return constant


def make_latitude(azimuth=180):
    """pv/orientation.py:82-88"""
    azimuth = np.radians(azimuth)

    def latitude(lon, lat, solar_position):
        return dict(slope=np.asarray(lat, dtype=np.float64), azimuth=azimuth)

    return latitude


def get_orientation(name, **params):
    """pv/orientation.py:13-23"""
    if isinstance(name, dict):
        params = dict(name)
        name = params.pop("name", "constant")
    return {
        "latitude_optimal": make_latitude_optimal,
        "constant": make_constant,
        "latitude": make_latitude,
    }[name](**params)


def surface_orientation(ds, solar_pos, orientation, tracking=None):
    """pv/orientation.py:91-196.  Returns dict(cosincidence, slope, azimuth)."""
    lon = np.radians(np.asarray(ds["lon"], dtype=np.float64))  # :104
    lat = np.radians(np.asarray(ds["lat"], dtype=np.float64))  # :105

    o = orientation(lon, lat, solar_pos)  # :107
    surface_slope = _Y(o["slope"])  # :108
    surface_azimuth = _Y(o["azimuth"])  # :109

    sun_altitude = solar_pos["altitude"]
    sun_azimuth = solar_pos["azimuth"]
    sin, cos = np.sin, np.cos

    with np.errstate(divide="ignore", invalid="ignore"):
        if tracking is None:  # :114-117
            cosincidence = sin(surface_slope) * cos(sun_altitude) * cos(
                surface_azimuth - sun_azimuth
            ) + cos(surface_slope) * sin(sun_altitude)
        elif tracking == "horizontal":  # :119-131
            axis_azimuth = surface_azimuth
            rotation = np.arctan(
                (cos(sun_altitude) / sin(sun_altitude))
                * sin(sun_azimuth - axis_azimuth)
            )
            surface_slope = abs(rotation)
            surface_azimuth = axis_azimuth + np.arcsin(
                sin(rotation) / sin(surface_slope)
            )
            cosincidence = cos(surface_slope) * sin(sun_altitude) + sin(
                surface_slope
            ) * cos(sun_altitude) * cos(sun_azimuth - surface_azimuth)
        elif tracking == "tilted_horizontal":  # :133-169
            axis_tilt = surface_slope
            rotation = np.arctan(
                (cos(sun_altitude) * sin(sun_azimuth - surface_azimuth))
                / (
                    cos(sun_altitude)
                    * cos(sun_azimuth - surface_azimuth)
                    * sin(axis_tilt)
                    + sin(sun_altitude) * cos(axis_tilt)
                )
            )
            surface_slope = np.arccos(cos(rotation) * cos(axis_tilt))
            azimuth_difference = sun_azimuth - surface_azimuth
            azimuth_difference = np.where(
                azimuth_difference > pi, azimuth_difference - 2 * pi, azimuth_difference
            )
            azimuth_difference = np.where(
                azimuth_difference < -pi,
                2 * pi + azimuth_difference,
                azimuth_difference,
            )
            rotation = np.where(
                np.logical_and(rotation < 0, azimuth_difference > 0),
                rotation + pi,
                rotation,
            )
            rotation = np.where(
                np.logical_and(rotation > 0, azimuth_difference < 0),
                rotation - pi,
                rotation,
            )
            cosincidence = cos(rotation) * (
                sin(axis_tilt) * cos(sun_altitude) * cos(sun_azimuth - surface_azimuth)
                + cos(axis_tilt) * sin(sun_altitude)
            ) + sin(rotation) * cos(sun_altitude) * sin(sun_azimuth - surface_azimuth)
        elif tracking == "vertical":  # :171-174
            cosincidence = sin(surface_slope) * cos(sun_altitude) + cos(
                surface_slope
            ) * sin(sun_altitude)
        elif tracking == "dual":  # :175-176
            cosincidence = np.float64(1.0)
        else:
            raise AssertionError("unknown tracking " + repr(tracking))

    # xarray .clip(min=0) keeps NaN  (:188)
    cosincidence = np.where(np.isnan(cosincidence), np.nan, np.maximum(cosincidence, 0))
    return {
        "cosincidence": cosincidence,
        "slope": surface_slope,
        "azimuth": surface_azimuth,
    }


# --------------------------------------------------------------------------
# pv/irradiation.py
# --------------------------------------------------------------------------


def _clip(influx, influx_max):
    """pv/irradiation.py:198-200  influx.clip(min=0, max=influx_max)"""
    return np.minimum(np.maximum(influx, 0), influx_max)


def diffuse_horizontal_irrad(ds, solar_pos, clearsky_model, influx):
    """pv/irradiation.py:13-73 (Reindl 1990)."""
    sinaltitude = np.sin(solar_pos["altitude"])
    influx_toa = ds["influx_toa"]
    if clearsky_model is None:  # :21-24
        clearsky_model = (
            "enhanced" if "temperature" in ds and "humidity" in ds else "simple"
        )
    with np.errstate(divide="ignore", invalid="ignore"):
        k = influx / influx_toa  # :28
    fmin, fmax = np.fmin, np.fmax  # dask.array.fmin/fmax: NaN-ignoring
    if clearsky_model == "simple":  # :33-42
        fraction = (
            ((k > 0.0) & (k <= 0.3))
            * fmin(1.0, 1.020 - 0.254 * k + 0.0123 * sinaltitude)
            + ((k > 0.3) & (k < 0.78))
            * fmin(0.97, fmax(0.1, 1.400 - 1.749 * k + 0.177 * sinaltitude))
            + (k >= 0.78) * fmax(0.1, 0.486 * k - 0.182 * sinaltitude)
        )
    elif clearsky_model == "enhanced":  # :43-65
        T = ds["temperature"]
        rh = ds["humidity"]
        fraction = (
            ((k > 0.0) & (k <= 0.3))
            * fmin(
                1.0,
                1.000 - 0.232 * k + 0.0239 * sinaltitude - 0.000682 * T + 0.0195 * rh,
            )
            + ((k > 0.3) & (k < 0.78))
            * fmin(
                0.97,
                fmax(
                    0.1,
                    1.329 - 1.716 * k + 0.267 * sinaltitude - 0.00357 * T + 0.106 * rh,
                ),
            )
            + (k >= 0.78)
            * fmax(0.1, 0.426 * k - 0.256 * sinaltitude + 0.00349 * T + 0.0734 * rh)
        )
    else:
        raise KeyError("`clearsky model` must be chosen from 'simple' and 'enhanced'")
    return influx * fraction  # :73


def _albedo(ds, influx):
    """pv/irradiation.py:128-139"""
    if "albedo" in ds:
        return ds["albedo"]
    elif "outflux" in ds:
        with np.errstate(divide="ignore", invalid="ignore"):
            a = ds["outflux"] / _where(influx, influx != 0)
        a = _fillna(a, 0)
        return np.minimum(a, 1)  # .clip(max=1)
    raise AssertionError(
        "Need either albedo or outflux as a variable in the dataset. "
        "Check your cutout and dataset module."
    )


def tilted_irradiation(
    ds,
    solar_pos,
    surf,
    trigon_model,
    clearsky_model,
    tracking=0,
    altitude_threshold=1.0,
    irradiation="total",
):
    """pv/irradiation.py:148-255."""
    influx_toa = ds["influx_toa"]
    sin, cos = np.sin, np.cos

    if "influx" in ds:  # :202-205
        influx = _clip(ds["influx"], influx_toa)
        diffuse = diffuse_horizontal_irrad(ds, solar_pos, clearsky_model, influx)
        direct = influx - diffuse
    elif "influx_direct" in ds and "influx_diffuse" in ds:  # :206-208
        direct = _clip(ds["influx_direct"], influx_toa)
        diffuse = _clip(ds["influx_diffuse"], influx_toa - direct)
    else:
        raise AssertionError(
            "Need either influx or influx_direct and influx_diffuse in the "
            "dataset. Check your cutout and dataset module."
        )

    with np.errstate(divide="ignore", invalid="ignore"):
        if trigon_model == "simple":  # :214-226
            k = surf["cosincidence"] / sin(solar_pos["altitude"])
            if tracking != "dual":
                cos_surface_slope = cos(surf["slope"])
            else:
                cos_surface_slope = sin(solar_pos["altitude"])
            influx = direct + diffuse
            direct_t = k * direct
            diffuse_t = (1.0 + cos_surface_slope) / 2.0 * diffuse
            ground_t = _albedo(ds, influx) * influx * ((1.0 - cos_surface_slope) / 2.0)
            total_t = _fillna(direct_t, 0.0) + _fillna(diffuse_t, 0.0) + _fillna(
                ground_t, 0.0
            )
        else:  # :227-236 -> Hay-Davies :76-115, :118-125, :142-145
            sinaltitude = sin(solar_pos["altitude"])
            cosincidence = surf["cosincidence"]
            surface_slope = surf["slope"]
            influx = direct + diffuse
            f = _fillna(np.sqrt(direct / influx), 0.0)  # :89
            A = direct / influx_toa  # :92
            R_b = cosincidence / sinaltitude  # :95
            diffuse_t = (
                (1.0 - A)
                * ((1 + cos(surface_slope)) / 2.0)
                * (1.0 + f * sin(surface_slope / 2.0) ** 3)
                + A * R_b
            ) * diffuse  # :97-102
            diffuse_t = _fillna(
                np.where(np.isnan(diffuse_t), np.nan, np.maximum(diffuse_t, 0)), 0
            )  # :112-113
            direct_t = R_b * direct  # :125
            ground_t = influx * _albedo(ds, influx) * (1.0 - cos(surface_slope)) / 2.0
            total_t = direct_t + diffuse_t + ground_t  # :236

    result = {
        "total": total_t,
        "direct": direct_t,
        "diffuse": diffuse_t,
        "ground": ground_t,
    }[irradiation]  # :238-245

    cap_alt = solar_pos["altitude"] < np.radians(altitude_threshold)  # :251
    result = np.where(~(cap_alt | (direct + diffuse <= 0.01)), result, 0)  # :252
    return result


# --------------------------------------------------------------------------
# pv/solar_panel_model.py
# --------------------------------------------------------------------------


def _power_huld(irradiance, t_amb, pc):
    """pv/solar_panel_model.py:12-44"""
    T_ = (pc["c_temp_amb"] * t_amb + pc["c_temp_irrad"] * irradiance) - pc["r_tmod"]
    G_ = irradiance / pc["r_irradiance"]
    with np.errstate(divide="ignore", invalid="ignore"):
        log_G_ = np.log(_where(G_, G_ > 0))
    eff = (
        1
        + pc["k_1"] * log_G_
        + pc["k_2"] * (log_G_) ** 2
        + T_ * (pc["k_3"] + pc["k_4"] * log_G_ + pc["k_5"] * log_G_**2)
        + pc["k_6"] * (T_**2)
    )
    eff = np.maximum(_fillna(eff, 0.0), 0)
    return G_ * eff * pc.get("inverter_efficiency", 1.0)


def _power_bofinger(irradiance, t_amb, pc):
    """pv/solar_panel_model.py:47-74"""
    fraction = (pc["NOCT"] - pc["Tamb"]) / pc["Intc"]
    with np.errstate(divide="ignore", invalid="ignore"):
        eta_ref = (
            pc["A"]
            + pc["B"] * irradiance
            + pc["C"] * np.log(_where(irradiance, irradiance != 0))
        )
        eta = _fillna(
            eta_ref
            * (1.0 + pc["D"] * (fraction * irradiance + (t_amb - pc["Tstd"])))
            / (1.0 + pc["D"] * fraction / pc["ta"] * eta_ref * irradiance),
            0,
        )
    capacity = (pc["A"] + pc["B"] * 1000.0 + pc["C"] * np.log(1000.0)) * 1e3
    power = irradiance * eta * (pc.get("inverter_efficiency", 1.0) / capacity)
    return np.where(irradiance >= pc["threshold"], power, 0)


def solar_panel_model(ds, irradiance, pc):
    """pv/solar_panel_model.py:77-85"""
    model = pc.get("model", "huld")
    if model == "huld":
        return _power_huld(irradiance, ds["temperature"], pc)
    elif model == "bofinger":
        return _power_bofinger(irradiance, ds["temperature"], pc)
    raise AssertionError(f"Unknown panel model: {model}")


def convert_pv(
    ds, panel, orientation, tracking=None, trigon_model="simple", clearsky_model="simple"
):
    """convert.py:840-854"""
    sp_ = solar_position(ds)
    surf = surface_orientation(ds, sp_, orientation, tracking)
    irr = tilted_irradiation(
        ds,
        sp_,
        surf,
        trigon_model=trigon_model,
        clearsky_model=clearsky_model,
        tracking=tracking,
    )
    return solar_panel_model(ds, irr, panel)


def convert_irradiation(ds, orientation, tracking=None, irradiation="total",
                        trigon_model="simple", clearsky_model="simple"):
    """convert.py:748-767"""
    sp_ = solar_position(ds)
    surf = surface_orientation(ds, sp_, orientation, tracking)
    return tilted_irradiation(ds, sp_, surf, trigon_model=trigon_model,
                              clearsky_model=clearsky_model, tracking=tracking,
                              irradiation=irradiation)


def convert_solar_thermal(ds, orientation, trigon_model, clearsky_model, c0, c1, t_store):
    """convert.py:550-573"""
    t_store = t_store + 273.15
    sp_ = solar_position(ds)
    surf = surface_orientation(ds, sp_, orientation)
    irr = tilted_irradiation(ds, sp_, surf, trigon_model, clearsky_model)
    with np.errstate(divide="ignore", invalid="ignore"):
        eta = c0 - c1 * _fillna((t_store - ds["temperature"]) / _where(irr, irr != 0), 0)
    output = irr * eta
    return np.where(output > 0.0, output, 0.0)


# --------------------------------------------------------------------------
# convert.py:292-401 temperature family, COP; 475-546 cooling demand; 1028-1034 runoff
# --------------------------------------------------------------------------


def convert_temperature(ds):
    """convert.py:292-298"""
    return ds["temperature"] - 273.15


def convert_soil_temperature(ds):
    """convert.py:306-316 (NaN over sea -> 0 so it does not contribute)"""
    return _fillna(ds["soil temperature"] - 273.15, 0.0)


def convert_dewpoint_temperature(ds):
    """convert.py:324-329"""
    return ds["dewpoint temperature"] - 273.15


def convert_coefficient_of_performance(ds, source, sink_T, c0, c1, c2):
    """convert.py:338-366"""
    assert source in ["air", "soil"]
    if source == "air":
        source_T = convert_temperature(ds)
        c0 = 6.81 if c0 is None else c0
        c1 = -0.121 if c1 is None else c1
        c2 = 0.000630 if c2 is None else c2
    else:
        source_T = convert_soil_temperature(ds)
        c0 = 8.77 if c0 is None else c0
        c1 = -0.150 if c1 is None else c1
        c2 = 0.000734 if c2 is None else c2
    delta_T = sink_T - source_T
    return c0 + c1 * delta_T + c2 * delta_T**2


def convert_cooling_demand(ds, threshold, a, constant, hour_shift):
    """convert.py:475-491.  Returns (values (days,ny,nx), day labels)."""
    T = ds["temperature"]
    labels, gid = day_bins(ds["time"], hour_shift)
    nd = len(labels)
    out = np.full((nd,) + T.shape[1:], np.nan, dtype=T.dtype)
    for d in range(nd):
        sel = T[gid == d]
        if sel.shape[0]:
            with np.errstate(invalid="ignore"):
                out[d] = np.nanmean(sel, axis=0)
    threshold = threshold + 273.15
    cool = a * (out - threshold)
    cool = np.where(np.isnan(cool), np.nan, np.maximum(cool, 0.0))
    return constant + cool, labels


def calculate_dni(ds, solar_pos, altitude_threshold=3.75):
    """csp.py:18-58"""
    thr = np.radians(altitude_threshold)
    altitude = solar_pos["altitude"]
    altitude = _where(altitude, altitude > 0, np.nan)
    altitude = _where(altitude, altitude > thr, thr)  # NaN > thr is False -> thr (sic, as the reference)
    with np.errstate(divide="ignore", invalid="ignore"):
        return ds["influx_direct"] / np.sin(altitude)


def convert_csp(ds, installation):
    """convert.py:940-972.  ``installation["efficiency"]``: object with .altitude, .azimuth (rad,
    ascending) and .values (p.u.); interpolation as xarray's DataArray.interp, i.e.
    scipy.interpolate.interpn(method="linear", bounds_error=False, fill_value=nan)."""
    from scipy.interpolate import interpn

    sp_ = solar_position(ds)
    tech = installation["technology"]
    if tech == "parabolic trough":
        irradiation = ds["influx_direct"]
    elif tech == "solar tower":
        irradiation = calculate_dni(ds, sp_)
    else:
        raise ValueError(f'Unknown CSP technology option "{tech}".')
    eff = installation["efficiency"]
    alt, az = np.broadcast_arrays(sp_["altitude"], sp_["azimuth"])
    xi = np.stack([np.asarray(alt, dtype=np.float64).ravel(), np.asarray(az, dtype=np.float64).ravel()], axis=-1)
    efficiency = interpn((np.asarray(eff.altitude, float), np.asarray(eff.azimuth, float)),
                         np.asarray(eff.values, float), xi, method="linear", bounds_error=False,
                         fill_value=np.nan).reshape(alt.shape)
    da = efficiency * irradiation
    da = da / installation["r_irradiance"]
    da = np.where(np.isnan(da), np.nan, np.minimum(da, 1.0))  # .clip(max=1.0)
    return _fillna(da, 0.0)


def convert_runoff(ds, weight_with_height=True):
    """convert.py:1028-1034"""
    runoff = ds["runoff"]
    if weight_with_height:
        runoff = runoff * ds["height"]
    return runoff


# --------------------------------------------------------------------------
# wind.py + convert.py:634-662
# --------------------------------------------------------------------------


def extrapolate_wind_speed(ds, to_height, from_height=None, method="logarithmic"):
    """wind.py:24-128"""
    import re

    to_name = f"wnd{int(to_height):0d}m"
    if to_name in ds:  # :75-78
        return ds[to_name]
    if from_height is None:  # :80-87
        heights = np.asarray([int(s[3:-1]) for s in ds if re.match(r"wnd\d+m", s)])
        if len(heights) == 0:
            raise AssertionError("Wind speed is not in dataset")
        from_height = heights[np.argmin(np.abs(heights - to_height))]
    from_name = f"wnd{int(from_height):0d}m"
    if method == "logarithmic":  # :91-102
        if "roughness" not in ds:
            raise RuntimeError("The logarithmic interpolation method requires roughness")
        roughness = ds["roughness"]
        with np.errstate(divide="ignore", invalid="ignore"):
            return ds[from_name] * (
                np.log(to_height / roughness) / np.log(from_height / roughness)
            )
    elif method == "power":  # :103-112
        if "wnd_shear_exp" not in ds:
            raise RuntimeError("The power law interpolation method requires wnd_shear_exp")
        return ds[from_name] * (to_height / from_height) ** ds["wnd_shear_exp"]
    raise ValueError(
        f"Interpolation method must be 'logarithmic' or 'power',  but is: {method}"
    )


def convert_wind(ds, turbine, interpolation_method="logarithmic"):
    """convert.py:634-662; np.interp returns float64 and clamps outside the knots."""
    V, POW, hub_height, P = (turbine[k] for k in ("V", "POW", "hub_height", "P"))
    wnd_hub = extrapolate_wind_speed(ds, to_height=hub_height, method=interpolation_method)
    return np.interp(wnd_hub, np.asarray(V, float), np.asarray(POW, float) / P)


# --------------------------------------------------------------------------
# convert.py:405-418 heat demand
# --------------------------------------------------------------------------


def day_bins(time, hour_shift):
    """Calendar-day bins of ``time + hour_shift`` as xarray ``resample(time="1D")``
    makes them (convert.py:408-412): left-closed days from the first to the
    last shifted timestamp.  Returns (labels DatetimeIndex, group id per step)."""
    t = pd.DatetimeIndex(time) + pd.Timedelta(hours=hour_shift)
    days = t.floor("D")
    labels = pd.date_range(days[0], days[-1], freq="D")
    gid = ((days - days[0]) // pd.Timedelta(days=1)).astype(np.int64)
    return labels, np.asarray(gid)


def convert_heat_demand(ds, threshold, a, constant, hour_shift):
    """convert.py:405-418.  Returns (values (days,ny,nx), day labels)."""
    T = ds["temperature"]
    labels, gid = day_bins(ds["time"], hour_shift)
    nd = len(labels)
    out = np.full((nd,) + T.shape[1:], np.nan, dtype=T.dtype)
    for d in range(nd):  # resample(...).mean(): skipna mean over present samples
        sel = T[gid == d]
        if sel.shape[0]:
            with np.errstate(invalid="ignore"):
                out[d] = np.nanmean(sel, axis=0)
    threshold = threshold + 273.15
    heat = a * (threshold - out)
    heat = np.where(np.isnan(heat), np.nan, np.maximum(heat, 0.0))  # .clip(min=0)
    return constant + heat, labels


# --------------------------------------------------------------------------
# resource.py pieces that shape the lookup tables
# --------------------------------------------------------------------------


def validate_turbine(turbine, add_cutout_windspeed):
    """resource.py:304-372 (only the table-shaping part)."""
    turbine = dict(turbine)
    turbine["V"] = np.asarray(turbine["V"], dtype=float)
    turbine["POW"] = np.asarray(turbine["POW"], dtype=float)
    if len(turbine["POW"]) != len(turbine["V"]):
        raise ValueError("turbine wind speed and power arrays do not have equal length.")
    if not np.all(np.diff(turbine["V"]) >= 0):
        raise ValueError("wind speed 'V' ... not in ascending order")
    max_v_zero = np.any(turbine["POW"][turbine["V"] == turbine["V"].max()] == 0)
    if add_cutout_windspeed is True and not max_v_zero:  # :357-363
        turbine["V"] = np.pad(turbine["V"], (0, 1), "maximum")
        turbine["POW"] = np.pad(turbine["POW"], (0, 1), "constant", constant_values=0)
    return turbine


def windturbine_smooth(turbine, params=None):
    """resource.py:227-297"""
    from scipy.signal import fftconvolve

    if params is None or params is True:
        params = {}
    eta = params.get("eta", 0.95)
    Delta_v = params.get("Delta_v", 1.27)
    sigma = params.get("sigma", 2.29)

    def kernel(v_0):
        return (
            1.0
            / np.sqrt(2 * np.pi * sigma * sigma)
            * np.exp(-(v_0 - Delta_v) * (v_0 - Delta_v) / (2 * sigma * sigma))
        )

    velocities_reg = np.linspace(-50.0, 50.0, 1001)
    power_reg = np.interp(velocities_reg, turbine["V"], turbine["POW"])
    kernel_reg = kernel(velocities_reg)
    convolution = 0.1 * fftconvolve(power_reg, kernel_reg, mode="same")
    velocities_new = np.linspace(0.0, 35.0, 72)
    power_new = eta * np.interp(velocities_new, velocities_reg, convolution)
    turbine = dict(turbine)
    turbine["V"], turbine["POW"] = velocities_new, power_new
    turbine["P"] = np.max(power_new)
    return turbine


# --------------------------------------------------------------------------
# aggregate.py + convert.py:59-276 orchestration
# --------------------------------------------------------------------------


def aggregate_matrix(da, matrix):
    """aggregate.py:16-35, dask branch: block(T,S) * matrix.T -> (T, n_bus) float64."""
    T = da.shape[0]
    flat = np.asarray(da).reshape(T, -1)
    return np.asarray(flat @ matrix.T) if not sp.issparse(matrix) else (matrix @ flat.T).T


def _aggregate_time(res, method, axis=0):
    """convert.py:51-56"""
    if method == "sum":
        return res.sum(axis=axis)
    elif method == "mean":
        return res.mean(axis=axis)
    return res


def convert_and_aggregate(
    ds,
    convert_func,
    matrix=None,
    layout=None,
    per_unit=False,
    return_capacity=False,
    aggregate_time="legacy",
    chunk=None,
    **convert_kwds,
):
    """convert.py:59-276 on plain arrays.

    ``matrix``: (n_bus, S) scipy sparse / ndarray; ``layout``: (ny, nx) ndarray.
    Returns ndarray: (time, n_bus) [dask-branch dim order], (n_bus,) after time
    aggregation, (time, ny, nx) / (ny, nx) without spatial aggregation; with
    ``return_capacity`` a tuple (result, capacity).
    ``chunk``: evaluate the physics in time slabs of that many steps (like the
    reference's dask ``{"time": 100}`` chunks) to bound memory.
    """
    if aggregate_time not in ("sum", "mean", "legacy", None):  # :160-164
        raise ValueError("aggregate_time must be 'sum', 'mean', 'legacy', or None")

    def _convert(sl):
        sub = {
            k: (v[sl] if (k == "time" or (hasattr(v, "ndim") and v.ndim == 3)) else v)
            for k, v in ds.items()
        }
        r = convert_func(sub, **convert_kwds)
        return r[0] if isinstance(r, tuple) else r

    nt = len(ds["time"])
    if chunk is None or convert_func in (convert_heat_demand, convert_cooling_demand):
        slabs = [slice(0, nt)]
    else:
        slabs = [slice(i, min(i + chunk, nt)) for i in range(0, nt, chunk)]

    no_args = matrix is None and layout is None
    if no_args:  # :200-211
        if per_unit or return_capacity:
            raise ValueError(
                "One of `matrix`, `shapes` and `layout` must be given for `per_unit` or `return_capacity`"
            )
        agg = "sum" if aggregate_time == "legacy" else aggregate_time
        da = np.concatenate([_convert(s) for s in slabs], axis=0)
        return _aggregate_time(da, agg)

    if matrix is not None:  # :213-233
        if np.ndim(matrix) != 2 and not sp.issparse(matrix):
            raise ValueError("Matrix not 2-dimensional.")
        matrix = sp.csr_matrix(matrix)
    if layout is not None:  # :242-249
        lay = np.asarray(layout, dtype=np.float64).reshape(-1)
        if matrix is None:
            matrix = sp.csr_matrix(lay[None, :])
        else:
            matrix = sp.csr_matrix(matrix) * sp.diags(lay).tocsr()
    matrix = sp.csr_matrix(matrix, dtype=np.float64)

    results = np.concatenate(
        [aggregate_matrix(_convert(s), matrix) for s in slabs], axis=0
    )  # :257

    if per_unit or return_capacity:  # :259-262
        capacity = np.asarray(matrix.sum(-1)).flatten()
    if per_unit:  # :264-266
        with np.errstate(divide="ignore", invalid="ignore"):
            results = _fillna(results / _where(capacity, capacity != 0)[None, :], 0.0)
    if aggregate_time != "legacy":  # :270-271
        results = _aggregate_time(results, aggregate_time)
    if return_capacity:
        return results, capacity
    return results
