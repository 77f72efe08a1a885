"""
Float64 restatement of the graded converters in torch  --  TEST INFRASTRUCTURE ONLY.

``atlite_oracle`` is the reference semantics, but NumPy on the CPU cannot evaluate the
graded year (1440 x 720 x 8760 cell-steps) in test time.  This module restates, operation
for operation, the parts of ``atlite_oracle`` the graded configurations use, in torch, so
that the same arithmetic runs on the GPU next to the kernels it checks:

  * ``solar_position``: Michalsky, with ``time_shift``;
  * ``pv``: ERA5 branch (influx_direct / influx_diffuse / influx_toa / albedo / temperature),
    no tracking, ``trigon_model="simple"``, the Huld panel, latitude_optimal or constant
    orientation;
  * ``wind``: log law from 100 m with roughness (or the 100 m fast lane), then ``np.interp``
    on the power curve;
  * ``heat_demand``: daily means over ``atlite_oracle.day_bins`` with ``hour_shift``, clip and
    constant.

It shares no code with the package (which must never import it) and keeps the oracle's dtypes:
under NumPy 2 a Python scalar times a float32 array stays float32, and torch promotes the same
way, so float32 roundings happen where the oracle has them.  tests/test_north_star_year.py pins
it to ``atlite_oracle`` at 1e-12.

Every converter works on slabs ``(t, ny, nx)`` on any device and returns ``(values,
allowance)``.  The allowance is the largest change a float32 decision can make to a cell at a
discontinuity of the float64 reference (0 where there is none):

  * PV: |the value without the altitude mask| where the float64 altitude lies within
    ``PV_ALTITUDE_WINDOW`` of the 1 degree threshold (about ten times the float32 error of a
    kernel's sin(altitude));
  * wind: |jump| where the hub speed lies within ``WIND_KNOT_WINDOW`` (relative) of a knot at
    which the power curve jumps (the cut-out);
  * heat: none, the clip is continuous.
"""

from __future__ import annotations

import math

import numpy as np
import pandas as pd
import torch

from atlite_oracle import day_bins

f64 = torch.float64
PV_ALTITUDE_WINDOW = 2e-6  # rad
WIND_KNOT_WINDOW = 1e-5  # relative to the knot


def _np_remainder(a, b):
    """NumPy's float ``%`` (npy_divmod): the exact fmod, moved into the divisor's sign."""
    m = torch.fmod(a, b)
    return torch.where((m != 0) & ((m < 0) != (b < 0)), m + b, m)


def solar_position(time, lon, lat, device, time_shift="0h"):
    """atlite_oracle.solar_position: dict(altitude, azimuth), float64 ``(t, ny, nx)``.
    ``lon`` / ``lat``: the grid's coordinates in degrees."""
    t = pd.DatetimeIndex(time) + pd.to_timedelta(time_shift)
    n = torch.as_tensor(np.asarray(t.to_julian_date(), dtype=np.float64) - 2451545.0, device=device)
    hour = torch.as_tensor(np.asarray(t.hour), dtype=f64, device=device)
    minute = torch.as_tensor(np.asarray(t.minute), dtype=f64, device=device)

    L = 280.460 + 0.9856474 * n
    g = torch.deg2rad(357.528 + 0.9856003 * n)
    l = torch.deg2rad(L + 1.915 * torch.sin(g) + 0.020 * torch.sin(2 * g))
    ep = torch.deg2rad(23.439 - 4e-7 * n)

    ra = torch.atan2(torch.cos(ep) * torch.sin(l), torch.cos(l))
    lon = torch.as_tensor(np.asarray(lon, dtype=np.float64), device=device)
    lmst = ((6.697375 + (hour + minute / 60.0) + 0.0657098242 * n) * 15.0)[:, None, None] + lon[None, None, :]
    h = _np_remainder(torch.deg2rad(lmst) - ra[:, None, None] + math.pi, 2 * math.pi) - math.pi

    dec = torch.asin(torch.sin(ep) * torch.sin(l))[:, None, None]

    lat = torch.deg2rad(torch.as_tensor(np.asarray(lat, dtype=np.float64), device=device))[None, :, None]
    alt = torch.asin(torch.clamp(torch.sin(dec) * torch.sin(lat) + torch.cos(dec) * torch.cos(lat) * torch.cos(h),
                                 -1.0, 1.0))
    az = torch.acos(torch.clamp((torch.sin(dec) * torch.cos(lat) - torch.cos(dec) * torch.sin(lat) * torch.cos(h))
                                / torch.cos(alt), -1.0, 1.0))
    az = torch.where(h <= 0, az, 2 * math.pi - az)
    return {"altitude": alt, "azimuth": az}


def orientation_table(orientation, lat, device):
    """The panel's (slope, azimuth) in radians, float64: per row ``(1, ny, 1)`` for
    ``"latitude_optimal"`` (atlite_oracle.make_latitude_optimal), ``(1, 1, 1)`` for
    ``{"slope": deg, "azimuth": deg}`` (make_constant)."""
    if isinstance(orientation, dict):  # NumPy float64 scalars, which promote float32 arrays to float64:
        # one-element tensors do too (a 0-d tensor would not)
        return tuple(torch.full((1, 1, 1), math.radians(orientation[k]), dtype=f64, device=device)
                     for k in ("slope", "azimuth"))
    if orientation != "latitude_optimal":
        raise ValueError(f"orientation {orientation!r} is not restated")
    lat = torch.deg2rad(torch.as_tensor(np.asarray(lat, dtype=np.float64), device=device))
    below_25 = torch.abs(lat) <= math.radians(25)
    below_50 = torch.abs(lat) <= math.radians(50)
    slope = torch.where(below_25, 0.87 * torch.abs(lat),
                        torch.where(below_50, 0.76 * torch.abs(lat) + math.radians(0.31),
                                    torch.full_like(lat, math.radians(40.0))))
    azimuth = torch.where(lat < 0, torch.zeros_like(lat), torch.full_like(lat, math.pi))
    return slope[None, :, None], azimuth[None, :, None]


def _fillna(a, value):
    return torch.where(torch.isnan(a), value, a)


def _clip(influx, influx_max):
    return torch.minimum(torch.maximum(influx, torch.zeros((), dtype=influx.dtype, device=influx.device)),
                         influx_max)


def pv(fields, time, lon, lat, panel, orientation, altitude_threshold=1.0):
    """atlite_oracle.convert_pv (ERA5 branch, no tracking, simple trigon model, Huld panel).

    ``fields``: float32 ``(t, ny, nx)`` tensors influx_toa, influx_direct, influx_diffuse, albedo,
    temperature.  Returns (capacity factors, allowance), float64 ``(t, ny, nx)``."""
    dev = fields["influx_toa"].device
    sp_ = solar_position(time, lon, lat, dev)
    alt, az = sp_["altitude"], sp_["azimuth"]
    surface_slope, surface_azimuth = orientation_table(orientation, lat, dev)

    # surface_orientation, tracking None
    sin_alt, cos_alt = torch.sin(alt), torch.cos(alt)
    cosincidence = (torch.sin(surface_slope) * cos_alt * torch.cos(surface_azimuth - az)
                    + torch.cos(surface_slope) * sin_alt)
    del az
    cosincidence = torch.where(torch.isnan(cosincidence), cosincidence, torch.clamp(cosincidence, min=0))

    # tilted_irradiation, influx_direct / influx_diffuse, trigon_model "simple"
    influx_toa = fields["influx_toa"]
    direct = _clip(fields["influx_direct"], influx_toa)
    diffuse = _clip(fields["influx_diffuse"], influx_toa - direct)
    k = cosincidence / sin_alt
    del cosincidence, sin_alt, cos_alt
    cos_surface_slope = torch.cos(surface_slope)
    influx = direct + diffuse
    direct_t = k * direct
    del k
    diffuse_t = (1.0 + cos_surface_slope) / 2.0 * diffuse
    ground_t = fields["albedo"] * influx * ((1.0 - cos_surface_slope) / 2.0)
    total_t = _fillna(direct_t, 0.0) + _fillna(diffuse_t, 0.0) + _fillna(ground_t, 0.0)
    del direct_t, diffuse_t, ground_t
    # result = where(~(cap_alt | dark), total, 0).  The altitude mask is applied after the panel
    # model instead: _huld is elementwise and _huld(0) == 0, so the values are the same, and the
    # panel output without the altitude mask is what the allowance needs.
    irr = torch.where(~(influx <= 0.01), total_t, 0.0)
    del total_t, influx, direct, diffuse
    unmasked = _huld(irr, fields["temperature"], panel)
    del irr
    cap_alt = alt < math.radians(altitude_threshold)
    value = torch.where(cap_alt, 0.0, unmasked)
    near = torch.abs(alt - math.radians(altitude_threshold)) < PV_ALTITUDE_WINDOW
    allowance = torch.where(near, torch.abs(unmasked), 0.0)
    return value, allowance


def _huld(irradiance, t_amb, pc):
    """atlite_oracle._power_huld"""
    T_ = (pc["c_temp_amb"] * t_amb + pc["c_temp_irrad"] * irradiance) - pc["r_tmod"]
    G_ = irradiance / pc["r_irradiance"]
    log_G_ = torch.log(torch.where(G_ > 0, G_, math.nan))
    eff = (
        1
        + pc["k_1"] * log_G_
        + pc["k_2"] * (log_G_) ** 2
        + T_ * (pc["k_3"] + pc["k_4"] * log_G_ + pc["k_5"] * log_G_**2)
        + pc["k_6"] * (T_**2)
    )
    eff = torch.clamp(_fillna(eff, 0.0), min=0)
    return G_ * eff * pc.get("inverter_efficiency", 1.0)


def _log_f32(x):
    """float32 log, correctly rounded (the float64 log rounded to float32).  NumPy's SIMD float32
    log is not: it is one ulp off for a few per cent of arguments, and torch's float32 logs differ
    between devices, so neither can be matched bit for bit; the pin test keeps the two apart."""
    return torch.log(x.to(f64)).to(torch.float32)


def wind_speed(wnd100m, roughness, hub_height):
    """atlite_oracle.extrapolate_wind_speed from 100 m with the log law (the fast lane for a hub
    at 100 m): the hub speed as ``np.interp`` sees it, float64.  The hub height is a Python float
    in the turbine configs and the oracle's ``from_height`` the NumPy int64 it picks among the
    dataset's heights, so the first quotient is float32 and the second float64."""
    if int(hub_height) == 100:  # wnd100m is in the dataset: returned as is
        return wnd100m.to(f64)
    if isinstance(hub_height, np.generic):
        to_log = torch.log(float(hub_height) / roughness.to(f64))
    else:
        to_log = _log_f32(hub_height / roughness)
    from_log = torch.log(100.0 / roughness.to(f64))
    return wnd100m * (to_log / from_log)


def interp(x, xp, fp):
    """``np.interp(x, xp, fp)`` for float64 ``x`` and ascending knots ``xp`` (duplicates allowed):
    clamped at both ends, a knot's value at the knot, and at a repeated knot the value of its
    last copy (the rightmost j with xp[j] <= x)."""
    xp = torch.as_tensor(np.asarray(xp, dtype=np.float64), device=x.device)
    fp = torch.as_tensor(np.asarray(fp, dtype=np.float64), device=x.device)
    n = xp.numel()
    j = torch.searchsorted(xp, x.contiguous(), right=True) - 1
    jc = j.clamp(0, n - 2)
    slope = (fp[jc + 1] - fp[jc]) / (xp[jc + 1] - xp[jc])
    out = torch.where(x == xp[jc], fp[jc], slope * (x - xp[jc]) + fp[jc])
    out = torch.where(j < 0, fp[0], torch.where(j >= n - 1, fp[-1], out))
    return torch.where(torch.isnan(x), x, out)


def wind(wnd100m, roughness, turbine):
    """atlite_oracle.convert_wind (log law): (capacity factors, allowance), float64 ``(t, ny, nx)``."""
    V = np.asarray(turbine["V"], dtype=np.float64)
    fp = np.asarray(turbine["POW"], dtype=np.float64) / turbine["P"]
    hub = wind_speed(wnd100m, roughness, turbine["hub_height"])
    value = interp(hub, V, fp)
    allowance = torch.zeros_like(value)
    for i in np.flatnonzero((V[1:] == V[:-1]) & (fp[1:] != fp[:-1])):  # knots where the curve jumps
        near = torch.abs(hub - V[i]) <= WIND_KNOT_WINDOW * abs(V[i])
        allowance = torch.where(near, torch.maximum(allowance, torch.full_like(allowance, abs(fp[i + 1] - fp[i]))),
                                allowance)
    return value, allowance


def heat_demand(temperature, time, threshold=15.0, a=1.0, constant=0.0, hour_shift=0.0):
    """atlite_oracle.convert_heat_demand: (daily values, allowance 0), float32 ``(days, ny, nx)``
    like the oracle's.  The daily mean is NumPy's ``nanmean`` over axis 0: a float32 sum, step
    after step, of the non-NaN values, divided by their count (in float64, rounded to float32)."""
    T = temperature
    _, gid = day_bins(time, hour_shift)
    nd = int(gid[-1]) + 1
    out = torch.full((nd,) + tuple(T.shape[1:]), math.nan, dtype=T.dtype, device=T.device)
    for d in range(nd):
        steps = np.flatnonzero(gid == d)
        if not len(steps):
            continue
        tot = torch.where(torch.isnan(T[steps[0]]), 0.0, T[steps[0]])
        cnt = (~torch.isnan(T[steps[0]])).to(torch.int64)
        for s in steps[1:]:
            tot = tot + torch.where(torch.isnan(T[s]), 0.0, T[s])
            cnt = cnt + (~torch.isnan(T[s])).to(torch.int64)
        out[d] = (tot.to(f64) / cnt).to(T.dtype)
    threshold = threshold + 273.15
    heat = a * (threshold - out)
    heat = torch.where(torch.isnan(heat), heat, torch.clamp(heat, min=0.0))
    return constant + heat, torch.zeros((), dtype=f64, device=T.device)
