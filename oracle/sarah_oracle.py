"""CPU oracle for ``atlite_b200.sarah`` (TEST INFRASTRUCTURE ONLY -- never imported by atlite_b200).

NumPy restatement of the SARAH semantics in DESIGN.md section 1:

  * gap filling per block of steps: in every (cell, block) series with some NaN and some valid
    values, the NaNs are replaced by ``np.interp`` of the valid values on the step index (linear
    between valid steps, the first / last valid value outside them), computed in float64 and
    stored back as float32; without interpolation NaN becomes 0;
  * the hourly mean: steps (2k, 2k + 1) averaged in float32 as (a + b) / 2, an odd last step dropped;
  * resampling onto a coarser grid with ``regrid_oracle.regrid`` (average), then
    ``influx_diffuse = SIS - SID`` and ``influx_direct = SID``.
"""

from __future__ import annotations

import numpy as np

import regrid_oracle


def fill_series(y, interpolate=True):
    """One float32 series of one block, filled."""
    y = np.array(y, dtype=np.float32)
    nan = np.isnan(y)
    if not interpolate:
        y[nan] = 0
        return y
    if nan.all() or not nan.any():
        return y
    y[nan] = np.interp(nan.nonzero()[0], (~nan).nonzero()[0], y[~nan])
    return y


def fill(a, starts, interpolate=True):
    """(nt, ...) float32 filled along axis 0 within the blocks beginning at ``starts``."""
    a = np.array(a, dtype=np.float32)
    bounds = list(starts) + [len(a)]
    flat = a.reshape(len(a), -1)
    for b0, b1 in zip(bounds[:-1], bounds[1:]):
        for c in range(flat.shape[1]):
            flat[b0:b1, c] = fill_series(flat[b0:b1, c], interpolate)
    return flat.reshape(a.shape)


def hourly_mean(a):
    n = len(a) - len(a) % 2
    return (a[0:n:2] + a[1:n:2]) / np.float32(2)


def influx(sis, sid, starts, interpolate=True, hourly=True, lon=None, lat=None, dst_lon=None, dst_lat=None):
    """(influx_direct, influx_diffuse) float32 from (nt, ny, nx) SIS / SID; resampled onto
    ``dst_lon`` / ``dst_lat`` when they are given."""
    sis, sid = fill(sis, starts, interpolate), fill(sid, starts, interpolate)
    if hourly:
        sis, sid = hourly_mean(sis), hourly_mean(sid)
    if dst_lon is not None:
        sis = regrid_oracle.regrid(sis, lon, lat, dst_lon, dst_lat, 5).astype(np.float32)
        sid = regrid_oracle.regrid(sid, lon, lat, dst_lon, dst_lat, 5).astype(np.float32)
    return sid, sis - sid
