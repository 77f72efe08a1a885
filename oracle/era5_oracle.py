"""CPU oracle for the ERA5 prepare-time derivations (TEST INFRASTRUCTURE ONLY -- never
imported by atlite_b200).  NumPy restatement of the arithmetic in atlite/datasets/era5.py,
each function citing the lines it follows.

The derivations are evaluated in the floating dtype of the inputs (float64 for lists and
integers), as the reference evaluates them in the dtype of the download: on float32 fields a
wind component above ~1.8e19 squares to inf in float32, and the wind speed, the shear exponent
and everything downstream follow from that inf, not from a finite float64 speed.  Only the
shear exponent's division by np.log(10 / 100), a float64 scalar, promotes to float64 there.

PARITY PINNING: **pinned against the reference's own source.**  The reference computes
these inside ``get_data_*`` after a CDS download; tests/golden/make_golden.py::era5_cases
loads datasets/era5.py from the reference's source tree under the xarray/dask stand-in
(tests/golden/xr_shim.py), replaces only ``retrieve_data`` (the download) and
``_rename_and_clean_coords`` (coordinate renaming) and records the outputs of
get_data_wind / sanitize_wind / get_data_influx / sanitize_influx (incl. the stored solar
position) in tests/golden/reference_era5.npz; make_golden.py::era5_edge_cases does the same at
the edges of the raw inputs (NaN, +-inf, 0, -0, negative values, calm and overflowing winds)
in tests/golden/reference_era5_edges.npz.  tests/test_era5.py and tests/test_era5_edges.py
hold this oracle to them (6e-7, identical NaN and +-inf positions; solar position 1e-12),
plus hand-computable known answers.  Not pinned against genuine xarray/dask (absent here).
"""

from __future__ import annotations

import numpy as np


def _inputs(*arrays):
    """The arrays in their common floating dtype (float32 stays float32)."""
    arrays = [np.asarray(a) for a in arrays]
    dt = np.result_type(*arrays, np.float32)
    return [a.astype(dt) for a in arrays]


def get_data_wind(u100, v100, u10, v10, fsr, sanitize=True):
    """era5.py:120-135 (+ sanitize_wind :141-146)."""
    u100, v100, u10, v10, fsr = _inputs(u100, v100, u10, v10, fsr)
    with np.errstate(over="ignore"):
        wnd100m = np.sqrt(u100**2 + v100**2)                               # :121
        wnd10m = np.sqrt(u10**2 + v10**2)
    with np.errstate(divide="ignore", invalid="ignore"):
        shear = np.log(wnd10m / wnd100m) / np.log(10 / 100)               # :124-126
    az = np.arctan2(u100, v100)                                            # :129
    az = np.where(az >= 0, az, az + 2 * np.pi)                             # :130 (NaN keeps NaN + 2 pi = NaN)
    rough = fsr.copy()
    if sanitize:
        rough = np.where(rough >= 0.0, rough, 2e-4)                        # :145
    return dict(wnd100m=wnd100m, wnd_shear_exp=shear, wnd_azimuth=az, roughness=rough)


def get_data_influx(ssrd, ssr, tisr, fdir, sanitize=True):
    """era5.py:163-175 (+ sanitize_influx :195-201)."""
    ssrd, ssr, tisr, fdir = _inputs(ssrd, ssr, tisr, fdir)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        albedo = (ssrd - ssr) / np.where(ssrd != 0, ssrd, np.nan)          # :165
        albedo = np.where(np.isnan(albedo), 0.0, albedo)                   # :166 fillna(0)
        out = dict(albedo=albedo, influx_diffuse=ssrd - fdir, influx_direct=fdir.copy(), influx_toa=tisr.copy())  # :168
    for a in ("influx_direct", "influx_diffuse", "influx_toa"):
        out[a] = out[a] / (60.0 * 60.0)                                    # :174-175
        if sanitize:
            out[a] = np.where(out[a] < 0.0, 0.0, out[a])                   # :199-200 clip(min=0), NaN stays
    return out
