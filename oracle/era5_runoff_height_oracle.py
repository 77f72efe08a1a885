"""CPU oracle for the ERA5 runoff and height derivations (TEST INFRASTRUCTURE ONLY -- never
imported by atlite_b200).  NumPy restatement of atlite/datasets/era5.py's get_data_runoff /
sanitize_runoff and _add_height, evaluated in the floating dtype of the inputs as the reference
evaluates them in the dtype of the download (the conventions of ``era5_oracle``).

PARITY PINNING: **pinned against the reference's own source.**
tests/golden/make_golden_era5_runoff_height.py loads datasets/era5.py from the reference's source
tree under the xarray stand-in (tests/golden/xr_shim.py), replaces only ``retrieve_data`` (the
download) and ``_rename_and_clean_coords`` (coordinate renaming), and records the outputs of
get_data_runoff, sanitize_runoff and get_data_height in
tests/golden/reference_era5_runoff_height.npz; tests/test_era5_raw_more.py holds this oracle to
them bit for bit.
"""

from __future__ import annotations

import numpy as np

from era5_oracle import _inputs


def get_data_runoff(ro, sanitize=True):
    """era5.py:228-238 (``ro`` renamed ``runoff``) + sanitize_runoff :241-246 (clip(min=0), NaN
    stays)."""
    (ro,) = _inputs(ro)
    runoff = ro.copy()
    if sanitize:
        runoff = np.where(runoff < 0.0, 0.0, runoff)
    return dict(runoff=runoff)


def get_data_height(z):
    """era5.py:65-81 (_add_height) / 247-256: ``z / g0`` (g0 = 9.80665) of the geopotential, its
    first step when it has a time axis (a leading axis of a 3-d array here)."""
    (z,) = _inputs(z)
    if z.ndim == 3:
        z = z[0]
    return dict(height=z / 9.80665)
