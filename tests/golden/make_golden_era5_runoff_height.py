#!/usr/bin/env python
"""Generate ``reference_era5_runoff_height.npz``: the REFERENCE'S OWN ``get_data_runoff``,
``sanitize_runoff`` and ``get_data_height`` (atlite/datasets/era5.py), loaded from the reference's
source file under the stand-ins of ``xr_shim.py`` as ``make_golden.py`` loads it for the wind and
influx derivations.  Only ``retrieve_data`` (the CDS download) and ``_rename_and_clean_coords``
(coordinate renaming) are replaced; every formula that executes is the reference's own line.

    python tests/golden/make_golden_era5_runoff_height.py   # writes tests/golden/reference_era5_runoff_height.npz

The output is committed; tests/test_era5_raw_more.py holds oracle/era5_runoff_height_oracle.py to it
on the CPU, so nothing reads the reference at test time.  The zip members carry no time stamps: the
same arrays give the same bytes.
"""

import os
import sys
import warnings
import zipfile

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import xr_shim  # noqa: E402

warnings.simplefilter("ignore")


def _savez_reproducible(path, arrays):
    """np.savez_compressed without the wall-clock time stamps of the zip members."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for k, v in arrays.items():
            zi = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            zi.compress_type = zipfile.ZIP_DEFLATED
            with zf.open(zi, "w", force_zip64=True) as fh:
                np.lib.format.write_array(fh, np.asanyarray(v), allow_pickle=False)


class _TimeArray(xr_shim.DataArray):
    """The stand-in's DataArray plus ``isel(time=i, drop=True)`` with an integer index, which
    _add_height (era5.py:76-78) calls and the stand-in does not provide: the axis goes away."""

    def isel(self, drop=False, **kw):
        (d, i), = kw.items()
        ax = self.dims.index(d)
        dims = self.dims[:ax] + self.dims[ax + 1:]
        return xr_shim.DataArray(np.take(self.values, i, axis=ax), {k: v for k, v in self._coords.items() if k in dims},
                                 dims, self.name, self.attrs)


class _ZDataset(xr_shim.Dataset):
    """The stand-in's Dataset whose ``z`` is a ``_TimeArray``."""

    def __getitem__(self, k):
        a = super().__getitem__(k)
        return _TimeArray(a.values, a._coords, a.dims, k, a.attrs) if k == "z" else a


def main():
    """get_data_runoff + sanitize_runoff (era5.py:228-246) and get_data_height (:65-81, 247-256)
    from the reference's own source, as make_golden.py::era5_cases runs get_data_wind: seeded float32 ``ro`` with negative values, NaN,
    +-0 and +-inf, and a geopotential ``z`` with a time axis whose steps differ (the height is the
    first step's) as well as a static one.  -> tests/golden/reference_era5_runoff_height.npz"""
    era5 = xr_shim.load_reference_era5()
    nx, ny, nt = 9, 6, 5
    rng = np.random.default_rng(57)
    x, y = np.arange(nx) * 0.5 + 3.0, np.arange(ny) * 0.5 + 45.0
    t = pd.date_range("2013-01-01 00:00", periods=nt, freq="h")
    co = dict(time=t, x=x, y=y, lon=x, lat=y)
    ro = rng.uniform(-2e-4, 3e-3, (nt, ny, nx)).astype(np.float32)
    ro[0, 0, :6] = [np.nan, np.inf, -np.inf, 0.0, -0.0, -1e-6]
    z = rng.uniform(-400.0, 4.0e4, (nt, ny, nx)).astype(np.float32)
    z[:, 1, 1] = [np.nan, 1.0, 2.0, 3.0, 4.0]
    z[0, 2, :3] = [0.0, -0.0, -98.0665]
    z_static = rng.uniform(-400.0, 4.0e4, (ny, nx)).astype(np.float32)
    units = {"units": "m**2 s**-2"}
    datasets = {
        "runoff": xr_shim.Dataset({"ro": xr_shim.DataArray(ro, co, ("time", "y", "x"), attrs={"units": "m"})},
                                  coords=co),
        "time": _ZDataset({"z": xr_shim.DataArray(z, co, ("time", "y", "x"), attrs=units)}, coords=co),
        "static": _ZDataset({"z": xr_shim.DataArray(z_static, co, ("y", "x"), attrs=units)}, coords=co)}
    era5._rename_and_clean_coords = lambda ds, add_lon_lat=True: ds  # noqa: E731
    out = {"x": x, "y": y, "time_ns": pd.DatetimeIndex(t).as_unit("ns").asi8, "raw|ro": ro, "raw|z": z,
           "raw|z_static": z_static}
    era5.retrieve_data = lambda **kw: datasets["runoff"]  # noqa: E731
    r = era5.get_data_runoff({})
    out["runoff|runoff"] = np.asarray(r["runoff"].values)
    out["runoff_sanitized|runoff"] = np.asarray(era5.sanitize_runoff(r)["runoff"].values)
    for tag in ("time", "static"):
        era5.retrieve_data = lambda tag=tag, **kw: datasets[tag]  # noqa: E731
        h = era5.get_data_height({})
        assert "z" not in h and h["height"].dims == ("y", "x")
        out[f"height|{tag}"] = np.asarray(h["height"].values)
    path = os.path.join(HERE, "reference_era5_runoff_height.npz")
    _savez_reproducible(path, out)
    print(f"era5 runoff and height -> {path} ({os.path.getsize(path) / 1e3:.0f} kB)")


if __name__ == "__main__":
    main()
