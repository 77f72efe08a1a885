"""ERA5 prepare-time derivations on the GPU (SURVEY section 8 f4).

Host-side mirror of the arithmetic in the reference's ``atlite/datasets/era5.py``
(the part after ``retrieve_data``): raw download variables in, cutout variables out,

    get_data_wind    (era5.py:104-137)  u100, v100, u10, v10, fsr
                                        -> wnd100m, wnd_shear_exp, wnd_azimuth, roughness
    get_data_influx  (era5.py:149-192)  ssrd, ssr, tisr, fdir
                                        -> influx_toa, influx_direct, influx_diffuse, albedo,
                                           solar_altitude, solar_azimuth (time shift -30 min)
    get_data_temperature (204-225)      t2m, stl4, d2m -> temperature, soil temperature,
                                           dewpoint temperature (renames)
    get_data_runoff  (228-238, 241-246) ro -> runoff (clipped at 0)
    get_data_height  (era5.py:65-81, 247-256)  z (geopotential) -> height = z / g0, static (y, x)
    sanitize_wind / sanitize_influx / sanitize_runoff (141-146, 195-201, 241-246)

The results are float32 torch CUDA tensors (float64 for the solar position, like the
reference's stored variables) in an ``atlite_b200.Dataset``: a device-resident cutout
ready for ``Cutout(data=...)``.  Kernels: csrc/era5.cu; no CPU fallback.
"""

from __future__ import annotations

import numpy as np
import pandas as pd

from . import _lib
from .engine import _dptr, _is_torch, _stream_ptr, _torch, current_device, time_ns
from .labelled import Dataset


def _dev_f32(a, device):
    torch = _torch()
    if _is_torch(a):
        return a.to(device=device, dtype=torch.float32).contiguous()
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(device)


def _raw(ds, name):
    if name not in ds:
        raise KeyError(f"raw ERA5 variable {name!r} missing")
    v = ds.raw(name) if hasattr(ds, "raw") else ds[name]
    if _is_torch(v):  # (torch.Tensor.values is a method: do not unwrap tensors)
        return v
    return getattr(v, "values", v)


def _coords(ds):
    c = dict(ds.coords) if hasattr(ds, "coords") else {k: ds[k] for k in ("time", "x", "y") if k in ds}
    out = {k: np.asarray(getattr(v, "values", v)) for k, v in c.items() if k in ("time", "x", "y", "lon", "lat")}
    out.setdefault("lon", out["x"])
    out.setdefault("lat", out["y"])
    return out


def _dims(t):
    return ("time", "y", "x")[-t.ndim:]


def get_data_wind(ds, sanitize=True, device=None):
    """era5.py:104-137 (+ sanitize_wind 141-146) on raw u100/v100/u10/v10/fsr."""
    torch = _torch()
    device = torch.device("cuda", current_device() if device is None else device)
    u100, v100, u10, v10, fsr = (_dev_f32(_raw(ds, n), device) for n in ("u100", "v100", "u10", "v10", "fsr"))
    if not (u100.shape == v100.shape == u10.shape == v10.shape == fsr.shape):
        raise ValueError("raw wind variables must share one shape")
    outs = [torch.empty_like(u100) for _ in range(4)]
    _lib.check(_lib.load().atl_era5_wind(device.index, u100.numel(), _dptr(u100), _dptr(v100), _dptr(u10), _dptr(v10),
                                         _dptr(fsr), 1 if sanitize else 0, *(_dptr(o) for o in outs), _stream_ptr()))
    names = ("wnd100m", "wnd_shear_exp", "wnd_azimuth", "roughness")
    return Dataset({n: (_dims(o), o) for n, o in zip(names, outs)}, coords=_coords(ds),
                   attrs={"module": "era5"})


def solar_position(time, lon, lat, time_shift="-30min", device=None):
    """pv/solar_position.py:69-116 materialised on the GPU: (altitude, azimuth), each a
    (time, y, x) float64 CUDA tensor."""
    torch = _torch()
    device = torch.device("cuda", current_device() if device is None else device)
    tns = np.ascontiguousarray(time_ns(time))
    lon = np.ascontiguousarray(lon, dtype=np.float64)
    lat = np.ascontiguousarray(lat, dtype=np.float64)
    shift = int(pd.to_timedelta(time_shift).value)
    alt = torch.empty((len(tns), len(lat), len(lon)), dtype=torch.float64, device=device)
    az = torch.empty_like(alt)
    _lib.check(_lib.load().atl_solar_position(device.index, _lib.ptr(tns), len(tns), shift, _lib.ptr(lon), len(lon),
                                              _lib.ptr(lat), len(lat), _dptr(alt), _dptr(az), _stream_ptr()))
    return alt, az


def get_data_influx(ds, sanitize=True, solar_position_vars=True, device=None):
    """era5.py:149-192 (+ sanitize_influx 195-201) on raw ssrd/ssr/tisr/fdir."""
    torch = _torch()
    device = torch.device("cuda", current_device() if device is None else device)
    ssrd, ssr, tisr, fdir = (_dev_f32(_raw(ds, n), device) for n in ("ssrd", "ssr", "tisr", "fdir"))
    if not (ssrd.shape == ssr.shape == tisr.shape == fdir.shape):
        raise ValueError("raw influx variables must share one shape")
    outs = [torch.empty_like(ssrd) for _ in range(4)]
    _lib.check(_lib.load().atl_era5_influx(device.index, ssrd.numel(), _dptr(ssrd), _dptr(ssr), _dptr(tisr), _dptr(fdir),
                                           1 if sanitize else 0, *(_dptr(o) for o in outs), _stream_ptr()))
    names = ("influx_toa", "influx_direct", "influx_diffuse", "albedo")
    co = _coords(ds)
    out = Dataset({n: (_dims(o), o) for n, o in zip(names, outs)}, coords=co, attrs={"module": "era5"})
    if solar_position_vars:  # era5.py:182-188
        alt, az = solar_position(co["time"], co["lon"], co["lat"], "-30min", device.index)
        out["solar_altitude"] = (("time", "y", "x"), alt)
        out["solar_azimuth"] = (("time", "y", "x"), az)
    return out


def get_data_temperature(ds, device=None):
    """era5.py:204-225: renames only."""
    torch = _torch()
    device = torch.device("cuda", current_device() if device is None else device)
    ren = {"t2m": "temperature", "stl4": "soil temperature", "d2m": "dewpoint temperature"}
    return Dataset({new: (("time", "y", "x"), _dev_f32(_raw(ds, old), device)) for old, new in ren.items() if old in ds},
                   coords=_coords(ds), attrs={"module": "era5"})


def get_data_runoff(ds, sanitize=True, device=None):
    """era5.py:228-238 (+ sanitize_runoff 241-246: clip(min=0))."""
    torch = _torch()
    device = torch.device("cuda", current_device() if device is None else device)
    ro = _dev_f32(_raw(ds, "ro"), device)
    if sanitize:
        ro = torch.where(ro < 0, torch.zeros_like(ro), ro)  # NaN stays NaN, like xarray's clip
    return Dataset({"runoff": (_dims(ro), ro)}, coords=_coords(ds), attrs={"module": "era5"})


def get_data_height(ds, device=None):
    """era5.py:65-81 (_add_height) / 247-256: geopotential ``z`` -> ``height = z / g0``
    (g0 = 9.80665), the first time step if ``z`` has a time axis; a static (y, x) field."""
    h = height_from_z(_raw(ds, "z"), device)
    return Dataset({"height": (("y", "x"), h)}, coords=_coords(ds), attrs={"module": "era5"})


def height_from_z(z, device=None):
    """era5.py:74-78: ``z / g0`` of the geopotential ``z`` ((y, x), or (time, y, x): its first
    step), as a float32 CUDA tensor.  The one definition of the height: the converters that read a
    raw cutout's ``z`` call it too, so they weight with exactly what ``get_data_height`` stores."""
    torch = _torch()
    device = torch.device("cuda", current_device() if device is None else device)
    z = _dev_f32(z[0] if z.ndim == 3 else z, device)
    return (z / 9.80665).contiguous()


def prepare(ds, features=("wind", "influx", "temperature", "runoff"), sanitize=True, device=None):
    """All requested features of one raw dataset merged into a device-resident cutout
    Dataset (what ``Cutout.prepare`` stores for ``module='era5'``).  The static
    ``height`` feature (era5.py:62) is added whenever the raw data carries ``z``."""
    fns = {"wind": get_data_wind, "influx": get_data_influx, "temperature": get_data_temperature,
           "runoff": get_data_runoff, "height": get_data_height}
    features = list(features)
    if "height" not in features and "z" in ds:
        features.append("height")
    merged = None
    for f in features:
        kw = {} if f in ("temperature", "height") else {"sanitize": sanitize}
        part = fns[f](ds, device=device, **kw)
        if merged is None:
            merged = part
        else:
            for n in part.data_vars:
                merged[n] = (part.dims_of(n), part.raw(n))
    return merged
