"""Reference-facing API of the hot path: ``convert_and_aggregate`` and the
``pv`` / ``wind`` / ``heat_demand`` wrappers, with the reference's signatures,
argument meaning, warnings and errors (convert.py:59-276, 421-471, 665-744,
857-936), executing on the GPU through ``libatlite_b200.so``.

Instead of building a lazy dask graph of ~60 ufunc passes and a per-chunk
``dense * csr.T`` product, a known ``convert_func`` is mapped to a fused
operator (physics + shape reduce in one kernel).  Unknown ``convert_func``
callables keep the reference's plugin protocol: they are evaluated by the
caller's code and only the aggregation runs on the GPU (``atl_spmm``).
"""

from __future__ import annotations

import inspect
import logging
import re
import threading
import types
import warnings
from collections.abc import Mapping
from pathlib import Path

import numpy as np
import pandas as pd
import scipy.sparse as sp

from . import _lib, engine
from .labelled import HAVE_XARRAY, DataArray, is_dataarray, make_dataarray
from .orientation import get_orientation
from .resource import (
    EfficiencyTable,
    get_cspinstallationconfig,
    get_solarpanelconfig,
    get_windturbineconfig,
    windturbine_smooth,
)

if HAVE_XARRAY:  # pragma: no cover
    import xarray as xr

logger = logging.getLogger(__name__)

_SOLAR_WARNING = """The calculation method and handling of solar position variables will change.
    The solar position will in the future be a permanent variables of a cutout.
    Recreate your cutout to remove this warning and permanently include the solar position variables into your cutout."""


# --------------------------------------------------------------------------
# dataset access helpers (xarray.Dataset or atlite_b200.labelled.Dataset)
# --------------------------------------------------------------------------


def _has(ds, name):
    return name in ds


def _coord(ds, name):
    v = ds[name]
    return np.asarray(getattr(v, "values", v))


def _raw(ds, name):
    """(time, y, x) array of a variable: torch CUDA tensor for a device-resident
    cutout, else a NumPy array."""
    if hasattr(ds, "raw"):
        arr = ds.raw(name)
        dims = ds.dims_of(name)
        if dims != ("time", "y", "x")[-len(dims):]:
            raise ValueError(f"variable {name!r} must have dims (time, y, x), has {dims}")
        return arr
    da = ds[name]
    if da.ndim == 3:
        da = da.transpose("time", "y", "x")
    return np.asarray(da.values)


# Raw ERA5 variables (CDS short names) a cutout may carry instead of the variables era5.prepare
# derives from them (datasets/era5.py:104-225).  A converter reads them directly only when its
# prepared inputs are absent and the raw set it needs is complete; everything else keeps its path.
_PV_PREPARED = ("influx_toa", "influx_direct", "influx_diffuse", "influx", "albedo", "outflux")
_PV_RAW = ("ssrd", "ssr", "tisr", "fdir")
_RAW_RENAMES = {"temperature": "t2m", "soil temperature": "stl4", "dewpoint temperature": "d2m"}


def _var(ds, name):
    """``name``, or the raw ERA5 variable era5.prepare renames to it (era5.py:204-225) when the
    dataset carries only that one."""
    raw = _RAW_RENAMES.get(name)
    if raw is not None and not _has(ds, name) and _has(ds, raw):
        return raw
    return name


def _pv_raw(ds):
    """Does the PV family read raw ssrd / ssr / tisr / fdir (no prepared irradiation variable)?"""
    return not any(_has(ds, n) for n in _PV_PREPARED) and all(_has(ds, n) for n in _PV_RAW)


_LR_PREPARED = ("wnd100m", "wnd_azimuth", "influx_direct")
_LR_RAW = ("u100", "v100", "fdir")


def _line_rating_raw(ds):
    """Does line_rating read raw u100 / v100 / fdir (no prepared wind or direct-influx variable)?"""
    return not any(_has(ds, n) for n in _LR_PREPARED) and all(_has(ds, n) for n in _LR_RAW)


def _csp_raw(ds):
    """Does csp read the raw fdir (no prepared influx_direct)?"""
    return not _has(ds, "influx_direct") and _has(ds, "fdir")


def _runoff_raw(ds):
    """Does runoff read the raw ro (no prepared runoff)?"""
    return not _has(ds, "runoff") and _has(ds, "ro")


def _dims_of(ds, name):
    return tuple(ds.dims_of(name)) if hasattr(ds, "dims_of") else tuple(ds[name].dims)


def _height(ds):
    """The static height (y, x): ``height`` (an integer height, such as GEBCO's int16, as float32),
    else ``z / g0`` of the geopotential ``z``'s first step as era5.prepare derives it
    (``era5.height_from_z``), else None.  A device tensor for a device-resident cutout, else a NumPy
    array.  Derive it on the WHOLE cutout: a time part of it starts at another step of a
    time-dependent ``z``."""
    if _has(ds, "height"):
        h = _raw(ds, "height")
        if engine._is_torch(h):
            return h if h.is_floating_point() else h.float()
        return h if np.asarray(h).dtype.kind == "f" else np.asarray(h, dtype=np.float32)
    if not _has(ds, "z"):
        return None
    from . import era5

    src = _time_slice(ds, 0, 1) if "time" in _dims_of(ds, "z") else ds  # only the first step is read
    z = _raw(src, "z")
    if engine._is_torch(z) and z.is_cuda:
        return era5.height_from_z(z, z.device.index)
    return _to_host(era5.height_from_z(z))


def _stored_solar_position(ds):
    """The stored solar position: (altitude, azimuth, solar source).  The kernels read both arrays
    with one width, so it is float64 (``SOLAR_STORED_F64``) only when both arrays are; otherwise
    both are taken as float32."""
    alt, az = _raw(ds, "solar_altitude"), _raw(ds, "solar_azimuth")
    if all(str(a.dtype).replace("torch.", "") == "float64" for a in (alt, az)):
        return alt, az, _lib.SOLAR_STORED_F64

    def f32(a):
        return a.to(engine._torch().float32) if engine._is_torch(a) else np.asarray(a, dtype=np.float32)

    return f32(alt), f32(az), _lib.SOLAR_STORED_F32


def _grid_shape(ds):
    return len(_coord(ds, "y")), len(_coord(ds, "x"))


def _is_dask_backed(ds):
    """Lazily loaded cutout: a dask-backed xarray dataset (what ``Cutout(path)`` opens,
    cutout.py:142-154) or an ``atlite_b200.LazyDataset``."""
    if getattr(ds, "lazy", False):
        return True
    if not HAVE_XARRAY or hasattr(ds, "raw"):
        return False
    try:
        from dask.array.core import Array

        return any(isinstance(ds[v].data, Array) for v in ds.data_vars)
    except Exception:  # noqa: BLE001
        return False


def _to_host(a):
    if engine._is_torch(a):
        return a.detach().cpu().numpy()
    return np.asarray(a)


# --------------------------------------------------------------------------
# fused operator specs
# --------------------------------------------------------------------------


class _Spec:
    """A known conversion bound to a cutout: can reduce to buses, or produce
    per-cell values / their time sum."""

    time_labels = None  # output time coordinate
    name = None
    units = None

    def _device_fields(self, fields):
        """Host arrays -> device tensors (per-cell output paths only)."""
        torch = engine._torch()
        dev = f"cuda:{engine.current_device()}"
        return {
            k: (v if v is None or engine._is_torch(v) else torch.from_numpy(np.ascontiguousarray(v)).to(dev))
            for k, v in fields.items()
        }

    def cells_timesum(self):
        """(NaN-skipping per-cell time sum, number of valid steps per cell), each (y, x)."""
        sc = self.cells(timesum=True)
        return sc[0], sc[1]


class _PvSpec(_Spec):
    name = "specific generation"

    def __init__(self, ds, panel, orientation, tracking=None, trigon_model="simple",
                 clearsky_model="simple", output="panel", thermal=(0.0, 0.0, 0.0)):
        ny, nx = _grid_shape(ds)
        self.ds = ds
        self.time_labels = pd.DatetimeIndex(_coord(ds, "time"))
        lon, lat = _coord(ds, "lon").astype(np.float64), _coord(ds, "lat").astype(np.float64)

        # SolarPosition: getter vs computation (pv/solar_position.py:54-67).  A raw ERA5 cutout gets
        # the position era5.prepare would have stored (time shift -30 min, era5.py:182-188), computed
        # in-kernel, so it does not warn.
        raw = _pv_raw(ds)
        solar = {}
        if _has(ds, "solar_azimuth") and _has(ds, "solar_altitude"):
            solar["solar_altitude"], solar["solar_azimuth"], solar_src = _stored_solar_position(ds)
        elif raw:
            solar_src = _lib.SOLAR_COMPUTED
        else:
            warnings.warn(_SOLAR_WARNING, DeprecationWarning)
            solar_src = _lib.SOLAR_COMPUTED

        # SurfaceOrientation (pv/orientation.py:104-109, 177-183)
        if tracking not in _lib.TRACKING:
            raise AssertionError(
                "Values describing tracking system must be None for no tracking,"
                "'horizontal' for 1-axis horizontal tracking,"
                "tilted_horizontal' for 1-axis horizontal tracking of tilted panle,"
                "vertical' for 1-axis vertical tracking, or 'dual' for 2-axis tracking"
            )
        lon_r = DataArray(np.radians(lon), {"x": _coord(ds, "x")}, ("x",), "lon")
        lat_r = DataArray(np.radians(lat), {"y": _coord(ds, "y")}, ("y",), "lat")
        o = orientation(lon_r, lat_r, None)

        def table(v, nm):
            """slope / azimuth of the callback (pv/orientation.py:107) -> scalar, (y,) or (y, x)."""
            if hasattr(v, "dims") and hasattr(v, "transpose") and getattr(v, "ndim", 0) >= 1:
                dims = tuple(v.dims)
                if not set(dims) <= {"y", "x"}:
                    raise NotImplementedError(
                        f"orientation {nm} varies along {dims}; only (y, x)-dependent orientations are "
                        "supported (the orientation may not depend on time / the solar position)")
                v = v.transpose(*[d for d in ("y", "x") if d in dims])
                arr = np.asarray(v.values, dtype=np.float64)
                return arr[None, :] * np.ones((ny, 1)) if dims == ("x",) else arr
            arr = np.asarray(getattr(v, "values", v), dtype=np.float64)
            if arr.ndim == 0 or arr.shape == (ny,) or arr.shape == (ny, nx):
                return arr
            if arr.shape == (nx,):
                return arr[None, :] * np.ones((ny, 1))
            raise NotImplementedError(
                f"orientation {nm} must be a scalar, vary with latitude (y), or be a (y, x) array; "
                f"got shape {arr.shape}")

        slope, azimuth = table(o["slope"], "slope"), table(o["azimuth"], "azimuth")

        # TiltedIrradiation inputs (pv/irradiation.py:202-213)
        if raw:  # derived in-kernel from ssrd / ssr / tisr / fdir as era5.prepare derives them
            irr_branch, clearsky, albedo_src = _lib.IRR_ERA5_RAW, 0, _lib.ALBEDO_VAR
        elif _has(ds, "influx"):
            irr_branch = _lib.IRR_INFLUX
            cm = clearsky_model
            if cm is None:
                cm = "enhanced" if _has(ds, "temperature") and _has(ds, "humidity") else "simple"
            if cm not in _lib.CLEARSKY:
                raise KeyError("`clearsky model` must be chosen from 'simple' and 'enhanced'")
            clearsky = _lib.CLEARSKY[cm]
        elif _has(ds, "influx_direct") and _has(ds, "influx_diffuse"):
            irr_branch, clearsky = _lib.IRR_DIRECT_DIFFUSE, 0
        else:
            raise AssertionError(
                "Need either influx or influx_direct and influx_diffuse in the "
                "dataset. Check your cutout and dataset module."
            )
        if raw:  # (the albedo is derived from ssrd / ssr)
            pass
        elif _has(ds, "albedo"):
            albedo_src = _lib.ALBEDO_VAR
        elif _has(ds, "outflux"):
            albedo_src = _lib.ALBEDO_OUTFLUX
        else:
            raise AssertionError(
                "Need either albedo or outflux as a variable in the dataset. "
                "Check your cutout and dataset module."
            )
        trigon = _lib.TRIGON_SIMPLE if trigon_model == "simple" else _lib.TRIGON_HAY_DAVIES

        # operator field slot -> dataset variable
        src = {"temperature": _var(ds, "temperature")}
        names = ["influx_toa", "temperature"]
        if output in ("total", "direct", "diffuse", "ground") and not _has(ds, src["temperature"]):
            names = ["influx_toa"]  # irradiation needs no temperature (convert.py:748-767)
        if raw:  # the slots of ATL_IRR_ERA5_RAW (include/atlite_b200.h)
            src.update(influx_toa="tisr", influx_direct="fdir", influx="ssrd", outflux="ssr")
            names += ["influx_direct", "influx", "outflux"]
        else:
            names += ["influx"] if irr_branch == _lib.IRR_INFLUX else ["influx_direct", "influx_diffuse"]
            if irr_branch == _lib.IRR_INFLUX and clearsky == 1:
                names.append("humidity")
            names.append("albedo" if albedo_src == _lib.ALBEDO_VAR else "outflux")
        self.fields = {n: _raw(ds, src.get(n, n)) for n in names}
        self.fields.update(solar)
        self.fields.setdefault("temperature", self.fields["influx_toa"])  # unused placeholder
        self.pitch = engine.pitch_of(self.fields.values(), nx)
        self.op = engine.PvOp(
            ny=ny, nx=nx, time=self.time_labels, lon=lon, lat=lat, slope=slope, azimuth=azimuth,
            tracking=tracking, trigon_model=trigon, clearsky_model=clearsky,
            irr_branch=irr_branch, albedo_src=albedo_src, solar_src=solar_src, panel=panel,
            output=output, thermal=thermal, pitch=self.pitch, time_shift="-30min" if raw else "0h",
        )

    def reduce(self, plan):
        return self.op.reduce(plan, self.fields)

    def job(self, plan):
        return engine.StreamJob(self.op, plan, self.fields)

    def cells(self, timesum=False):
        return self.op.cells(self._device_fields(self.fields), timesum=timesum)


class _IrradiationSpec(_PvSpec):
    """convert_irradiation (convert.py:748-767): the PV operator without the panel."""

    units = "W m**-2"

    def __init__(self, ds, orientation, tracking=None, irradiation="total", trigon_model="simple",
                 clearsky_model="simple"):
        if irradiation not in ("total", "direct", "diffuse", "ground"):
            raise ValueError(f"irradiation must be total, direct, diffuse or ground, not {irradiation!r}")
        super().__init__(ds, None, orientation, tracking, trigon_model, clearsky_model, output=irradiation)
        self.name = f"{irradiation} tilted"


class _SolarThermalSpec(_PvSpec):
    """convert_solar_thermal (convert.py:550-573)."""

    def __init__(self, ds, orientation, trigon_model, clearsky_model, c0, c1, t_store):
        super().__init__(ds, None, orientation, None, trigon_model, clearsky_model,
                         output="solar_thermal", thermal=(c0, c1, t_store))
        self.name = None


class _PointwiseSpec(_Spec):
    """Pointwise function of one (time, y, x) variable."""

    def __init__(self, ds, var, shift=0.0, nan_to_zero=False, poly=None, cell_scale=None, name=None,
                 clip_min_zero=False):
        ny, nx = _grid_shape(ds)
        if not _has(ds, var):
            raise KeyError(var)
        self.field = _raw(ds, var)
        self.time_labels = pd.DatetimeIndex(_coord(ds, "time"))
        self.name = name
        self.pitch = engine.pitch_of([self.field], nx)
        kw = {"clip_min_zero": True} if clip_min_zero else {}
        self.op = engine.PointwiseOp(ny=ny, nx=nx, shift=shift, nan_to_zero=nan_to_zero, poly=poly,
                                     cell_scale=cell_scale, pitch=self.pitch, **kw)

    def reduce(self, plan):
        return self.op.reduce(plan, self.field)

    def job(self, plan):
        return engine.StreamJob(self.op, plan, self.field)

    def cells(self, timesum=False):
        f = self._device_fields({"f": self.field})
        return self.op.cells(f["f"], timesum=timesum)


def _temperature_spec(ds):
    return _PointwiseSpec(ds, _var(ds, "temperature"), shift=-273.15, name="temperature")


def _soil_temperature_spec(ds):
    return _PointwiseSpec(ds, _var(ds, "soil temperature"), shift=-273.15, nan_to_zero=True, name="soil temperature")


def _dewpoint_temperature_spec(ds):
    return _PointwiseSpec(ds, _var(ds, "dewpoint temperature"), shift=-273.15, name="dewpoint temperature")


def _cop_spec(ds, source, sink_T, c0, c1, c2):
    assert source in ["air", "soil"], NotImplementedError("'source' must be one of  ['air', 'soil']")
    if source == "air":  # convert.py:343-350
        d = (6.81, -0.121, 0.000630)
        var, nz = "temperature", False
    else:  # convert.py:351-358
        d = (8.77, -0.150, 0.000734)
        var, nz = "soil temperature", True
    c0, c1, c2 = (dv if v is None else v for v, dv in zip((c0, c1, c2), d))
    return _PointwiseSpec(ds, _var(ds, var), shift=-273.15, nan_to_zero=nz, poly=(sink_T, c0, c1, c2))


def _runoff_spec(ds, weight_with_height=True, height=None):
    """``height``: the static height of the whole cutout when ``ds`` is one time part of it.  A raw
    ERA5 cutout (``ro``, no ``runoff``) is read directly: ``ro`` clipped at 0 as sanitize_runoff
    does (era5.py:241-246), weighted with ``height`` or, without it, ``z / g0``."""
    raw = _runoff_raw(ds)
    scale = None
    if weight_with_height:
        h = height
        if h is None and raw:
            h = _height(ds)
        elif h is None and _has(ds, "height"):
            h = _height(ds)
        if h is None:
            raise KeyError(
                "runoff(weight_with_height=True) needs the static 'height' variable (datasets/era5.py:65-81: "
                "geopotential z / g0); prepare the cutout with the 'height' feature "
                "(atlite_b200.era5.get_data_height) or pass weight_with_height=False"
            )
        scale = _to_host(h)
        if scale.ndim == 3:
            scale = scale[0]
        scale = np.ascontiguousarray(scale[:, : _grid_shape(ds)[1]])  # drop row padding
    if raw:
        return _PointwiseSpec(ds, "ro", cell_scale=scale, name="runoff", clip_min_zero=True)
    return _PointwiseSpec(ds, "runoff", cell_scale=scale, name="runoff")


class _CspSpec(_Spec):
    """convert_csp (convert.py:940-972)."""

    name = "specific generation"
    units = "kWh/kW_ref"

    def __init__(self, ds, installation):
        ny, nx = _grid_shape(ds)
        self.time_labels = pd.DatetimeIndex(_coord(ds, "time"))
        tech = installation["technology"]
        if tech not in _lib.CSP_TECH:
            raise ValueError(f'Unknown CSP technology option "{tech}".')
        # a raw ERA5 cutout: the kernel derives influx_direct from fdir, and the solar position is
        # the one era5.prepare would have stored (-30 min, era5.py:182-188), without the warning
        self.raw = _csp_raw(ds)
        solar = {}
        if _has(ds, "solar_azimuth") and _has(ds, "solar_altitude"):
            solar["solar_altitude"], solar["solar_azimuth"], solar_src = _stored_solar_position(ds)
        elif self.raw:
            solar_src = _lib.SOLAR_COMPUTED
        else:
            warnings.warn(_SOLAR_WARNING, DeprecationWarning)
            solar_src = _lib.SOLAR_COMPUTED
        eff = EfficiencyTable.from_any(installation["efficiency"])
        self.fields = {"influx_direct": _raw(ds, "fdir" if self.raw else "influx_direct"), **solar}
        self.pitch = engine.pitch_of(self.fields.values(), nx)
        self.op = engine.CspOp(
            ny=ny, nx=nx, time=self.time_labels, lon=_coord(ds, "lon").astype(np.float64),
            lat=_coord(ds, "lat").astype(np.float64), solar_src=solar_src,
            technology=_lib.CSP_TECH[tech], r_irradiance=installation["r_irradiance"],
            altitude=eff.altitude, azimuth=eff.azimuth, efficiency=eff.values, pitch=self.pitch,
            raw=self.raw, time_shift="-30min" if self.raw and solar_src == _lib.SOLAR_COMPUTED else "0h",
        )

    def reduce(self, plan):
        return self.op.reduce(plan, self.fields)

    def job(self, plan):
        return engine.StreamJob(self.op, plan, self.fields)

    def cells(self, timesum=False):
        return self.op.cells(self._device_fields(self.fields), timesum=timesum)


class _WindSpec(_Spec):
    name = "specific generation"
    units = "MWh/MWp"

    def __init__(self, ds, turbine, interpolation_method="logarithmic"):
        ny, nx = _grid_shape(ds)
        self.time_labels = pd.DatetimeIndex(_coord(ds, "time"))
        V, POW, hub_height, P = (turbine[k] for k in ("V", "POW", "hub_height", "P"))
        to_name = f"wnd{int(hub_height):0d}m"
        aux = None
        from_height = hub_height
        self.raw = _wind_raw_fields(ds, hub_height, interpolation_method)
        if self.raw is not None:
            # raw ERA5 u100 / v100 (+ fsr | u10, v10): the speed, roughness and shear exponent are
            # derived in-kernel; era5.prepare stores wnd100m only, so 100 m is the height to
            # extrapolate from, and a hub at 100 m is the fast lane
            method = _lib.WIND_NONE if int(hub_height) == 100 else (
                _lib.WIND_LOG if interpolation_method == "logarithmic" else _lib.WIND_POWER)
            from_height = 100
            wnd = None
        elif _has(ds, to_name):  # fast lane, wind.py:75-78
            method = _lib.WIND_NONE
            wnd = _raw(ds, to_name)
        else:
            names = list(ds.data_vars) if hasattr(ds, "data_vars") else list(ds)
            heights = np.asarray([int(s[3:-1]) for s in names if re.match(r"wnd\d+m", str(s))])
            if len(heights) == 0:
                raise AssertionError("Wind speed is not in dataset")
            from_height = heights[np.argmin(np.abs(heights - hub_height))]
            wnd = _raw(ds, f"wnd{int(from_height):0d}m")
            if interpolation_method == "logarithmic":
                if not _has(ds, "roughness"):
                    raise RuntimeError(
                        "The logarithmic interpolation method requires surface roughness (roughness);\n"
                        "make sure you choose a compatible dataset like ERA5"
                    )
                method, aux = _lib.WIND_LOG, _raw(ds, "roughness")
            elif interpolation_method == "power":
                if not _has(ds, "wnd_shear_exp"):
                    raise RuntimeError(
                        "The power law interpolation method requires a wind shear exponent (wnd_shear_exp);\n"
                        "make sure you choose a compatible dataset like ERA5 and update your cutout"
                    )
                method, aux = _lib.WIND_POWER, _raw(ds, "wnd_shear_exp")
            else:
                raise ValueError(
                    f"Interpolation method must be 'logarithmic' or 'power',  but is: {interpolation_method}"
                )
        self.wnd, self.aux = wnd, aux
        self.pitch = engine.pitch_of(list(self.raw.values()) if self.raw is not None else [wnd, aux], nx)
        self.op = engine.WindOp(
            ny=ny, nx=nx, V=np.asarray(V, float), POW_norm=np.asarray(POW, float) / P,
            method=method, from_height=from_height, to_height=hub_height, pitch=self.pitch,
        )

    def reduce(self, plan):
        if self.raw is not None:
            return self.op.reduce_raw(plan, self.raw)
        return self.op.reduce(plan, self.wnd, self.aux)

    def job(self, plan):
        if self.raw is not None:
            return engine.StreamJob(self.op, plan, self.raw, abi="wind_raw")
        return engine.StreamJob(self.op, plan, {"wnd": self.wnd, "aux": self.aux})

    def cells(self, timesum=False):
        if self.raw is not None:
            return self.op.cells_raw(self._device_fields(self.raw), timesum=timesum)
        f = self._device_fields({"wnd": self.wnd, "aux": self.aux})
        return self.op.cells(f["wnd"], f["aux"], timesum=timesum)


def _wind_raw_fields(ds, hub_height, interpolation_method):
    """The raw ERA5 variables wind reads when the dataset has no ``wnd{h}m`` variable: u100 and
    v100, plus fsr for the logarithmic law or u10 and v10 for the power law (none of these for a
    hub at 100 m).  None when a prepared wind speed exists or the raw set is incomplete."""
    names = list(ds.data_vars) if hasattr(ds, "data_vars") else list(ds)
    if any(re.match(r"wnd\d+m", str(s)) for s in names):
        return None
    need = ["u100", "v100"]
    if int(hub_height) != 100:  # (the fast lane reads wnd{int(hub_height)}m)
        if interpolation_method == "logarithmic":
            need.append("fsr")
        elif interpolation_method == "power":
            need += ["u10", "v10"]
        else:
            return None
    if not all(_has(ds, n) for n in need):
        return None
    return {n: _raw(ds, n) for n in need}


def day_bins(time, hour_shift):
    """Calendar-day bins of ``time + hour_shift`` (``resample(time="1D")``,
    convert.py:408-412).  Returns (day labels, offsets[n_days+1] into time)."""
    t = pd.DatetimeIndex(time) + pd.Timedelta(hours=hour_shift)
    if len(t) == 0:
        return pd.DatetimeIndex([]), np.zeros(1, dtype=np.int64)
    if not t.is_monotonic_increasing:
        raise ValueError("time axis must be sorted for the daily heat-demand bins")
    days = t.floor("D")
    labels = pd.date_range(days[0], days[-1], freq="D")
    offsets = np.searchsorted(days.values, labels.values, side="left")
    offsets = np.append(offsets, len(t)).astype(np.int64)
    return labels, offsets


class _HeatSpec(_Spec):
    name = "heat_demand"
    cooling = False

    def __init__(self, ds, threshold, a, constant, hour_shift):
        ny, nx = _grid_shape(ds)
        self.temp = _raw(ds, _var(ds, "temperature"))
        self.time_labels, self.day_start = day_bins(_coord(ds, "time"), hour_shift)
        self.pitch = engine.pitch_of([self.temp], nx)
        self.op = engine.HeatOp(ny=ny, nx=nx, threshold=threshold, a=a, constant=constant,
                                cooling=self.cooling, pitch=self.pitch)

    def reduce(self, plan):
        return self.op.reduce(plan, self.temp, self.day_start)

    def job(self, plan):
        return engine.StreamJob(self.op, plan, self.temp, day_start=self.day_start)

    def cells(self, timesum=False):
        f = self._device_fields({"t": self.temp})
        return self.op.cells(f["t"], self.day_start, timesum=timesum)


class _CoolingSpec(_HeatSpec):
    """convert_cooling_demand (convert.py:475-491): a * (Tmean - threshold)."""

    name = "cooling_demand"
    cooling = True


# --------------------------------------------------------------------------
# convert_* callables (plugin protocol, convert.py:198)
# --------------------------------------------------------------------------


def _wrap_cells(ds, spec, values):
    coords = {"time": spec.time_labels, "y": _coord(ds, "y"), "x": _coord(ds, "x")}
    attrs = {"units": spec.units} if spec.units else {}
    return make_dataarray(_to_host(values), ("time", "y", "x"), coords, attrs, spec.name)


def convert_pv(ds, panel, orientation, tracking=None, trigon_model="simple", clearsky_model="simple"):
    """Per-cell PV capacity factors (time, y, x); convert.py:840-854."""
    spec = _PvSpec(ds, panel, orientation, tracking, trigon_model, clearsky_model)
    return _wrap_cells(ds, spec, spec.cells())


def convert_wind(ds, turbine, interpolation_method="logarithmic"):
    """Per-cell wind capacity factors (time, y, x); convert.py:634-662."""
    spec = _WindSpec(ds, turbine, interpolation_method)
    return _wrap_cells(ds, spec, spec.cells())


def convert_heat_demand(ds, threshold, a, constant, hour_shift):
    """Per-cell daily heat demand (day, y, x); convert.py:405-418."""
    spec = _HeatSpec(ds, threshold, a, constant, hour_shift)
    return _wrap_cells(ds, spec, spec.cells())


def convert_irradiation(ds, orientation, tracking=None, irradiation="total", trigon_model="simple",
                        clearsky_model="simple"):
    """Per-cell tilted irradiation (time, y, x); convert.py:748-767."""
    spec = _IrradiationSpec(ds, orientation, tracking, irradiation, trigon_model, clearsky_model)
    return _wrap_cells(ds, spec, spec.cells())


def convert_solar_thermal(ds, orientation, trigon_model, clearsky_model, c0, c1, t_store):
    """Per-cell solar thermal collector output; convert.py:550-573."""
    spec = _SolarThermalSpec(ds, orientation, trigon_model, clearsky_model, c0, c1, t_store)
    return _wrap_cells(ds, spec, spec.cells())


def convert_temperature(ds):
    """Outside temperature in deg C; convert.py:292-298."""
    spec = _temperature_spec(ds)
    return _wrap_cells(ds, spec, spec.cells())


def convert_soil_temperature(ds):
    """Soil temperature in deg C, 0 over sea; convert.py:306-316."""
    spec = _soil_temperature_spec(ds)
    return _wrap_cells(ds, spec, spec.cells())


def convert_dewpoint_temperature(ds):
    """Dewpoint temperature in deg C; convert.py:324-329."""
    spec = _dewpoint_temperature_spec(ds)
    return _wrap_cells(ds, spec, spec.cells())


def convert_coefficient_of_performance(ds, source, sink_T, c0, c1, c2):
    """Heat pump COP; convert.py:338-366."""
    spec = _cop_spec(ds, source, sink_T, c0, c1, c2)
    return _wrap_cells(ds, spec, spec.cells())


def convert_cooling_demand(ds, threshold, a, constant, hour_shift):
    """Per-cell daily cooling demand; convert.py:475-491."""
    spec = _CoolingSpec(ds, threshold, a, constant, hour_shift)
    return _wrap_cells(ds, spec, spec.cells())


def convert_csp(ds, installation):
    """Per-cell CSP specific generation; convert.py:940-972."""
    spec = _CspSpec(ds, installation)
    return _wrap_cells(ds, spec, spec.cells())


def convert_runoff(ds, weight_with_height=True):
    """Runoff (optionally weighted with height); convert.py:1028-1034."""
    spec = _runoff_spec(ds, weight_with_height)
    return _wrap_cells(ds, spec, spec.cells())


_SPECS = {
    "convert_pv": _PvSpec, "convert_wind": _WindSpec, "convert_heat_demand": _HeatSpec,
    "convert_irradiation": _IrradiationSpec, "convert_solar_thermal": _SolarThermalSpec,
    "convert_temperature": _temperature_spec, "convert_soil_temperature": _soil_temperature_spec,
    "convert_dewpoint_temperature": _dewpoint_temperature_spec,
    "convert_coefficient_of_performance": _cop_spec, "convert_cooling_demand": _CoolingSpec,
    "convert_runoff": _runoff_spec, "convert_csp": _CspSpec,
}


# identity -> spec: this package's own convert_* objects ...
_REGISTRY = {globals()[_n]: _s for _n, _s in _SPECS.items()}


def _reference_registry():
    """... plus the reference's, when the caller has imported it (``atlite.convert``
    in sys.modules): a script written against the reference passes
    ``atlite.convert.convert_pv`` etc. as ``convert_func``."""
    import sys

    mod = sys.modules.get("atlite.convert")
    if mod is None:
        return {}
    return {getattr(mod, n): s for n, s in _SPECS.items() if callable(getattr(mod, n, None))}


def _known_spec(convert_func):
    """Fused operator for a KNOWN converter, matched by identity (never by name: a user
    plugin that happens to be called ``convert_pv`` keeps the plugin protocol)."""
    try:
        spec = _REGISTRY.get(convert_func)
        return spec if spec is not None else _reference_registry().get(convert_func)
    except TypeError:  # unhashable callable
        return None


# --------------------------------------------------------------------------
# time-partitioned execution: several GPUs from one process, lazily loaded cutouts
# --------------------------------------------------------------------------


PART_BYTES = 1 << 30  # input bytes per time part of a lazily loaded cutout


def _time_slice(ds, lo, hi):
    """Steps [lo, hi) of a cutout dataset (views for in-memory data; for a dask-backed
    xarray dataset still lazy: only these steps are read when the part is converted)."""
    if hasattr(ds, "isel_time"):
        return ds.isel_time(lo, hi)
    return ds.isel(time=slice(lo, hi))


def _bytes_per_step(ds):
    ny, nx = _grid_shape(ds)
    names = list(ds.data_vars) if hasattr(ds, "data_vars") else list(ds)
    if hasattr(ds, "dims_of"):
        n3 = sum(1 for n in names if len(ds.dims_of(n)) == 3)
    else:
        n3 = sum(1 for n in names if len(ds[n].dims) == 3)  # xarray: metadata only, nothing is read
    return max(1, n3) * ny * nx * 4


def _is_host_resident(ds):
    """No variable lives on a GPU (device-resident cutouts are single-device objects)."""
    if not hasattr(ds, "raw") or getattr(ds, "lazy", False):
        return True
    return not any(engine._is_torch(ds.raw(n)) and ds.raw(n).is_cuda for n in ds.keys())


def _partition(ds, n_time, devices, lazy, day_offsets=None):
    """Contiguous time parts [(lo, hi, device)], in time order.  In-memory cutouts get one
    part per device; lazily loaded ones (dask-backed) parts of ~1 GiB of input, cut on the
    dataset's own time chunks (cutout.py:143: {"time": 100}), so a cutout that does not
    fit the host memory streams through it.  ``day_offsets`` (heat / cooling demand):
    part boundaries are snapped to calendar-day starts of the shifted axis."""
    from .dist import shard_bounds

    n_dev = len(devices)
    if n_time == 0:
        return [(0, 0, devices[0])]
    cuts = [0]
    if lazy:
        unit = 100
        try:
            ch = ds.chunks.get("time") if hasattr(ds.chunks, "get") else None
            if ch:
                unit = max(1, int(ch[0]))
        except Exception:  # noqa: BLE001
            pass
        k = max(1, int(round(PART_BYTES / (unit * _bytes_per_step(ds)))))
        per_dev = [shard_bounds(n_time, n_dev, r, align=unit) for r in range(n_dev)]
        for lo, hi in per_dev:
            for c in range(lo + unit * k, hi, unit * k):
                cuts.append(c)
            if hi > cuts[-1]:
                cuts.append(hi)
        owner_of = lambda lo: next(devices[r] for r, (a, b) in enumerate(per_dev) if a <= lo < b)  # noqa: E731
    else:
        per_dev = [shard_bounds(n_time, n_dev, r) for r in range(n_dev)]
        cuts += [hi for lo, hi in per_dev if hi > lo]
        owner_of = lambda lo: next(devices[r] for r, (a, b) in enumerate(per_dev) if a <= lo < b)  # noqa: E731
    if day_offsets is not None:  # snap to day starts (first step of a day of the shifted axis)
        offs = np.asarray(day_offsets)
        snapped = sorted({int(offs[np.argmin(np.abs(offs - c))]) for c in cuts[1:-1]} | {0, n_time})
        cuts = snapped
    cuts = sorted(set(cuts))
    return [(lo, hi, owner_of(min(lo, n_time - 1))) for lo, hi in zip(cuts[:-1], cuts[1:]) if hi > lo]


def _whole_cutout_kwds(spec_cls, ds, convert_kwds):
    """Inputs a time part's spec must take from the whole cutout, not from its part: the height a
    raw cutout's runoff derives from the first step of a time-dependent geopotential ``z``."""
    if (spec_cls is _runoff_spec and convert_kwds.get("weight_with_height", True) and _runoff_raw(ds)
            and convert_kwds.get("height") is None):
        h = _height(ds)
        return {} if h is None else {"height": _to_host(h)}
    return {}


def _run_partitioned(ds, spec_cls, convert_kwds, parts, run, workers_per_device):
    """Convert every time part on its device and return the per-part results in time order:
    ``_run_parts`` with one spec, ``spec_cls(part, **convert_kwds)``, whose per-part work is
    ``run(spec, device) -> result``."""
    return _run_parts(ds, lambda part: [lambda: spec_cls(part, **convert_kwds)], parts,
                      lambda specs, dev: [run(specs[0], dev)], workers_per_device)[0]


def _run_parts(ds, make, parts, run, workers_per_device):
    """Convert every time part on its device (one host thread per device, two for lazily
    loaded data so that reading part i+1 overlaps the GPU work on part i).  Each part is loaded
    once (one ``_time_slice``), and ``make(part)`` returns one builder per spec that reads it;
    ``run(specs, device)`` does the part's work and returns one result per spec.  Returns, per spec,
    its per-part (result, labels) in time order.  Warnings are re-issued by the caller's thread,
    each once per spec that raised it while being built (once in all for the others)."""
    from concurrent.futures import ThreadPoolExecutor

    torch = engine._torch()
    devices = sorted({d for _, _, d in parts})
    pools = {d: ThreadPoolExecutor(workers_per_device, thread_name_prefix=f"atl-dev{d}") for d in devices}
    caught = warnings.catch_warnings()  # restores the filters and showwarning on exit
    caught.__enter__()
    warnings.simplefilter("always")
    log = []  # (spec whose building raised it, or None; the warning)
    building = threading.local()  # the spec this thread is building, if any

    def record(message, category, filename, lineno, file=None, line=None):
        # a warning is shown on the thread that raised it, so the owner is exact
        log.append((getattr(building, "spec", None), warnings.WarningMessage(message, category, filename, lineno)))

    warnings.showwarning = record

    def work(lo, hi, dev):
        torch.cuda.set_device(dev)  # per-thread current device
        specs = []
        for k, build in enumerate(make(_time_slice(ds, lo, hi))):
            building.spec = k
            try:
                specs.append(build())
            finally:
                building.spec = None
        res = run(specs, dev)
        # only the labels travel on: the spec owns the part's input (up to PART_BYTES of decoded
        # fields, or its device copy), which must not outlive the part -- a lazily loaded cutout
        # larger than the host memory is the point of converting part by part
        return [(r, types.SimpleNamespace(units=getattr(sp_, "units", None), name=sp_.name,
                                          time_labels=sp_.time_labels)) for r, sp_ in zip(res, specs)]

    try:
        futs = [pools[d].submit(work, lo, hi, d) for lo, hi, d in parts]
        out = [f.result() for f in futs]
    finally:
        for p in pools.values():
            p.shutdown(wait=True)
        caught.__exit__(None, None, None)
    one = len(out[0]) == 1 if out else True
    seen = set()
    for owner, w in log:
        key = (0 if one else owner, w.category, str(w.message))
        if key not in seen:
            seen.add(key)
            warnings.warn_explicit(w.message, w.category, w.filename, w.lineno)
    return [[part[k] for part in out] for k in range(len(out[0]))] if out else []


def _concat_parts(res):
    """Per-part (result, labels) of one spec -> (results concatenated along time, time labels, name)."""
    time_labels = pd.Index(np.concatenate([np.asarray(sp_.time_labels) for _, sp_ in res]))
    if isinstance(res[0][1].time_labels, pd.DatetimeIndex):
        time_labels = pd.DatetimeIndex(time_labels)
    return np.concatenate([v for v, _ in res], axis=0), time_labels, res[0][1].name


# --------------------------------------------------------------------------
# orchestration
# --------------------------------------------------------------------------


def _aggregate_time_np(values, method, axis):
    if method == "sum":
        return np.nansum(values, axis=axis)
    if method == "mean":
        return np.nanmean(values, axis=axis)
    return values


def _finish_results(res, caps, agg, bus_major):
    """The tail of convert_and_aggregate (convert.py:259-271) on a (time, bus) float32 result:
    float64, ``/ capacity.where(capacity != 0)`` then ``fillna(0)`` when ``caps`` is given
    (per_unit), time aggregation (``agg`` = "sum" / "mean", NaN-skipping like xarray's) or the
    (bus, time) layout of NumPy-backed cutouts.  A device result is finished ON the device --
    for a year x 3000 buses these are four passes over 210 MB and a strided transpose that cost
    the host several times the conversion kernel -- and only the final array crosses PCIe."""
    if engine._is_torch(res):
        torch = engine._torch()
        r = res.to(torch.float64)
        if caps is not None:
            c = torch.as_tensor(np.where(caps != 0, caps, np.nan), dtype=torch.float64, device=r.device)
            r = r / c[None, :]
            r = torch.where(torch.isnan(r), torch.zeros((), dtype=r.dtype, device=r.device), r)
        if agg == "sum":
            r = torch.nansum(r, dim=0)
        elif agg == "mean":
            r = torch.nanmean(r, dim=0)
        elif bus_major:
            r = r.T.contiguous()
        return r.cpu().numpy()
    results = np.asarray(res).astype(np.float64)
    if caps is not None:
        with np.errstate(divide="ignore", invalid="ignore"):
            results = results / np.where(caps != 0, caps, np.nan)[None, :]
        results = np.where(np.isnan(results), 0.0, results)
    if agg is not None:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)  # mean of an all-NaN column is NaN, silently
            return _aggregate_time_np(results, agg, 0)
    return np.ascontiguousarray(results.T) if bus_major else results


def _ensure_index(index, n):
    """utils.py:22-36 ensure_coords: pandas Index -> (dim name, Index)."""
    if index is None:
        index = pd.RangeIndex(n)
    if isinstance(index, pd.MultiIndex):
        return index.name or "dim_0", index
    if isinstance(index, pd.Index):
        return index.name or "dim_0", index
    if HAVE_XARRAY and isinstance(index, xr.Coordinates):
        if len(index.dims) > 1:
            raise ValueError(f"index must have a single dimension, not: {index.dims}")
        d = list(index.dims)[0]
        return d, index.to_index()
    raise ValueError(f"index must be a pandas index or xarray coordinates, not: {index}")


def _layout_values(layout, ds):
    """layout.reindex_like(cutout.data).stack(spatial=[y, x])  (convert.py:244)."""
    y, x = _coord(ds, "y"), _coord(ds, "x")
    if HAVE_XARRAY and isinstance(layout, xr.DataArray):
        lay = layout.reindex(y=y, x=x).transpose("y", "x")
        return np.asarray(lay.values, dtype=np.float64).reshape(-1)
    lay = layout.transpose("y", "x")
    iy = pd.Index(np.asarray(lay.coords["y"])).get_indexer(y)
    ix = pd.Index(np.asarray(lay.coords["x"])).get_indexer(x)
    vals = np.asarray(lay.values, dtype=np.float64)
    out = vals[np.clip(iy, 0, None)][:, np.clip(ix, 0, None)]
    out[iy < 0, :] = np.nan
    out[:, ix < 0] = np.nan
    return out.reshape(-1)


def scale_columns(matrix, lay):
    """``csr_matrix(matrix) * spdiag(lay)`` (convert.py:249): column j scaled by lay[j].

    Done on the entries directly (6 ms instead of the 44 ms sparse product at 1440 x 720 ->
    3000 shapes).  The sparse product stores no entry whose value is 0 -- a layout 0, or a
    stored 0 of ``matrix`` -- so neither does this: a CSR reduce multiplies every stored entry,
    and a stored 0 on a NaN cell (ERA5 soil temperature over the sea, where layouts are 0)
    would make its bus NaN where the reference's is finite."""
    if engine._is_torch(matrix):
        return _scale_columns_device(matrix, lay)
    m0 = sp.csr_matrix(matrix)
    if not m0.has_canonical_format:  # the product sums duplicates (a +w / -w pair is no entry)
        m0 = m0.copy()
        m0.sum_duplicates()
    data = m0.data.astype(np.float64) * lay[m0.indices]
    if (data != 0).all():
        return sp.csr_matrix((data, m0.indices, m0.indptr), shape=m0.shape)
    m = sp.csr_matrix((data, m0.indices.copy(), m0.indptr.copy()), shape=m0.shape)  # m0's arrays may be the caller's
    m.eliminate_zeros()
    return m


def _scale_columns_device(m, lay):
    """``scale_columns`` of a canonical CUDA ``torch.sparse_csr`` matrix, on its device: the same
    float64 products, and the entries that become 0 dropped."""
    torch = engine._torch()
    crow, col = m.crow_indices(), m.col_indices()
    data = m.values().to(torch.float64) * torch.as_tensor(lay, dtype=torch.float64, device=m.device)[col]
    keep = data != 0
    if bool(keep.all()):
        return torch.sparse_csr_tensor(crow, col, data, m.shape)
    rows = torch.repeat_interleave(torch.arange(m.shape[0], device=m.device), crow.diff())
    counts = torch.bincount(rows[keep], minlength=m.shape[0])
    crow = torch.cat([counts.new_zeros(1), counts.cumsum(0)]).to(col.dtype)
    return torch.sparse_csr_tensor(crow, col[keep], data[keep], m.shape)


def _row_sums(matrix):
    """``matrix.sum(-1)`` as scipy computes it.  A CUDA matrix is summed by scipy too, after a copy
    to the host: NumPy adds a row's entries in blocks (``np.add.reduceat``), and the capacity is
    meant to be the scipy path's bit for bit."""
    if engine._is_torch(matrix):
        matrix = sp.csr_matrix((matrix.values().cpu().numpy(), matrix.col_indices().cpu().numpy(),
                                matrix.crow_indices().cpu().numpy()), shape=tuple(matrix.shape))
    return np.asarray(matrix.sum(-1)).flatten()


def _resolve_aggregate_time(aggregate_time, capacity_factor, capacity_factor_timeseries, stacklevel):
    """``aggregate_time`` after the deprecated flags, with their warnings (``stacklevel``: that of
    the caller of the public call)."""
    if aggregate_time not in ("sum", "mean", "legacy", None):
        raise ValueError(
            f"aggregate_time must be 'sum', 'mean', 'legacy', or None, got {aggregate_time!r}"
        )
    if aggregate_time == "legacy":
        warnings.warn(
            "aggregate_time='legacy' is deprecated and will be removed in a "
            "future release. Pass 'sum', 'mean', or None explicitly.",
            FutureWarning,
            stacklevel=stacklevel,
        )
    if capacity_factor or capacity_factor_timeseries:
        if aggregate_time != "legacy":
            raise ValueError(
                "Cannot use 'aggregate_time' together with deprecated "
                "'capacity_factor' or 'capacity_factor_timeseries'."
            )
        if capacity_factor:
            warnings.warn(
                "capacity_factor is deprecated. Use aggregate_time='mean' instead.",
                FutureWarning,
                stacklevel=stacklevel,
            )
            aggregate_time = "mean"
        if capacity_factor_timeseries:
            warnings.warn(
                "capacity_factor_timeseries is deprecated. Use aggregate_time=None instead.",
                FutureWarning,
                stacklevel=stacklevel,
            )
            aggregate_time = None
    return aggregate_time


def _resolve_matrix(cutout, ds, matrix, index, layout, shapes, shapes_crs):
    """``matrix``, ``shapes`` or ``layout`` (convert.py:213-254) as one CSR matrix -- scipy, or a
    CUDA tensor that stays on its device -- and the bus (dim, index)."""
    if matrix is not None:
        if shapes is not None:
            raise ValueError("Passing matrix and shapes is ambiguous. Pass only one of them.")
        if is_dataarray(matrix):
            coords = matrix.indexes[matrix.dims[1]].to_frame(index=False)
            if not np.array_equal(coords[["x", "y"]], cutout.grid[["x", "y"]]):
                raise ValueError(
                    "Matrix spatial coordinates not aligned with cutout spatial coordinates."
                )
            if index is None:
                index = matrix
            matrix = matrix.values
        if not matrix.ndim == 2:
            raise ValueError("Matrix not 2-dimensional.")
        # a CUDA matrix stays on the device; its plan is built there
        matrix = engine.device_csr(matrix) if engine._is_torch(matrix) else sp.csr_matrix(matrix)

    if shapes is not None:
        if isinstance(shapes, pd.Series) or hasattr(shapes, "geometry"):
            if index is None:
                index = shapes.index
        matrix = cutout.indicatormatrix(shapes, shapes_crs).tocsr()

    if layout is not None:
        assert is_dataarray(layout)
        lay = _layout_values(layout, ds)
        if matrix is None:
            matrix = sp.csr_matrix(lay[None, :])
        else:
            matrix = scale_columns(matrix, lay)

    assert isinstance(matrix, sp.csr_matrix) or engine._is_torch(matrix)
    dim, idx = _ensure_index(index, matrix.shape[0])
    return matrix, dim, idx


class _Request(types.SimpleNamespace):
    """One ``convert_and_aggregate`` call with its arguments resolved: ``convert_func``, its
    fused ``spec_cls`` (None for a plugin) and ``convert_kwds``; ``aggregate_time`` after the
    deprecated flags; ``per_unit`` / ``return_capacity``; and how the cutout runs: ``shard``,
    ``devices``, ``lazy`` and ``partitioned``.  ``aggregated`` requests also carry the CSR
    ``matrix`` and the bus ``dim`` / ``idx`` (``_Request.resolve_matrix``)."""

    @classmethod
    def resolve(cls, cutout, convert_func, per_unit, return_capacity, aggregate_time, capacity_factor,
                capacity_factor_timeseries, aggregated, convert_kwds, stacklevel):
        """Everything but the matrix: no GPU work."""
        aggregate_time = _resolve_aggregate_time(aggregate_time, capacity_factor, capacity_factor_timeseries,
                                                 stacklevel + 1)
        ds = cutout.data
        spec_cls = _known_spec(convert_func)
        shard = getattr(cutout, "time_shard", None)  # multi-GPU time sharding (dist.py)
        devices = list(getattr(cutout, "devices", None) or [])
        lazy = _is_dask_backed(ds)
        # several GPUs from this one process, and/or a lazily loaded (dask-backed) cutout that
        # is converted time part by time part instead of being materialised whole
        partitioned = spec_cls is not None and (len(devices) > 1 or lazy) and _is_host_resident(ds)
        if partitioned and shard is not None:
            raise ValueError("a cutout is either time-sharded across processes (time_shard=) or fanned "
                             "out to several devices by one process (devices=), not both")
        return cls(cutout=cutout, ds=ds, convert_func=convert_func, spec_cls=spec_cls,
                   convert_kwds=dict(convert_kwds), aggregate_time=aggregate_time, per_unit=per_unit,
                   return_capacity=return_capacity, aggregated=aggregated, shard=shard, devices=devices,
                   lazy=lazy, partitioned=partitioned, matrix=None, dim=None, idx=None)

    def check_per_cell(self):
        if not self.aggregated and (self.per_unit or self.return_capacity):
            raise ValueError(
                "One of `matrix`, `shapes` and `layout` must be "
                "given for `per_unit` or `return_capacity`"
            )

    def resolve_matrix(self, matrix, index, layout, shapes, shapes_crs):
        if self.aggregated:
            self.matrix, self.dim, self.idx = _resolve_matrix(self.cutout, self.ds, matrix, index, layout, shapes,
                                                              shapes_crs)

    def select_device(self):
        if len(self.devices) == 1 and not self.partitioned:
            engine._torch().cuda.set_device(self.devices[0])

    def parts(self):
        """The time parts of a partitioned run: [(lo, hi, device)], snapped to the day starts of a
        heat / cooling demand request's own day table."""
        n_time = len(_coord(self.ds, "time"))
        day_offsets = None
        if self.spec_cls in (_HeatSpec, _CoolingSpec):
            day_offsets = day_bins(_coord(self.ds, "time"), self.convert_kwds.get("hour_shift", 0.0))[1]
        return _partition(self.ds, n_time, self.devices or [engine.current_device()], self.lazy, day_offsets)

    def part_kwds(self):
        return dict(self.convert_kwds, **_whole_cutout_kwds(self.spec_cls, self.ds, self.convert_kwds))


def _run_cells(req, spec):
    """The per-cell result (no matrix, shapes or layout) of ``req``: values (time, y, x), or their
    time sum / mean (y, x).  ``spec``: the spec or the plugin's DataArray, None when partitioned."""
    ds, shard = req.ds, req.shard
    agg = "sum" if req.aggregate_time == "legacy" else req.aggregate_time
    coords_yx = {"y": _coord(ds, "y"), "x": _coord(ds, "x")}
    if req.partitioned:
        parts, wpd, kwds = req.parts(), 2 if req.lazy else 1, req.part_kwds()
        if agg is None:
            res = _run_partitioned(ds, req.spec_cls, kwds, parts, lambda sp_, dev: _to_host(sp_.cells()), wpd)
            sp0 = res[0][1]
            attrs = {"units": sp0.units} if sp0.units else {}
            labels = pd.Index(np.concatenate([np.asarray(sp_.time_labels) for _, sp_ in res]))
            vals = np.concatenate([v for v, _ in res], axis=0)
            return make_dataarray(vals, ("time", "y", "x"), {"time": labels, **coords_yx}, attrs, sp0.name)
        res = _run_partitioned(ds, req.spec_cls, kwds, parts,
                               lambda sp_, dev: tuple(_to_host(a).astype(np.float64) for a in sp_.cells_timesum()), wpd)
        sp0 = res[0][1]
        attrs = {"units": sp0.units} if sp0.units else {}
        total = sum(v[0] for v, _ in res)
        count = sum(v[1] for v, _ in res)
        if agg == "mean":
            with np.errstate(divide="ignore", invalid="ignore"):
                total = np.where(count > 0, total / count, np.nan)
        return make_dataarray(total, ("y", "x"), coords_yx, attrs, sp0.name)
    if req.spec_cls is None:
        da = spec
        if agg == "sum":
            return da.sum("time", keep_attrs=True)
        if agg == "mean":
            return da.mean("time", keep_attrs=True)
        return da
    attrs = {"units": spec.units} if spec.units else {}
    if agg is None:
        vals = _to_host(spec.cells())
        labels = spec.time_labels
        if shard is not None:
            vals, labels = shard.gather_time(vals, labels)
        return make_dataarray(vals, ("time", "y", "x"), {"time": labels, **coords_yx}, attrs, spec.name)
    # NaN-skipping time sum and the number of valid steps per cell (da.sum / da.mean
    # over "time" skip NaN, convert.py:51-56; an all-NaN cell has mean NaN, sum 0)
    total, count = spec.cells_timesum()
    if shard is not None:
        total, count = shard.sum_planes(total, count)
    vals = _to_host(total).astype(np.float64)
    if agg == "mean":
        cnt = _to_host(count).astype(np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            vals = np.where(cnt > 0, vals / cnt, np.nan)
    return make_dataarray(vals, ("y", "x"), coords_yx, attrs, spec.name)


def _run_reduce(req, spec):
    """The (time, bus) float32 result of an aggregated ``req``, its time labels and its name.
    ``spec``: the spec or the plugin's DataArray, None when partitioned."""
    ds, matrix = req.ds, req.matrix
    ny, nx = _grid_shape(ds)
    if req.partitioned:
        digest = None if engine._is_torch(matrix) else engine.matrix_digest(matrix)
        res = _run_partitioned(
            ds, req.spec_cls, req.part_kwds(), req.parts(),
            lambda sp_, dev: _to_host(sp_.reduce(engine.get_plan(matrix, ny, nx, device=dev, pitch=sp_.pitch,
                                                                 digest=digest))), 2 if req.lazy else 1)
        res, time_labels, name = _concat_parts(res)
    elif req.spec_cls is not None:
        plan = engine.get_plan(matrix, ny, nx, pitch=spec.pitch)
        res = spec.reduce(plan)  # (time, bus) float32
        time_labels, name = spec.time_labels, spec.name
    else:
        da = spec
        pitch = None
        vals0 = da if engine._is_torch(da) else getattr(da, "values", da)
        if engine._is_torch(vals0) and vals0.ndim == 3 and vals0.shape[-1] != nx:
            pitch = int(vals0.shape[-1])  # plugin result computed from a row-padded device cutout
        plan = engine.get_plan(matrix, ny, nx, pitch=pitch)
        vals = da if engine._is_torch(da) else getattr(da, "values", da)
        res = plan.spmm(np.asarray(vals) if not engine._is_torch(vals) else vals)
        time_labels = pd.Index(np.asarray(da.coords["time"])) if hasattr(da, "coords") else pd.RangeIndex(len(vals))
        name = getattr(da, "name", None)
    if req.shard is not None:
        res, time_labels = req.shard.gather_time(res, time_labels)
    return res, time_labels, name


def _finish(req, res, time_labels, name):
    """Labelled result (and capacity) of an aggregated ``req`` from its (time, bus) result."""
    capacity = caps = None
    if req.per_unit or req.return_capacity:
        caps = _row_sums(req.matrix)
        capacity = make_dataarray(caps, (req.dim,), {req.dim: req.idx}, {"units": "MW"})
    units = "p.u." if req.per_unit else "MW"
    dim, idx = req.dim, req.idx

    # dim order mirrors aggregate.py: (time, bus) for dask-backed cutouts
    # (:24-32), (bus, time) for NumPy-backed ones (:34-35)
    agg = req.aggregate_time if req.aggregate_time != "legacy" else None
    bus_major = agg is None and not _is_dask_backed(req.ds)
    results = _finish_results(res, caps if req.per_unit else None, agg, bus_major)
    if agg is not None:
        out = make_dataarray(results, (dim,), {dim: idx}, {"units": units}, name)
    elif not bus_major:
        out = make_dataarray(results, ("time", dim), {"time": time_labels, dim: idx}, {"units": units}, name)
    else:
        out = make_dataarray(results, (dim, "time"), {dim: idx, "time": time_labels}, {"units": units}, name)
    if req.return_capacity:
        return out, capacity
    return out


def _spec_of(req):
    """The spec of a request that is not partitioned (the plugin's DataArray for a plugin)."""
    if req.partitioned:
        return None
    if req.spec_cls is not None:
        return req.spec_cls(req.ds, **req.convert_kwds)
    return req.convert_func(req.ds, **req.convert_kwds)  # plugin protocol: the callable produces the field


def convert_and_aggregate(
    cutout,
    convert_func,
    matrix=None,
    index=None,
    layout=None,
    shapes=None,
    shapes_crs=4326,
    per_unit=False,
    return_capacity=False,
    aggregate_time="legacy",
    capacity_factor=False,
    capacity_factor_timeseries=False,
    show_progress=False,
    dask_kwargs={},
    **convert_kwds,
):
    """Convert and aggregate a weather-based renewable generation time-series.

    Same contract as the reference (convert.py:59-276): ``matrix`` (N x S, in
    ``cutout.grid`` order), ``shapes`` or ``layout`` select spatial
    aggregation; ``per_unit`` / ``return_capacity``; ``aggregate_time`` in
    {"sum", "mean", "legacy", None}; deprecated ``capacity_factor*`` flags.
    ``show_progress`` and ``dask_kwargs`` are accepted and ignored (the result
    is computed eagerly on the GPU and returned loaded).
    """
    aggregated = not all(v is None for v in [layout, shapes, matrix])
    req = _Request.resolve(cutout, convert_func, per_unit, return_capacity, aggregate_time, capacity_factor,
                           capacity_factor_timeseries, aggregated, convert_kwds, stacklevel=3)
    func_name = convert_func.__name__.replace("convert_", "")
    logger.info(f"Convert and aggregate '{func_name}'.")
    req.select_device()
    spec = _spec_of(req)
    req.check_per_cell()
    if not aggregated:
        return _run_cells(req, spec)
    req.resolve_matrix(matrix, index, layout, shapes, shapes_crs)
    return _finish(req, *_run_reduce(req, spec))


# --------------------------------------------------------------------------
# technology wrappers
# --------------------------------------------------------------------------
#
# Each wrapper resolves its own arguments into those of ``convert_and_aggregate`` with one helper
# (``_<wrapper>_kwds``), which ``convert_many`` calls too; the wrapper's signature holds the defaults.


def _heat_demand_kwds(threshold, a, constant, hour_shift, **params):
    return dict(convert_func=convert_heat_demand, threshold=threshold, a=a, constant=constant,
                hour_shift=hour_shift, **params)


def heat_demand(cutout, threshold=15.0, a=1.0, constant=0.0, hour_shift=0.0, **params):
    """Daily heat demand by the degree-day approximation (convert.py:421-471)."""
    return cutout.convert_and_aggregate(**_heat_demand_kwds(threshold, a, constant, hour_shift, **params))


def _wind_kwds(turbine, smooth, add_cutout_windspeed, interpolation_method, **params):
    turbine = get_windturbineconfig(turbine, add_cutout_windspeed=add_cutout_windspeed)
    if smooth:
        turbine = windturbine_smooth(turbine, params=smooth)
    return dict(convert_func=convert_wind, turbine=turbine, interpolation_method=interpolation_method, **params)


def wind(cutout, turbine, smooth=False, add_cutout_windspeed=False,
         interpolation_method="logarithmic", **params):
    """Wind generation time-series (convert.py:665-744)."""
    return cutout.convert_and_aggregate(
        **_wind_kwds(turbine, smooth, add_cutout_windspeed, interpolation_method, **params))


def _orientation(orientation):
    return orientation if callable(orientation) else get_orientation(orientation)


def _pv_kwds(panel, orientation, tracking, clearsky_model, **params):
    if isinstance(panel, (str, Path)):
        panel = get_solarpanelconfig(panel)
    return dict(convert_func=convert_pv, panel=panel, orientation=_orientation(orientation), tracking=tracking,
                clearsky_model=clearsky_model, **params)


def pv(cutout, panel, orientation, tracking=None, clearsky_model=None, **params):
    """PV generation time-series (convert.py:857-936)."""
    return cutout.convert_and_aggregate(**_pv_kwds(panel, orientation, tracking, clearsky_model, **params))


# --------------------------------------------------------------------------
# further technology wrappers on the same path (SURVEY.md section 8 f3)
# --------------------------------------------------------------------------


def _temperature_kwds(**params):
    return dict(convert_func=convert_temperature, **params)


def temperature(cutout, **params):
    """convert.py:301-302"""
    return cutout.convert_and_aggregate(**_temperature_kwds(**params))


def _soil_temperature_kwds(**params):
    return dict(convert_func=convert_soil_temperature, **params)


def soil_temperature(cutout, **params):
    """convert.py:319-320"""
    return cutout.convert_and_aggregate(**_soil_temperature_kwds(**params))


def _dewpoint_temperature_kwds(**params):
    return dict(convert_func=convert_dewpoint_temperature, **params)


def dewpoint_temperature(cutout, **params):
    """convert.py:332-335"""
    return cutout.convert_and_aggregate(**_dewpoint_temperature_kwds(**params))


def _coefficient_of_performance_kwds(source, sink_T, c0, c1, c2, **params):
    return dict(convert_func=convert_coefficient_of_performance, source=source, sink_T=sink_T, c0=c0, c1=c1,
                c2=c2, **params)


def coefficient_of_performance(cutout, source="air", sink_T=55.0, c0=None, c1=None, c2=None, **params):
    """Air- or ground-sourced heat pump COP (convert.py:369-401)."""
    return cutout.convert_and_aggregate(**_coefficient_of_performance_kwds(source, sink_T, c0, c1, c2, **params))


def _cooling_demand_kwds(threshold, a, constant, hour_shift, **params):
    return dict(convert_func=convert_cooling_demand, threshold=threshold, a=a, constant=constant,
                hour_shift=hour_shift, **params)


def cooling_demand(cutout, threshold=23.0, a=1.0, constant=0.0, hour_shift=0.0, **params):
    """Daily cooling demand by the degree-day approximation (convert.py:494-546)."""
    return cutout.convert_and_aggregate(**_cooling_demand_kwds(threshold, a, constant, hour_shift, **params))


def _solar_thermal_kwds(orientation, trigon_model, clearsky_model, c0, c1, t_store, **params):
    return dict(convert_func=convert_solar_thermal, orientation=_orientation(orientation),
                trigon_model=trigon_model, clearsky_model=clearsky_model, c0=c0, c1=c1, t_store=t_store, **params)


def solar_thermal(cutout, orientation={"slope": 45.0, "azimuth": 180.0}, trigon_model="simple",
                  clearsky_model="simple", c0=0.8, c1=3.0, t_store=80.0, **params):
    """Solar thermal collector time series (convert.py:576-630)."""
    return cutout.convert_and_aggregate(
        **_solar_thermal_kwds(orientation, trigon_model, clearsky_model, c0, c1, t_store, **params))


def _irradiation_kwds(orientation, irradiation, tracking, clearsky_model, **params):
    return dict(convert_func=convert_irradiation, orientation=_orientation(orientation), tracking=tracking,
                irradiation=irradiation, clearsky_model=clearsky_model, **params)


def irradiation(cutout, orientation, irradiation="total", tracking=None, clearsky_model=None, **params):
    """Total / direct / diffuse / ground irradiation on a tilted surface (convert.py:770-836)."""
    return cutout.convert_and_aggregate(
        **_irradiation_kwds(orientation, irradiation, tracking, clearsky_model, **params))


def _csp_kwds(installation, technology, **params):
    if isinstance(installation, (str, Path)):
        installation = get_cspinstallationconfig(installation)
    if technology is not None:
        installation = dict(installation, technology=technology)
    return dict(convert_func=convert_csp, installation=installation, **params)


def csp(cutout, installation, technology=None, **params):
    """CSP generation time-series from direct radiation (convert.py:975-1024)."""
    return cutout.convert_and_aggregate(**_csp_kwds(installation, technology, **params))


def _runoff_kwds(smooth, lower_threshold_quantile, normalize_using_yearly, **params):
    return dict(convert_func=convert_runoff, **params)


def runoff(cutout, smooth=None, lower_threshold_quantile=None, normalize_using_yearly=None, **params):
    """Runoff aggregated to buses with the reference's optional post-processing
    (rolling mean, lower-quantile cut, yearly normalisation; convert.py:1037-1084)."""
    result = cutout.convert_and_aggregate(
        **_runoff_kwds(smooth, lower_threshold_quantile, normalize_using_yearly, **params))
    return _runoff_post(result, smooth, lower_threshold_quantile, normalize_using_yearly)


def _runoff_post(result, smooth, lower_threshold_quantile, normalize_using_yearly):
    """runoff's post-processing of the ``convert_and_aggregate`` result."""
    res, cap = (result if isinstance(result, tuple) else (result, None))
    if "time" not in res.dims or (smooth is None and lower_threshold_quantile is None
                                  and normalize_using_yearly is None):
        return result
    tax = list(res.dims).index("time")
    vals = np.asarray(res.values, dtype=np.float64)
    if smooth is not None:
        if smooth is True:
            smooth = 24 * 7
        frame = pd.DataFrame(np.moveaxis(vals, tax, 0).reshape(vals.shape[tax], -1))
        sm = frame.rolling(smooth, min_periods=1).mean().values
        vals = np.moveaxis(sm.reshape(np.moveaxis(vals, tax, 0).shape), 0, tax)
    if lower_threshold_quantile is not None:
        if lower_threshold_quantile is True:
            lower_threshold_quantile = 5e-3
        lower = pd.Series(vals.ravel()).quantile(lower_threshold_quantile)
        vals = np.where(vals >= lower, vals, 0.0)
    if normalize_using_yearly is not None:
        idx = normalize_using_yearly.index
        idx = idx.year if isinstance(idx, pd.DatetimeIndex) else idx.astype(int)
        tyears = pd.DatetimeIndex(np.asarray(res.coords["time"])).year
        full = pd.Series(tyears).value_counts().loc[lambda x: x > 8700].index.intersection(idx)
        assert len(full), "Need at least a full year of data (more is better)"
        sel = (tyears >= min(full)) & (tyears <= max(full))
        norm = normalize_using_yearly.copy()
        norm.index = idx
        target = norm.loc[min(full):max(full)].sum()
        other = [d for d in res.dims if d != "time"][0]
        target = target.reindex(pd.Index(np.asarray(res.coords[other]))).values
        have = np.take(vals, np.flatnonzero(sel), axis=tax).sum(axis=tax)
        factor = target / have
        vals = vals * (factor[:, None] if tax == 1 else factor[None, :])
    out = make_dataarray(vals, tuple(res.dims), {d: np.asarray(res.coords[d]) for d in res.dims},
                         dict(res.attrs), getattr(res, "name", None))
    return (out, cap) if cap is not None else out


# --------------------------------------------------------------------------
# several conversions from one pass over the cutout
# --------------------------------------------------------------------------


# Cutout conversion method -> (the public call, the helper that resolves its arguments into those
# of convert_and_aggregate; None: they already are)
_CONVERSIONS = {
    "convert_and_aggregate": (convert_and_aggregate, None), "pv": (pv, _pv_kwds), "wind": (wind, _wind_kwds),
    "irradiation": (irradiation, _irradiation_kwds), "solar_thermal": (solar_thermal, _solar_thermal_kwds),
    "csp": (csp, _csp_kwds), "temperature": (temperature, _temperature_kwds),
    "soil_temperature": (soil_temperature, _soil_temperature_kwds),
    "dewpoint_temperature": (dewpoint_temperature, _dewpoint_temperature_kwds),
    "coefficient_of_performance": (coefficient_of_performance, _coefficient_of_performance_kwds),
    "heat_demand": (heat_demand, _heat_demand_kwds), "cooling_demand": (cooling_demand, _cooling_demand_kwds),
    "runoff": (runoff, _runoff_kwds),
}
_RUNOFF_POST = ("smooth", "lower_threshold_quantile", "normalize_using_yearly")


def _bind(func, *args, **kwargs):
    """The arguments ``func(*args, **kwargs)`` would get, defaults applied, found without calling
    it.  Arguments that do not bind raise TypeError, as the call would."""
    try:  # the signature Python binds a call against: not that of a function it wraps
        sig = inspect.signature(func, follow_wrapped=False)
    except (TypeError, ValueError):  # no signature to check against (a builtin plugin)
        return None
    try:
        ba = sig.bind(*args, **kwargs)
    except TypeError as e:
        raise TypeError(f"{getattr(func, '__qualname__', func)}(): {e}") from None
    ba.apply_defaults()
    var_kw = next((p.name for p in sig.parameters.values() if p.kind is p.VAR_KEYWORD), None)
    out = dict(ba.arguments)
    out.update(out.pop(var_kw, {}) if var_kw else {})
    return out


def _many_request(cutout, name, request):
    """One request of ``convert_many`` resolved as its own call resolves it, with its warnings and
    errors, and nothing sent to the GPU: (the ``_Request``, the arguments of its matrix, runoff's
    post-processing arguments or None)."""
    if not isinstance(request, Mapping):
        raise TypeError(f"request {name!r} must be a dict of 'method' and the method's keyword arguments, "
                        f"not {type(request).__name__}")
    kw = dict(request)
    if "method" not in kw:
        raise TypeError(f"request {name!r} has no 'method'")
    method = kw.pop("method")
    if method not in _CONVERSIONS:
        getattr(cutout, method)  # a name the cutout does not have raises the AttributeError of its call
        raise ValueError(f"request {name!r}: {method!r} is not a conversion method; one of "
                         f"{', '.join(_CONVERSIONS)}")
    call, helper = _CONVERSIONS[method]
    args = _bind(call, cutout, **kw)
    del args["cutout"]
    post = {k: args[k] for k in _RUNOFF_POST} if method == "runoff" else None
    ca = _bind(convert_and_aggregate, cutout, **(helper(**args) if helper else args))
    del ca["cutout"]
    matrix_args = [ca.pop(k) for k in ("matrix", "index", "layout", "shapes", "shapes_crs")]
    for k in ("show_progress", "dask_kwargs"):
        del ca[k]
    req = _Request.resolve(cutout, ca.pop("convert_func"), ca.pop("per_unit"), ca.pop("return_capacity"),
                           ca.pop("aggregate_time"), ca.pop("capacity_factor"), ca.pop("capacity_factor_timeseries"),
                           aggregated=any(v is not None for v in matrix_args[0:1] + matrix_args[2:4]),
                           convert_kwds=ca, stacklevel=4)
    _bind(req.spec_cls or req.convert_func, req.ds, **req.convert_kwds)
    req.check_per_cell()
    return req, matrix_args, post


def _run_own(req):
    """A request run as its own ``convert_and_aggregate`` call runs."""
    req.select_device()
    spec = _spec_of(req)
    if not req.aggregated:
        return _run_cells(req, spec)
    return _finish(req, *_run_reduce(req, spec))


def _run_shared(reqs):
    """The aggregated fused requests of a host-resident cutout on one device, from one pass of its
    fields (``engine.reduce_host_many``)."""
    reqs[0].select_device()
    ny, nx = _grid_shape(reqs[0].ds)
    specs = [_spec_of(r) for r in reqs]
    jobs = [sp_.job(engine.get_plan(r.matrix, ny, nx, pitch=sp_.pitch)) for r, sp_ in zip(reqs, specs)]
    outs, _ = engine.reduce_host_many(jobs)
    return [_finish(r, out, sp_.time_labels, sp_.name) for r, out, sp_ in zip(reqs, outs, specs)]


def _run_shared_parts(reqs, parts):
    """The aggregated fused requests of a lazily loaded cutout, or of one spread over several
    devices, that are cut into the same time ``parts``: each part is loaded once, and its specs are
    reduced in one shared pass."""
    r0 = reqs[0]
    ny, nx = _grid_shape(r0.ds)
    kwds = [r.part_kwds() for r in reqs]
    digests = [None if engine._is_torch(r.matrix) else engine.matrix_digest(r.matrix) for r in reqs]

    def make(part):
        return [lambda r=r, kw=kw: r.spec_cls(part, **kw) for r, kw in zip(reqs, kwds)]

    def run(specs, dev):
        jobs = [sp_.job(engine.get_plan(r.matrix, ny, nx, device=dev, pitch=sp_.pitch, digest=dg))
                for r, sp_, dg in zip(reqs, specs, digests)]
        return engine.reduce_host_many(jobs)[0]

    per_req = _run_parts(r0.ds, make, parts, run, 2 if r0.lazy else 1)
    return [_finish(r, *_concat_parts(res)) for r, res in zip(reqs, per_req)]


def convert_many(cutout, requests):
    """Several conversions of one cutout: ``requests`` maps a name to a dict of ``method`` (a
    ``Cutout`` conversion method: ``convert_and_aggregate``, ``pv``, ``wind``, ``irradiation``,
    ``solar_thermal``, ``csp``, ``temperature``, ``soil_temperature``, ``dewpoint_temperature``,
    ``coefficient_of_performance``, ``heat_demand``, ``cooling_demand`` or ``runoff``) and that
    method's keyword arguments; returns a dict of the same names.

    ``res[name]`` is what ``getattr(cutout, method)(**kwargs)`` returns (bit for bit under
    ``set_deterministic(True)``), with the warnings that call raises, and each request's argument
    errors are raised before anything reaches the GPU.  What differs is the input cost: on a
    host-resident cutout, every aggregated request (``matrix``, ``shapes`` or ``layout``) of a
    fused converter reads its fields from one pass of the cutout's time slabs to the GPU, each
    variable copied once however many requests read it; a lazily loaded cutout, or one spread
    over several devices, is loaded once per time part for the requests cut into the same parts
    (heat / cooling demand cuts its parts at its own day starts, so each further day table loads
    the cutout once more).  Per-cell requests, plugin converters, device-resident and time-sharded
    cutouts run each request as its own call."""
    if not isinstance(requests, Mapping):
        raise TypeError(f"requests must be a dict of name -> request, not {type(requests).__name__}")
    resolved = {name: _many_request(cutout, name, r) for name, r in requests.items()}
    for req, matrix_args, _ in resolved.values():
        req.resolve_matrix(*matrix_args)
    shared = [r for r, _, _ in resolved.values()
              if r.aggregated and r.spec_cls is not None and r.shard is None and _is_host_resident(r.ds)]
    out = {}
    if shared and not shared[0].partitioned:
        out.update({id(r): v for r, v in zip(shared, _run_shared(shared))})
    elif shared:  # requests cut into the same time parts share their loads
        groups = {}
        for r in shared:
            parts = r.parts()
            groups.setdefault(tuple(parts), (parts, []))[1].append(r)
        for parts, group in groups.values():
            out.update({id(r): v for r, v in zip(group, _run_shared_parts(group, parts))})
    results = {}
    for name, (req, _, post) in resolved.items():
        res = out[id(req)] if id(req) in out else _run_own(req)
        results[name] = res if post is None else _runoff_post(res, **post)
    return results


def hydro(cutout, plants, hydrobasins, flowspeed=1, weight_with_height=False, show_progress=False, **kwargs):
    """Inflow time-series of ``plants`` from the runoff of their catchment basins
    (convert.py:1087-1149, hydro.py), (plant, time) float64.

    ``plants``: DataFrame with ``lon`` and ``lat`` columns, its index becomes the ``plant``
    coordinate.  ``hydrobasins``: one level of HydroBASINS as a (Geo)DataFrame with ``HYBAS_ID``,
    ``DIST_MAIN``, ``NEXT_DOWN`` and ``geometry``, or a path geopandas reads.  Each plant drains its
    basin and every basin upstream of it; a basin's runoff is the mean over its cells
    (``runoff`` with the row-normalised indicator matrix; ``weight_with_height`` and ``**kwargs``
    such as ``smooth`` or ``lower_threshold_quantile`` go there), times its cylindrical
    equal-area area, and reaches the plant ``int(dDIST_MAIN / (flowspeed * 3.6) + 0.5)`` time
    steps later (the roll wraps around the series).  The per-plant sum of the rolled series runs
    on the GPU (csrc/hydro.cu).  ``show_progress`` is accepted and unused."""
    from . import hydro as hy

    if getattr(cutout, "time_shard", None) is not None:
        raise NotImplementedError(
            "hydro on a time-sharded cutout: the roll wraps over the whole series, and routing the "
            "gathered runoff is not implemented; convert the cutout in one process (devices= spreads "
            "the runoff over several GPUs)")
    r = hy.route(plants, hydrobasins)
    basins = r.basins
    matrix = hy.normalise_rows(cutout.indicatormatrix(basins.shapes))
    runoff = cutout.runoff(matrix=matrix, index=basins.shapes.index, weight_with_height=weight_with_height,
                           show_progress=show_progress, **kwargs)
    if isinstance(runoff, tuple) or "time" not in runoff.dims:
        raise KeyError("hydro needs the runoff of every basin as a time series (aggregate_time=None)")
    R = np.asarray(runoff.transpose("hid", "time").values, dtype=np.float64)
    time = runoff.indexes["time"]
    area = hy.basin_areas(basins.shapes)
    dist = basins.meta["DIST_MAIN"].to_numpy(dtype=np.float64)
    rows = r.rows
    plant_of = np.repeat(np.arange(len(r.ptr) - 1), np.diff(r.ptr))
    plant_dist = dist[rows[r.ptr[:-1]]] if len(rows) else np.zeros(0)  # each walk starts at the plant's basin
    shifts = hy.travel_steps(dist[rows], plant_dist[plant_of], flowspeed)
    devs = list(getattr(cutout, "devices", None) or [])
    out = engine.hydro_shift_sum(R, r.ptr, rows, shifts, area[rows],
                                 device=devs[0] if devs else engine.current_device())
    return make_dataarray(out.cpu().numpy(), ("plant", "time"), {"plant": plants.index, "time": time})


# --------------------------------------------------------------------------
# dynamic line rating (convert.py:1152-1367)
# --------------------------------------------------------------------------


_LINE_RATING_VARS = ("temperature", "wnd100m", "wnd_azimuth", "influx_direct", "height")


class _LineRatingSpec(_Spec):
    """convert_line_rating of every line of an intersection matrix, min-reduced over its cells.
    ``params``: the six per-line arrays of ``_lib.LINE_PARAMS``.  A raw ERA5 cutout (u100, v100,
    fdir and no prepared wind or direct influx) hands t2m (or temperature), u100, v100 and fdir to
    the kernel, which derives wind speed, wind azimuth and direct influx as era5.prepare does.
    ``height``: the static height of the whole cutout when ``ds`` is one time part of it (a raw
    cutout may carry only a time-dependent geopotential ``z``)."""

    units = "A"

    def __init__(self, ds, params, height=None):
        ny, nx = _grid_shape(ds)
        self.time_labels = pd.DatetimeIndex(_coord(ds, "time"))
        self.raw = _line_rating_raw(ds)
        if self.raw:  # operator slot -> dataset variable (include/atlite_b200.h: AtlLineRatingRawFields)
            src = {"t2m": _var(ds, "temperature"), "u100": "u100", "v100": "v100", "fdir": "fdir"}
            self.fields = {k: _raw(ds, v) for k, v in src.items()}
            self.fields["height"] = _height(ds) if height is None else height
            self._lead = "t2m"
        else:
            self.fields = {n: (_height(ds) if n == "height" else _raw(ds, n)) for n in _LINE_RATING_VARS}
            self._lead = "temperature"
        # SolarPosition (pv/solar_position.py:54-67): the stored position as it is, else computed at
        # the default shift of 0 h, with the reference's warning; a raw cutout gets the position
        # era5.prepare would have stored (-30 min, era5.py:182-188), without the warning
        if _has(ds, "solar_azimuth") and _has(ds, "solar_altitude"):
            self.fields["solar_altitude"], self.fields["solar_azimuth"], solar_src = _stored_solar_position(ds)
        elif self.raw:
            solar_src = _lib.SOLAR_COMPUTED
        else:
            warnings.warn(_SOLAR_WARNING, DeprecationWarning)
            solar_src = _lib.SOLAR_COMPUTED
        first = self.fields[self._lead]
        self.device = first.device.index if engine._is_torch(first) else engine.current_device()
        self.pitch = engine.pitch_of([v for k, v in self.fields.items() if k != "height"], nx)
        shift = "-30min" if self.raw and solar_src == _lib.SOLAR_COMPUTED else "0h"
        self.op = engine.LineRatingOp(ny=ny, nx=nx, time=self.time_labels, lon=_coord(ds, "lon"),
                                      lat=_coord(ds, "lat"), solar_src=solar_src, params=params,
                                      time_shift=shift, device=self.device, pitch=self.pitch)

    def reduce(self, plan):
        """(time, line) float32: a torch tensor for a device-resident cutout, else NumPy (the host
        fields go to the device in parts of about PART_BYTES)."""
        f = self.fields
        first = f[self._lead]
        nt = first.shape[0]
        reduce = self.op.reduce_raw if self.raw else self.op.reduce
        if engine._is_torch(first):
            if nt == 0:
                return engine._torch().zeros((0, plan.n_bus), dtype=engine._torch().float32, device=first.device)
            return reduce(plan, f)
        out = np.empty((nt, plan.n_bus), dtype=np.float32)
        if nt == 0:
            return out
        torch = engine._torch()
        dev = f"cuda:{plan.device}"

        def up(name, a):
            """float32 on the device, the solar position in the operator's width; fields are cast on
            the host, as the other operators' host paths do"""
            f64 = self.op.solar_f64 and name.startswith("solar_")
            a = np.ascontiguousarray(a, dtype=np.float64) if f64 else engine.host_f32(a)
            return torch.from_numpy(a).to(dev)

        step = max(1, PART_BYTES // (sum(a[:1].nbytes for k, a in f.items() if k != "height") or 1))
        height = up("height", f["height"])
        for lo in range(0, nt, step):
            hi = min(nt, lo + step)
            part = {k: (height if k == "height" else up(k, a[lo:hi])) for k, a in f.items()}
            out[lo:hi] = reduce(plan, part, t0=lo).cpu().numpy()
        return out


def convert_line_rating(ds, psi, R, D=0.028, Ts=373, epsilon=0.6, alpha=0.6, per_unit=False):
    """IEEE-738 maximal current in A (convert.py:1152-1252) of a dict of scalars or arrays that
    broadcast together: ``temperature``, ``wnd100m``, ``height``, ``wnd_azimuth``,
    ``influx_direct``, ``solar_altitude``, ``solar_azimuth`` (radians).  ``psi`` is taken through
    ``radians()`` as in the reference.  Evaluated elementwise on the GPU; ``per_unit`` is
    accepted and unused, as in the reference.  For a cutout use ``line_rating``."""
    if not isinstance(ds, dict):
        raise TypeError("convert_line_rating evaluates a dict of arrays; use line_rating for a cutout")
    vals = {n: ds[n] for n in _lib.LINE_RATING_FIELDS}
    vals.update(psi=psi, R=R, D=D, Ts=Ts, epsilon=epsilon, alpha=alpha)
    return engine.line_rating_eval(vals).astype(np.float64)


def _line_shapes(shapes):
    """``shapes`` as a pandas Series: ``GeoSeries(shapes).rename_axis("dim_0")`` for anything but a
    GeoSeries (convert.py:1325-1326), a GeoSeries with its own index."""
    if hasattr(shapes, "columns") and hasattr(shapes, "geometry"):  # GeoDataFrame: its geometry column
        shapes = shapes.geometry
    if type(shapes).__name__ == "GeoSeries":
        return pd.Series(list(shapes.values), index=shapes.index, dtype=object)
    if isinstance(shapes, pd.Series):
        s = pd.Series(list(shapes.values), index=shapes.index, dtype=object)
    elif isinstance(shapes, dict):
        s = pd.Series(list(shapes.values()), index=list(shapes.keys()), dtype=object)
    else:
        s = pd.Series(list(shapes), dtype=object)
    return s.rename_axis("dim_0")


def _line_parameters(shapes, line_resistance, params):
    """(shapes as a Series, line dimension name, the per-line DataFrame psi, R, D, Ts, epsilon,
    alpha) as convert.py:1325-1350 builds them, with the reference's two assertions.  The line
    dimension is named as ``xr.concat(..., dim=df.index)`` names it (convert.py:1367): the name of
    the table's index -- which pandas drops when the shapes' and a Series parameter's index names
    differ -- or ``"concat_dim"`` when it has none."""
    from . import gis

    s = _line_shapes(shapes)
    azimuth = pd.Series([gis.line_azimuth(g) for g in s.values], index=s.index, dtype=np.float64)
    azimuth = azimuth.where(azimuth >= 0, azimuth + np.pi)  # convert.py:1340
    params = dict(params)
    params.setdefault("D", 0.028)
    params.setdefault("Ts", 373)
    params.setdefault("epsilon", 0.6)
    params.setdefault("alpha", 0.6)
    # the azimuth (radians) goes in as psi, which convert_line_rating passes through radians()
    # again (convert.py:1347, 1215): reproduced
    df = pd.DataFrame({"psi": azimuth, "R": line_resistance}).assign(**params)
    assert df.notnull().all().all(), "Nan values encountered."
    assert df.columns.equals(pd.Index(["psi", "R", "D", "Ts", "epsilon", "alpha"]))
    dim = df.index.name if df.index.name is not None else "concat_dim"
    return s, dim, df


def line_rating(cutout, shapes, line_resistance, show_progress=False, dask_kwargs={}, **params):
    """Dynamic line rating of every line in A, (line, time), by the IEEE-738 heat balance
    (convert.py:1255-1367).  ``shapes``: LineStrings (shapely / geopandas objects or GeoJSON
    dicts) in the cutout's CRS; ``line_resistance`` and ``params`` (D, Ts, epsilon, alpha) are
    scalars or pandas Series aligned with the shapes by index.  Per step a line gets the min over
    the cells it intersects (``Cutout.intersectionmatrix``), NaN cells skipped; a line that
    touches no cell, or only NaN cells, gets NaN.  The cutout needs ``temperature``,
    ``wnd100m``, ``wnd_azimuth``, ``influx_direct`` and ``height``; a stored solar position is
    used as it is, else it is computed (0 h shift) with a ``DeprecationWarning``.  A raw ERA5
    cutout without ``wnd100m``, ``wnd_azimuth`` and ``influx_direct`` is read directly when it has
    ``u100``, ``v100`` and ``fdir``, with ``temperature`` or ``t2m``, and ``height`` or the
    geopotential ``z``: the result is the prepared cutout's, and an absent solar position is
    computed as era5.prepare stores it (-30 min shift), without the warning.
    ``show_progress`` and ``dask_kwargs`` are accepted and unused."""
    if getattr(cutout, "time_shard", None) is not None:
        raise NotImplementedError(
            "line_rating on a time-sharded cutout: gathering the per-rank line results is not "
            "implemented; convert the cutout in one process (devices= spreads it over several GPUs)")
    ds = cutout.data
    raw = _line_rating_raw(ds)
    for n in ((_var(ds, "temperature"),) + _LR_RAW if raw else _LINE_RATING_VARS):
        if not _has(ds, n):
            raise KeyError(f"line_rating needs the variable {n!r} in the cutout")
    if raw and not (_has(ds, "height") or _has(ds, "z")):
        raise KeyError("line_rating needs the variable 'height' (or the geopotential 'z') in the cutout")
    s, dim, df = _line_parameters(shapes, line_resistance, params)
    lp = {k: df[k].to_numpy(dtype=np.float64) for k in _lib.LINE_PARAMS}

    I = cutout.intersectionmatrix(list(s.values)).tocsr()  # noqa: E741
    ny, nx = _grid_shape(ds)
    kw = {"params": lp}
    if raw:  # from the whole cutout: a time part would start at another step of a time-dependent z
        kw["height"] = _height(ds)
    if not _is_host_resident(ds):
        spec = _LineRatingSpec(ds, **kw)
        plan = engine.get_plan(I, ny, nx, device=spec.device, pitch=spec.pitch, entries=True)
        res = spec.reduce(plan)  # (time, line) float32 on the device: widened and transposed there
        res = res.to(engine._torch().float64).T.contiguous().cpu().numpy()
        time_labels = spec.time_labels
    else:
        # host-resident, pinned and lazily loaded cutouts, on one or several devices: the min is
        # per step, so the results of time parts simply concatenate
        lazy = _is_dask_backed(ds)
        n_time = len(_coord(ds, "time"))
        devices = list(cutout.devices or [engine.current_device()])
        parts = _partition(ds, n_time, devices, lazy)
        digest = engine.matrix_digest(I)
        out = _run_partitioned(
            ds, _LineRatingSpec, kw, parts,
            lambda sp_, dev: _to_host(sp_.reduce(engine.get_plan(I, ny, nx, device=dev, pitch=sp_.pitch,
                                                                 digest=digest, entries=True))),
            2 if lazy else 1)
        res = np.ascontiguousarray(np.concatenate([v for v, _ in out], axis=0).T, dtype=np.float64)
        time_labels = pd.DatetimeIndex(np.concatenate([np.asarray(sp_.time_labels) for _, sp_ in out]))
    return make_dataarray(res, (dim, "time"), {dim: df.index, "time": time_labels}, {"units": "A"})
