"""SARAH satellite irradiance for a cutout (datasets/sarah.py of the reference).

``get_data`` reads a directory of daily SARAH files (``SIS*.nc`` global and ``SID*.nc`` direct
surface irradiance, half-hourly at 0.05 degrees), crops them to the cutout, fills the dawn and dusk
gaps along time, averages half-hours into hours, resamples onto the cutout grid when it is coarser,
and adds the solar position.  The gap filling and the pair mean run in one kernel
(``engine.SarahOp``, csrc/sarah.cu), the resampling is ``gis.regrid``'s (``gis.regrid_op``), the
solar position ``era5.solar_position``.  Files go to the GPU a few days at a time, so the half-hourly
input is never held whole; the result is host-resident, ready to be merged with an ERA5 cutout
(``Cutout.merge``).  Semantics and deviations: DESIGN.md section 1.
"""

from __future__ import annotations

import glob
import logging
import os

import numpy as np
import pandas as pd

logger = logging.getLogger(__name__)

# Model, CRS and resolution settings (datasets/sarah.py:28-39)
crs = 4326
dx = 0.05
dy = 0.05
dt = "30min"
features = {
    "influx": [
        "influx_direct",
        "influx_diffuse",
        "solar_altitude",
        "solar_azimuth",
    ],
}
static_features = {}

_FILES_PER_LAUNCH = 4  # days read, filled and regridded together


def get_filenames(sarah_dir, coords):
    """DataFrame with columns ``sis`` and ``sid``, indexed by day, of the files under ``sarah_dir``
    (searched recursively) whose day lies in the span of ``coords["time"]``.  Only days with both
    files are kept.  Files that do not cover the span are logged as an error, not raised."""

    def starting_with(name):
        pattern = os.path.join(sarah_dir, "**", f"{name}*.nc")
        files = pd.Series(glob.glob(pattern, recursive=True), dtype=object)
        assert not files.empty, f"No files found at {pattern}. Make sure sarah_dir points to the correct directory!"
        files.index = pd.to_datetime(files.str.extract(r"SI.in(\d{8})", expand=False))
        return files.sort_index()

    files = pd.concat(dict(sis=starting_with("SIS"), sid=starting_with("SID")), join="inner", axis=1)
    time = pd.DatetimeIndex(np.asarray(coords["time"]))
    start, end = time[0].floor("D"), time[-1].floor("D")
    if start < files.index[0] or end > files.index[-1]:
        logger.error(f"Files in {sarah_dir} do not cover the whole time span:\t{start} until {end}")
    return files.loc[(files.index >= start) & (files.index <= end)].sort_index()


def as_slice(bounds, pad=True):
    """Coordinate bounds (lo, hi) -> ``slice(lo - 0.01, hi + 0.01)``; a slice is returned as is."""
    if not isinstance(bounds, slice):
        bounds = np.asarray(bounds) + (-0.01, 0.01)
        bounds = slice(*bounds)
    return bounds


def block_starts(lengths, chunk=None):
    """Start steps of the gap-filling blocks for files of ``lengths`` steps laid end to end: every
    file is cut into runs of ``chunk`` steps (the whole file when ``chunk`` is None), as dask chunks
    files opened with ``chunks={"time": chunk}``."""
    out, off = [], 0
    for n in lengths:
        step = int(chunk) if chunk else max(int(n), 1)
        out.extend(range(off, off + int(n), step))
        off += int(n)
    return out


# ---------------------------------------------------------------- gap filling and hourly mean

def _time_first(dims, arr, dim="time"):
    """(values as (nt, 1, cells) float32, permutation applied, shape after it)."""
    if np.asarray(arr).dtype != np.float32:
        raise TypeError(f"SARAH fields are float32, not {np.asarray(arr).dtype}")
    perm = [dims.index(dim)] + [i for i, d in enumerate(dims) if d != dim]
    a = np.transpose(np.asarray(arr), perm)
    return np.ascontiguousarray(a.reshape(a.shape[0], 1, -1)), perm, a.shape


def _apply(ds, fill, hourly, dim="time"):
    from .engine import SarahOp
    from .labelled import DataArray, Dataset

    if isinstance(ds, DataArray):
        named = [(ds.name, ds.dims, ds.values)]
    elif isinstance(ds, Dataset) and not getattr(ds, "lazy", False):
        named = [(n, ds.dims_of(n), ds.raw(n)) for n in ds.keys() if dim in ds.dims_of(n)]
    else:
        raise TypeError(f"takes this package's DataArray or in-memory Dataset, not {type(ds).__name__}")
    if any(not isinstance(a, np.ndarray) for _, _, a in named):
        raise TypeError("the fields must be host (NumPy) arrays")
    res = {}
    for k in range(0, len(named), 2):  # the kernel fills two fields per launch
        pair = named[k:k + 2]
        prepared = [_time_first(dims, arr, dim) for _, dims, arr in pair]
        a, b = prepared[0][0], prepared[-1][0]
        nt = a.shape[0]
        op = SarahOp(1, a.shape[2])
        outs = op(a, b, [0] if nt else [], fill=fill, hourly=hourly)
        for (n, dims, _), (_, perm, shape), o in zip(pair, prepared, outs):
            o = o.reshape((o.shape[0],) + shape[1:])
            res[n] = (dims, np.transpose(o, np.argsort(perm)))
    nt = len(next(iter(named))[2]) if named else 0
    sel = slice(0, nt - nt % 2, 2) if hourly else slice(None)

    def coords_of(coords):
        return {k: (v[sel] if k == dim else v) for k, v in coords.items()}

    if isinstance(ds, DataArray):
        dims, vals = res[ds.name]
        return DataArray(vals, coords_of(ds.coords), dims, ds.name, ds.attrs)
    out = Dataset(coords=coords_of(ds.coords), attrs=ds.attrs)
    for n in ds.keys():
        out._vars[n] = res.get(n, ds._vars[n])
    return out


def interpolate(ds, dim="time"):
    """NaNs of ``ds`` (this package's float32 DataArray or in-memory Dataset) filled along ``dim``
    as ``np.interp`` fills them on the step index: linearly between valid steps, with the first /
    last valid value before / after them; an all-NaN series stays NaN.  An in-memory array is one
    block (``get_data`` fills file by file).  Runs on the GPU."""
    from .engine import SarahOp

    return _apply(ds, SarahOp.FILL_INTERP, False, dim)


def hourly_mean(ds):
    """Steps (2k, 2k + 1) of ``ds`` averaged in float32 as (a + b) / 2 and labelled with step 2k's
    time; NaN propagates and an odd last step is dropped.  Runs on the GPU."""
    from .engine import SarahOp

    return _apply(ds, SarahOp.FILL_NONE, True)


# ---------------------------------------------------------------- reading the files

def _cf_field(ds, name, ys, xs):
    """Variable ``name`` of one opened file, cropped to rows ``ys`` / columns ``xs``, CF-decoded:
    ``_FillValue`` / ``missing_value`` -> NaN, then ``scale_factor`` and ``add_offset`` in float32."""
    f = getattr(ds, "_file", None)
    if f is None:  # NetCDF-4 / chunk container: the native decoder unpacks and masks _FillValue
        return np.ascontiguousarray(ds.isel_time(0, len(ds.coords["time"])).raw(name)[:, ys, xs])
    v = f.variables[name]  # NetCDF-3: scipy's memory map of the raw values
    raw = np.asarray(v[:, ys, xs])
    a = raw.astype(np.float32)
    for attr in ("_FillValue", "missing_value"):
        fv = getattr(v, attr, None)
        if fv is not None:
            a[raw == np.asarray(fv, dtype=raw.dtype)] = np.nan
    sf, ao = getattr(v, "scale_factor", None), getattr(v, "add_offset", None)
    if sf is not None:
        a *= np.float32(sf)
    if ao is not None:
        a += np.float32(ao)
    return a


def _crop(index, bounds):
    loc = pd.Index(index).slice_indexer(bounds.start, bounds.stop)
    return slice(loc.start, loc.stop)


def get_data(cutout, feature, tmpdir, lock=None, monthly_requests=False, **creation_parameters):
    """SARAH ``influx`` for ``cutout``: a host-resident Dataset with ``influx_direct`` and
    ``influx_diffuse`` (float32) and ``solar_altitude`` / ``solar_azimuth`` (float64, time shift 0),
    coordinates ``time, y, x, lon, lat`` and ``attrs["module"] = "sarah"`` (datasets/sarah.py:162-244);
    an xarray Dataset when the cutout's data is one.  It covers the whole days of the files
    that ``get_filenames`` selects; select the cutout's times with ``Cutout.sel`` afterwards.

    ``creation_parameters``: ``sarah_dir`` (required), ``sarah_interpolate`` (default True: fill
    NaNs along time within each block of ``cutout.chunks["time"]`` steps of a file, else set them
    to 0) and ``parallel`` (accepted, unused).  ``tmpdir``, ``lock`` and ``monthly_requests`` are
    accepted and unused.  ``feature`` must be ``"influx"``, SARAH's only feature."""
    from . import era5, gis, ingest
    from .engine import SarahOp, _torch, current_device
    from .labelled import HAVE_XARRAY, Dataset, xr

    assert cutout.dt in ("30min", "30T", "h", "1h")
    if feature != "influx":
        raise ValueError(f"SARAH provides the feature 'influx' only, not {feature!r}")
    sarah_dir = creation_parameters["sarah_dir"]
    creation_parameters.setdefault("parallel", False)
    interp = creation_parameters.setdefault("sarah_interpolate", True)
    hourly = cutout.dt not in ("30min", "30T")
    chunk = (cutout.chunks or {}).get("time")

    files = get_filenames(sarah_dir, cutout.coords)
    opened = [(ingest.open_cutout(a), ingest.open_cutout(b)) for a, b in zip(files["sis"], files["sid"])]
    lengths = []
    for sis, sid in opened:
        if not np.array_equal(np.asarray(sis.coords["time"]), np.asarray(sid.coords["time"])):
            raise ValueError("a SIS file and its SID file have different time steps")
        lengths.append(len(sis.coords["time"]))
    time = pd.DatetimeIndex(np.concatenate([np.asarray(s.coords["time"]) for s, _ in opened])
                            if opened else np.array([], dtype="datetime64[ns]"))
    ext = np.asarray(cutout.extent, dtype=np.float64)
    lon0 = np.asarray(opened[0][0].coords["lon"], dtype=np.float64) if opened else np.zeros(0)
    lat0 = np.asarray(opened[0][0].coords["lat"], dtype=np.float64) if opened else np.zeros(0)
    xs, ys = _crop(lon0, as_slice(ext[:2])), _crop(lat0, as_slice(ext[2:]))
    lon, lat = lon0[xs].round(4), lat0[ys].round(4)

    torch = _torch()
    device = current_device()
    op = SarahOp(len(lat), len(lon), device)
    regrid = cutout.dx != dx or cutout.dy != dy
    if regrid:
        dst_lon = pd.Index(np.asarray(cutout.coords["lon"], dtype=np.float64), name="lon")
        dst_lat = pd.Index(np.asarray(cutout.coords["lat"], dtype=np.float64), name="lat")
        rop = gis.regrid_op(lon, lat, dst_lon, dst_lat, gis.RESAMPLING_AVERAGE, device)
        out_lon, out_lat = np.asarray(dst_lon), np.asarray(dst_lat)
    else:
        out_lon, out_lat = lon, lat
    out_time = time[0:len(time) - len(time) % 2:2] if hourly else time
    shape = (len(out_time), len(out_lat), len(out_lon))
    direct, diffuse = np.empty(shape, dtype=np.float32), np.empty(shape, dtype=np.float32)
    alt, az = np.empty(shape, dtype=np.float64), np.empty(shape, dtype=np.float64)

    # groups of files launched together: a cut needs an even step when pairs are averaged
    offs = np.concatenate([[0], np.cumsum(lengths)]).astype(int)
    groups, i = [], 0
    while i < len(opened):
        j = min(i + _FILES_PER_LAUNCH, len(opened))
        while hourly and j < len(opened) and offs[j] % 2:
            j += 1
        groups.append((i, j))
        i = j
    fill = SarahOp.FILL_INTERP if interp else SarahOp.FILL_ZERO
    for i, j in groups:
        lo, hi = int(offs[i]), int(offs[j])
        fields = []
        for k in (0, 1):
            name = ("SIS", "SID")[k]
            host = np.concatenate([_cf_field(opened[f][k], name, ys, xs) for f in range(i, j)])
            fields.append(torch.from_numpy(host).to(f"cuda:{device}"))
        sis, sid = op(fields[0], fields[1], block_starts(lengths[i:j], chunk), fill=fill,
                      hourly=hourly)
        if regrid:
            sis, sid = rop(sis), rop(sid)
        olo, ohi = (lo // 2, hi // 2) if hourly else (lo, hi)
        direct[olo:ohi] = sid.cpu().numpy()
        diffuse[olo:ohi] = (sis - sid).cpu().numpy()
        a, z = era5.solar_position(out_time[olo:ohi], out_lon, out_lat, "0h", device)
        alt[olo:ohi], az[olo:ohi] = a.cpu().numpy(), z.cpu().numpy()

    coords = {"time": out_time, "x": out_lon, "y": out_lat, "lon": out_lon, "lat": out_lat}
    values = {"influx_direct": direct, "influx_diffuse": diffuse, "solar_altitude": alt, "solar_azimuth": az}
    if HAVE_XARRAY and isinstance(cutout.data, xr.Dataset):  # pragma: no cover - xarray is optional
        ds = xr.Dataset({n: (("time", "y", "x"), v) for n, v in values.items()},
                        coords={"time": out_time, "x": out_lon, "y": out_lat, "lon": ("x", out_lon),
                                "lat": ("y", out_lat)}, attrs={"module": "sarah"})
        ds["influx_diffuse"].attrs.update(long_name="Surface Diffuse Shortwave Flux", units="W m-2")
        return ds
    return Dataset({n: (("time", "y", "x"), v) for n, v in values.items()}, coords=coords, attrs={"module": "sarah"})
