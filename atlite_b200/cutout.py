"""``Cutout``: the container the conversion methods are bound to.

The reference's ``Cutout`` (cutout.py:61-689) also creates/downloads/prepares
NetCDF cutouts and does GIS work; none of that is on the hot path.  This class
keeps what ``convert_and_aggregate`` consumes -- ``.data`` (variables as
``(time, y, x)`` arrays with ``x, y, time, lon, lat`` coordinates), ``.grid``
(cells in y-major / x-minor order, cutout.py:355-376) -- binds the same
conversion methods (cutout.py:653-689), and adds device residency:
``to_device()`` uploads the fields once so repeated pv / wind / heat_demand
calls read them straight from HBM.
"""

from __future__ import annotations

from collections import namedtuple
from pathlib import Path

import numpy as np
import pandas as pd

from . import convert as _convert
from .gis import compute_indicatormatrix  # noqa: F401  (re-exported as the reference's atlite.cutout does)
from .labelled import HAVE_XARRAY, Dataset, make_dataarray

if HAVE_XARRAY:  # pragma: no cover
    import xarray as xr


_AffineTuple = namedtuple("Affine", "a b c d e f")


def _affine(a, b, c, d, e, f):
    """x = a*col + b*row + c, y = d*col + e*row + f (rasterio.Affine when rasterio is there)."""
    try:
        from rasterio import Affine  # pragma: no cover

        return Affine(a, b, c, d, e, f)  # pragma: no cover
    except ImportError:
        return _AffineTuple(float(a), float(b), float(c), float(d), float(e), float(f))


class _Registered:
    """Owns a cudaHostRegister'ed NumPy array (unregisters it when collected)."""

    def __init__(self, arr):
        self.arr = arr

    def __del__(self):
        try:
            import torch

            torch.cuda.cudart().cudaHostUnregister(self.arr.ctypes.data)
        except Exception:  # noqa: BLE001
            pass


def _numa_sharded_copy(a, devices, shard_bounds, local_cpus):
    """Copy ``a`` (time, y, x) into a fresh page-aligned array whose time shard r is written
    -- first touched -- by a thread pinned to the CPUs local to devices[r]."""
    import os
    import threading

    nbytes = a.nbytes
    raw = np.empty(nbytes + 4096, dtype=np.uint8)  # untouched pages: placement happens at first write
    off = (-raw.ctypes.data) % 4096
    dst = raw[off:off + nbytes].view(a.dtype).reshape(a.shape)
    nt = a.shape[0]

    def work(r, dev):
        lo, hi = shard_bounds(nt, len(devices), r)
        old = None
        try:
            cpus = local_cpus(dev)
            if cpus:
                old = os.sched_getaffinity(0)
                both = set(cpus) & set(old)
                if both:
                    os.sched_setaffinity(0, both)  # pid 0 = the calling thread
            dst[lo:hi] = a[lo:hi]
        finally:
            if old is not None:
                os.sched_setaffinity(0, old)

    ths = [threading.Thread(target=work, args=(r, d)) for r, d in enumerate(devices)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    return dst


def _host_slice(arr, lo, hi):
    """Steps [lo, hi) of a NumPy array or torch tensor, as a NumPy array."""
    part = arr[lo:hi]
    return part.detach().cpu().numpy() if hasattr(part, "detach") else np.asarray(part)


def _same_values(a, b, name):
    """Variable ``name`` equal in the Datasets ``a`` and ``b`` (NaN equal to NaN), lazy ones read
    part by part."""
    if a.dims_of(name) != b.dims_of(name):
        return False
    if name not in getattr(a, "_loaders", {}) and name not in getattr(b, "_loaders", {}):
        return np.array_equal(_host_slice(a.raw(name), 0, None), _host_slice(b.raw(name), 0, None), equal_nan=True)
    nt, step = len(a.coords["time"]), min(getattr(d, "time_chunk", 1 << 30) for d in (a, b))

    def part(d, lo, hi):
        return d.isel_time(lo, hi).raw(name) if name in getattr(d, "_loaders", {}) else _host_slice(d.raw(name), lo, hi)

    return all(np.array_equal(np.asarray(part(a, lo, min(nt, lo + step))), np.asarray(part(b, lo, min(nt, lo + step))),
                              equal_nan=True) for lo in range(0, nt, step))


class Cutout:
    """``devices``: which GPUs of this process convert the cutout.  ``None`` = the current
    CUDA device; ``"all"`` or a list of device indices = the time axis of a HOST-resident
    cutout (NumPy / pinned / lazily loaded xarray data) is cut into one contiguous shard per
    device, every device streams and converts its shard from its own host thread, and the
    shard results land in one host array -- the reference's single call in a single process
    (convert.py:59-75), no ``torchrun`` needed.  (``time_shard=`` is the other multi-GPU mode:
    one PROCESS per GPU under ``torchrun``, results gathered over NCCL, see dist.py.)"""

    def __init__(self, path=None, data=None, time_shard=None, devices=None, **kwargs):
        if data is None:
            if path is None:
                raise ValueError("Cutout needs `data=` (or a NetCDF `path` when xarray is installed)")
            if HAVE_XARRAY:  # the reference's own way in (cutout.py:142-154): lazy, {"time": 100} chunks
                chunks = kwargs.pop("chunks", {"time": 100})
                data = xr.open_dataset(str(path), chunks=chunks)
            else:  # without xarray: this package's readers (chunk container, NetCDF-4 via h5py, NetCDF-3)
                from . import ingest

                data = ingest.open_cutout(path)
        elif isinstance(data, dict):
            data = Dataset(
                {k: v for k, v in data.items() if k not in ("time", "x", "y", "lon", "lat")},
                coords={k: data[k] for k in ("time", "x", "y", "lon", "lat") if k in data},
            )
        for c in ("x", "y", "time"):
            if c not in data.coords:
                raise ValueError(f"cutout data lacks coordinate {c!r}")
        if isinstance(data, Dataset):
            if "lon" not in data.coords:
                data.coords["lon"] = data.coords["x"]
            if "lat" not in data.coords:
                data.coords["lat"] = data.coords["y"]
        self.path = path
        self.data = data
        self._devices = devices
        # set by atlite_b200.dist.TimeShard: this process holds one contiguous
        # time shard of the cutout and results are gathered across ranks
        self.time_shard = time_shard

    @property
    def devices(self):
        """Resolved list of CUDA device indices, or None (= the current device)."""
        d = self._devices
        if d is None:
            return None
        if isinstance(d, str):
            if d != "all":
                raise ValueError(f"devices must be None, 'all' or a list of device indices, not {d!r}")
            import torch

            d = list(range(torch.cuda.device_count()))
        d = [int(k) for k in (d if hasattr(d, "__iter__") else [d])]
        if not d:
            raise RuntimeError("no CUDA device visible (atlite_b200 has no CPU fallback)")
        return d

    # ---- identity (cutout.py:211-256)
    @property
    def name(self):
        """Stem of the cutout's path (cutout.py:212-216); None for a cutout built from data only."""
        return None if self.path is None else Path(self.path).stem

    @property
    def module(self):
        return getattr(self.data, "attrs", {}).get("module")  # cutout.py:219-223

    @property
    def chunks(self):
        """{dim: size} from the ``chunksize_*`` attributes of a prepared cutout (cutout.py:240-249)."""
        attrs = getattr(self.data, "attrs", {})
        chunks = {k[len("chunksize_"):]: v for k, v in attrs.items() if k.startswith("chunksize_")}
        return chunks or None

    @property
    def dt(self):
        """Time resolution as a pandas frequency string (cutout.py:328-332)."""
        return pd.infer_freq(pd.DatetimeIndex(np.asarray(self.coords["time"])))

    # ---- geometry (cutout.py:300-376)
    @property
    def coords(self):
        return self.data.coords

    @property
    def shape(self):
        return len(self.coords["y"]), len(self.coords["x"])

    @property
    def dx(self):
        x = np.asarray(self.coords["x"])
        return float(np.round(x[1] - x[0], 8)) if len(x) > 1 else 0.0

    @property
    def dy(self):
        y = np.asarray(self.coords["y"])
        return float(np.round(y[1] - y[0], 8)) if len(y) > 1 else 0.0

    @property
    def crs(self):
        return getattr(self.data, "attrs", {}).get("crs", "EPSG:4326")

    @property
    def extent(self):
        x, y = np.asarray(self.coords["x"]), np.asarray(self.coords["y"])
        return np.array([x.min() - self.dx / 2, x.max() + self.dx / 2,
                         y.min() - self.dy / 2, y.max() + self.dy / 2])

    @property
    def bounds(self):
        """(x, y, X, Y) of the covered area (cutout.py:277-281)."""
        return self.extent[[0, 2, 1, 3]]

    @property
    def transform(self):
        """Affine coefficients (a, b, c, d, e, f) of the grid, cell (col, row) -> (x, y) of its lower-left
        corner (cutout.py:284-295; a ``rasterio.Affine`` when rasterio is installed)."""
        x, y = np.asarray(self.coords["x"]), np.asarray(self.coords["y"])
        return _affine(self.dx, 0.0, x[0] - self.dx / 2, 0.0, self.dy, y[0] - self.dy / 2)

    @property
    def transform_r(self):
        """The same with the y axis reversed (cutout.py:298-309)."""
        x, y = np.asarray(self.coords["x"]), np.asarray(self.coords["y"])
        return _affine(self.dx, 0.0, x[0] - self.dx / 2, 0.0, -self.dy, y[-1] + self.dy / 2)

    def area(self, crs=None):
        """Area per grid cell in the units of the cutout's CRS (cutout.py:539-562: ``grid.to_crs(crs).area``
        with crs = the cutout's own -- for a regular grid every cell is dx * dy).  Another CRS needs
        a reprojection library, which is outside this package."""
        if crs is not None and str(crs).upper().replace("EPSG:", "") != str(self.crs).upper().replace("EPSG:", ""):
            raise NotImplementedError(f"area(crs={crs!r}): reprojection is outside this package; cutout CRS is {self.crs}")
        ny, nx = self.shape
        return make_dataarray(np.full((ny, nx), abs(self.dx * self.dy)), ("y", "x"),
                              {"y": np.asarray(self.coords["y"]), "x": np.asarray(self.coords["x"])})

    def uniform_density_layout(self, capacity_density, crs=None):
        """capacity_density * area per cell (cutout.py:570-589)."""
        return capacity_density * self.area(crs)

    def layout_from_capacity_list(self, data, col="Capacity"):
        """(y, x) capacity layout from a table with columns ``x``, ``y`` and ``col``: every entry is
        added to its nearest grid cell (cutout.py:600-651).  Follows the reference's index
        arithmetic step by step -- searchsorted(left), clip, "move to best distance" with
        ``x_grid[ix - 1]`` -- including its wrap-around for entries at or left of the first
        coordinate (ix - 1 = -1 there), so that layouts agree cell by cell; NaN capacities count
        as 0 (pandas' groupby sum)."""
        xg, yg = np.asarray(self.coords["x"], dtype=np.float64), np.asarray(self.coords["y"], dtype=np.float64)
        px, py = np.asarray(data["x"], dtype=np.float64), np.asarray(data["y"], dtype=np.float64)
        cap = np.nan_to_num(np.asarray(data[col], dtype=np.float64), nan=0.0)
        ix = np.clip(np.searchsorted(xg, px, side="left"), 0, len(xg) - 1)
        iy = np.clip(np.searchsorted(yg, py, side="left"), 0, len(yg) - 1)
        ix = ix - (px - xg[ix - 1] < xg[ix] - px)
        iy = iy - (py - yg[iy - 1] < yg[iy] - py)
        ok = ~(np.isnan(px) | np.isnan(py))  # groupby drops NaN keys
        lay = np.zeros(self.shape)
        np.add.at(lay, (iy[ok] % len(yg), ix[ok] % len(xg)), cap[ok])
        return make_dataarray(lay, ("y", "x"), {"y": yg, "x": xg})

    def sel(self, path=None, bounds=None, buffer=0, **kwargs):
        """Sub-cutout (cutout.py:378-413): ``bounds`` = (x1, y1, x2, y2), widened by ``buffer``;
        further keyword arguments select by coordinate labels with inclusive slices, e.g.
        ``time=slice("2013-01", "2013-03")``.  Host-resident data is sliced as views, lazily
        loaded data stays lazy."""
        if bounds is not None:
            x1, y1, x2, y2 = (float(v) for v in np.asarray(bounds, dtype=np.float64).ravel())
            if buffer > 0:  # box(*bounds).buffer(buffer).bounds
                x1, y1, x2, y2 = x1 - buffer, y1 - buffer, x2 + buffer, y2 + buffer
            kwargs.update(x=slice(x1, x2), y=slice(y1, y2))
        return Cutout(path, data=self.data.sel(**kwargs), devices=self._devices)

    def merge(self, other, path=None, **kwargs):
        """One cutout with the variables of both (cutout.py:415-451); attrs are combined, with
        ``module`` the union of both cutouts' modules.  xarray data is merged by
        ``xarray.Dataset.merge(other.data, **kwargs)``.  For this package's Dataset / LazyDataset,
        ``x``, ``y`` and ``time`` must be identical (no outer join: select first with ``sel``), only
        ``compat`` is accepted, and a variable in both cutouts must be equal in both (NaN equals NaN)
        unless ``compat="override"``, which takes it from this cutout.  When either side is lazy the
        result is lazy: in-memory variables are served time slice by time slice."""
        from .labelled import LazyDataset

        if not isinstance(other, Cutout):
            raise TypeError(f"can only merge a Cutout, not {type(other).__name__}")
        modules = []
        for m in (self.module, other.module):
            modules += [] if m is None else [m] if isinstance(m, str) else list(m)
        attrs = {**getattr(self.data, "attrs", {}), **getattr(other.data, "attrs", {})}
        attrs["module"] = list(dict.fromkeys(modules))
        a, b = self.data, other.data
        if not (isinstance(a, Dataset) and isinstance(b, Dataset)):
            if isinstance(a, Dataset) or isinstance(b, Dataset):
                raise TypeError("cannot merge xarray data with this package's Dataset")
            return Cutout(path, data=a.merge(b, **kwargs).assign_attrs(**attrs))  # pragma: no cover

        unknown = sorted(set(kwargs) - {"compat"})
        if unknown:
            raise TypeError(f"merge got unsupported keyword argument(s) {unknown}; only compat is supported")
        override = kwargs.get("compat") == "override"
        for c in ("x", "y", "time"):
            if not np.array_equal(np.asarray(a.coords[c]), np.asarray(b.coords[c])):
                raise ValueError(f"coordinate {c!r} differs between the cutouts; select matching ones with sel() first")
        shared = [n for n in b.keys() if n in a.keys()]
        if not override:
            for n in shared:
                if not _same_values(a, b, n):
                    raise ValueError(f"variable {n!r} differs between the cutouts; pass compat='override' to take "
                                     "this cutout's")
        coords = {**b.coords, **a.coords}
        lazy = getattr(a, "lazy", False) or getattr(b, "lazy", False)
        if not lazy:
            out = Dataset(coords=coords, attrs=attrs)
            for src in (b, a):
                out._vars.update(src._vars)
            return Cutout(path, data=out, devices=self._devices)
        loaders, static, dtypes, tc = {}, {}, {}, []
        nx = len(a.coords["x"])
        for src in (b, a):  # this cutout's variables last: they win
            for n in src.keys():
                loaders.pop(n, None)
                static.pop(n, None)
                dims = src.dims_of(n)
                if n in getattr(src, "_loaders", {}):
                    loaders[n], dtypes[n] = src._loaders[n], src.dtype_of(n)
                elif dims[:1] == ("time",):  # a device cutout's rows may be padded: crop them
                    arr = src.raw(n)
                    loaders[n] = (lambda lo, hi, arr=arr: _host_slice(arr, lo, hi)[..., :nx])
                    dtypes[n] = np.dtype(str(arr.dtype).replace("torch.", ""))
                else:
                    static[n] = (dims, src.raw(n))
            if getattr(src, "lazy", False):
                tc.append(src.time_chunk)
        out = LazyDataset(loaders, coords, attrs=attrs, time_chunk=min(tc), dtypes=dtypes)
        out._vars.update(static)
        return Cutout(path, data=out, devices=self._devices)

    def equals(self, other):
        """Same coordinates and variables, the path aside (cutout.py:591-598)."""
        if not isinstance(other, Cutout):
            return NotImplemented
        if hasattr(self.data, "equals") and not isinstance(self.data, Dataset):
            return bool(self.data.equals(other.data))
        a, b = self.data, other.data
        if not isinstance(b, Dataset) or getattr(a, "lazy", False) or getattr(b, "lazy", False):
            return False
        if set(a.keys()) != set(b.keys()) or set(a.coords) != set(b.coords):
            return False
        if any(not np.array_equal(np.asarray(a.coords[k]), np.asarray(b.coords[k])) for k in a.coords):
            return False
        host = lambda v: v.detach().cpu().numpy() if hasattr(v, "detach") else np.asarray(v)  # noqa: E731
        return all(a.dims_of(k) == b.dims_of(k) and np.array_equal(host(a.raw(k)), host(b.raw(k)), equal_nan=True)
                   for k in a.keys())

    def to_file(self, fn=None):
        """Save the cutout (cutout.py:453-465): NetCDF through xarray when the data is an xarray
        dataset, else this package's chunk container (zlib + byte shuffle, ``ingest.write_chunked``),
        which ``Cutout(path)`` opens lazily."""
        fn = self.path if fn is None else fn
        if fn is None:
            raise ValueError("no file name: the cutout has no path")
        if not isinstance(self.data, Dataset):
            self.data.to_netcdf(fn)
            return
        from . import ingest

        d = self.data
        if getattr(d, "lazy", False):
            d = d.isel_time(0, len(np.asarray(d.coords["time"])))
        host = lambda v: v.detach().cpu().numpy() if hasattr(v, "detach") else np.asarray(v)  # noqa: E731
        nx = len(np.asarray(d.coords["x"]))
        var3 = {k: host(d.raw(k))[..., :nx] for k in d.keys() if len(d.dims_of(k)) == 3}
        static = {k: host(d.raw(k))[..., :nx] for k in d.keys() if len(d.dims_of(k)) == 2}
        ingest.write_chunked(fn, var3, {k: np.asarray(v) for k, v in d.coords.items()}, static=static,
                             attrs=dict(getattr(d, "attrs", {})))

    @property
    def grid(self):
        """Cell centres in y-major, x-minor order: flat index s = iy*nx + ix."""
        x, y = np.asarray(self.coords["x"]), np.asarray(self.coords["y"])
        xs, ys = np.meshgrid(x, y)
        return pd.DataFrame({"x": xs.ravel(), "y": ys.ravel()})

    def uniform_layout(self):
        ny, nx = self.shape
        return make_dataarray(
            np.ones((ny, nx)), ("y", "x"),
            {"y": np.asarray(self.coords["y"]), "x": np.asarray(self.coords["x"])},
        )

    def indicatormatrix(self, shapes, shapes_crs=4326):
        """Cell x shape overlap matrix (cutout.py:492-515 -> gis.py:104-145): entry
        [i, j] is the fraction of grid cell j (``cutout.grid`` order) inside shape i.
        Computed on the GPU from the polygon edges (csrc/indicator.cu); shapes may be
        shapely / geopandas objects, GeoJSON dicts or coordinate arrays (see gis.py).
        Shapes must be in the cutout's CRS (no reprojection here)."""
        from . import gis

        self._require_own_crs(shapes_crs)
        return gis.compute_indicatormatrix(self.coords["x"], self.coords["y"], shapes)

    def intersectionmatrix(self, shapes, shapes_crs=4326):
        """Cell x shape incidence matrix (cutout.py:517-537 -> gis.py:148-183): entry
        [i, j] is 1.0 when shape i intersects the closed box of grid cell j
        (``cutout.grid`` order), a boundary contact included.  The boxes are the
        reference grid's own float64 boxes and the test is exact (csrc/indicator.cu).
        Shapes may be points, lines, polygons or collections of them, as shapely /
        geopandas objects, GeoJSON dicts or coordinate arrays (see gis.py).  Shapes
        must be in the cutout's CRS (no reprojection here)."""
        from . import gis

        self._require_own_crs(shapes_crs)
        return gis.compute_intersectionmatrix(self.coords["x"], self.coords["y"], shapes)

    def availabilitymatrix(self, shapes, excluder, nprocesses=None, disable_progressbar=True, shapes_crs=None):
        """(shape, y, x) share of each grid cell that is eligible land inside each shape
        (cutout.py:517 -> gis.py:586-661), computed on the GPU (``gis.compute_availabilitymatrix``):
        ``excluder`` is a ``gis.ExclusionContainer``; shapes take their CRS from ``.crs``, else
        ``shapes_crs``, else the cutout's.  ``nprocesses`` and ``disable_progressbar`` are unused."""
        from . import gis

        return gis.compute_availabilitymatrix(self, shapes, excluder, nprocesses, disable_progressbar, shapes_crs)

    def _require_own_crs(self, shapes_crs):
        if str(shapes_crs).upper().replace("EPSG:", "") != str(self.crs).upper().replace("EPSG:", ""):
            raise NotImplementedError(
                f"shapes_crs={shapes_crs!r}: reprojection is outside this package; "
                f"pass shapes in the cutout's CRS ({self.crs})"
            )

    # ---- host residency
    def pin_host(self, variables=None, devices=None):
        """Return a Cutout whose (time, y, x) variables live in page-locked host memory
        (float32 NumPy arrays).  Host-streamed conversions then DMA the time slabs directly at
        PCIe rate instead of staging pageable memory through the library's pinned ring.

        With ``devices`` (default: this cutout's ``devices``) the copy is NUMA-aware: the steps
        each GPU will stream (``dist.shard_bounds``) are first touched -- hence physically
        placed -- by a thread running on the CPUs next to that GPU, so that on a two-socket box
        no shard crosses the inter-socket link on its way to its GPU."""
        import torch

        from . import _lib
        from .dist import shard_bounds

        ds = self.data
        devs = self.devices if devices is None else Cutout(data=ds, devices=devices).devices
        names = list(ds.data_vars) if variables is None else list(variables)
        out = Dataset(coords={k: np.asarray(getattr(v, "values", v)) for k, v in dict(ds.coords).items()
                              if k in ("time", "x", "y", "lon", "lat")},
                      attrs=dict(getattr(ds, "attrs", {})))
        keep = []
        for n in names:
            a = _convert._to_host(_convert._raw(ds, n))
            if not (n.startswith("solar_") and a.dtype == np.float64):
                a = np.asarray(a, dtype=np.float32)
            if devs and len(devs) > 1 and a.ndim == 3:
                dst = _numa_sharded_copy(a, devs, shard_bounds, _lib.device_local_cpus)
                rc = torch.cuda.cudart().cudaHostRegister(dst.ctypes.data, dst.nbytes, 0)
                if int(rc) != 0:
                    raise RuntimeError(f"cudaHostRegister failed ({rc}) for variable {n!r}")
                keep.append(_Registered(dst))
                out[n] = (("time", "y", "x"), dst)
                continue
            t = torch.empty(a.shape, dtype=torch.from_numpy(a[:0].copy()).dtype, pin_memory=True)
            t.numpy()[...] = a
            keep.append(t)
            out[n] = (("time", "y", "x")[-a.ndim:], t.numpy())
        res = Cutout(data=out, time_shard=self.time_shard, devices=self._devices if devices is None else devices)
        res._pinned = keep  # these objects own the page-locked memory
        return res

    # ---- device residency
    def to_device(self, device=None, variables=None, pad=True):
        """Return a Cutout whose (time, y, x) variables live in GPU memory as
        float32 torch tensors (solar position variables keep float64).  With
        ``pad`` (default) rows are zero-padded to a multiple of 4 elements when
        the width is not one already, so that the 128-bit kernels apply (the
        padding is invisible: coordinates and results keep the logical width)."""
        import torch

        dev = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        ds = self.data
        names = list(ds.data_vars) if variables is None else list(variables)
        out = Dataset(coords={k: np.asarray(getattr(v, "values", v)) for k, v in dict(ds.coords).items()
                              if k in ("time", "x", "y", "lon", "lat")},
                      attrs=dict(getattr(ds, "attrs", {})))
        for n in names:
            arr = _convert._raw(ds, n)
            if not _convert.engine._is_torch(arr):
                a = np.asarray(arr)
                if not (n.startswith("solar_") and a.dtype == np.float64):
                    a = np.ascontiguousarray(a, dtype=np.float32)
                arr = torch.from_numpy(np.ascontiguousarray(a)).to(dev, non_blocking=False)
            nx = len(out.coords["x"])
            if pad and arr.shape[-1] == nx and nx % 4:
                arr = torch.nn.functional.pad(arr, (0, 4 - nx % 4))
            dims = ("time", "y", "x")[-arr.ndim:]
            out[n] = (dims, arr.contiguous())
        return Cutout(data=out, time_shard=self.time_shard)

    def __repr__(self):
        ny, nx = self.shape
        return f"<atlite_b200.Cutout {nx} x {ny} x {len(self.coords['time'])}>"

    # ---- conversion and aggregation (cutout.py:653-689)
    convert_and_aggregate = _convert.convert_and_aggregate
    convert_many = _convert.convert_many
    heat_demand = _convert.heat_demand
    cooling_demand = _convert.cooling_demand
    temperature = _convert.temperature
    soil_temperature = _convert.soil_temperature
    dewpoint_temperature = _convert.dewpoint_temperature
    coefficient_of_performance = _convert.coefficient_of_performance
    solar_thermal = _convert.solar_thermal
    irradiation = _convert.irradiation
    wind = _convert.wind
    pv = _convert.pv
    csp = _convert.csp
    runoff = _convert.runoff
    hydro = _convert.hydro
    line_rating = _convert.line_rating
