"""Minimal labelled-array containers used when ``xarray`` is not installed.

The reference returns ``xarray.DataArray`` objects (convert.py:132-151).  If
xarray is importable the public API returns genuine xarray objects; otherwise
these light stand-ins carry the same information (``.values``, ``.dims``,
``.coords``, ``.attrs``, ``.name``) and the handful of methods the reference's
tests and typical user code touch (``sum``/``mean`` over a dim, ``sel``/``isel``,
``transpose``, ``notnull``, ``to_pandas``, element-wise arithmetic).
"""

from __future__ import annotations

import numbers

import numpy as np
import pandas as pd

try:  # pragma: no cover - depends on the environment
    import xarray as xr

    HAVE_XARRAY = True
except Exception:  # noqa: BLE001
    xr = None
    HAVE_XARRAY = False


class DataArray:
    __array_priority__ = 50

    def __init__(self, data, coords=None, dims=None, name=None, attrs=None):
        self.values = np.asarray(data)
        if dims is None:
            if coords is not None and not isinstance(coords, dict):
                raise TypeError("coords must be a dict when dims is not given")
            dims = tuple(coords) if coords else tuple(f"dim_{i}" for i in range(self.values.ndim))
        self.dims = tuple(dims)
        if len(self.dims) != self.values.ndim:
            raise ValueError(f"dims {self.dims} do not match data of ndim {self.values.ndim}")
        self.coords = {}
        for k, v in (coords or {}).items():
            self.coords[k] = v if isinstance(v, pd.Index) else np.asarray(v)
        self.name = name
        self.attrs = dict(attrs or {})

    # ---- basic protocol
    data = property(lambda self: self.values)
    shape = property(lambda self: self.values.shape)
    ndim = property(lambda self: self.values.ndim)
    dtype = property(lambda self: self.values.dtype)
    size = property(lambda self: self.values.size)

    @property
    def sizes(self):
        return dict(zip(self.dims, self.values.shape))

    @property
    def indexes(self):
        return {d: pd.Index(self.coords[d], name=d) for d in self.dims if d in self.coords}

    def __array__(self, dtype=None, copy=None):
        return np.asarray(self.values, dtype=dtype)

    def __len__(self):
        return len(self.values)

    def __repr__(self):
        return (
            f"<atlite_b200.DataArray {self.name or ''} "
            f"({', '.join(f'{d}: {n}' for d, n in self.sizes.items())}) {self.dtype}>\n"
            f"{self.values!r}\nattrs: {self.attrs}"
        )

    def __float__(self):
        return float(self.values)

    def __bool__(self):
        return bool(self.values)

    def item(self):
        return self.values.item()

    def load(self, **kwargs):
        return self

    def copy(self):
        return DataArray(self.values.copy(), dict(self.coords), self.dims, self.name, self.attrs)

    def rename(self, name):
        out = self.copy()
        out.name = name
        return out

    def _like(self, values, dims=None, drop=()):
        dims = self.dims if dims is None else tuple(dims)
        coords = {k: v for k, v in self.coords.items() if k in dims and k not in drop}
        return DataArray(values, coords, dims, self.name, self.attrs)

    # ---- reductions / selection
    def _reduce(self, fn, dim, keep_attrs):
        if dim is None:
            out = DataArray(fn(self.values, axis=None), {}, (), self.name)
        else:
            dims = [dim] if isinstance(dim, str) else list(dim)
            axes = tuple(self.dims.index(d) for d in dims)
            rest = tuple(d for d in self.dims if d not in dims)
            out = self._like(fn(self.values, axis=axes), rest)
        if not keep_attrs:
            out.attrs = {}
        return out

    def sum(self, dim=None, keep_attrs=False):
        return self._reduce(np.nansum, dim, keep_attrs)

    def mean(self, dim=None, keep_attrs=False):
        return self._reduce(np.nanmean, dim, keep_attrs)

    def max(self, dim=None, keep_attrs=False):
        return self._reduce(np.nanmax, dim, keep_attrs)

    def min(self, dim=None, keep_attrs=False):
        return self._reduce(np.nanmin, dim, keep_attrs)

    def all(self):
        return bool(np.all(self.values))

    def any(self):
        return bool(np.any(self.values))

    def notnull(self):
        return self._like(~pd.isnull(self.values))

    def isnull(self):
        return self._like(pd.isnull(self.values))

    def round(self, n=0):
        return self._like(np.round(self.values, n))

    def fillna(self, v):
        return self._like(np.where(np.isnan(self.values), v, self.values))

    def transpose(self, *dims):
        dims = tuple(dims) if dims else self.dims[::-1]
        perm = [self.dims.index(d) for d in dims]
        return self._like(self.values.transpose(perm), dims)

    T = property(lambda self: self.transpose())

    def isel(self, **idx):
        values, dims = self.values, list(self.dims)
        coords = dict(self.coords)
        for d, i in idx.items():
            ax = dims.index(d)
            values = np.take(values, i, axis=ax) if not isinstance(i, slice) else values[
                (slice(None),) * ax + (i,)
            ]
            if d in coords:
                coords[d] = np.asarray(coords[d])[i]
            if isinstance(i, numbers.Integral):
                dims.pop(ax)
                coords.pop(d, None)
        return DataArray(values, {k: v for k, v in coords.items() if k in dims}, dims, self.name, self.attrs)

    def sel(self, method=None, **labels):
        idx = {}
        for d, lab in labels.items():
            index = pd.Index(self.coords[d])
            if isinstance(index, pd.DatetimeIndex) or np.issubdtype(index.dtype, np.datetime64):
                lab = pd.Timestamp(lab)
            if method == "nearest":
                i = int(index.get_indexer([lab], method="nearest")[0])
            else:
                i = index.get_loc(lab)
            idx[d] = i
        return self.isel(**idx)

    def to_pandas(self):
        if self.ndim == 0:
            return self.values.item()
        if self.ndim == 1:
            return pd.Series(self.values, index=pd.Index(self.coords[self.dims[0]], name=self.dims[0]), name=self.name)
        if self.ndim == 2:
            return pd.DataFrame(
                self.values,
                index=pd.Index(self.coords[self.dims[0]], name=self.dims[0]),
                columns=pd.Index(self.coords[self.dims[1]], name=self.dims[1]),
            )
        raise ValueError("to_pandas supports at most 2 dimensions")

    # ---- arithmetic (same-dims or scalar / ndarray operands)
    def _binary(self, other, fn, reflexive=False):
        if isinstance(other, DataArray):
            if other.dims != self.dims:
                if set(other.dims) <= set(self.dims) or set(self.dims) <= set(other.dims):
                    big, small = (self, other) if len(self.dims) >= len(other.dims) else (other, self)
                    shape = [small.sizes.get(d, 1) for d in big.dims]
                    sv = small.transpose(*[d for d in big.dims if d in small.dims]).values.reshape(shape)
                    a, b = (self.values, sv) if big is self else (sv, other.values)
                    return big._like(fn(a, b))
                raise ValueError(f"cannot align dims {self.dims} and {other.dims}")
            o = other.values
        else:
            o = other
        return self._like(fn(o, self.values) if reflexive else fn(self.values, o))

    def __add__(self, o): return self._binary(o, np.add)
    def __radd__(self, o): return self._binary(o, np.add, True)
    def __sub__(self, o): return self._binary(o, np.subtract)
    def __rsub__(self, o): return self._binary(o, np.subtract, True)
    def __mul__(self, o): return self._binary(o, np.multiply)
    def __rmul__(self, o): return self._binary(o, np.multiply, True)
    def __truediv__(self, o): return self._binary(o, np.divide)
    def __rtruediv__(self, o): return self._binary(o, np.divide, True)
    def __gt__(self, o): return self._binary(o, np.greater)
    def __ge__(self, o): return self._binary(o, np.greater_equal)
    def __lt__(self, o): return self._binary(o, np.less)
    def __le__(self, o): return self._binary(o, np.less_equal)
    def __eq__(self, o): return self._binary(o, np.equal)  # noqa: E704
    def __ne__(self, o): return self._binary(o, np.not_equal)
    __hash__ = None


class Dataset:
    """name -> (time, y, x) arrays plus 1-D coordinates; the shape of ``cutout.data``."""

    def __init__(self, data_vars=None, coords=None, attrs=None):
        self.coords = {}
        for k, v in (coords or {}).items():
            self.coords[k] = v if isinstance(v, pd.Index) else np.asarray(v)
        self._vars = {}
        self.attrs = dict(attrs or {})
        for k, v in (data_vars or {}).items():
            self[k] = v

    def __setitem__(self, name, value):
        if isinstance(value, DataArray):
            self._vars[name] = (value.dims, value.values)
        elif isinstance(value, tuple):
            dims, arr = value
            self._vars[name] = (tuple(dims), arr if hasattr(arr, "ndim") else np.asarray(arr))
        else:
            arr = value if hasattr(value, "ndim") else np.asarray(value)
            dims = {3: ("time", "y", "x"), 2: ("y", "x"), 1: ("time",)}.get(arr.ndim)
            if dims is None:
                raise ValueError("cannot infer dims; pass (dims, array)")
            self._vars[name] = (dims, arr)

    def __contains__(self, name):
        return name in self._vars or name in self.coords

    def __iter__(self):
        return iter(self._vars)

    def keys(self):
        return self._vars.keys()

    @property
    def data_vars(self):
        return dict(self._vars)

    def raw(self, name):
        """The stored array object (NumPy or torch), without wrapping."""
        return self._vars[name][1]

    def dims_of(self, name):
        return self._vars[name][0]

    def isel_time(self, lo, hi):
        """Steps [lo, hi) of every variable that has a time axis (views, no copies);
        static (y, x) variables and the other coordinates are shared."""
        out = Dataset(coords={k: (v[lo:hi] if k == "time" else v) for k, v in self.coords.items()},
                      attrs=self.attrs)
        for name, (dims, arr) in self._vars.items():
            out._vars[name] = (dims, arr[lo:hi] if dims and dims[0] == "time" else arr)
        return out

    # ---- selection (what Cutout.sel needs of xarray.Dataset.sel: cutout.py:378-413)
    _AXIS_COORDS = {"time": ("time",), "y": ("y", "lat"), "x": ("x", "lon")}

    def _positions(self, indexers):
        """{dim: slice of integer positions} from integer slices (isel)."""
        out = {}
        for d, sl in indexers.items():
            if d not in self._AXIS_COORDS:
                raise KeyError(f"cannot select along {d!r}; dimensions are time, y, x")
            if not isinstance(sl, slice):
                raise TypeError(f"{d}: pass a slice (single labels would drop the dimension a cutout needs)")
            out[d] = slice(*sl.indices(len(self.coords[d])))
            if out[d].step != 1:
                raise ValueError(f"{d}: only contiguous selections keep the regular grid")
        return out

    def _sel_coords(self, pos):
        coords = {}
        for k, v in self.coords.items():
            dim = next((d for d, names in self._AXIS_COORDS.items() if k in names), None)
            coords[k] = v[pos[dim]] if dim in pos and np.ndim(v) == 1 else v
        return coords

    def isel(self, **indexers):
        """Contiguous positional selection along time / y / x (views of host arrays and of time
        slices of device tensors).  A device-resident cutout can only be cut along time: its
        rows may be padded to the kernels' pitch -- select before ``to_device()``."""
        pos = self._positions(indexers)
        out = Dataset(coords=self._sel_coords(pos), attrs=self.attrs)
        for name, (dims, arr) in self._vars.items():
            if any(d in pos and d in dims for d in ("y", "x")) and not isinstance(arr, np.ndarray):
                raise NotImplementedError("spatial selection of a device-resident cutout: select first, then to_device()")
            out._vars[name] = (dims, arr[tuple(pos.get(d, slice(None)) for d in dims)])
        return out

    def sel(self, **indexers):
        """Label-based selection with INCLUSIVE slice ends (xarray / pandas semantics) along
        time / y / x, e.g. ``ds.sel(x=slice(5, 15), y=slice(47, 55), time=slice("2013-01", "2013-02"))``."""
        pos = {}
        for d, sl in indexers.items():
            if d not in self._AXIS_COORDS:
                raise KeyError(f"cannot select along {d!r}; dimensions are time, y, x")
            idx = self.coords[d] if isinstance(self.coords[d], pd.Index) else pd.Index(self.coords[d])
            if not isinstance(sl, slice):
                sl = slice(sl, sl)
            loc = idx.slice_indexer(sl.start, sl.stop)
            pos[d] = slice(loc.start, loc.stop)
        return self.isel(**pos)

    def __getitem__(self, name):
        if name in self._vars:
            dims, arr = self._vars[name]
            coords = {d: self.coords[d] for d in dims if d in self.coords}
            return DataArray(np.asarray(arr), coords, dims, name)
        if name in self.coords:
            v = self.coords[name]
            dim = {"lon": "x", "lat": "y"}.get(name, name)
            return DataArray(np.asarray(v), {dim: self.coords.get(dim, v)}, (dim,), name)
        raise KeyError(name)

    @property
    def sizes(self):
        out = {}
        for dims, arr in self._vars.values():
            out.update(dict(zip(dims, arr.shape)))
        for d in ("time", "y", "x"):
            if d in self.coords and d not in out:
                out[d] = len(self.coords[d])
        return out

    @property
    def indexes(self):
        return {d: pd.Index(self.coords[d], name=d) for d in ("time", "y", "x") if d in self.coords}

    def __repr__(self):
        return f"<atlite_b200.Dataset vars={list(self._vars)} sizes={self.sizes}>"


class LazyDataset(Dataset):
    """A cutout whose (time, y, x) variables are read on demand: ``loaders`` maps a variable
    name to ``load(lo, hi) -> ndarray`` returning steps [lo, hi) (a NetCDF / HDF5 / zarr
    reader, a memory map ...).  ``convert_and_aggregate`` converts such a cutout time part
    by time part (``time_chunk`` steps at a time, the reference opens cutouts with
    ``chunks={"time": 100}``, cutout.py:143), so it never has to fit the host memory;
    static (y, x) variables are passed as arrays in ``static``.  ``sources`` maps a variable to
    the chunk window it reads (``ingest.ChunkSource``), which ``Cutout.to_device()`` decodes on
    the GPU; it follows ``isel`` / ``sel`` as the loaders do."""

    lazy = True

    def __init__(self, loaders, coords, static=None, attrs=None, time_chunk=100, dtypes=None, sources=None):
        super().__init__(static or {}, coords=coords, attrs=attrs)
        self._loaders = dict(loaders)
        self._sources = {n: s for n, s in (sources or {}).items() if n in self._loaders}
        self._dtypes = dict(dtypes or {})
        self.time_chunk = int(time_chunk)
        self.chunks = {"time": (self.time_chunk,)}
        self.loaded_steps = 0  # bookkeeping for tests: steps read so far / largest single read
        self.largest_read = 0

    def __contains__(self, name):
        return name in self._loaders or super().__contains__(name)

    def __iter__(self):
        return iter(list(self._loaders) + list(self._vars))

    def keys(self):
        return list(self._loaders) + list(self._vars)

    @property
    def data_vars(self):
        out = {n: (("time", "y", "x"), None) for n in self._loaders}
        out.update(self._vars)
        return out

    def dims_of(self, name):
        return ("time", "y", "x") if name in self._loaders else super().dims_of(name)

    def dtype_of(self, name):
        return np.dtype(self._dtypes.get(name, np.float32))

    def raw(self, name):
        if name in self._loaders:
            raise RuntimeError(f"variable {name!r} of a LazyDataset is only readable through isel_time(lo, hi)")
        return super().raw(name)

    def __getitem__(self, name):
        if name in self._loaders:
            n = len(self.coords["time"])
            return self.isel_time(0, n)[name]
        return super().__getitem__(name)

    def isel(self, **indexers):
        """Still lazy: the loaders of the selection read [lo + t0, hi + t0) and crop y / x."""
        pos = self._positions(indexers)
        t0 = pos["time"].start if "time" in pos else 0
        ys, xs = pos.get("y", slice(None)), pos.get("x", slice(None))

        def cropped(load):
            return lambda lo, hi: np.asarray(load(lo + t0, hi + t0))[:, ys, xs]

        static = {n: (dims, arr[tuple(pos.get(d, slice(None)) for d in dims)]) for n, (dims, arr) in self._vars.items()}
        out = LazyDataset({n: cropped(ld) for n, ld in self._loaders.items()}, self._sel_coords(pos),
                          attrs=self.attrs, time_chunk=self.time_chunk, dtypes=self._dtypes,
                          sources={n: s.isel(pos) for n, s in self._sources.items()})
        out._vars.update(static)
        return out

    def isel_time(self, lo, hi):
        out = Dataset(coords={k: (v[lo:hi] if k == "time" else v) for k, v in self.coords.items()},
                      attrs=self.attrs)
        for name, load in self._loaders.items():
            arr = np.asarray(load(lo, hi))
            if arr.shape[0] != hi - lo:
                raise ValueError(f"loader of {name!r} returned {arr.shape[0]} steps for [{lo}, {hi})")
            out._vars[name] = (("time", "y", "x"), arr)
        for name, (dims, arr) in self._vars.items():
            out._vars[name] = (dims, arr)
        self.loaded_steps += hi - lo
        self.largest_read = max(self.largest_read, hi - lo)
        return out


def make_dataarray(values, dims, coords, attrs=None, name=None):
    """Return an xarray.DataArray when xarray is installed, else the stand-in."""
    if HAVE_XARRAY:
        return xr.DataArray(values, coords=coords, dims=dims, attrs=attrs, name=name)
    return DataArray(values, coords, dims, name, attrs)


def is_dataarray(obj):
    return isinstance(obj, DataArray) or (HAVE_XARRAY and isinstance(obj, xr.DataArray))
