"""Cutout ingest without xarray: lazily loaded cutouts whose chunks are decoded by the
library's parallel chunk decoder (``atl_decode_chunks``, csrc/decode.cu).

The reference writes cutouts as NetCDF-4 (HDF5) with zlib level 9 + byte shuffle
(data.py:139,245-248) and opens them lazily with ``chunks={"time": 100}``
(cutout.py:142-154); every read then inflates chunk by chunk on one thread inside libhdf5.
Here a variable is described by a CHUNK INDEX -- where each compressed chunk sits in the
file -- and the time parts ``convert_and_aggregate`` asks for are decoded on all host cores
(pread + inflate + un-shuffle + scatter), optionally straight into page-locked memory, from
where the host-streaming entry points DMA them to the GPU.

Where the index comes from:
  * ``open_netcdf4(path)``   -- an HDF5 / NetCDF-4 file, index read with h5py's low-level
                                chunk query (``dataset.id.get_chunk_info``).  h5py is not part
                                of the build image, so this path is exercised only where it is
                                installed; there is no own HDF5 metadata parser (DESIGN.md).
  * ``open_chunked(path)``   -- the container ``write_chunked`` produces: the same chunk
                                encoding (zlib + HDF5 byte shuffle), chunks back to back in one
                                file and a kerchunk-style JSON index next to it.
  * ``open_netcdf3(path)``   -- NetCDF-3 classic files through scipy's memory map (no
                                compression in that format).
All three return an ``atlite_b200.LazyDataset`` ready for ``Cutout(data=...)``.

``open_grid(path)`` reads 2-D grids (GEBCO terrain) window by window instead: it returns the
coordinates and a variable that copies out only the rows and columns it is sliced at.
"""

from __future__ import annotations

import ctypes as C
import json
import os
import zlib

import numpy as np
import pandas as pd

from . import _lib
from .labelled import LazyDataset


class ChunkedVariable:
    """One (time, y, x) variable stored as compressed chunks in a file.  ``load`` decodes steps into
    host memory on host threads; ``load_device`` decodes them on the GPU into a device tensor, bit
    for bit the same values.  ``device_batch_bytes`` bounds the compressed and the decoded bytes of
    one batch of chunks on the device (a batch holds one chunk at least); None sizes the batches
    from the free device memory (``load_device_many``), so that one launch of the decoder gets
    many chunks."""

    device_batch_bytes = None

    def __init__(self, path, shape, chunk, dtype, offsets, sizes, origins, shuffle=True, deflate=True,
                 scale_factor=None, add_offset=None, fill_value=None, threads=0):
        self.path = os.fspath(path)
        self.shape = tuple(int(v) for v in shape)
        self.chunk = tuple(int(v) for v in chunk)
        self.dtype = np.dtype(dtype)
        self.offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        self.sizes = np.ascontiguousarray(sizes, dtype=np.int64)
        self.origins = np.ascontiguousarray(origins, dtype=np.int64).reshape(-1, 3)
        if not (len(self.offsets) == len(self.sizes) == len(self.origins)):
            raise ValueError("chunk index arrays differ in length")
        if len(self.shape) != 3 or len(self.chunk) != 3:
            raise ValueError("ChunkedVariable describes (time, y, x) variables")
        self.shuffle, self.deflate = bool(shuffle), bool(deflate)
        self.scale_factor, self.add_offset, self.fill_value = scale_factor, add_offset, fill_value
        self.threads = int(threads)
        order = np.argsort(self.origins[:, 0], kind="stable")  # by first time step: parts select a contiguous run
        self.offsets, self.sizes, self.origins = self.offsets[order], self.sizes[order], self.origins[order]

    def load(self, lo, hi, pinned=False):
        """Steps [lo, hi) decoded into a float32 (nt, ny, nx) array (native byte order; packed
        integer variables are unpacked with scale_factor / add_offset, the fill value -> NaN)."""
        lo, hi = int(lo), int(hi)
        nt, (_, ny, nx) = hi - lo, self.shape
        raw_dt = self.dtype.newbyteorder("=")
        if pinned:
            import torch

            t = torch.empty((nt, ny, nx), dtype=getattr(torch, raw_dt.name), pin_memory=True)
            out = t.numpy()
        else:
            out = np.empty((nt, ny, nx), dtype=raw_dt)
        if nt > 0:
            sel = np.flatnonzero((self.origins[:, 0] < hi) & (self.origins[:, 0] + self.chunk[0] > lo))
            spec = _lib.ChunkSpec()
            spec.ny, spec.nx, spec.elem_bytes = ny, nx, self.dtype.itemsize
            spec.shuffle, spec.deflate = int(self.shuffle), int(self.deflate)
            for i in range(3):
                spec.chunk[i] = self.chunk[i]
            offs, sizes = np.ascontiguousarray(self.offsets[sel]), np.ascontiguousarray(self.sizes[sel])
            orig = np.ascontiguousarray(self.origins[sel])
            covered = self._covers(orig, lo, hi)
            if not covered:
                out[...] = 0  # chunks never written (HDF5 leaves them out): fill value below
            _lib.check(_lib.load().atl_decode_chunks(self.path.encode(), C.byref(spec), len(sel), _lib.ptr(offs),
                                                     _lib.ptr(sizes), _lib.ptr(orig), lo, nt,
                                                     out.ctypes.data_as(C.c_void_p), self.threads))
        if self.dtype.byteorder == ">" or (self.dtype.byteorder == "=" and not np.little_endian):
            out.byteswap(inplace=True)
        if out.dtype == np.float32 and self.scale_factor is None and self.add_offset is None and self.fill_value is None:
            res = out
        else:
            res = out.astype(np.float32)
            if self.fill_value is not None:
                res[out == self.fill_value] = np.nan
            if self.scale_factor is not None:
                res *= np.float32(self.scale_factor)
            if self.add_offset is not None:
                res += np.float32(self.add_offset)
        return res  # a page-locked `out` stays alive through the array's base (the tensor's storage)

    def load_device(self, lo, hi, rows=None, cols=None, device=None, pitch=None):
        """Steps [lo, hi) x rows [r0, r1) x columns [c0, c1) (default: all) as a float32 CUDA tensor of
        shape (nt, r1 - r0, pitch) (pitch >= c1 - c0, default c1 - c0; the columns past the window
        are zero), equal bit for bit to ``load(lo, hi)[:, r0:r1, c0:c1]``.  Only the chunks that meet
        the window are read; they cross PCIe compressed and are inflated on the GPU."""
        return load_device_many([(self, lo, hi, rows, cols, pitch)], device)[0]

    def _window(self, lo, hi, rows, cols, pitch):
        lo, hi = int(lo), int(hi)
        nt, ny, nx = self.shape
        r0, r1 = (0, ny) if rows is None else (int(rows[0]), int(rows[1]))
        c0, c1 = (0, nx) if cols is None else (int(cols[0]), int(cols[1]))
        pitch = c1 - c0 if pitch is None else int(pitch)
        if not (0 <= lo <= hi <= nt and 0 <= r0 <= r1 <= ny and 0 <= c0 <= c1 <= nx and pitch >= c1 - c0):
            raise ValueError(f"window [{lo}, {hi}) x [{r0}, {r1}) x [{c0}, {c1}) (pitch {pitch}) outside "
                             f"the variable's {self.shape}")
        return lo, hi, r0, r1, c0, c1, pitch

    def _decode_device(self, out, lo, hi, r0, r1, c0, c1, pitch, batch_bytes):
        """Decode the window into ``out`` on the current stream (synchronous)."""
        from .engine import _stream_ptr

        _, ny, nx = self.shape
        sel = np.flatnonzero((self.origins[:, 0] < hi) & (self.origins[:, 0] + self.chunk[0] > lo))
        spec = _lib.ChunkSpec()
        spec.ny, spec.nx, spec.elem_bytes = ny, nx, self.dtype.itemsize
        spec.shuffle, spec.deflate = int(self.shuffle), int(self.deflate)
        for i in range(3):
            spec.chunk[i] = self.chunk[i]
        offs, sizes = np.ascontiguousarray(self.offsets[sel]), np.ascontiguousarray(self.sizes[sel])
        orig = np.ascontiguousarray(self.origins[sel])
        conv = self._device_convert()
        _lib.check(_lib.load().atl_decode_chunks_device(
            out.device.index, self.path.encode(), C.byref(spec), len(sel), _lib.ptr(offs), _lib.ptr(sizes),
            _lib.ptr(orig), lo, hi - lo, r0, r1 - r0, c0, c1 - c0, C.byref(conv), C.c_void_p(out.data_ptr()),
            pitch, int(batch_bytes), self.threads, _stream_ptr()))

    def _device_convert(self):
        """The ChunkConvert that makes the device path compute what ``load`` computes."""
        dt = self.dtype
        kinds = {"f": _lib.RAW_FLOAT, "i": _lib.RAW_INT, "u": _lib.RAW_UINT}
        if dt.kind not in kinds or (dt.kind == "f" and dt.itemsize == 2):
            raise NotImplementedError(f"chunks of dtype {dt} are not decoded on the device")
        c = _lib.ChunkConvert()
        c.kind = kinds[dt.kind]
        c.big_endian = int(dt.byteorder == ">" or (dt.byteorder == "=" and not np.little_endian))
        native = dt.newbyteorder("=")
        c.convert = int(not (native == np.float32 and self.scale_factor is None and self.add_offset is None
                             and self.fill_value is None))
        if self.fill_value is not None:
            try:  # `raw == fill` compares in NumPy's promoted type
                cmp = np.result_type(native, self.fill_value)
                fill = np.asarray(self.fill_value).astype(cmp).reshape(-1)[0]
            except (OverflowError, TypeError, ValueError):
                cmp = None  # an integer fill outside the raw type's range matches no element
            if cmp is not None:
                c.has_fill = 1
                if cmp.kind in "iu":
                    c.fill_as_int, c.fill_int = 1, int(fill)
                else:
                    c.fill = float(fill)
        if self.scale_factor is not None:
            c.has_scale, c.scale = 1, float(np.float32(self.scale_factor))
        if self.add_offset is not None:
            c.has_offset, c.offset = 1, float(np.float32(self.add_offset))
        return c

    def _covers(self, orig, lo, hi):
        nty = -(-(min(hi, self.shape[0]) - (lo // self.chunk[0]) * self.chunk[0]) // self.chunk[0])
        want = nty * -(-self.shape[1] // self.chunk[1]) * -(-self.shape[2] // self.chunk[2])
        return len(orig) >= want


# host staging of all concurrent device loads together: each keeps up to two batches of compressed
# chunks in page-locked memory
DEVICE_STAGING_BYTES = 4 << 30


def load_device_many(jobs, device=None):
    """Windows of several ChunkedVariables decoded on the GPU at the same time: ``jobs`` is a list of
    (variable, lo, hi, rows, cols, pitch) as ``ChunkedVariable.load_device`` takes them; returns
    their tensors in order.  Each variable is decoded on a stream of its own from a host thread of
    its own, so the decoder's launches of different variables run side by side; batches are sized
    from the device memory left free by the results (a variable's ``device_batch_bytes`` overrides
    that), so that a launch gets as many chunks as fit.  The values do not depend on either."""
    import torch

    if device is None:
        device = torch.cuda.current_device()
    dev = device if isinstance(device, torch.device) else torch.device("cuda", int(device))
    wins = [var._window(*rest) for var, *rest in jobs]
    outs = [torch.empty((w[1] - w[0], w[3] - w[2], w[6]), dtype=torch.float32, device=dev) for w in wins]
    todo = [k for k, o in enumerate(outs) if o.numel()]
    if not todo:
        return outs
    with torch.cuda.device(dev):
        torch.cuda.current_stream().synchronize()  # the results are allocated before the side streams write
        free = torch.cuda.mem_get_info()[0]
    n = len(todo)
    # scratch per load: up to two batches of compressed and of decoded bytes
    auto = max(64 << 20, min(free * 3 // 4 // (4 * n), DEVICE_STAGING_BYTES // n))

    def run(k):
        var = jobs[k][0]
        bb = auto if var.device_batch_bytes is None else var.device_batch_bytes
        with torch.cuda.device(dev):
            stream = torch.cuda.Stream(dev)
            with torch.cuda.stream(stream):
                var._decode_device(outs[k], *wins[k], bb)

    if n == 1:
        run(todo[0])
    else:
        from concurrent.futures import ThreadPoolExecutor

        with ThreadPoolExecutor(n) as ex:
            for f in [ex.submit(run, k) for k in todo]:
                f.result()
    return outs


class ChunkSource:
    """A window of a ``ChunkedVariable``: steps from ``t0`` on, rows [r0, r1), columns [c0, c1).
    ``LazyDataset`` keeps one per chunked variable through ``isel`` / ``sel``, so that
    ``Cutout.to_device()`` can decode exactly the selection on the GPU."""

    def __init__(self, var, t0=0, rows=None, cols=None):
        self.var, self.t0 = var, int(t0)
        self.rows = (0, var.shape[1]) if rows is None else tuple(int(v) for v in rows)
        self.cols = (0, var.shape[2]) if cols is None else tuple(int(v) for v in cols)

    def isel(self, pos):
        """The source of the selection ``pos`` ({dim: slice of positions within this window})."""
        def sub(span, sl):
            if sl is None:
                return span
            return span[0] + sl.start, span[0] + max(sl.start, sl.stop)

        t = pos.get("time")
        return ChunkSource(self.var, self.t0 + (t.start if t is not None else 0), sub(self.rows, pos.get("y")),
                           sub(self.cols, pos.get("x")))

    def job(self, nt, pitch=None):
        """The (variable, lo, hi, rows, cols, pitch) job of ``load_device_many`` for nt steps."""
        return (self.var, self.t0, self.t0 + nt, self.rows, self.cols, pitch)


def _lazy(variables, coords, static, attrs, time_chunk, pinned=False):
    loaders = {n: (lambda lo, hi, v=v: v.load(lo, hi, pinned=pinned)) for n, v in variables.items()}
    sources = {n: ChunkSource(v) for n, v in variables.items()}
    return LazyDataset(loaders, coords, static=static, attrs=attrs, time_chunk=time_chunk, sources=sources)


# ----------------------------------------------------------------------------------------
# the chunk container (tests, benchmarks, fast re-load of a prepared cutout)
# ----------------------------------------------------------------------------------------


def shuffle_bytes(a):
    """HDF5 shuffle filter: all first bytes of the elements, then all second bytes, ..."""
    a = np.ascontiguousarray(a)
    return a.view(np.uint8).reshape(-1, a.dtype.itemsize).T.copy().tobytes()


def write_chunked(path, data_vars, coords, chunk=(100, None, None), complevel=9, shuffle=True, static=None,
                  attrs=None):
    """Write (time, y, x) variables as zlib (+ byte shuffle) chunks, the encoding the reference
    uses for cutouts (data.py:245-248), plus ``<path>.index.json`` with the chunk index."""
    path = os.fspath(path)
    index = {"format": "atlite_b200-chunks-1", "variables": {}, "attrs": dict(attrs or {}), "static": {},
             "coords": {k: (pd.DatetimeIndex(v).as_unit("ns").asi8.tolist() if k == "time" else np.asarray(v).tolist())
                        for k, v in coords.items()}}
    with open(path, "wb") as fh:
        for name, arr in data_vars.items():
            arr = np.asarray(arr)
            nt, ny, nx = arr.shape
            c = tuple(int(min(s, n) if s else n) for s, n in zip(chunk, arr.shape))
            offs, sizes, orig = [], [], []
            for t in range(0, nt, c[0]):
                for y in range(0, ny, c[1]):
                    for x in range(0, nx, c[2]):
                        blk = np.zeros(c, dtype=arr.dtype)  # edge chunks are stored whole
                        part = arr[t:t + c[0], y:y + c[1], x:x + c[2]]
                        blk[:part.shape[0], :part.shape[1], :part.shape[2]] = part
                        raw = shuffle_bytes(blk) if shuffle else blk.tobytes()
                        comp = zlib.compress(raw, complevel) if complevel else raw
                        offs.append(fh.tell())
                        sizes.append(len(comp))
                        orig.append([t, y, x])
                        fh.write(comp)
            index["variables"][name] = dict(shape=list(arr.shape), chunk=list(c), dtype=arr.dtype.str,
                                            shuffle=bool(shuffle), deflate=bool(complevel), offsets=offs, sizes=sizes,
                                            origins=orig)
        for name, arr in (static or {}).items():
            index["static"][name] = np.asarray(arr).tolist()
    with open(path + ".index.json", "w") as fh:
        json.dump(index, fh)
    return path


def open_chunked(path, threads=0, pinned=False):
    path = os.fspath(path)
    with open(path + ".index.json") as fh:
        idx = json.load(fh)
    if idx.get("format") != "atlite_b200-chunks-1":
        raise ValueError(f"{path}.index.json is not a chunk index of this package")
    coords = {k: (pd.DatetimeIndex(np.asarray(v, dtype="int64").astype("datetime64[ns]")) if k == "time"
                  else np.asarray(v, dtype=np.float64)) for k, v in idx["coords"].items()}
    variables = {n: ChunkedVariable(path, v["shape"], v["chunk"], v["dtype"], v["offsets"], v["sizes"], v["origins"],
                                    v["shuffle"], v["deflate"], threads=threads) for n, v in idx["variables"].items()}
    static = {n: np.asarray(a, dtype=np.float32) for n, a in idx.get("static", {}).items()}
    tc = min((v.chunk[0] for v in variables.values()), default=100)
    return _lazy(variables, coords, static, idx.get("attrs", {}), tc, pinned)


# ----------------------------------------------------------------------------------------
# NetCDF-4 (HDF5) through h5py's chunk query; NetCDF-3 classic through scipy
# ----------------------------------------------------------------------------------------


def _cf_time(values, units, calendar="standard"):
    """CF 'units since epoch' -> DatetimeIndex (the encodings xarray writes for hourly data)."""
    unit, _, epoch = units.partition(" since ")
    scale = {"seconds": "s", "second": "s", "minutes": "m", "minute": "m", "hours": "h", "hour": "h",
             "days": "D", "day": "D"}[unit.strip().lower()]
    if calendar not in ("standard", "gregorian", "proleptic_gregorian"):
        raise NotImplementedError(f"calendar {calendar!r}")
    return pd.Timestamp(epoch.strip()) + pd.to_timedelta(np.asarray(values, dtype="float64"), unit=scale)


def open_netcdf4(path, threads=0, pinned=False):
    """A NetCDF-4 / HDF5 cutout as the reference writes it.  Needs h5py for the METADATA only
    (shapes, attributes, where every chunk sits); the chunk payloads are read and decoded by
    this package's native decoder."""
    try:
        import h5py
    except ImportError as e:  # pragma: no cover - h5py is not in the build image
        raise ImportError(
            "reading the chunk index of a NetCDF-4 / HDF5 cutout needs h5py (metadata only); "
            "without it, open the cutout with xarray or convert it once with ingest.write_chunked") from e
    path = os.fspath(path)
    variables, static, coords, attrs = {}, {}, {}, {}
    with h5py.File(path, "r") as f:  # pragma: no cover
        attrs = {k: (v.decode() if isinstance(v, bytes) else v) for k, v in f.attrs.items()}

        def decode(a):
            return a.decode() if isinstance(a, bytes) else a

        for name, d in f.items():
            if not isinstance(d, h5py.Dataset):
                continue
            if name in ("x", "y", "lon", "lat"):
                coords[name] = np.asarray(d[...], dtype=np.float64)
            elif name == "time":
                coords[name] = _cf_time(d[...], decode(d.attrs["units"]), decode(d.attrs.get("calendar", "standard")))
            elif d.ndim == 3:
                if d.chunks is None:
                    raise NotImplementedError(f"variable {name!r} is stored contiguously; use xarray for this file")
                other = [k for k in (d.compression, d.scaleoffset, d.fletcher32) if k not in (None, False, "gzip")]
                if other:
                    raise NotImplementedError(f"variable {name!r} uses filters {other}; only shuffle + gzip are decoded")
                n = d.id.get_num_chunks()
                info = [d.id.get_chunk_info(i) for i in range(n)]
                variables[name] = ChunkedVariable(
                    path, d.shape, d.chunks, d.dtype, [c.byte_offset for c in info], [c.size for c in info],
                    [list(c.chunk_offset) for c in info], shuffle=bool(d.shuffle), deflate=d.compression == "gzip",
                    scale_factor=d.attrs.get("scale_factor"), add_offset=d.attrs.get("add_offset"),
                    fill_value=d.attrs.get("_FillValue"), threads=threads)
            elif d.ndim == 2:
                static[name] = np.asarray(d[...], dtype=np.float32)
    coords.setdefault("lon", coords.get("x"))
    coords.setdefault("lat", coords.get("y"))
    tc = min((v.chunk[0] for v in variables.values()), default=100)
    return _lazy(variables, coords, static, attrs, max(tc, 1), pinned)


def open_netcdf3(path):
    """NetCDF-3 classic (no compression in this format): variables are memory-mapped by
    scipy and converted to native float32 part by part."""
    from scipy.io import netcdf_file

    f = netcdf_file(os.fspath(path), "r", mmap=True)
    coords, loaders, static = {}, {}, {}
    for name, v in f.variables.items():
        if name in ("x", "y", "lon", "lat"):
            coords[name] = np.array(v[:], dtype=np.float64)
        elif name == "time":
            cal = getattr(v, "calendar", b"standard")
            coords[name] = _cf_time(np.array(v[:]), v.units.decode(), cal.decode() if isinstance(cal, bytes) else cal)
        elif len(v.shape) == 3:
            sf, ao = getattr(v, "scale_factor", None), getattr(v, "add_offset", None)

            def load(lo, hi, v=v, sf=sf, ao=ao):
                a = np.array(v[lo:hi], dtype=np.float32)
                if sf is not None:
                    a *= np.float32(sf)
                if ao is not None:
                    a += np.float32(ao)
                return a

            loaders[name] = load
        elif len(v.shape) == 2:
            static[name] = np.array(v[:], dtype=np.float32)
    coords.setdefault("lon", coords.get("x"))
    coords.setdefault("lat", coords.get("y"))
    ds = LazyDataset(loaders, coords, static=static, attrs={}, time_chunk=100)
    ds._file = f  # keeps the memory map alive
    return ds


# ----------------------------------------------------------------------------------------
# 2-D grids read window by window (GEBCO terrain: 86400 x 43200 int16)
# ----------------------------------------------------------------------------------------


class GridVariable:
    """The 2-D (lat, lon) variable of a grid file, read only where it is sliced: ``v[r0:r1, c0:c1]``
    is a native-order NumPy copy of those rows and columns, in the file's dtype.  ``fill`` is the
    ``_FillValue`` (else ``missing_value``) in that dtype, or None; ``attrs`` the variable's
    attributes."""

    def __init__(self, var, shape, dtype, fill, attrs, owner):
        self._var, self.shape, self.dtype = var, tuple(int(n) for n in shape), np.dtype(dtype).newbyteorder("=")
        self.fill, self.attrs, self._owner = fill, attrs, owner  # the owner keeps the file open

    def read(self, rows, cols, out=None):
        """Rows ``rows`` x columns ``cols`` (slices) into ``out`` (a fresh array when None)."""
        part = self._var[rows, cols]
        if out is None:
            return np.array(part, dtype=self.dtype)
        np.copyto(out, part)
        return out

    def __getitem__(self, key):
        rows, cols = key
        return self.read(rows, cols)

    def window(self, r0, r1, c0, c1):
        return GridWindow(self, r0, r1, c0, c1)


class GridWindow:
    """Rows [r0, r1) x columns [c0, c1) of a ``GridVariable``, read row range by row range
    (``engine.RegridOp.window`` streams it to the GPU this way)."""

    def __init__(self, var, r0, r1, c0, c1):
        self.var, self.r0, self.c0 = var, int(r0), int(c0)
        self.shape, self.dtype = (int(r1) - int(r0), int(c1) - int(c0)), var.dtype

    def read(self, lo, hi, out=None):
        """Window rows [lo, hi) into ``out`` (a fresh array when None)."""
        return self.var.read(slice(self.r0 + lo, self.r0 + hi), slice(self.c0, self.c0 + self.shape[1]), out)

    def __array__(self, dtype=None, copy=None):
        a = self.read(0, self.shape[0])
        return a if dtype is None else a.astype(dtype)


def _attr(v):
    if isinstance(v, bytes):
        return v.decode()
    v = np.asarray(v)
    return v.item() if v.size == 1 else v


def _grid_parts(names, dims_of):
    """(variable name, lon name, lat name) of a grid file: ``elevation``, else its only 2-D variable."""
    lon = next((n for n in ("lon", "x") if n in names), None)
    lat = next((n for n in ("lat", "y") if n in names), None)
    if lon is None or lat is None:
        raise ValueError("a grid file needs 'lon' and 'lat' coordinate variables")
    two = [n for n in names if len(dims_of(n)) == 2]
    name = "elevation" if "elevation" in two else (two[0] if len(two) == 1 else None)
    if name is None:
        raise ValueError(f"no 'elevation' variable and not exactly one 2-D variable among {sorted(two)}")
    if tuple(dims_of(name)) != (lat, lon):
        raise ValueError(f"variable {name!r} has dims {tuple(dims_of(name))}, expected ({lat!r}, {lon!r})")
    return name, lon, lat


def open_grid(path):
    """(lon, lat, GridVariable) of a 2-D grid file such as GEBCO's: the ``lon`` / ``lat`` centres
    (float64, as stored) and its ``elevation`` variable (else its only 2-D variable), read only where
    it is sliced.  NetCDF-3 through scipy's memory map (big-endian on disk, converted while a window is
    copied out); NetCDF-4 through h5py, else xarray, for any storage layout.  Packed variables
    (``scale_factor`` / ``add_offset``) are refused."""
    path = os.fspath(path)
    with open(path, "rb") as fh:
        magic = fh.read(8)
    if magic[:3] == b"CDF":
        from scipy.io import netcdf_file

        f = netcdf_file(path, "r", mmap=True)
        name, lon, lat = _grid_parts(list(f.variables), lambda n: f.variables[n].dimensions)
        v = f.variables[name]
        var, dtype, attrs = v.data, v.data.dtype, {k: _attr(a) for k, a in v._attributes.items()}
        coords = np.array(f.variables[lon].data, dtype=np.float64), np.array(f.variables[lat].data, dtype=np.float64)
    elif magic == b"\x89HDF\r\n\x1a\n":  # pragma: no cover - needs h5py or xarray, not in the build image
        try:
            import h5py

            f = h5py.File(path, "r")
            names = [n for n in f if isinstance(f[n], h5py.Dataset)]
            # NetCDF-4 dims are HDF5 dimension scales; a coordinate variable is its own scale
            name, lon, lat = _grid_parts(names, lambda n: tuple(d[0].name.rsplit("/", 1)[-1] if len(d) else ""
                                                                for d in f[n].dims))
            var = f[name]
            attrs = {k: _attr(a) for k, a in var.attrs.items() if k not in ("DIMENSION_LIST", "REFERENCE_LIST")}
        except ImportError:
            import xarray as xr

            f = xr.open_dataset(path, mask_and_scale=False, decode_times=False)
            name, lon, lat = _grid_parts(list(f.variables), lambda n: f[n].dims)
            var, attrs = f[name].variable, {k: _attr(a) for k, a in f[name].attrs.items()}
        dtype = var.dtype
        coords = np.asarray(f[lon][...], dtype=np.float64), np.asarray(f[lat][...], dtype=np.float64)
    else:
        raise ValueError(f"{path}: neither a NetCDF-3 nor a NetCDF-4 / HDF5 file")
    if "scale_factor" in attrs or "add_offset" in attrs:
        raise ValueError(f"variable {name!r} is packed (scale_factor / add_offset); only unpacked grids are read")
    fill = next((attrs[k] for k in ("_FillValue", "missing_value") if k in attrs), None)
    if fill is not None:
        fill = np.asarray(fill).astype(dtype).item()
    shape = (len(coords[1]), len(coords[0]))
    return coords[0], coords[1], GridVariable(var, shape, dtype, fill, attrs, f)


def open_cutout(path, **kw):
    """Pick the reader by what the file is: chunk container (side-car index), HDF5 signature,
    NetCDF-3 classic magic."""
    path = os.fspath(path)
    if os.path.exists(path + ".index.json"):
        return open_chunked(path, **kw)
    with open(path, "rb") as fh:
        magic = fh.read(8)
    if magic == b"\x89HDF\r\n\x1a\n":
        return open_netcdf4(path, **kw)
    if magic[:3] == b"CDF":
        return open_netcdf3(path)
    raise ValueError(f"{path}: neither a chunk container, an HDF5 / NetCDF-4 file nor a NetCDF-3 file")
