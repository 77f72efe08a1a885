"""Handle wrappers over the C ABI: aggregation plans and the pv / wind / heat
operators.  Arrays may be NumPy (host) or torch CUDA tensors (device-resident
cutout); host arrays go through the library's streaming entry points
(``atl_*_reduce_host``), device tensors through the kernel entry points.
"""

from __future__ import annotations

import ctypes as C
import os
import threading
from collections import OrderedDict

import numpy as np
import pandas as pd
import scipy.sparse as sp

from . import _lib


def _is_torch(x):
    return type(x).__module__.startswith("torch")


def _torch():
    import torch

    return torch


def current_device():
    try:
        torch = _torch()
        if torch.cuda.is_available():
            return torch.cuda.current_device()
    except Exception:  # noqa: BLE001
        pass
    return 0


def _stream_ptr():
    torch = _torch()
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dptr(x):
    if x is None:
        return None
    if _is_torch(x):
        assert x.is_cuda and x.is_contiguous()
        return C.c_void_p(x.data_ptr())
    raise TypeError("device pointer requested for a non-torch array")


def _hptr(x):
    if x is None:
        return None
    assert isinstance(x, np.ndarray) and x.flags["C_CONTIGUOUS"]
    return C.c_void_p(x.ctypes.data)


def host_f32(a):
    """C-contiguous float32 view/copy of a host array."""
    a = np.asarray(a)
    if a.dtype != np.float32 or not a.flags["C_CONTIGUOUS"]:
        a = np.ascontiguousarray(a, dtype=np.float32)
    return a


def pitch_of(arrays, nx):
    """Row pitch (elements) of a set of (time, y, x) fields: the last dimension of
    device tensors (``Cutout.to_device`` pads rows to a multiple of 4), ``nx`` for
    host arrays."""
    p = None
    for a in arrays:
        if a is None or getattr(a, "ndim", 0) != 3:
            continue
        w = int(a.shape[-1])
        if p is not None and w != p:
            raise ValueError("fields of one call must share the same row pitch")
        p = w
    p = nx if p is None else p
    if p < nx:
        raise ValueError(f"fields are narrower ({p}) than the grid ({nx})")
    if p != nx and not any(_is_torch(a) for a in arrays if a is not None):
        raise ValueError("host arrays must be unpadded (last dimension == nx)")
    return p


def time_ns(time):
    """datetime-like sequence -> contiguous int64 nanoseconds since the epoch (UTC)."""
    idx = pd.DatetimeIndex(np.asarray(time))
    return np.ascontiguousarray(idx.as_unit("ns").asi8, dtype=np.int64)


def device_csr(matrix):
    """A 2-D CUDA tensor as a canonical ``torch.sparse_csr`` tensor on its device.

    A dense tensor stores its nonzeros, NaN included, as ``sp.csr_matrix(dense)`` does.  A sparse
    CSR tensor must already be canonical (column indices strictly ascending within each row, so no
    duplicates): then its entries, their order and its row sums are those of the same scipy matrix.
    The check runs on the device."""
    torch = _torch()
    if not (_is_torch(matrix) and matrix.is_cuda):
        raise TypeError(f"expected a CUDA tensor, got {type(matrix).__name__}")
    if matrix.ndim != 2:
        raise ValueError("Matrix not 2-dimensional.")
    if matrix.layout == torch.strided:
        return matrix.to_sparse_csr()
    if matrix.layout != torch.sparse_csr:
        raise TypeError(f"a CUDA matrix must be dense or torch.sparse_csr, not {matrix.layout}")
    crow, col = matrix.crow_indices(), matrix.col_indices()
    nnz = col.numel()
    if nnz > 1:
        bad = col[1:] <= col[:-1]
        starts = crow[1:-1]
        bad[starts[(starts > 0) & (starts < nnz)] - 1] = False  # a row's first entry follows another row
        if bool(bad.any()):
            raise ValueError(
                "the sparse CSR matrix is not canonical: column indices must be strictly ascending within "
                "each row.  Canonicalise it through COO, .to_sparse_coo().coalesce().to_sparse_csr(); torch "
                "marks a COO tensor converted from CSR as coalesced, so rebuild it first: "
                "c = m.to_sparse_coo(); torch.sparse_coo_tensor(c.indices(), c.values(), c.shape)"
                ".coalesce().to_sparse_csr()")
    return matrix


class Plan:
    """Device-side aggregation plan built from an (n_bus, S) CSR matrix: a scipy matrix (or
    anything ``sp.csr_matrix`` takes), or a CUDA tensor (``device_csr``) whose plan is built
    without leaving the device."""

    def __init__(self, matrix, ny, nx, device=None, pitch=None, entries=False):
        """``entries``: keep the per-slot entry lists on the device even when the matrix does
        not tile well (``atl_plan_create_entries``; the line-rating kernel needs them)."""
        lib = _lib.load()
        self.grid = (ny, nx)
        self.device = current_device() if device is None else device
        self.pitch = nx if pitch is None else int(pitch)
        h = C.c_void_p()
        if _is_torch(matrix):
            torch = _torch()
            m = device_csr(matrix).to(f"cuda:{self.device}")
            self._check_columns(m.shape, ny, nx)
            self._matrix = m
            indptr = m.crow_indices().to(torch.int64).contiguous()
            indices = m.col_indices().to(torch.int32).contiguous()
            data = m.values().to(torch.float64).contiguous()
            stream = torch.cuda.current_stream(self.device).cuda_stream
            _lib.check(
                lib.atl_plan_create_device(
                    self.device, ny, nx, self.pitch, m.shape[0], data.numel(),
                    _dptr(indptr), _dptr(indices), _dptr(data), 1 if entries else 0, C.c_void_p(stream),
                    C.byref(h),
                )
            )
        else:
            m = sp.csr_matrix(matrix)
            m.sum_duplicates()
            self._check_columns(m.shape, ny, nx)
            self._matrix = None
            self._indptr = np.ascontiguousarray(m.indptr, dtype=np.int64)
            self._indices = np.ascontiguousarray(m.indices, dtype=np.int32)
            self._data = np.ascontiguousarray(m.data, dtype=np.float64)
            create = lib.atl_plan_create_entries if entries else lib.atl_plan_create_pitched
            _lib.check(
                create(
                    self.device, ny, nx, self.pitch, m.shape[0],
                    _lib.ptr(self._indptr), _lib.ptr(self._indices), _lib.ptr(self._data),
                    C.byref(h),
                )
            )
        self.shape = tuple(m.shape)
        self.handle = h
        info = _lib.PlanInfo()
        _lib.check(lib.atl_plan_info(h, C.byref(info)))
        self.info = {f[0]: getattr(info, f[0]) for f in _lib.PlanInfo._fields_}
        self.n_bus = m.shape[0]

    @staticmethod
    def _check_columns(shape, ny, nx):
        if shape[1] != ny * nx:
            raise ValueError(
                f"matrix has {shape[1]} columns but the cutout grid has {ny}x{nx}={ny * nx} cells"
            )

    def __del__(self):
        h = getattr(self, "handle", None)
        if h:
            try:
                _lib.load().atl_plan_destroy(h)
            except Exception:  # noqa: BLE001
                pass
            self.handle = None

    def spmm(self, dense):
        """(nt, ny, nx) | (nt, S) per-cell values (host or device) -> (nt, n_bus) float32."""
        torch = _torch()
        if not _is_torch(dense):
            dense = torch.from_numpy(host_f32(dense)).to(f"cuda:{self.device}")
        dense = dense.contiguous().to(torch.float32)
        nt = dense.shape[0]
        ny, nx = self.grid
        ok = (dense.ndim == 3 and tuple(dense.shape[1:]) == (ny, self.pitch)) or \
             (dense.ndim == 2 and dense.shape[1] == ny * self.pitch)
        if not ok:
            raise ValueError(f"per-cell values have shape {tuple(dense.shape)}; this plan expects "
                             f"(time, {ny}, {self.pitch}) or (time, {ny * self.pitch})")
        if dense.device.type != "cuda" or dense.device.index != self.device:
            raise ValueError(f"per-cell values live on {dense.device}, the plan on cuda:{self.device}")
        if self.pitch != nx and not self.info["fused"]:
            # a plan that does not tile gathers with the CSR indices, which address unpadded rows
            if getattr(self, "_flat", None) is None:
                m = self._matrix if self._matrix is not None else \
                    sp.csr_matrix((self._data, self._indices, self._indptr), shape=self.shape)
                self._flat = Plan(m, ny, nx, self.device)
            return self._flat.spmm(dense.reshape(nt, ny, self.pitch)[:, :, :nx].contiguous())
        out = torch.zeros((nt, self.n_bus), dtype=torch.float32, device=dense.device)
        if nt == 0:
            return out
        _lib.check(_lib.load().atl_spmm(self.handle, _dptr(dense), nt, _dptr(out), _stream_ptr()))
        return out


_PLAN_CACHE: "OrderedDict[tuple, Plan]" = OrderedDict()
_PLAN_LOCK = threading.Lock()
_PLAN_CACHE_SIZE = 4  # per device


def matrix_digest(m):
    """Content key of a CSR matrix for the plan cache: three 128-bit hashes (indptr, indices,
    data; ``atl_hash128``) next to shape, nnz and dtypes.  A collision would silently reuse a
    wrong plan, hence 3 x 128 bits; the hash sits on the critical path of every call, hence
    not hashlib (blake2b: 23 ms for the 15 MB of 1440 x 720 -> 3000 shapes; this: ~3 ms)."""
    lib = _lib.load()
    parts = []
    for seed, a in enumerate((m.indptr, m.indices, m.data)):
        b = np.ascontiguousarray(a)
        out = (C.c_uint64 * 2)()
        _lib.check(lib.atl_hash128(b.ctypes.data_as(C.c_void_p), b.nbytes, seed, out))
        parts += [int(out[0]), int(out[1]), b.nbytes, str(b.dtype)]
    return (m.shape, m.nnz, tuple(parts))


def get_plan(matrix, ny, nx, device=None, pitch=None, digest=None, entries=False):
    """Plans are cached (LRU, 4 entries per device): the typical workflow evaluates many
    technologies against the same shapes.  Thread-safe (one host thread per GPU in the
    single-process multi-GPU path); ``digest`` = a precomputed ``matrix_digest``;
    ``entries``: see ``Plan``.  A CUDA matrix is not cached: its plan is built on the device at
    every call."""
    device = current_device() if device is None else device
    pitch = nx if pitch is None else int(pitch)
    if _is_torch(matrix):
        return Plan(matrix, ny, nx, device, pitch, entries)
    m = sp.csr_matrix(matrix)
    key = (device, ny, nx, pitch) + (matrix_digest(m) if digest is None else digest) + (("entries",) if entries else ())
    with _PLAN_LOCK:
        plan = _PLAN_CACHE.get(key)
        if plan is not None:
            _PLAN_CACHE.move_to_end(key)
            return plan
    plan = Plan(m, ny, nx, device, pitch, entries)  # built outside the lock: devices build concurrently
    with _PLAN_LOCK:
        _PLAN_CACHE[key] = plan
        mine = [k for k in _PLAN_CACHE if k[0] == device]
        for k in mine[:-_PLAN_CACHE_SIZE]:
            del _PLAN_CACHE[k]
    return plan


# The field struct of each ``atl_<abi>_*`` family whose calls take one; the others take the
# pointer of their one field.
_FIELD_STRUCTS = {"pv": _lib.PvFields, "wind": _lib.WindFields, "wind_raw": _lib.WindRawFields,
                  "csp": _lib.CspFields, "line_rating": _lib.LineRatingFields,
                  "line_rating_raw": _lib.LineRatingRawFields}


class _Op:
    """Handle of an ``atl_<abi>_*`` operator (``abi`` = ``_abi``) on one GPU and grid.  Its calls
    take the fields as a dict (name -> array, None = absent) where the C calls take a field
    struct, as one array otherwise; all fields of a call are NumPy arrays (host, streamed) or
    CUDA tensors (device)."""

    _abi = None
    solar_f64 = False  # the stored solar position is read as float64 (ATL_SOLAR_STORED_F64)

    def _grid(self, ny, nx, device, pitch):
        self.device = current_device() if device is None else device
        self.ny, self.nx = ny, nx
        self.pitch = int(pitch) or nx

    def _create(self, create, cfg):
        h = C.c_void_p()
        _lib.check(create(self.device, C.byref(cfg), C.byref(h)))
        self.handle = h

    def __del__(self):
        h = getattr(self, "handle", None)
        if h:
            try:
                getattr(_lib.load(), f"atl_{self._abi}_destroy")(h)
            except Exception:  # noqa: BLE001
                pass
            self.handle = None

    @staticmethod
    def _all_device(arrs):
        kinds = {_is_torch(a) for a in arrs if a is not None}
        if len(kinds) > 1:
            raise ValueError("mixing host (NumPy) and device (torch) fields in one call")
        return kinds.pop() if kinds else False

    def _out(self, shape, like):
        torch = _torch()
        return torch.empty(shape, dtype=torch.float32, device=like.device)

    def _dev(self, a, f64=False):
        """Device field -> contiguous tensor, after checking what the kernels assume
        about it: (time, ny, pitch) layout on this operator's GPU, float32 (float64
        with ``f64``: a stored solar position the operator reads as float64).  The C
        ABI takes raw pointers, so this is the only place a wrong shape or width can
        be caught."""
        torch = _torch()
        pitch = getattr(self, "pitch", 0) or self.nx
        if a.ndim != 3 or tuple(a.shape[1:]) != (self.ny, pitch):
            raise ValueError(f"field has shape {tuple(a.shape)}, expected (time, {self.ny}, {pitch})")
        want = torch.float64 if f64 else torch.float32
        if a.dtype != want:
            raise TypeError(f"this device field must be {want}, got {a.dtype}")
        if a.device.type != "cuda" or a.device.index != self.device:
            raise ValueError(f"field lives on {a.device}, operator on cuda:{self.device}")
        return a.contiguous()

    def _host(self, a, f64=False):
        """Host field -> C-contiguous float32 array (float64 with ``f64``), copied when it is not one."""
        a = np.asarray(a)
        if a.ndim != 3 or a.shape[1:] != (self.ny, self.nx):
            raise ValueError(f"field has shape {a.shape}, expected (time, {self.ny}, {self.nx})")
        return np.ascontiguousarray(a, dtype=np.float64) if f64 else host_f32(a)

    @staticmethod
    def _empty_like(first, shape):
        """Result for an empty time axis (e.g. a rank whose time shard is empty): no
        kernel is launched (empty tensors have NULL data pointers)."""
        if _is_torch(first):
            torch = _torch()
            return torch.zeros(shape, dtype=torch.float32, device=first.device)
        return np.zeros(shape, dtype=np.float32)

    @staticmethod
    def _pack(struct, fields, conv):
        """``fields`` as the ctypes ``struct`` of field pointers (``conv(name, array)`` gives the
        array a pointer is taken from), and the arrays, which must outlive the call."""
        f, keep = struct(), []
        for n, _ in struct._fields_:
            a = fields.get(n)
            if a is not None:
                a = conv(n, a)
                keep.append(a)
                setattr(f, n, a.data_ptr() if _is_torch(a) else a.ctypes.data)
        return f, keep

    def _args(self, abi, fields, host):
        """The field argument of an ``atl_<abi>_*`` call, and what it points into.  The stored
        solar position has the operator's width (``solar_f64``): host arrays are converted to it,
        device tensors must have it; every other field is float32."""
        check = self._host if host else self._dev
        struct = _FIELD_STRUCTS.get(abi)
        if struct is None:
            a = check(fields)
            return C.c_void_p(a.ctypes.data if host else a.data_ptr()), [a]
        f, keep = self._pack(struct, fields, lambda n, a: check(a, f64=self.solar_f64 and n.startswith("solar_")))
        return C.byref(f), keep + [f]

    @staticmethod
    def _check_steps(fields, nt):
        """Every field must hold the ``nt`` steps a call reads: the C calls take raw pointers and
        would read past a shorter one."""
        items = fields.items() if isinstance(fields, dict) else [("field", fields)]
        for n, a in items:
            if a is not None and a.shape[0] < nt:
                raise ValueError(f"field {n!r} has {a.shape[0]} steps, the call reads {nt}")

    @staticmethod
    def _lead(fields, lead):
        if not isinstance(fields, dict):
            return fields
        return fields[lead] if lead else next(a for a in fields.values() if a is not None)

    def _reduce(self, plan, fields, nt=None, start=None, chunk_steps=0, lead=None, abi=None, steps=None):
        """(nt, n_bus) float32: torch CUDA tensor for device fields, ndarray for host fields.
        ``nt`` defaults to the steps of the ``lead`` field (the first one given); ``start`` is the
        time argument in front of ``nt``, if the call has one: t0, or heat's day table; ``steps``
        is the number of steps the call reads from every field (default ``nt``)."""
        abi = abi or self._abi
        dev = self._all_device(fields.values() if isinstance(fields, dict) else [fields])
        first = self._lead(fields, lead)
        nt = first.shape[0] if nt is None else nt
        self._check_steps(fields, nt if steps is None else steps)
        if nt == 0:
            return self._empty_like(first, (0, plan.n_bus))
        f, keep = self._args(abi, fields, host=not dev)
        targs = (nt,) if start is None else (start, nt)
        lib = _lib.load()
        if dev:
            out = self._out((nt, plan.n_bus), first)
            _lib.check(getattr(lib, f"atl_{abi}_reduce")(self.handle, plan.handle, f, *targs, _dptr(out), _stream_ptr()))
            return out
        out = np.empty((nt, plan.n_bus), dtype=np.float32)
        _lib.check(getattr(lib, f"atl_{abi}_reduce_host")(self.handle, plan.handle, f, *targs, _hptr(out), chunk_steps))
        return out

    def _cells(self, fields, timesum, nt=None, start=None, lead=None, abi=None, steps=None):
        """Per-cell values (nt, ny, nx), or with ``timesum`` their time sum and the count of valid
        steps as one (2, ny, nx) tensor; device fields only.  Arguments as for ``_reduce``."""
        abi = abi or self._abi
        first = self._lead(fields, lead)
        nt = first.shape[0] if nt is None else nt
        self._check_steps(fields, nt if steps is None else steps)
        if nt == 0:
            return self._empty_like(first, (2, self.ny, self.nx) if timesum else (0, self.ny, self.nx))
        f, keep = self._args(abi, fields, host=False)
        targs = (nt,) if start is None else (start, nt)
        lib = _lib.load()
        if timesum:
            torch = _torch()
            out = torch.zeros((2, self.ny, self.nx), dtype=torch.float32, device=first.device)  # sum | valid steps
            _lib.check(getattr(lib, f"atl_{abi}_timesum")(self.handle, f, *targs, _dptr(out[0]), _dptr(out[1]), _stream_ptr()))
        else:
            out = self._out((nt, self.ny, self.nx), first)
            _lib.check(getattr(lib, f"atl_{abi}_cells")(self.handle, f, *targs, _dptr(out), _stream_ptr()))
        return out


class PvOp(_Op):
    """convert_pv (convert.py:840-854) operator; see include/atlite_b200.h."""

    _abi = "pv"
    FIELD_NAMES = tuple(n for n, _ in _lib.PvFields._fields_)

    def __init__(self, *, ny, nx, time, lon, lat, slope, azimuth, tracking, trigon_model,
                 clearsky_model, irr_branch, albedo_src, solar_src, panel=None, time_shift="0h",
                 altitude_threshold=1.0, output="panel", thermal=(0.0, 0.0, 0.0), device=None, pitch=0):
        self._grid(ny, nx, device, pitch)
        self._time = time_ns(time)
        self.nt = len(self._time)
        self._lon, self._lat = _lib.as_f64(lon), _lib.as_f64(lat)
        slope, azimuth = np.asarray(slope, dtype=np.float64), np.asarray(azimuth, dtype=np.float64)
        self.orientation_2d = slope.ndim == 2 or azimuth.ndim == 2
        oshape = (ny, nx) if self.orientation_2d else (ny,)
        # (ny,) tables broadcast along x when the other one is 2-D
        self._slope = np.ascontiguousarray(np.broadcast_to(slope[:, None] if (self.orientation_2d and slope.ndim == 1) else slope, oshape))
        self._az = np.ascontiguousarray(np.broadcast_to(azimuth[:, None] if (self.orientation_2d and azimuth.ndim == 1) else azimuth, oshape))
        cfg = _lib.PvConfig()
        cfg.ny, cfg.nx, cfg.nt = ny, nx, self.nt
        cfg.time_ns = _lib.ptr(self._time).value
        cfg.time_shift_ns = int(pd.to_timedelta(time_shift).value)
        cfg.lon_deg, cfg.lat_deg = _lib.ptr(self._lon).value, _lib.ptr(self._lat).value
        cfg.slope_rad, cfg.azimuth_rad = _lib.ptr(self._slope).value, _lib.ptr(self._az).value
        cfg.tracking = _lib.TRACKING[tracking]
        cfg.trigon_model = trigon_model
        cfg.clearsky_model = clearsky_model
        cfg.irr_branch, cfg.albedo_src, cfg.solar_src = irr_branch, albedo_src, solar_src
        self.solar_f64 = solar_src == _lib.SOLAR_STORED_F64
        cfg.pitch = int(pitch)
        cfg.orientation_2d = 1 if self.orientation_2d else 0
        cfg.output = _lib.OUTPUT[output]
        for i, v in enumerate(thermal):
            cfg.thermal[i] = float(v)
        cfg.altitude_threshold_deg = altitude_threshold
        model = "huld" if panel is None else panel.get("model", "huld")
        if model not in _lib.PANEL:
            raise AssertionError(f"Unknown panel model: {model}")
        cfg.panel_model = _lib.PANEL[model]
        if panel is None:
            vals = []
        elif model == "huld":
            vals = [panel["c_temp_amb"], panel["c_temp_irrad"], panel["r_tmod"], panel["r_irradiance"]]
            vals += [panel[f"k_{i}"] for i in range(1, 7)]
            vals += [panel.get("inverter_efficiency", 1.0)]
        else:
            vals = [panel[k] for k in ("A", "B", "C", "D", "NOCT", "Tamb", "Intc", "Tstd", "ta", "threshold")]
            vals += [panel.get("inverter_efficiency", 1.0)]
        for i, v in enumerate(vals):
            cfg.panel[i] = float(v)
        self._create(_lib.load().atl_pv_create, cfg)

    def reduce(self, plan, fields, t0=0, nt=None, chunk_steps=0):
        """(nt, n_bus) float32: torch CUDA tensor for device fields, ndarray for host fields."""
        return self._reduce(plan, fields, nt, t0, chunk_steps)

    def cells(self, fields, t0=0, timesum=False):
        """Per-cell values (nt, ny, nx) or their time sum (ny, nx); device fields only."""
        return self._cells(fields, timesum, start=t0)


class WindOp(_Op):
    """convert_wind (convert.py:634-662) operator."""

    _abi = "wind"

    def __init__(self, *, ny, nx, V, POW_norm, method, from_height, to_height, device=None, pitch=0):
        self._grid(ny, nx, device, pitch)
        self._V, self._P = _lib.as_f64(V), _lib.as_f64(POW_norm)
        cfg = _lib.WindConfig()
        cfg.ny, cfg.nx, cfg.method = ny, nx, method
        cfg.from_height, cfg.to_height = float(from_height), float(to_height)
        cfg.pitch = int(pitch)
        cfg.n_knots = len(self._V)
        cfg.V, cfg.POW_norm = _lib.ptr(self._V).value, _lib.ptr(self._P).value
        self._create(_lib.load().atl_wind_create, cfg)

    def reduce_raw(self, plan, fields, chunk_steps=0):
        """``reduce`` on raw ERA5 variables: ``fields`` maps u100, v100 and, for the log / power
        law, fsr / u10, v10 to (time, y, x) arrays (host or device); see atl_wind_raw_reduce."""
        return self._reduce(plan, fields, chunk_steps=chunk_steps, lead="u100", abi="wind_raw")

    def cells_raw(self, fields, timesum=False):
        """``cells`` on raw ERA5 variables (device fields only)."""
        return self._cells(fields, timesum, lead="u100", abi="wind_raw")

    def reduce(self, plan, wnd, aux=None, chunk_steps=0):
        return self._reduce(plan, {"wnd": wnd, "aux": aux}, chunk_steps=chunk_steps, lead="wnd")

    def cells(self, wnd, aux=None, timesum=False):
        return self._cells({"wnd": wnd, "aux": aux}, timesum, lead="wnd")


class HeatOp(_Op):
    """convert_heat_demand (convert.py:405-418) operator."""

    _abi = "heat"

    def __init__(self, *, ny, nx, threshold, a, constant, cooling=False, device=None, pitch=0):
        self._grid(ny, nx, device, pitch)
        cfg = _lib.HeatConfig()
        cfg.ny, cfg.nx = ny, nx
        cfg.threshold_c, cfg.a, cfg.constant = float(threshold), float(a), float(constant)
        cfg.cooling = 1 if cooling else 0
        cfg.pitch = int(pitch)
        self._create(_lib.load().atl_heat_create, cfg)

    def _days(self, temperature, day_start):
        """The day table as int64, its number of days and the step its last day ends at, after
        checking that ``temperature`` holds that step: the C calls see the offsets, not the
        field's length."""
        ds = np.ascontiguousarray(day_start, dtype=np.int64)
        end = int(ds[-1]) if len(ds) else 0
        self._check_steps(temperature, end)
        return ds, len(ds) - 1, end

    def reduce(self, plan, temperature, day_start, chunk_days=0):
        ds, nd, end = self._days(temperature, day_start)
        if nd == 0 or temperature.shape[0] == 0:
            return self._empty_like(temperature, (nd, plan.n_bus))
        return self._reduce(plan, temperature, nd, _lib.ptr(ds), chunk_days, steps=end)

    def cells(self, temperature, day_start, timesum=False):
        ds, nd, end = self._days(temperature, day_start)
        if nd == 0 or temperature.shape[0] == 0:
            return self._empty_like(temperature, (2, self.ny, self.nx) if timesum else (nd, self.ny, self.nx))
        return self._cells(temperature, timesum, nd, _lib.ptr(ds), steps=end)


class PointwiseOp(_Op):
    """Pointwise function of one field (temperature family, COP, runoff x height);
    see include/atlite_b200.h."""

    _abi = "pointwise"

    def __init__(self, *, ny, nx, shift=0.0, nan_to_zero=False, poly=None, cell_scale=None, clip_min_zero=False,
                 device=None, pitch=0):
        """``clip_min_zero``: clip the field at 0 first (NaN stays), as sanitize_runoff clips the raw
        ERA5 runoff ``ro`` (datasets/era5.py:241-246)."""
        self._grid(ny, nx, device, pitch)
        cfg = _lib.PointwiseConfig()
        cfg.ny, cfg.nx = ny, nx
        cfg.shift = float(shift)
        cfg.pitch = int(pitch)
        cfg.nan_to_zero = 1 if nan_to_zero else 0
        cfg.poly = 0 if poly is None else 1
        if poly is not None:
            cfg.sink, cfg.c0, cfg.c1, cfg.c2 = (float(v) for v in poly)
        self._scale = None
        if cell_scale is not None:
            self._scale = host_f32(cell_scale)
            if self._scale.shape != (ny, nx):
                raise ValueError(f"cell_scale must have shape {(ny, nx)}, has {self._scale.shape}")
            cfg.cell_scale = self._scale.ctypes.data
        lib = _lib.load()
        if clip_min_zero:
            self._create(lib.atl_pointwise_create_ex, _lib.PointwiseConfigEx(base=cfg, clip_min_zero=1))
        else:
            self._create(lib.atl_pointwise_create, cfg)

    def reduce(self, plan, field, chunk_steps=0):
        return self._reduce(plan, field, chunk_steps=chunk_steps)

    def cells(self, field, timesum=False):
        return self._cells(field, timesum)


class CspOp(_Op):
    """convert_csp (convert.py:940-972) operator.  ``raw``: the ``influx_direct`` field is the raw
    ERA5 ``fdir`` (hourly J m-2), from which the kernel derives the direct influx as era5.prepare
    does (``atl_csp_raw_create``)."""

    _abi = "csp"

    def __init__(self, *, ny, nx, time, lon, lat, solar_src, technology, r_irradiance, altitude, azimuth,
                 efficiency, time_shift="0h", dni_altitude_threshold=3.75, raw=False, device=None, pitch=0):
        self._grid(ny, nx, device, pitch)
        self._time = time_ns(time)
        self._lon, self._lat = _lib.as_f64(lon), _lib.as_f64(lat)
        self._alt, self._az, self._eff = _lib.as_f64(altitude), _lib.as_f64(azimuth), _lib.as_f64(efficiency)
        cfg = _lib.CspConfig()
        cfg.ny, cfg.nx, cfg.nt = ny, nx, len(self._time)
        cfg.time_ns = _lib.ptr(self._time).value
        cfg.time_shift_ns = int(pd.to_timedelta(time_shift).value)
        cfg.lon_deg, cfg.lat_deg = _lib.ptr(self._lon).value, _lib.ptr(self._lat).value
        cfg.solar_src = solar_src
        self.solar_f64 = solar_src == _lib.SOLAR_STORED_F64
        cfg.pitch = int(pitch)
        cfg.technology = technology
        cfg.r_irradiance = float(r_irradiance)
        cfg.dni_altitude_threshold_deg = float(dni_altitude_threshold)
        cfg.n_alt, cfg.n_az = len(self._alt), len(self._az)
        cfg.altitude_rad, cfg.azimuth_rad = _lib.ptr(self._alt).value, _lib.ptr(self._az).value
        cfg.efficiency = _lib.ptr(self._eff).value
        lib = _lib.load()
        self._create(lib.atl_csp_raw_create if raw else lib.atl_csp_create, cfg)

    def reduce(self, plan, fields, t0=0, chunk_steps=0):
        return self._reduce(plan, fields, start=t0, chunk_steps=chunk_steps, lead="influx_direct")

    def cells(self, fields, t0=0, timesum=False):
        return self._cells(fields, timesum, start=t0, lead="influx_direct")


class LineRatingOp(_Op):
    """convert_line_rating (convert.py:1152-1252) of every line of a plan, min-reduced over the
    line's cells; see include/atlite_b200.h.  ``params``: dict of the six per-line arrays
    psi, R, D, Ts, epsilon, alpha (psi as convert_line_rating takes it)."""

    _abi = "line_rating"

    def __init__(self, *, ny, nx, time, lon, lat, solar_src, params, time_shift="0h", device=None, pitch=0):
        self._grid(ny, nx, device, pitch)
        self._time = time_ns(time)
        self.nt = len(self._time)
        self._lon, self._lat = _lib.as_f64(lon), _lib.as_f64(lat)
        self._params = {k: _lib.as_f64(params[k]) for k in _lib.LINE_PARAMS}
        self.n_lines = len(self._params["psi"])
        cfg = _lib.LineRatingConfig()
        cfg.ny, cfg.nx, cfg.pitch, cfg.nt = ny, nx, int(pitch), self.nt
        cfg.time_ns = _lib.ptr(self._time).value
        cfg.time_shift_ns = int(pd.to_timedelta(time_shift).value)
        cfg.lon_deg, cfg.lat_deg = _lib.ptr(self._lon).value, _lib.ptr(self._lat).value
        cfg.solar_src = solar_src
        self.solar_f64 = solar_src == _lib.SOLAR_STORED_F64
        cfg.n_lines = self.n_lines
        for k, v in self._params.items():
            setattr(cfg, k, _lib.ptr(v).value)
        self._create(_lib.load().atl_line_rating_create, cfg)

    def reduce(self, plan, fields, t0=0):
        """(nt, n_lines) float32 torch CUDA tensor from DEVICE fields (time, ny, pitch); height is
        (ny, pitch).  NaN where a line has no valid cell."""
        return self._line_reduce(plan, fields, t0, "line_rating", "temperature")

    def reduce_raw(self, plan, fields, t0=0):
        """``reduce`` on raw ERA5 variables: ``fields`` maps t2m, u100, v100, fdir (time, ny, pitch),
        height (ny, pitch) and a stored solar position (if any) to DEVICE tensors; the wind speed,
        wind azimuth and direct influx are derived in-kernel (atl_line_rating_raw_reduce)."""
        return self._line_reduce(plan, fields, t0, "line_rating_raw", "t2m")

    def _line_reduce(self, plan, fields, t0, abi, lead):
        torch = _torch()
        first = fields[lead]
        nt = first.shape[0]

        def conv(n, a):
            if n == "height":
                if tuple(a.shape) != (self.ny, self.pitch) or a.dtype != torch.float32 or a.device != first.device:
                    raise ValueError(f"height must be a float32 ({self.ny}, {self.pitch}) tensor on {first.device}")
                return a.contiguous()
            a = self._dev(a, f64=self.solar_f64 and n.startswith("solar_"))
            if a.shape[0] != nt:
                raise ValueError(f"field {n!r} has {a.shape[0]} steps, {lead} {nt}")
            return a

        f, keep = self._pack(_FIELD_STRUCTS[abi], fields, conv)
        out = self._out((nt, plan.n_bus), first)
        _lib.check(getattr(_lib.load(), f"atl_{abi}_reduce")(self.handle, plan.handle, C.byref(f), t0, nt, _dptr(out),
                                                             _stream_ptr()))
        return out


class StreamJob:
    """One reduce of a shared pass over host fields (``reduce_host_many``): what ``op.reduce(plan,
    fields, ...)`` takes, with ``abi`` the job's field family (default the operator's), ``t0`` the
    PV / CSP time offset, ``day_start`` heat demand's day table and ``chunk`` the slab length of the
    job's own call (steps, or days for heat; 0: that call's default), which it keeps in the pass."""

    def __init__(self, op, plan, fields, abi=None, t0=0, day_start=None, chunk=0):
        self.op, self.plan, self.fields = op, plan, fields
        self.abi = abi or op._abi
        self.t0, self.chunk = int(t0), int(chunk)
        self.day_start = None if day_start is None else np.ascontiguousarray(day_start, dtype=np.int64)
        if self.abi not in _lib.JOB:
            raise ValueError(f"no shared host pass for {self.abi!r} operators")
        if (self.abi == "heat") != (self.day_start is not None):
            raise ValueError("heat jobs, and only they, take a day table")
        arrs = list(fields.values()) if isinstance(fields, dict) else [fields]
        if any(_is_torch(a) for a in arrs if a is not None):
            raise ValueError("a shared host pass takes host (NumPy) fields")
        if self.day_start is None:
            self.rows = self.steps = op._lead(fields, None).shape[0]
        else:
            self.rows = len(self.day_start) - 1
            self.steps = int(self.day_start[-1]) if len(self.day_start) else 0


def reduce_host_many(jobs, chunk_units=0):
    """Run ``jobs`` (StreamJob) over their host fields in one pass of their time slabs through the
    device ring (atl_reduce_host_many): each distinct host array is copied host -> device once per
    slab, however many jobs read it, and each job reduces the slabs its own call would, so its result
    is that call's bit for bit.  Returns the (rows, n_bus) float32 result of every job (rows: days of
    a heat job, steps otherwise) and the pass's ``{"h2d_bytes", "n_slabs"}``.  ``chunk_units``: the
    ring's slab length in steps; 0 picks ~192 MiB of the jobs' input per slab."""
    stats = {"h2d_bytes": 0, "n_slabs": 0}
    if not jobs:
        return [], stats
    nt = {j.steps for j in jobs if j.day_start is None}
    if len(nt) > 1:
        raise ValueError(f"the step jobs of one pass must read the same steps, not {sorted(nt)}")
    # the steps every field of the pass holds: the step jobs' own, or enough for every day table
    nt = nt.pop() if nt else min(j.fields.shape[0] for j in jobs)
    conv = {}  # one converted copy per source array, so that jobs reading one field share its host pointer

    def host(op, name, a):
        f64 = op.solar_f64 and name.startswith("solar_")
        key = (id(a), f64)
        if key not in conv:
            conv[key] = (a, op._host(a, f64=f64))
        return conv[key][1]

    keep, arr, outs = [], (_lib.StreamJob * len(jobs))(), []
    for k, j in enumerate(jobs):
        j.op._check_steps(j.fields, j.steps)
        if isinstance(j.fields, dict):
            f, kp = j.op._pack(_FIELD_STRUCTS[j.abi], j.fields, lambda n, a, op=j.op: host(op, n, a))
            ptr = C.addressof(f)
        else:
            f = host(j.op, "field", j.fields)
            kp, ptr = [], f.ctypes.data
        out = np.empty((max(j.rows, 0), j.plan.n_bus), dtype=np.float32)
        outs.append(out)
        keep += [f, kp]
        arr[k] = _lib.StreamJob(_lib.JOB[j.abi], j.op.handle.value, j.plan.handle.value, ptr, j.t0,
                                None if j.day_start is None else j.day_start.ctypes.data,
                                0 if j.day_start is None else len(j.day_start) - 1, j.chunk, out.ctypes.data)
    op0 = jobs[0].op
    st = _lib.StreamStats()
    _lib.check(_lib.load().atl_reduce_host_many(op0.device, op0.ny, op0.nx, nt, arr, len(jobs), chunk_units,
                                                C.byref(st)))
    stats.update(h2d_bytes=st.h2d_bytes, n_slabs=st.n_slabs)
    return outs, stats


def hydro_shift_sum(runoff, entry_ptr, rows, shifts, weights, device=None):
    """(n_plants, nt) float64 torch CUDA tensor: per plant p the sum, in entry order, of
    ``weights[e] * runoff[rows[e]]`` rolled forward in time by ``shifts[e]`` steps (np.roll
    semantics: any integer, negative and >= nt wrap), e in ``entry_ptr[p]:entry_ptr[p + 1]``
    (atl_hydro_shift_sum).  ``runoff``: (n_rows, nt) NumPy array or torch tensor, taken as float64."""
    torch = _torch()
    device = current_device() if device is None else device
    dev = f"cuda:{device}"
    entry_ptr = np.ascontiguousarray(entry_ptr, dtype=np.int64)
    rows = np.ascontiguousarray(rows, dtype=np.int32)
    n_plants = len(entry_ptr) - 1
    R = runoff if _is_torch(runoff) else torch.from_numpy(np.ascontiguousarray(runoff, dtype=np.float64))
    R = R.to(device=dev, dtype=torch.float64).contiguous()
    if R.ndim != 2:
        raise ValueError("runoff must be (n_rows, nt)")
    n_rows, nt = int(R.shape[0]), int(R.shape[1])
    if entry_ptr.ndim != 1 or n_plants < 0 or entry_ptr[0] != 0 or (np.diff(entry_ptr) < 0).any() or not (
            len(rows) == len(shifts) == len(weights) == entry_ptr[-1]):
        raise ValueError("entry_ptr must be a CSR row pointer over rows, shifts and weights")
    n_ent = int(entry_ptr[-1])
    if n_ent and (rows.min() < 0 or rows.max() >= n_rows):
        raise ValueError(f"entry rows must lie in [0, {n_rows})")

    def up(a, dt):
        return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(dev)

    ptr_d, rows_d = up(entry_ptr, np.int64), up(rows, np.int32)
    shifts_d, w_d = up(shifts, np.int64), up(weights, np.float64)
    out = torch.empty((n_plants, nt), dtype=torch.float64, device=dev)
    with torch.cuda.device(device):
        _lib.check(_lib.load().atl_hydro_shift_sum(device, n_rows, nt, _dptr(R), n_plants, _dptr(ptr_d),
                                                   _dptr(rows_d), _dptr(shifts_d), _dptr(w_d), _dptr(out),
                                                   _stream_ptr()))
    return out


def line_rating_eval(values, device=None):
    """Elementwise convert_line_rating: ``values`` maps the names of ``_lib.LineRatingFlat`` to
    arrays (or scalars) of one broadcast shape; returns float32 NumPy values of that shape."""
    torch = _torch()
    device = current_device() if device is None else device
    arrs = np.broadcast_arrays(*[np.asarray(values[n], dtype=np.float64) for n, _ in _lib.LineRatingFlat._fields_])
    shape = arrs[0].shape
    f = _lib.LineRatingFlat()
    keep = []
    for (n, _), a in zip(_lib.LineRatingFlat._fields_, arrs):
        dt = torch.float64 if n in _lib.LINE_PARAMS else torch.float32
        t = torch.from_numpy(np.ascontiguousarray(a.reshape(-1))).to(device=f"cuda:{device}", dtype=dt)
        keep.append(t)
        setattr(f, n, t.data_ptr())
    out = torch.empty(int(np.prod(shape)), dtype=torch.float32, device=f"cuda:{device}")
    with torch.cuda.device(device):
        _lib.check(_lib.load().atl_line_rating_eval(device, out.numel(), C.byref(f), _dptr(out), _stream_ptr()))
    return out.cpu().numpy().reshape(shape)


def _batched(src, src_shape, dst_shape, slab_bytes, device, run):
    """``run`` on a (batch, *src_shape) CUDA tensor as it is; a NumPy array goes to ``device`` in batch
    slabs of at most ``slab_bytes`` source bytes (one entry at least) and comes back as NumPy."""
    if _is_torch(src):
        return run(src)
    torch = _torch()
    src = np.asarray(src)
    out = np.empty((src.shape[0],) + tuple(dst_shape), dtype=src.dtype)
    step = max(1, slab_bytes // max(1, src_shape[0] * src_shape[1] * src.itemsize))
    for b0 in range(0, src.shape[0], step):
        part = torch.from_numpy(np.ascontiguousarray(src[b0:b0 + step])).to(f"cuda:{device}")
        out[b0:b0 + step] = run(part).cpu().numpy()
    return out


def _device_field(t, ny, nx, device):
    """A (batch, ny, nx) CUDA tensor on ``device`` whose rows the kernels can read with strides."""
    if t.ndim != 3 or tuple(t.shape[1:]) != (ny, nx):
        raise ValueError(f"field has shape {tuple(t.shape)}, expected (batch, {ny}, {nx})")
    if t.device.type != "cuda" or t.device.index != device:
        raise ValueError(f"field lives on {t.device}, operator on cuda:{device}")
    if t.stride(2) != 1 or t.stride(1) < nx or (t.shape[0] > 1 and t.stride(0) < ny * t.stride(1)):
        t = t.contiguous()
    return t


class RegridOp(_Op):
    """Separable regrid tables on one GPU (atl_regrid_create).  ``ytab`` / ``xtab`` are
    ``(first, count, weights)`` per destination row / column: int32 (n,), int32 (n,) and float64
    (n, k), weights[j, :count[j]] for source indices first[j] ... first[j] + count[j] - 1."""

    _abi = "regrid"
    HOST_SLAB_BYTES = 256 << 20  # source bytes per host -> device slab
    RING_STAGES, SMEM_MAX = 4, 160 << 10  # csrc/regrid.cu: RG_STAGES, RG_SMEM_MAX

    @classmethod
    def ring_fits(cls, xtab):
        """Whether atl_regrid_create accepts the x table ``xtab``: the shared memory of a column tile
        one destination column wide (its x weights, then the ring of float64 source rows; regrid.cu's
        regrid_smem), the narrowest tile the plan splits a row into, must fit in SMEM_MAX.  Computed
        on the host, so a caller can choose another kernel before any device work."""
        _, count, w = xtab
        kx = max(1, np.shape(w)[1])
        span = max(1, int(np.max(count, initial=0)))
        slot = (span * 8 + 15) // 16 * 16 + 16
        return (kx * 8 + 15) // 16 * 16 + cls.RING_STAGES * slot <= cls.SMEM_MAX

    def __init__(self, src_shape, ytab, xtab, device=None):
        lib = _lib.load()
        self.device = current_device() if device is None else int(device)
        self.ny, self.nx = (int(n) for n in src_shape)
        (yf, yc, yw), (xf, xc, xw) = ([np.ascontiguousarray(a, dtype=dt) for a, dt in
                                       zip(tab, (np.int32, np.int32, np.float64))] for tab in (ytab, xtab))
        self.dst_shape = (len(yf), len(xf))
        h = C.c_void_p()
        _lib.check(lib.atl_regrid_create(self.device, self.ny, self.nx, len(yf), len(xf), yw.shape[1], _lib.ptr(yf),
                                         _lib.ptr(yc), _lib.ptr(yw), xw.shape[1], _lib.ptr(xf), _lib.ptr(xc),
                                         _lib.ptr(xw), C.byref(h)))
        self.handle = h
        v = [C.c_int32() for _ in range(4)]
        _lib.check(lib.atl_regrid_info(h, *[C.byref(x) for x in v]))
        self.info = dict(zip(("n_bands", "n_ctiles", "tile_cols", "max_span"), (x.value for x in v)))

    def __call__(self, src, nodata=None, empty=None):
        """(batch, ny, nx) float32 / float64 values -> (batch, ny_dst, nx_dst) of the same dtype.  A CUDA
        tensor (on this operator's device; its rows may be strided) is resampled in place into a
        tensor on that device; a NumPy array goes through in slabs of HOST_SLAB_BYTES and comes back
        as a NumPy array.  ``nodata`` (atl_regrid_nodata): values equal to it are skipped like NaN;
        ``empty``: the value of a cell without a valid value (default NaN)."""
        return _batched(src, (self.ny, self.nx), self.dst_shape, self.HOST_SLAB_BYTES, self.device,
                        lambda t: self._device(t, nodata, empty))

    def _device(self, t, nodata=None, empty=None):
        torch = _torch()
        lib = _lib.load()
        fn = {torch.float32: lib.atl_regrid_f32, torch.float64: lib.atl_regrid_f64}.get(t.dtype)
        if fn is None:
            raise TypeError(f"regrid supports float32 and float64, not {t.dtype}")
        t = _device_field(t, self.ny, self.nx, self.device)
        out = torch.empty((t.shape[0],) + self.dst_shape, dtype=t.dtype, device=t.device)
        strides = (t.stride(1), max(t.stride(0), self.ny * t.stride(1)))
        with torch.cuda.device(self.device):
            if nodata is None and empty is None:
                _lib.check(fn(self.handle, t.shape[0], C.c_void_p(t.data_ptr()), *strides, _dptr(out), _stream_ptr()))
            else:
                has = nodata is not None and not np.isnan(nodata)
                _lib.check(lib.atl_regrid_nodata(self.handle, _lib.REGRID_DTYPE[str(t.dtype)[6:]], t.shape[0],
                                                 C.c_void_p(t.data_ptr()), *strides, int(has),
                                                 float(nodata) if has else 0.0,
                                                 np.nan if empty is None else float(empty), _dptr(out), _stream_ptr()))
        return out

    WINDOW_SLAB_BYTES = 64 << 20  # source bytes per host -> device band of a 2-D window

    def window(self, src, fill=None):
        """(ny_dst, nx_dst) average of one 2-D (ny, nx) int16 / float32 / float64 window
        (atl_regrid_window): values equal to ``fill`` are skipped like NaN and a cell without a valid
        value gets ``fill`` (else NaN); int16 results are rounded half away from zero.  A CUDA tensor
        (on this operator's device, rows may be strided) gives a tensor on that device.  Host input,
        a NumPy array or a reader with ``shape``, ``dtype`` and ``read(lo, hi, out)`` (rows [lo, hi)
        into ``out``, like ``ingest.GridWindow``), gives a NumPy array: it goes to the device in bands
        of destination rows whose source rows fit in WINDOW_SLAB_BYTES, the next band's read and copy
        overlapping the current band's kernel."""
        torch = _torch()
        dtype = np.dtype(str(src.dtype).replace("torch.", "")).newbyteorder("=")
        if dtype.name not in _lib.REGRID_DTYPE:
            raise TypeError(f"a window must be int16, float32 or float64, not {dtype}")
        if tuple(src.shape) != (self.ny, self.nx):
            raise ValueError(f"window has shape {tuple(src.shape)}, expected ({self.ny}, {self.nx})")
        if fill is not None and dtype.kind == "i" and not (np.iinfo(dtype).min <= fill <= np.iinfo(dtype).max):
            fill = None  # no int16 pixel can equal it
        code, fv = _lib.REGRID_DTYPE[dtype.name], (0.0 if fill is None else float(fill))
        lib = _lib.load()
        dev = f"cuda:{self.device}"

        def launch(t, out, band0, n_bands, row0, n_rows):
            _lib.check(lib.atl_regrid_window(self.handle, code, band0, n_bands, C.c_void_p(t.data_ptr()), row0,
                                             n_rows, t.stride(0), int(fill is not None), fv, _dptr(out), _stream_ptr()))

        n_bands = self.info["n_bands"]
        if _is_torch(src):
            if src.device.type != "cuda" or src.device.index != self.device:
                raise ValueError(f"window lives on {src.device}, operator on cuda:{self.device}")
            if src.stride(1) != 1:
                src = src.contiguous()
            out = torch.empty(self.dst_shape, dtype=src.dtype, device=src.device)
            with torch.cuda.device(self.device):
                launch(src, out, 0, n_bands, 0, self.ny)
            return out
        read = src.read if hasattr(src, "read") else (lambda lo, hi, out: np.copyto(out, src[lo:hi]))
        groups = self._window_bands(self.nx * dtype.itemsize)
        rows = max([hi - lo for _, _, lo, hi in groups] + [1])
        tdt = getattr(torch, dtype.name)
        out = torch.empty(self.dst_shape, dtype=tdt, device=dev)
        with torch.cuda.device(self.device):
            compute, copy = torch.cuda.current_stream(), torch.cuda.Stream()
            pinned = [torch.empty((rows, self.nx), dtype=tdt, pin_memory=True) for _ in range(2)]
            staged = [torch.empty((rows, self.nx), dtype=tdt, device=dev) for _ in range(2)]
            copied = [torch.cuda.Event() for _ in range(2)]
            used = [torch.cuda.Event() for _ in range(2)]
            for k, (band0, nb, lo, hi) in enumerate(groups):
                s = k % 2
                if k >= 2:
                    copied[s].synchronize()  # the pinned buffer's previous copy has left it
                read(lo, hi, pinned[s].numpy()[:hi - lo])
                copy.wait_event(used[s])  # the device buffer's previous kernel is done with it
                with torch.cuda.stream(copy):
                    staged[s][:hi - lo].copy_(pinned[s][:hi - lo], non_blocking=True)
                    copied[s].record(copy)
                compute.wait_event(copied[s])
                launch(staged[s], out, band0, nb, lo, hi - lo)
                used[s].record(compute)
            res = out.cpu().numpy()
        return res

    def _window_bands(self, row_bytes):
        """[(first band, bands, first source row, end row)]: consecutive kernel bands grouped so that
        each group's source rows fit in WINDOW_SLAB_BYTES (one band at least)."""
        n = self.info["n_bands"]
        lo, hi = np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32)
        _lib.check(_lib.load().atl_regrid_band_rows(self.handle, _lib.ptr(lo), _lib.ptr(hi)))
        limit = max(1, self.WINDOW_SLAB_BYTES // max(1, row_bytes))
        groups = []
        for b in range(n):
            if hi[b] == lo[b]:  # reads no row: joins any group
                lo[b], hi[b] = (groups[-1][2], groups[-1][3]) if groups else (0, 0)
            if groups:
                b0, nb, glo, ghi = groups[-1]
                nlo, nhi = (min(glo, lo[b]), max(ghi, hi[b])) if ghi > glo else (lo[b], hi[b])
                if nhi - nlo <= limit:
                    groups[-1] = (b0, nb + 1, int(nlo), int(nhi))
                    continue
            groups.append((b, 1, int(lo[b]), int(hi[b])))
        return groups


class ReprojectOp:
    """A warp between two axis-aligned grids in CRSs of ``proj.SUPPORTED`` on one GPU (atl_reproject).
    ``src`` / ``dst``: (transform, (ny, nx), CRS key); a transform is the 6-tuple (a, 0, c, 0, e, f),
    either sign of a and e.  ``resampling`` 0 (nearest), 5 (average) or one of the statistics 6
    (mode), 8 (max), 9 (min), 10 (med), 11 (q1), 12 (q3), 13 (sum), 14 (rms) (rasterio's values;
    DESIGN.md section 1).  NaN and ``src_nodata`` are skipped; a cell without a valid pixel gets
    ``dst_nodata``.  Nothing is built per destination cell: the kernel computes each footprint.  The
    pair of CRSs may be the same one (the identity projection); ``tables`` builds the operator on
    regrid's tables instead."""

    HOST_SLAB_BYTES = 256 << 20  # source bytes per host -> device slab
    # the selections (med, q1, q3, mode): device scratch per band of cells (0: the library's 1 GiB)
    # and the largest box one thread selects (-1: the library's 32 pixels; 0: every box goes through
    # the scratch)
    SELECT_SCRATCH_BYTES = 0
    SELECT_SMALL = -1

    def __init__(self, src, dst, resampling, src_nodata=None, dst_nodata=np.nan, device=None, tile=None):
        from . import proj

        self.device = current_device() if device is None else int(device)
        (sa, _, sc, _, se, sf), (self.ny, self.nx), skey = src
        (da, _, dc, _, de, df), self.dst_shape, dkey = dst
        self.dst_shape = tuple(int(n) for n in self.dst_shape)
        r = _lib.Reproject()
        r.src = _lib.Lattice(float(sc), float(sa), float(sf), float(se), int(self.nx), int(self.ny))
        r.dst = _lib.Lattice(float(dc), float(da), float(df), float(de), self.dst_shape[1], self.dst_shape[0])
        r.proj = proj.device_projection(dkey, skey)  # destination points into the source CRS
        r.resampling = int(resampling)
        r.has_nodata = int(src_nodata is not None and not np.isnan(src_nodata))
        r.src_nodata = float(src_nodata) if r.has_nodata else 0.0
        r.dst_nodata = float(dst_nodata)
        r.tile_y, r.tile_x = tile if tile is not None else self._tile(src, dst)
        self.desc = r
        self.spans = None

    @classmethod
    def tables(cls, src_shape, ytab, xtab, resampling, src_nodata=None, dst_nodata=np.nan, device=None):
        """The warp whose boxes are regrid's average tables ``ytab`` / ``xtab`` (``(first, count,
        weights)`` per destination row / column over the stored source order, ``regrid_axis``), for
        every resampling but nearest: cell (i, j) takes the source rows and columns of ``ytab[i]`` and
        ``xtab[j]`` with the product of their weights.  Such a table is a box: every weight between
        its first and last is 1 (padded pixels fold into the border pixels, which are first or last)."""
        ny, nx = (int(n) for n in src_shape)
        dst_shape = (len(ytab[0]), len(xtab[0]))
        unit = (1.0, 0.0, 0.0, 0.0, 1.0, 0.0)
        op = cls((unit, (ny, nx), 4326), (unit, dst_shape, 4326), resampling, src_nodata, dst_nodata, device,
                 tile=cls._table_tile(ytab, xtab))
        op.spans = (cls._spans(ytab), cls._spans(xtab))
        return op

    @staticmethod
    def _spans(tab):
        first, count, w = (np.asarray(a) for a in tab)
        spans = (_lib.Span * max(1, len(first)))()
        for k, (f, c) in enumerate(zip(first.tolist(), count.tolist())):
            if c <= 0:
                continue
            if c > 2 and not (w[k, 1:c - 1] == 1.0).all():
                raise ValueError("a regrid table entry is not a box: weights between its ends differ from 1")
            spans[k].lo, spans[k].hi, spans[k].w_lo, spans[k].w_hi = f, f + c, float(w[k, 0]), float(w[k, c - 1])
        return spans

    @staticmethod
    def _table_tile(ytab, xtab):
        """``_tile``'s rule on the median table box."""
        yc, xc = np.asarray(ytab[1]), np.asarray(xtab[1])
        px = float(np.median(yc)) * float(np.median(xc)) if len(yc) and len(xc) else 1.0
        if px <= 32:
            return 8, 32
        cells = 1 << int(np.clip(np.floor(np.log2(ReprojectOp.TILE_PIXELS / px)), 0, 8))
        return max(1, cells // 32), min(cells, 32)

    TILE_PIXELS = 4096  # source pixels per CTA and batch entry the average kernel aims at

    @staticmethod
    def _tile(src, dst):
        """The average kernel's CTA tile (tile_y, tile_x): 8 x 32 cells when the typical footprint is
        small enough for one thread (32 pixels), else fewer cells, so that a CTA still sums about
        TILE_PIXELS pixels per batch entry and large footprints spread over many CTAs.  The median
        footprint comes from 17 x 17 cells sampled across the destination with proj.py."""
        from . import proj

        (sa, _, sc, _, se, sf), (sny, snx), skey = src
        (da, _, dc, _, de, df), (dny, dnx), dkey = dst
        if dny == 0 or dnx == 0:
            return 8, 32
        ii = np.unique(np.linspace(0, dny - 1, 17).astype(np.int64))[:, None]
        jj = np.unique(np.linspace(0, dnx - 1, 17).astype(np.int64))[None, :]
        with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
            u0, v0 = proj.transform(dc + jj * da + 0 * ii, df + ii * de + 0 * jj, dkey, skey)
            u1, v1 = proj.transform(dc + (jj + 1) * da + 0 * ii, df + (ii + 1) * de + 0 * jj, dkey, skey)
            w = np.clip(np.ceil(np.fmax((u0 - sc) / sa, (u1 - sc) / sa)), 0, snx) - \
                np.clip(np.floor(np.fmin((u0 - sc) / sa, (u1 - sc) / sa)), 0, snx)
            h = np.clip(np.ceil(np.fmax((v0 - sf) / se, (v1 - sf) / se)), 0, sny) - \
                np.clip(np.floor(np.fmin((v0 - sf) / se, (v1 - sf) / se)), 0, sny)
        n = (w * h)[np.isfinite(w * h) & (w * h > 0)]
        px = float(np.median(n)) if len(n) else 1.0
        if px <= 32:
            return 8, 32
        cells = 1 << int(np.clip(np.floor(np.log2(ReprojectOp.TILE_PIXELS / px)), 0, 8))
        return max(1, cells // 32), min(cells, 32)

    def __call__(self, src):
        """(batch, ny, nx) float32 / float64 values -> (batch, *dst_shape) of the same dtype.  A CUDA
        tensor (on this operator's device; its rows may be strided) is read in place and gives a
        tensor on that device; a NumPy array goes through in batch slabs of HOST_SLAB_BYTES and comes
        back as a NumPy array.  Each slab is one launch over whole 2-D entries, so a host entry must
        fit on the device."""
        return _batched(src, (self.ny, self.nx), self.dst_shape, self.HOST_SLAB_BYTES, self.device, self._device)

    def _device(self, t):
        torch = _torch()
        code = {torch.float32: 1, torch.float64: 2}.get(t.dtype)  # ATL_REGRID_F32 / _F64
        if code is None:
            raise TypeError(f"reproject supports float32 and float64, not {t.dtype}")
        t = _device_field(t, self.ny, self.nx, self.device)
        out = torch.empty((t.shape[0],) + self.dst_shape, dtype=t.dtype, device=t.device)
        o = _lib.ReprojectOptions()
        if self.spans is not None:
            o.row_spans, o.col_spans = C.addressof(self.spans[0]), C.addressof(self.spans[1])
        o.scratch_bytes, o.select_small = int(self.SELECT_SCRATCH_BYTES), int(self.SELECT_SMALL)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().atl_reproject_ex(self.device, C.byref(self.desc), C.byref(o), code, t.shape[0],
                                                    C.c_void_p(t.data_ptr()), t.stride(1),
                                                    max(t.stride(0), self.ny * t.stride(1)), _dptr(out), _stream_ptr()))
        return out


class SarahOp(_Op):
    """SARAH's gap filling and pair mean on one GPU (atl_sarah_fill) for (time, ny, nx) float32 SIS and
    SID fields.  A call fills NaNs within the time blocks starting at ``block_starts`` (``fill`` one
    of FILL_INTERP, FILL_ZERO, FILL_NONE) and, with ``hourly``, averages steps (2k, 2k + 1) into step k."""

    _abi = "sarah"
    MAX_BLOCKS = 512  # ATL_SARAH_MAX_BLOCKS
    FILL_NONE, FILL_ZERO, FILL_INTERP = 0, 1, 2  # ATL_SARAH_FILL_*

    def __init__(self, ny, nx, device=None):
        self._grid(int(ny), int(nx), device, 0)

    def launches(self, block_starts, nt, hourly, batch=None):
        """[(lo, hi, block starts relative to lo)] of the launches a call makes: at most ``batch``
        (default MAX_BLOCKS) blocks each, cut at block starts only, and with ``hourly`` at even steps
        only, so that no block and no pair spans two launches."""
        starts = [int(s) for s in block_starts]
        if nt and (not starts or starts[0] != 0 or any(b <= a for a, b in zip(starts, starts[1:])) or starts[-1] >= nt):
            raise ValueError(f"block starts must ascend strictly from 0 and lie below {nt}")
        batch = self.MAX_BLOCKS if batch is None else int(batch)
        if not 1 <= batch <= self.MAX_BLOCKS:
            raise ValueError(f"batch must be in [1, {self.MAX_BLOCKS}]")
        out, i = [], 0
        while i < len(starts):
            j = min(i + batch, len(starts))
            while hourly and j < len(starts) and starts[j] % 2:
                j -= 1  # back to an even cut
            if j == i:
                raise ValueError(f"no even block start within {batch} blocks of step {starts[i]}")
            hi = starts[j] if j < len(starts) else nt
            out.append((starts[i], hi, [s - starts[i] for s in starts[i:j]]))
            i = j
        return out

    def __call__(self, sis, sid, block_starts, fill=2, hourly=True, batch=None):
        """(filled SIS, filled SID), each (nt // 2 if hourly else nt, ny, nx) float32: CUDA tensors
        on this operator's device for CUDA tensors, NumPy arrays for NumPy arrays (moved one
        launch at a time).  ``batch``: blocks per launch (see ``launches``); the result does not
        depend on it."""
        torch = _torch()
        device = self._all_device([sis, sid])
        nt = sis.shape[0]
        for a in (sis, sid):
            if tuple(a.shape) != (nt, self.ny, self.nx):
                raise ValueError(f"field has shape {tuple(a.shape)}, expected ({nt}, {self.ny}, {self.nx})")
        if device:
            sis, sid = self._dev(sis), self._dev(sid)
        n_out = nt // 2 if hourly else nt
        kw = dict(dtype=torch.float32, device=sis.device) if device else dict(dtype=np.float32)
        outs = [(torch.empty if device else np.empty)((n_out, self.ny, self.nx), **kw) for _ in range(2)]
        for lo, hi, starts in self.launches(block_starts, nt, hourly, batch):
            if device:
                parts = [sis[lo:hi], sid[lo:hi]]
            else:
                parts = [torch.from_numpy(host_f32(a[lo:hi])).to(f"cuda:{self.device}") for a in (sis, sid)]
            olo, ohi = (lo // 2, hi // 2) if hourly else (lo, hi)
            res = [o[olo:ohi] if device else torch.empty((ohi - olo, self.ny, self.nx), dtype=torch.float32,
                                                          device=parts[0].device) for o in outs]
            st = np.ascontiguousarray(starts, dtype=np.int32)
            with torch.cuda.device(self.device):
                _lib.check(_lib.load().atl_sarah_fill(self.device, hi - lo, self.ny * self.nx, _dptr(parts[0]),
                                                      _dptr(parts[1]), len(st), _lib.ptr(st), int(fill),
                                                      int(bool(hourly)), _dptr(res[0]), _dptr(res[1]), _stream_ptr()))
            if not device:
                for o, r in zip(outs, res):
                    o[olo:ohi] = r.cpu().numpy()
        return tuple(outs)


class GeoTiffOp:
    """Segment decode of a GeoTIFF band on one GPU (atl_geotiff_read).  ``op(info, rows, cols)``
    returns the image window ``[rows[0], rows[1]) x [cols[0], cols[1])`` of the file ``info``
    describes (a ``geotiff.TiffInfo``) as a (ny, nx) CUDA tensor of the file's dtype, reading and
    decoding only the segments that intersect it.  Segments cross PCIe in batches of at most
    ``batch_bytes``; the result does not depend on it.  ``stats`` holds the last call's segments,
    bytes read, bytes copied to the device and batches.  A corrupt segment raises ``ValueError``
    naming it."""

    BATCH_BYTES = 64 << 20

    def __init__(self, device=None, batch_bytes=None, n_threads=0):
        self.device = current_device() if device is None else int(device)
        self.batch_bytes = int(self.BATCH_BYTES if batch_bytes is None else batch_bytes)
        if self.batch_bytes <= 0:
            raise ValueError("batch_bytes must be positive")
        self.n_threads = int(n_threads)
        self.stats = None

    def __call__(self, info, rows, cols):
        torch = _torch()
        (r0, r1), (c0, c1) = (int(v) for v in rows), (int(v) for v in cols)
        ny, nx = info.shape
        if not (0 <= r0 < r1 <= ny and 0 <= c0 < c1 <= nx):
            raise ValueError(f"window rows [{r0}, {r1}) x columns [{c0}, {c1}) is not inside the {ny} x {nx} image")
        seg = np.ascontiguousarray(info.segments_in(r0, r1, c0, c1), dtype=np.int64)
        off = np.ascontiguousarray(info.offsets[seg], dtype=np.int64)
        cnt = np.ascontiguousarray(info.byte_counts[seg], dtype=np.int64)
        order = np.argsort(off, kind="stable")  # file order: sequential reads
        seg, off, cnt = seg[order], off[order], cnt[order]
        L = _lib.TiffLayout()
        L.compression = {1: _lib.TIFF_NONE, 5: _lib.TIFF_LZW, 8: _lib.TIFF_DEFLATE, 32946: _lib.TIFF_DEFLATE}[
            info.compression]
        L.predictor, L.sample_bytes = info.predictor, info.dtype.itemsize
        L.big_endian, L.tiled = int(info.byteorder == ">"), int(info.tiled)
        L.width, L.height = nx, ny
        L.seg_h, L.seg_w = info.block
        L.win_r0, L.win_c0, L.win_ny, L.win_nx = r0, c0, r1 - r0, c1 - c0
        udt = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[info.dtype.itemsize]
        out = torch.empty((r1 - r0, c1 - c0), dtype=udt, device=f"cuda:{self.device}")
        bad, st = C.c_int64(-1), _lib.TiffStats()
        lib = _lib.load()
        with torch.cuda.device(self.device):
            rc = lib.atl_geotiff_read(self.device, os.fsencode(info.path), C.byref(L), len(seg), _lib.ptr(seg),
                                      _lib.ptr(off), _lib.ptr(cnt), self.batch_bytes, self.n_threads, _dptr(out),
                                      C.byref(bad), C.byref(st), _stream_ptr())
        if rc != _lib.ATL_OK and bad.value >= 0:
            raise ValueError(f"{info.path}: corrupt {lib.atl_last_error().decode()}")
        _lib.check(rc)
        self.stats = {n: int(getattr(st, n)) for n, _ in _lib.TiffStats._fields_}
        return out.view(getattr(torch, info.dtype.name))
