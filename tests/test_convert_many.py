"""Cutout.convert_many: several conversions from one pass over the cutout.

Every result must be the separate call's (``getattr(cutout, method)(**kwargs)``) bit for bit under
``set_deterministic``: values (NaN equal), dims, coords, attrs, name and capacity, with the same
warnings -- on every residency: pageable NumPy, pin_host(), partly pinned, a chunk-container lazy
cutout cut into several time parts, devices=[0], devices="all" and to_device().  The shared host
pass is also checked at engine level, slab length by slab length, against each operator's own
``atl_*_reduce_host`` call, and for what it copies: each distinct host array once per pass.
Argument errors are raised before anything reaches the GPU, so those cases run without one."""

import functools
import warnings

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

import atlite_b200 as ab
from atlite_b200 import _lib, convert, engine, ingest, synthetic as syn

NX, NY, NT = 70, 45, 37
CSP = "SAM_solar_tower"
gpu = pytest.mark.gpu


def _chunks(n):
    """The slab lengths test_host_stream streams every operator at."""
    return sorted({c for c in (1, 2, 3, 7, n - 1, n, n + 5) if c > 0}) + [0]


def _box(x0, y0, x1, y1):
    return {"type": "Polygon", "coordinates": [[(x0, y0), (x1, y0), (x1, y1), (x0, y1), (x0, y0)]]}


def _plugin(ds):
    """A converter the package does not know: the plugin protocol, aggregated by atl_spmm."""
    return ds["temperature"]


def _layout(ds):
    x, y = np.asarray(ds.coords["x"]), np.asarray(ds.coords["y"])
    vals = np.linspace(0.0, 3.0, len(y) * len(x)).reshape(len(y), len(x))
    vals[:3, :4] = 0.0
    return ab.DataArray(vals, {"y": y, "x": x}, ("y", "x"))


def _prepared():
    """Prepared ERA5 variables with a stored (float64) solar position, and NaN steps at slab edges."""
    ds = syn.make_dataset(NX, NY, NT, x0=-10.0, y0=-20.0, dx=0.5, dy=1.0, extra=("runoff", "wnd_shear_exp"))
    rng = np.random.default_rng(3)
    for name, steps in (("temperature", (0, 6, 7)), ("influx_direct", (13, 14)), ("wnd100m", (20, 36)),
                        ("runoff", (2, 3))):
        a = ds.raw(name)
        for t in steps:
            a[t, rng.integers(0, NY, 9), rng.integers(0, NX, 9)] = np.nan
    t = pd.DatetimeIndex(np.asarray(ds.coords["time"]))
    lon, lat = np.meshgrid(np.radians(np.asarray(ds.coords["x"])), np.radians(np.asarray(ds.coords["y"])))
    hour = (t.hour.values + t.dayofyear.values * 24.0)[:, None, None]
    alt = np.sin(hour / 24.0 * 2 * np.pi + lon[None]) * np.cos(lat[None]) * 1.2
    az = np.pi + 0.8 * np.cos(hour / 24.0 * 2 * np.pi + lon[None])
    out = ab.Dataset({k: (ds.dims_of(k), ds.raw(k)) for k in ds.keys()}, coords=dict(ds.coords), attrs=dict(ds.attrs))
    out["solar_altitude"] = (("time", "y", "x"), alt.astype(np.float64))
    out["solar_azimuth"] = (("time", "y", "x"), az.astype(np.float64))
    return out


def _raw():
    """Raw ERA5 variables only (PV and wind derive their inputs in-kernel)."""
    x, y = syn.make_coords(NX, NY, -10.0, 35.0, 0.5, 0.5)
    rng = np.random.default_rng(5)
    shp = (NT, NY, NX)
    f = lambda lo, hi: rng.uniform(lo, hi, shp).astype(np.float32)  # noqa: E731
    d = dict(u100=f(-15, 15), v100=f(-15, 15), u10=f(-8, 8), v10=f(-8, 8), fsr=f(1e-4, 2.0),
             ssrd=f(0, 3.0e6), tisr=f(0, 4.5e6), t2m=f(250, 305))
    d["ssr"] = (d["ssrd"] * rng.uniform(0.6, 1.0, shp)).astype(np.float32)
    d["fdir"] = (d["ssrd"] * rng.uniform(0.0, 1.1, shp)).astype(np.float32)
    d["t2m"][8] = np.nan
    coords = dict(time=syn.make_time(NT + 24 * 40)[24 * 40:], x=x, y=y, lon=x, lat=y)
    return ab.Dataset({k: (("time", "y", "x"), v) for k, v in d.items()}, coords=coords, attrs={"module": "era5"})


def _requests(ds, raw):
    m = syn.make_shapes(NX, NY, 11)
    x, y = np.asarray(ds.coords["x"]), np.asarray(ds.coords["y"])
    regions = pd.Series([_box(x[3], y[2], x[30], y[20]), _box(x[25], y[10], x[60], y[40])],
                        index=pd.Index(["north", "south"], name="region"))
    lay = _layout(ds)
    req = {
        "wind_log": dict(method="wind", turbine="Vestas_V112_3MW", layout=lay, aggregate_time="sum"),
        "wind_pow": dict(method="wind", turbine="Vestas_V112_3MW", interpolation_method="power", matrix=m,
                         per_unit=True, aggregate_time=None),
        "temperature": dict(method="temperature", shapes=regions, aggregate_time=None),
        "cop": dict(method="coefficient_of_performance", matrix=m, aggregate_time="mean"),
        "heat": dict(method="heat_demand", hour_shift=5, matrix=m, aggregate_time=None),
        "cooling": dict(method="cooling_demand", shapes=regions, aggregate_time=None),
        "cells": dict(method="temperature", aggregate_time="mean"),
        "plugin": dict(method="convert_and_aggregate", convert_func=_plugin, matrix=m, aggregate_time=None),
    }
    if raw:
        req["pv_dual"] = dict(method="pv", panel="CSi", orientation="latitude_optimal", tracking="dual",
                              matrix=m, layout=lay, per_unit=True, return_capacity=True, aggregate_time=None)
        req["wind_raw"] = dict(method="wind", turbine="Vestas_V112_3MW", matrix=m, return_capacity=True,
                               aggregate_time="legacy")
        req["plugin"] = dict(method="convert_and_aggregate", convert_func=lambda d: d["t2m"], matrix=m,
                             aggregate_time=None)
    else:
        req["pv"] = dict(method="pv", panel="CSi", orientation="latitude_optimal", matrix=m, per_unit=True,
                         return_capacity=True, aggregate_time=None)
        req["irradiation"] = dict(method="irradiation", orientation="latitude_optimal", layout=lay,
                                  aggregate_time="mean")
        req["csp"] = dict(method="csp", installation=CSP, matrix=m, aggregate_time="legacy")
        req["runoff"] = dict(method="runoff", smooth=3, matrix=m, aggregate_time=None)
    return req


def _same(got, want, what):
    if isinstance(want, tuple):
        assert isinstance(got, tuple) and len(got) == len(want), what
        for k, (g, w) in enumerate(zip(got, want)):
            _same(g, w, f"{what}[{k}]")
        return
    assert type(got) is type(want), (what, type(got), type(want))
    assert tuple(got.dims) == tuple(want.dims), (what, got.dims, want.dims)
    assert set(got.coords) == set(want.coords), what
    for c in want.coords:
        assert np.array_equal(np.asarray(got.coords[c]), np.asarray(want.coords[c])), (what, c)
    assert dict(got.attrs) == dict(want.attrs), (what, got.attrs, want.attrs)
    assert got.name == want.name, (what, got.name, want.name)
    g, w = np.asarray(got.values), np.asarray(want.values)
    assert g.dtype == w.dtype and g.shape == w.shape, (what, g.dtype, w.dtype, g.shape, w.shape)
    assert np.array_equal(g, w, equal_nan=True), (what, np.nanmax(np.abs(g - w)))


def _recorded(fn):
    with warnings.catch_warnings(record=True) as log:
        warnings.simplefilter("always")
        out = fn()
    return out, sorted((w.category.__name__, str(w.message)) for w in log)


def _separately(cutout, requests):
    def run():
        return {n: getattr(cutout, r["method"])(**{k: v for k, v in r.items() if k != "method"})
                for n, r in requests.items()}

    return _recorded(run)


def _check_all(cutout, requests, what):
    want, want_w = _separately(cutout, requests)
    got, got_w = _recorded(lambda: cutout.convert_many(requests))
    assert list(got) == list(requests)
    for n in requests:
        _same(got[n], want[n], f"{what} {n}")
    assert got_w == want_w, what
    return got


@pytest.fixture
def deterministic():
    prev = ab.set_deterministic(True)
    yield
    ab.set_deterministic(prev)


def _lazy(ds, tmp_path, name):
    three = {k: ds.raw(k) for k in ds.keys() if ds.dims_of(k) == ("time", "y", "x")}
    static = {k: ds.raw(k) for k in ds.keys() if ds.dims_of(k) == ("y", "x")}
    coords = {k: np.asarray(v) for k, v in ds.coords.items()}
    p = ingest.write_chunked(tmp_path / f"{name}.bin", three, coords, chunk=(5, None, None), static=static or None,
                             attrs=dict(ds.attrs))
    return ab.Cutout(data=ingest.open_cutout(p))


def _residencies(ds, tmp_path, name):
    host = ab.Cutout(data=ds)
    yield "host", host
    yield "pin_host", host.pin_host()
    keep = [k for k in ds.keys() if ds.dims_of(k) == ("time", "y", "x")][::2]
    part = host.pin_host(variables=keep).data
    mixed = ab.Dataset({k: (ds.dims_of(k), part.raw(k) if k in keep else ds.raw(k)) for k in ds.keys()},
                       coords=dict(ds.coords), attrs=dict(ds.attrs))
    yield "partly pinned", ab.Cutout(data=mixed)
    yield "lazy", _lazy(ds, tmp_path, name)
    yield "devices=[0]", ab.Cutout(data=ds, devices=[0])
    yield "devices=all", ab.Cutout(data=ds, devices="all")
    yield "to_device", host.to_device()


# ---------------------------------------------------------------------------------- 1. equality


@gpu
@pytest.mark.parametrize("kind", ["prepared", "raw"])
def test_equal_to_separate_calls_on_every_residency(kind, deterministic, tmp_path, monkeypatch):
    # time parts of ~8 steps, so the lazy cutout streams several parts, snapped to the heat days
    monkeypatch.setattr(convert, "PART_BYTES", 8 * NY * NX * 4 * (14 if kind == "prepared" else 10))
    ds = _prepared() if kind == "prepared" else _raw()
    requests = _requests(ds, raw=kind == "raw")
    for residency, cutout in _residencies(ds, tmp_path, kind):
        if residency == "to_device":  # a Dataset of CUDA tensors gives a plugin no DataArray to work on
            requests = {k: v for k, v in requests.items() if k != "plugin"}
        _check_all(cutout, requests, f"{kind} {residency}")


@gpu
def test_warnings_once_per_request(deterministic, tmp_path):
    """Computed solar positions (no stored one) warn once per PV / CSP request, in every time part
    of a lazy cutout as once in all; legacy aggregation once per request."""
    ds = syn.make_dataset(NX, NY, NT, x0=-10.0, y0=-20.0, dx=0.5, dy=1.0)
    m = syn.make_shapes(NX, NY, 5)
    requests = {"pv": dict(method="pv", panel="CSi", orientation="latitude_optimal", matrix=m),
                "pv2": dict(method="pv", panel="CdTe", orientation="latitude_optimal", matrix=m,
                            aggregate_time=None),
                "csp": dict(method="csp", installation=CSP, matrix=m, aggregate_time="sum")}
    for cutout in (ab.Cutout(data=ds), _lazy(ds, tmp_path, "warn")):
        _check_all(cutout, requests, "warnings")


# ---------------------------------------------------------------------------------- 2. the shared ring


def _ops(ds):
    """One spec of every job kind, host fields: pv, wind, wind_raw, csp, pointwise, heat."""
    panel, orient = ab.get_solarpanelconfig("CSi"), ab.get_orientation("latitude_optimal")
    turbine = ab.get_windturbineconfig("Vestas_V112_3MW")
    raw = _raw()
    return {
        "pv": convert._PvSpec(ds, panel, orient),
        "wind": convert._WindSpec(ds, turbine),
        "wind_raw": convert._WindSpec(raw, turbine),
        "csp": convert._CspSpec(ds, ab.get_cspinstallationconfig(CSP)),
        "pointwise": convert._temperature_spec(ds),
        "heat": convert._HeatSpec(ds, 15.0, 1.0, 0.0, 5.0),
    }


def _own_call(spec, plan, chunk):
    """The job's single-operator host call (atl_*_reduce_host) with slabs of ``chunk``."""
    job = spec.job(plan)
    if job.abi == "heat":
        return spec.op.reduce(plan, spec.temp, spec.day_start, chunk_days=chunk)
    if job.abi == "wind_raw":
        return spec.op.reduce_raw(plan, spec.raw, chunk_steps=chunk)
    if job.abi == "wind":
        return spec.op.reduce(plan, spec.wnd, spec.aux, chunk_steps=chunk)
    return spec.op.reduce(plan, job.fields, chunk_steps=chunk)


@gpu
def test_shared_ring_equals_each_operators_own_call(deterministic):
    """Every job keeps its own call's slabs, whatever the ring's: bitwise that call, NaN steps at
    slab edges included (a NaN pairs differently with its neighbour in another slab layout)."""
    ds = _prepared()
    plan = engine.get_plan(syn.make_shapes(NX, NY, 9), NY, NX)
    specs = _ops(ds)
    specs["cooling"] = convert._CoolingSpec(ds, 23.0, 1.0, 0.0, -3.0)  # a second day table, same pass
    for chunk in _chunks(NT):
        own = {k: _own_call(s, plan, chunk) for k, s in specs.items()}
        for ring in (1, 7, chunk, 0):
            jobs = [s.job(plan) for s in specs.values()]
            for j in jobs:
                j.chunk = chunk
            outs, stats = engine.reduce_host_many(jobs, chunk_units=ring)
            assert stats["n_slabs"] == (-(-NT // ring) if ring else 1), (chunk, ring)
            for (k, want), got in zip(own.items(), outs):
                assert got.dtype == np.float32 and got.shape == want.shape, (k, chunk, ring)
                assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (k, chunk, ring)


@gpu
def test_step_jobs_alone_and_heat_alone(deterministic):
    ds = _prepared()
    plan = engine.get_plan(syn.make_shapes(NX, NY, 4), NY, NX)
    specs = _ops(ds)
    heat = specs.pop("heat")
    outs, stats = engine.reduce_host_many([s.job(plan) for s in specs.values()], chunk_units=3)
    assert stats["n_slabs"] == -(-NT // 3)
    for (k, s), got in zip(specs.items(), outs):
        assert np.array_equal(got, s.reduce(plan), equal_nan=True), k
    (got,), stats = engine.reduce_host_many([heat.job(plan)], chunk_units=2)
    assert np.array_equal(got, heat.reduce(plan), equal_nan=True)
    steps = int(heat.day_start[-1] - heat.day_start[0])
    assert stats == {"h2d_bytes": steps * NY * NX * 4, "n_slabs": -(-steps // 2)}
    assert engine.reduce_host_many([]) == ([], {"h2d_bytes": 0, "n_slabs": 0})


# ---------------------------------------------------------------------------------- 3. sharing is real


@gpu
def test_each_host_array_is_copied_once_per_pass(deterministic):
    ds = _prepared()
    plan = engine.get_plan(syn.make_shapes(NX, NY, 4), NY, NX)
    pv = convert._PvSpec(ds, ab.get_solarpanelconfig("CSi"), ab.get_orientation("latitude_optimal"))
    temp = convert._temperature_spec(ds)
    heat = convert._HeatSpec(ds, 15.0, 1.0, 0.0, 0.0)
    jobs = [pv.job(plan), temp.job(plan), heat.job(plan)]
    _, stats = engine.reduce_host_many(jobs, chunk_units=2)
    # PV reads influx_toa, influx_direct, influx_diffuse, albedo, temperature and the float64 solar
    # position; temperature and heat read the same temperature array
    distinct = {id(a): a for a in list(pv.fields.values()) + [temp.field, heat.temp] if a is not None}
    want = sum(a.dtype.itemsize for a in distinct.values()) * NT * NY * NX
    assert len(distinct) == 7
    assert stats == {"h2d_bytes": want, "n_slabs": -(-NT // 2)}


@gpu
def test_lazy_cutout_loads_each_variable_once_per_part(deterministic, tmp_path, monkeypatch):
    """Every variable is loaded once per part of each distinct cut: one for the step conversions,
    and one per heat / cooling day table, which cuts at its own day starts."""
    ds = _prepared()
    cutout = _lazy(ds, tmp_path, "count")
    loads = {}
    lz = cutout.data
    for name, load in list(lz._loaders.items()):
        def counted(lo, hi, load=load, name=name):
            loads.setdefault(name, []).append((lo, hi))  # (two loader threads: in no particular order)
            return load(lo, hi)
        lz._loaders[name] = counted
    monkeypatch.setattr(convert, "PART_BYTES", 10 * NY * NX * 4 * 14)
    requests = {k: v for k, v in _requests(ds, raw=False).items() if k not in ("cells", "plugin")}
    cutout.convert_many(requests)
    time = np.asarray(ds.coords["time"])
    cuts = {tuple(convert._partition(lz, NT, [0], True, offs)) for offs in (
        None, convert.day_bins(time, 5)[1], convert.day_bins(time, 0.0)[1])}  # steps, heat, cooling
    assert len(cuts) == 3 and all(len(c) > 1 for c in cuts)
    want = sorted((lo, hi) for c in cuts for lo, hi, _ in c)
    assert set(loads) == set(lz._loaders)
    for name, got in loads.items():
        assert sorted(got) == want, name


@gpu
def test_a_launch_start_next_to_a_nan_can_change_a_step_by_one_ulp(deterministic):
    """Why a job in a shared pass keeps its own call's slabs: the fused kernels walk a launch's steps
    in batches counted from its first step, and a NaN that reaches a batch's result sends the whole
    batch down the exact path, which may round the other steps of the batch differently.  So the same
    step, next to a NaN, is not always bitwise the same when a launch starts at it."""
    ds = _prepared()
    m = sp.csr_matrix(convert._layout_values(_layout(ds), ds)[None, :])
    plan = engine.get_plan(m, NY, NX)
    w = convert._WindSpec(ds, ab.get_windturbineconfig("Vestas_V112_3MW"))
    whole = w.op.reduce(plan, w.wnd, w.aux, chunk_steps=NT)  # one launch from step 0
    nan_steps = set(np.flatnonzero(np.isnan(w.wnd).any(axis=(1, 2))).tolist())
    differ = set()
    for s in range(1, NT):
        part = w.op.reduce(plan, w.wnd[s:], w.aux[s:], chunk_steps=NT)  # one launch from step s
        same = (part == whole[s:]) | (np.isnan(part) & np.isnan(whole[s:]))
        differ |= {int(t) + s for t in np.flatnonzero(~same.all(axis=1))}
    assert differ, "no step changed with the launch start"
    assert all(t - 1 in nan_steps or t + 1 in nan_steps for t in differ), (sorted(differ), sorted(nan_steps))


NXL, NYL, NTL = 400, 300, 73


@gpu
def test_equal_to_separate_calls_when_jobs_assemble_their_slabs(deterministic, monkeypatch):
    """A cutout large enough that the ring takes several slabs (~192 MiB of the union's input each)
    while every job keeps its own, longer or shorter, slabs: each job builds them in its own window
    from the ring slots, across ring slab boundaries, with NaN steps on both sides of one."""
    ds = syn.make_dataset(NXL, NYL, NTL, x0=-10.0, y0=35.0, dx=0.1, dy=0.1, extra=("runoff", "wnd_shear_exp"))
    rng = np.random.default_rng(9)
    for name, steps in (("wnd100m", (44, 45, 46, 47)), ("temperature", (23, 45, 46)), ("influx_direct", (45,))):
        a = ds.raw(name)
        for t in steps:
            a[t, rng.integers(0, NYL, 50), rng.integers(0, NXL, 50)] = np.nan
    m = syn.make_shapes(NXL, NYL, 40)
    requests = {
        "pv": dict(method="pv", panel="CSi", orientation="latitude_optimal", matrix=m, aggregate_time=None),
        "wind_log": dict(method="wind", turbine="Vestas_V112_3MW", matrix=m, aggregate_time=None),
        "wind_pow": dict(method="wind", turbine="Vestas_V112_3MW", interpolation_method="power", matrix=m,
                         aggregate_time="sum"),
        "temperature": dict(method="temperature", matrix=m, aggregate_time=None),
        "cop": dict(method="coefficient_of_performance", matrix=m, aggregate_time=None),
        "heat": dict(method="heat_demand", hour_shift=5, matrix=m, aggregate_time=None),
        "runoff": dict(method="runoff", matrix=m, aggregate_time=None),
    }
    passes = []
    shared = engine.reduce_host_many

    def counted(jobs, chunk_units=0):
        outs, stats = shared(jobs, chunk_units)
        passes.append(stats)
        return outs, stats

    monkeypatch.setattr(engine, "reduce_host_many", counted)
    host = ab.Cutout(data=ds)
    for residency, cutout in (("host", host), ("pin_host", host.pin_host())):
        passes.clear()
        _check_all(cutout, requests, f"large {residency}")
        assert len(passes) == 1 and passes[0]["n_slabs"] >= 2, passes


@gpu
def test_per_unit_without_a_matrix_raises_what_the_separate_call_raises():
    c = ab.Cutout(data=syn.make_dataset(12, 8, 5))
    for request in (dict(method="heat_demand", per_unit=True), dict(method="temperature", return_capacity=True)):
        kw = {k: v for k, v in request.items() if k != "method"}
        with pytest.raises(ValueError) as want:
            getattr(c, request["method"])(**kw)
        with pytest.raises(ValueError) as got:
            c.convert_many({"a": request})
        assert str(got.value) == str(want.value)


# ---------------------------------------------------------------------------------- 4. errors before launch


@gpu
def test_jobs_on_another_grid_are_refused_before_launch():
    ds = _prepared()
    plan = engine.get_plan(syn.make_shapes(NX, NY, 4), NY, NX)
    small = syn.make_dataset(NX - 1, NY, NT)
    jobs = [convert._temperature_spec(ds).job(plan), convert._temperature_spec(small).job(
        engine.get_plan(syn.make_shapes(NX - 1, NY, 4), NY, NX - 1))]
    before = _lib.launch_count()
    with pytest.raises(_lib.AtlError, match="job 1: operator on device 0 with grid 45x69"):
        engine.reduce_host_many(jobs)
    assert _lib.launch_count() == before
    job = _lib.StreamJob(_lib.JOB["pointwise"], jobs[0].op.handle.value, plan.handle.value,
                         jobs[0].fields.ctypes.data, 0, None, 0, 0, np.empty((NT, 4), np.float32).ctypes.data)
    arr = (_lib.StreamJob * 1)(job)
    lib = _lib.load()
    assert lib.atl_reduce_host_many(1, NY, NX, NT, arr, 1, 0, None) == -1  # ATL_ERR_INVALID
    assert lib.atl_reduce_host_many(0, NY + 1, NX, NT, arr, 1, 0, None) == -1  # ATL_ERR_INVALID
    arr[0].kind = 17
    assert lib.atl_reduce_host_many(0, NY, NX, NT, arr, 1, 0, None) == -1  # ATL_ERR_INVALID
    assert _lib.launch_count() == before


@pytest.fixture(scope="module")
def cpu_cutout():
    return ab.Cutout(data=syn.make_dataset(12, 8, 5))


def _same_error(cutout, request, separate, names=()):
    """convert_many raises what the separate call raises, before anything reaches the GPU: the
    valid request in front of the bad one must not run.  Arguments that do not bind are found
    without calling anything, so their TypeError names the arguments (``names``) in its own words."""
    with pytest.raises(Exception) as want:
        separate()
    fine = dict(method="temperature", matrix=sp.identity(96, format="csr"), aggregate_time=None)
    with pytest.raises(type(want.value)) as got:
        cutout.convert_many({"fine": fine, "bad": request})
    if names:
        assert all(f"'{n}'" in str(got.value) and f"'{n}'" in str(want.value) for n in names), (got.value, want.value)
    else:
        assert str(got.value) == str(want.value)


def test_argument_errors_match_the_separate_call(cpu_cutout, monkeypatch):
    c = cpu_cutout

    def no_gpu(*a, **k):
        raise AssertionError("reached the GPU")

    for name in ("get_plan", "reduce_host_many", "device_csr"):
        monkeypatch.setattr(engine, name, no_gpu)
    monkeypatch.setattr(type(c), "indicatormatrix", no_gpu)
    _same_error(c, dict(method="nope"), lambda: c.nope)
    _same_error(c, dict(method="pv", panel="CSi", orientation="latitude_optimal", bogus=1),
                lambda: c.pv(panel="CSi", orientation="latitude_optimal", bogus=1), names=["bogus"])
    _same_error(c, dict(method="wind"), lambda: c.wind(), names=["turbine"])
    _same_error(c, dict(method="wind", turbine="no such turbine"), lambda: c.wind(turbine="no such turbine"))
    _same_error(c, dict(method="temperature", aggregate_time="daily"), lambda: c.temperature(aggregate_time="daily"))
    _same_error(c, dict(method="convert_and_aggregate", convert_func=_plugin, factor=3),
                lambda: c.convert_and_aggregate(convert_func=_plugin, factor=3), names=["factor"])
    with pytest.raises(ValueError, match="One of `matrix`, `shapes` and `layout` must be given"):
        c.convert_many({"a": dict(method="heat_demand", per_unit=True)})
    _same_error(c, dict(method="temperature", aggregate_time="sum", capacity_factor=True),
                lambda: c.temperature(aggregate_time="sum", capacity_factor=True))
    with pytest.raises(ValueError, match="not a conversion method"):
        c.convert_many({"a": dict(method="indicatormatrix", shapes=[])})
    with pytest.raises(TypeError, match="must be a dict"):
        c.convert_many({"a": ["pv"]})
    with pytest.raises(TypeError, match="has no 'method'"):
        c.convert_many({"a": dict(panel="CSi")})
    with pytest.raises(TypeError, match="must be a dict"):
        c.convert_many([("a", dict(method="pv"))])
    assert c.convert_many({}) == {}
    assert ab.convert_many(c, {}) == {}


def test_plugin_arguments_are_checked_without_calling_the_plugin(cpu_cutout):
    calls = []

    def plugin(ds):
        calls.append("plugin")
        return ds["temperature"]

    @functools.wraps(plugin)
    def wrapped(ds, **kw):  # takes any keyword, as Python binds it (not as its __wrapped__ would)
        calls.append("wrapped")
        return plugin(ds)

    with pytest.raises(TypeError, match="'factor'"):
        cpu_cutout.convert_many({"a": dict(method="convert_and_aggregate", convert_func=plugin, factor=3)})
    assert convert._bind(wrapped, cpu_cutout.data, factor=3) == {"ds": cpu_cutout.data, "factor": 3}
    assert calls == []
