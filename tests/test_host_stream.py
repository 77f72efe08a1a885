"""The host-streaming path (csrc/host_stream.cu) slab by slab, for every operator ABI.

A host-resident or pin_host() cutout reaches the GPU through ``atl_*_reduce_host``: the (time, y, x)
fields are copied in time slabs into a two-slot device ring, each slab is reduced by the operator's
device call at its own time offset (or day cursor, for heat demand) and its rows are written into
one output.  Every case here streams the same fields at many slab lengths -- 1 and 2 reuse both ring
slots at every step, nt + 5 and 0 (the default sizing) take one slab -- and holds each result

- bitwise equal to the same fields reduced on the device in the unpadded layout (the layout host
  streaming uses; ``set_deterministic`` fixes the summation order, which does not depend on where
  a slab starts), and
- to the parity bar (conftest.assert_parity) against the float64 oracle.

The grid (70 x 45) is no multiple of 4 or 32 and the time axis (37 steps) is prime, so slabs are
ragged.  Further cases: windows [t0, nt) of the operator's time axis, partial heat days and day
tables that start past step 0, pinned / pageable / non-contiguous / float64 fields in one call,
staging buffers reused at other sizes, two threads streaming at once, NaN at slab edges, the
default slab sizing at full ERA5 scale, the public converters on every host residency, and the
argument checks that must stop a call before anything is launched."""

import threading
import time
import warnings

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp
from conftest import assert_parity, oracle_ds

import atlite_oracle as O
import era5_oracle as EO
import era5_runoff_height_oracle as ERH
import line_rating_oracle as LO
import atlite_b200 as ab
from atlite_b200 import _lib, convert, engine, gis, synthetic as syn

pytestmark = pytest.mark.gpu

warnings.filterwarnings("ignore", category=DeprecationWarning)

NX, NY, NT = 70, 45, 37
G0 = 9.80665


def cap_of(m):
    return np.asarray(sp.csr_matrix(m).sum(-1)).flatten()


def bt(res):
    """public API result (bus, time) -> oracle layout (time, bus)"""
    assert res.dims[1] == "time"
    return np.asarray(res.values).T


def _chunks(n):
    """Slab lengths: every step its own slab (both ring slots reused at every step), ragged slabs,
    one step short of the axis, exactly the axis, longer than the axis, and the default sizing."""
    return sorted({c for c in (1, 2, 3, 7, n - 1, n, n + 5) if c > 0}) + [0]


def _np(x):
    return x.cpu().numpy() if engine._is_torch(x) else np.asarray(x)


def _dev(x):
    """Host field(s) -> CUDA tensors in the unpadded layout, as ``to_device(pad=False)`` stores them."""
    import torch

    if isinstance(x, dict):
        return {k: _dev(v) for k, v in x.items()}
    return None if x is None else torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _same_bits(got, want, what):
    got, want = _np(got), _np(want)
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    bits = np.dtype(f"u{got.dtype.itemsize}")
    diff = got.view(bits) != want.view(bits)
    assert not diff.any(), (f"{what}: {diff.sum()} of {diff.size} values differ from the device result; "
                            f"first at {tuple(np.argwhere(diff)[0])}")


def _ring(reduce, host, want, cap, what, chunks, **parity):
    """``reduce(fields, chunk)`` of the host ``fields`` at every slab length in ``chunks``: bitwise the
    device reduce of the same fields, and within the parity bar of the oracle's ``want``."""
    ref = _np(reduce(_dev(host), 0))
    assert_parity(ref, want, cap, what=f"{what} device", **parity)
    for c in chunks:
        got = reduce(host, c)
        assert isinstance(got, np.ndarray)
        _same_bits(got, ref, f"{what} chunk {c}")
        assert_parity(got, want, cap, what=f"{what} chunk {c}", **parity)
    return ref


@pytest.fixture
def deterministic():
    prev = ab.set_deterministic(True)
    yield
    ab.set_deterministic(prev)


def _with_vars(ds, **new):
    """A copy of the dataset ``ds`` (arrays shared) with the variables ``new`` added or replaced."""
    out = ab.Dataset({k: (ds.dims_of(k), ds.raw(k)) for k in ds.keys()}, coords=dict(ds.coords),
                     attrs=dict(ds.attrs))
    for k, v in new.items():
        out[k] = (("time", "y", "x")[-v.ndim:], v)
    return out


def _with_solar(ds, alt_dtype, az_dtype):
    """``ds`` with a stored solar position (the oracle's, at 0 h) in the given dtypes."""
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sp_ = O.solar_position(oracle_ds(ds))
    return _with_vars(ds, solar_altitude=np.asarray(sp_["altitude"], dtype=alt_dtype),
                      solar_azimuth=np.asarray(sp_["azimuth"], dtype=az_dtype))


@pytest.fixture(scope="module")
def ds_full():
    # 70 x 45 cells, 37 steps (prime), both hemispheres, day, night and the terminator
    return syn.make_dataset(NX, NY, NT, x0=-10.0, y0=-20.0, dx=0.5, dy=1.0, extra=("wnd_shear_exp", "humidity"))


@pytest.fixture(scope="module")
def shapes():
    return syn.make_shapes(NX, NY, 23)


@pytest.fixture(scope="module")
def plan(shapes):
    return engine.get_plan(shapes, NY, NX)


# ---------------------------------------------------------------------------------- raw ERA5 case


def _raw_arrays(nx, ny, nt, seed=0):
    """Seeded raw ERA5 fields with edge cells: zero ssrd (albedo 0), NaN ssr (albedo 0), NaN and
    negative fsr (roughness 2e-4), negative accumulations, negative runoff, and a geopotential that
    changes from step to step (the height is its first step's)."""
    rng = np.random.default_rng(seed)
    shp = (nt, ny, nx)
    f = lambda lo, hi: rng.uniform(lo, hi, shp).astype(np.float32)  # noqa: E731
    d = dict(u100=f(-15, 15), v100=f(-15, 15), u10=f(-8, 8), v10=f(-8, 8), fsr=f(-0.05, 2.0),
             ssrd=f(0, 3.0e6), tisr=f(0, 4.5e6), t2m=f(250, 305), ro=f(-1e-4, 2e-3))
    d["ssr"] = (d["ssrd"] * rng.uniform(0.6, 1.0, shp)).astype(np.float32)
    d["fdir"] = (d["ssrd"] * rng.uniform(0.0, 1.1, shp)).astype(np.float32)
    base = rng.uniform(0.0, 1500.0 * G0, (ny, nx)).astype(np.float32)
    d["z"] = (base[None] + (np.arange(nt, dtype=np.float32) * 40.0 * G0)[:, None, None]).astype(np.float32)
    d["ssrd"][:, 0, :5] = 0.0
    d["ssr"][:, 1, 2] = np.nan
    d["fsr"][:, 2, 2] = np.nan
    d["fsr"][:, 3, 1] = -0.3
    d["ssrd"][:, 2, 4] = -40.0
    d["fdir"][:, 3, 3] = -25.0
    d["tisr"][:, 1, 6] = -3.6
    d["ro"][:, 1, 4] = -3e-5
    return d


def _raw_oracle(d, co):
    """What era5.prepare stores, from the ERA5 oracles, with the solar position at -30 min."""
    ow = EO.get_data_wind(d["u100"], d["v100"], d["u10"], d["v10"], d["fsr"])
    oi = EO.get_data_influx(d["ssrd"], d["ssr"], d["tisr"], d["fdir"])
    c = dict(time=co["time"], lon=co["x"], lat=co["y"])
    sol = O.solar_position(c, time_shift="-30min")
    od = dict(c, solar_altitude=sol["altitude"], solar_azimuth=sol["azimuth"], temperature=d["t2m"].astype(np.float64),
              runoff=ERH.get_data_runoff(d["ro"])["runoff"], height=ERH.get_data_height(d["z"])["height"])
    od.update({k: ow[k] for k in ("wnd100m", "roughness", "wnd_shear_exp")})
    od.update({k: oi[k] for k in ("influx_toa", "influx_direct", "influx_diffuse", "albedo")})
    return od


@pytest.fixture(scope="module")
def raw():
    x, y = syn.make_coords(NX, NY, -10.0, 35.0, 0.5, 0.5)
    co = dict(time=syn.make_time(NT + 24 * 40)[24 * 40:], x=x, y=y, lon=x, lat=y)  # February
    d = _raw_arrays(NX, NY, NT, seed=5)
    ds = ab.Dataset({k: (("time", "y", "x"), v) for k, v in d.items()}, coords=dict(co))
    return dict(ds=ds, od=_raw_oracle(d, co))


# ---------------------------------------------------------------------------------- 1. the ring, per ABI


def _pv_spec(ds, **case):
    case = dict(dict(panel="CSi", orientation="latitude_optimal"), **case)
    return convert._PvSpec(ds, ab.get_solarpanelconfig(case.pop("panel")), ab.get_orientation(case.pop("orientation")),
                           **case)


def _oracle_pv(od, matrix, **case):
    case = dict(dict(panel="CSi", orientation="latitude_optimal"), **case)
    return O.convert_and_aggregate(od, O.convert_pv, matrix=matrix, aggregate_time=None,
                                   panel=ab.get_solarpanelconfig(case.pop("panel")),
                                   orientation=O.get_orientation(case.pop("orientation")), **case)


@pytest.mark.parametrize("variant", ["prepared", "raw", "stored_f32", "stored_f64"])
def test_pv_ring(ds_full, raw, shapes, plan, deterministic, variant):
    if variant == "raw":
        ds, od = raw["ds"], raw["od"]
    else:
        dt = {"prepared": None, "stored_f32": np.float32, "stored_f64": np.float64}[variant]
        ds = ds_full if dt is None else _with_solar(ds_full, dt, dt)
        od = oracle_ds(ds)
    spec = _pv_spec(ds)
    assert spec.op.solar_f64 == (variant == "stored_f64")
    want = _oracle_pv(od, shapes)
    assert want.sum() > 0
    _ring(lambda f, c: spec.op.reduce(plan, f, chunk_steps=c), spec.fields, want, cap_of(shapes),
          f"stream-pv {variant}", _chunks(NT))


def _turbine(hub):
    return dict(ab.get_windturbineconfig("Vestas_V112_3MW"), hub_height=hub)


@pytest.mark.parametrize("variant,hub,method", [("wnd", 100, "logarithmic"), ("aux", 80, "logarithmic"),
                                                ("aux", 80, "power"), ("raw", 100, "logarithmic"),
                                                ("raw", 80, "logarithmic"), ("raw", 120, "power")])
def test_wind_ring(ds_full, raw, shapes, plan, deterministic, variant, hub, method):
    ds, od = (raw["ds"], raw["od"]) if variant == "raw" else (ds_full, oracle_ds(ds_full))
    spec = convert._WindSpec(ds, _turbine(hub), method)
    if variant == "raw":
        fields = spec.raw
        assert set(fields) == {"u100", "v100"} | ({"fsr"} if hub == 80 else {"u10", "v10"} if hub == 120 else set())

        def reduce(f, c):
            return spec.op.reduce_raw(plan, f, chunk_steps=c)
    else:
        fields = {"wnd": spec.wnd, "aux": spec.aux}
        assert (spec.aux is None) == (variant == "wnd")

        def reduce(f, c):
            return spec.op.reduce(plan, f["wnd"], f["aux"], chunk_steps=c)
    want = O.convert_and_aggregate(od, O.convert_wind, matrix=shapes, aggregate_time=None, turbine=_turbine(hub),
                                   interpolation_method=method)
    _ring(reduce, fields, want, cap_of(shapes), f"stream-wind {variant} {hub} {method}", _chunks(NT))


CSP = "SAM_solar_tower"


@pytest.mark.parametrize("variant", ["computed", "stored_f64", "raw"])
def test_csp_ring(ds_full, raw, shapes, plan, deterministic, variant):
    if variant == "raw":
        ds, od = raw["ds"], raw["od"]
    else:
        ds = ds_full if variant == "computed" else _with_solar(ds_full, np.float64, np.float64)
        od = oracle_ds(ds)
    cfg = ab.get_cspinstallationconfig(CSP)
    spec = convert._CspSpec(ds, cfg)
    assert spec.raw == (variant == "raw") and spec.op.solar_f64 == (variant == "stored_f64")
    want = O.convert_and_aggregate(od, O.convert_csp, matrix=shapes, aggregate_time=None, installation=cfg)
    assert want.sum() > 0
    _ring(lambda f, c: spec.op.reduce(plan, f, chunk_steps=c), spec.fields, want, cap_of(shapes),
          f"stream-csp {variant}", _chunks(NT))


@pytest.mark.parametrize("variant", ["temperature", "cop", "runoff"])
def test_pointwise_ring(ds_full, raw, shapes, plan, deterministic, variant):
    od = oracle_ds(ds_full)
    if variant == "temperature":
        spec, kw = convert._temperature_spec(ds_full), dict(convert_func=O.convert_temperature)
        parity = dict(additive=True)  # signed deg C values: bus sums cancel
        cap = cap_of(shapes) * 300.0
    elif variant == "cop":
        spec = convert._cop_spec(ds_full, "air", 55.0, None, None, None)
        kw = dict(convert_func=O.convert_coefficient_of_performance, source="air", sink_T=55.0, c0=None, c1=None,
                  c2=None)
        parity, cap = {}, cap_of(shapes) * 10.0
    else:  # raw ro clipped at 0, times the height of z's first step
        spec, od = convert._runoff_spec(raw["ds"]), raw["od"]
        kw, parity = dict(convert_func=O.convert_runoff, weight_with_height=True), {}
        assert spec.op._scale is not None
    want = O.convert_and_aggregate(od, matrix=shapes, aggregate_time=None, **kw)
    if variant == "runoff":
        cap = np.abs(want).max(0) * 10
    _ring(lambda f, c: spec.op.reduce(plan, f, chunk_steps=c), spec.field, want, cap,
          f"stream-pointwise {variant}", _chunks(NT), **parity)


# ---------------------------------------------------------------------------------- 3. heat day tables

HEAT_NT = 103  # hourly steps: four full days and partial ones, whatever the hour shift


@pytest.fixture(scope="module")
def ds_heat():
    return syn.make_dataset(NX, NY, HEAT_NT, x0=-10.0, y0=-20.0, dx=0.5, dy=1.0, kinds=("temperature",))


@pytest.mark.parametrize("cooling", [False, True], ids=["heating", "cooling"])
@pytest.mark.parametrize("hour_shift", [0.0, 3.0, -5.5])
def test_heat_ring(ds_heat, shapes, plan, deterministic, cooling, hour_shift):
    """Heat and cooling demand stream whole days: the ring runs in days with a day cursor, and each
    slab's day offsets are taken relative to its first step.  Shifts of 3 h and -5.5 h make the first
    and the last day partial; a table without the first and last day starts past step 0 and ends
    before the last step."""
    threshold, a, constant = (5.0, 1.7, 0.3) if cooling else (17.0, 1.3, 0.2)
    spec = (convert._CoolingSpec if cooling else convert._HeatSpec)(ds_heat, threshold, a, constant, hour_shift)
    want = O.convert_and_aggregate(oracle_ds(ds_heat), O.convert_cooling_demand if cooling else O.convert_heat_demand,
                                   matrix=shapes, aggregate_time=None, threshold=threshold, a=a, constant=constant,
                                   hour_shift=hour_shift)
    days = spec.day_start
    nd = len(days) - 1
    assert nd == want.shape[0] and days[-1] == HEAT_NT
    if hour_shift:
        assert days[1] - days[0] < 24 and days[-1] - days[-2] < 24  # partial first and last day
    what = f"stream-{'cooling' if cooling else 'heat'} {hour_shift}"
    cap = cap_of(shapes) * 50.0
    _ring(lambda f, c: spec.op.reduce(plan, f, days, chunk_days=c), spec.temp, want, cap, what, _chunks(nd))
    inner = days[1:-1]
    assert inner[0] > 0 and inner[-1] < HEAT_NT
    _ring(lambda f, c: spec.op.reduce(plan, f, inner, chunk_days=c), spec.temp, want[1:-1], cap, f"{what} inner days",
          [1, 2, 3, nd - 2])


# ---------------------------------------------------------------------------------- 2. time offsets


def _offset_case(name, ds_full):
    if name == "pv":
        spec = _pv_spec(ds_full)
        return spec, lambda p, f, t0, c: spec.op.reduce(p, f, t0=t0, chunk_steps=c)
    spec = convert._CspSpec(ds_full, ab.get_cspinstallationconfig(CSP))
    return spec, lambda p, f, t0, c: spec.op.reduce(p, f, t0=t0, chunk_steps=c)


@pytest.mark.parametrize("name", ["pv", "csp"])
def test_time_windows_end_at_the_axis_end(ds_full, plan, deterministic, name):
    """A window [t0, nt) of the operator's time axis, streamed in several slabs, equals the same rows of
    the whole axis: each slab runs at t0 plus its own offset.  A window one step longer fails with the
    library's error, raised on the host before the slab's launch."""
    spec, reduce = _offset_case(name, ds_full)
    whole = reduce(plan, spec.fields, 0, 0)
    _same_bits(whole, reduce(plan, _dev(spec.fields), 0, 0), f"{name} whole axis")
    for t0 in (1, 11, NT - 3):
        part = {k: v[t0:] for k, v in spec.fields.items()}
        for c in (1, 4, 0):
            _same_bits(reduce(plan, part, t0, c), whole[t0:], f"{name} t0={t0} chunk {c}")
        _same_bits(reduce(plan, _dev(part), t0, 0), whole[t0:], f"{name} t0={t0} device")
        over = {k: v[t0 - 1:] for k, v in spec.fields.items()}  # NT - t0 + 1 steps from t0
        for f in (over, _dev(over)):
            with pytest.raises(_lib.AtlError, match="slab outside the operator's time axis"):
                reduce(plan, f, t0, 4)


# ---------------------------------------------------------------------------------- 4. memory kinds


def _pinned(a):
    import torch

    t = torch.empty(a.shape, dtype=torch.float32, pin_memory=True)
    t.numpy()[...] = a
    return t


def test_memory_kinds_and_the_staging_pool(ds_full, plan, deterministic):
    """Pinned fields are DMA'd directly, pageable ones staged through the pooled pinned buffers, a
    non-contiguous or float64 field is first copied to contiguous float32: all in one call, with
    slab sizes that grow and shrink so pooled buffers serve requests of other sizes, with and
    without the pool released in between."""
    spec = _pv_spec(ds_full)
    f = spec.fields
    ref = spec.op.reduce(plan, f)  # all pageable
    keep = [_pinned(f["influx_toa"]), _pinned(f["temperature"])]
    wide = np.repeat(f["influx_diffuse"], 2, axis=2)
    mixed = dict(f, influx_toa=keep[0].numpy(), temperature=keep[1].numpy(), influx_diffuse=wide[:, :, ::2],
                 albedo=f["albedo"].astype(np.float64))
    assert not mixed["influx_diffuse"].flags["C_CONTIGUOUS"]
    np.testing.assert_array_equal(mixed["influx_diffuse"], f["influx_diffuse"])
    pinned = {k: (v if v is None else _pinned(v)) for k, v in f.items()}
    keep += [v for v in pinned.values() if v is not None]
    pinned = {k: v.numpy() for k, v in pinned.items()}
    for i, c in enumerate((1, 3, 7, NT, 0, 5, 2, 1, NT + 5)):
        if i in (4, 7):
            ab.release_host_staging()
        for what, fields in (("mixed", mixed), ("pinned", pinned), ("pageable", f)):
            _same_bits(spec.op.reduce(plan, fields, chunk_steps=c), ref, f"{what} chunk {c}")


def test_two_threads_stream_at_once(ds_full, plan, deterministic):
    """Two host threads stream different operators on the same GPU at once (the C calls release the
    GIL): each gets the result it gets alone."""
    pv = _pv_spec(ds_full)
    wind = convert._WindSpec(ds_full, _turbine(80), "logarithmic")
    calls = {"pv": lambda: pv.op.reduce(plan, pv.fields, chunk_steps=3),
             "wind": lambda: wind.op.reduce(plan, wind.wnd, wind.aux, chunk_steps=2)}
    serial = {k: fn() for k, fn in calls.items()}
    got, errors = {}, []

    def run(name):
        try:
            got[name] = [calls[name]() for _ in range(4)]
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    threads = [threading.Thread(target=run, args=(n,)) for n in calls]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for name, results in got.items():
        for r in results:
            _same_bits(r, serial[name], f"thread {name}")


# ---------------------------------------------------------------------------------- 5. NaN at slab edges

NAN_STEPS = (6, 7, 13, NT - 1)  # for chunk 7: a slab's last, first, last step; the axis' last step


@pytest.mark.parametrize("kind", ["wind", "pv", "pointwise"])
def test_nan_through_slab_boundaries(ds_full, shapes, plan, deterministic, kind):
    var = {"wind": "wnd100m", "pv": "albedo", "pointwise": "temperature"}[kind]
    a = ds_full.raw(var).copy()
    for i, t in enumerate(NAN_STEPS):
        a[t, 10 + 3 * i, 60 - 5 * i] = np.nan  # lit cells at every one of these steps
    ds = _with_vars(ds_full, **{var: a})
    od = oracle_ds(ds)
    if kind == "wind":
        spec = convert._WindSpec(ds, _turbine(100), "logarithmic")
        fields, reduce = spec.wnd, lambda f, c: spec.op.reduce(plan, f, chunk_steps=c)
        want = O.convert_and_aggregate(od, O.convert_wind, matrix=shapes, aggregate_time=None, turbine=_turbine(100))
        cap, parity = cap_of(shapes), {}
    elif kind == "pv":  # a NaN albedo makes the Hay-Davies ground term, and the bus, NaN
        spec = _pv_spec(ds, trigon_model="other")
        fields, reduce = spec.fields, lambda f, c: spec.op.reduce(plan, f, chunk_steps=c)
        want = _oracle_pv(od, shapes, trigon_model="other")
        cap, parity = cap_of(shapes), {}
    else:
        spec = convert._temperature_spec(ds)
        fields, reduce = spec.field, lambda f, c: spec.op.reduce(plan, f, chunk_steps=c)
        want = O.convert_and_aggregate(od, O.convert_temperature, matrix=shapes, aggregate_time=None)
        cap, parity = cap_of(shapes) * 300.0, dict(additive=True)
    nan_rows = np.flatnonzero(np.isnan(want).any(axis=1))
    np.testing.assert_array_equal(nan_rows, NAN_STEPS)
    _ring(reduce, fields, want, cap, f"stream-{kind} nan", _chunks(NT), **parity)


# ---------------------------------------------------------------------------------- 6. full scale


def test_default_slabs_at_full_scale(deterministic):
    """One pageable temperature reduce at 1440 x 720 x 100 with the default slab sizing: about 48
    steps (192 MiB) per slab, so three slabs, the last one 4 steps.  Bitwise the device reduce, and
    at the parity bar of scipy's sparse product in float64 (computed in blocks to keep the host
    footprint under 1 GB)."""
    import torch

    nx, ny, nt = 1440, 720, 100
    rng = np.random.default_rng(17)
    field = np.empty((nt, ny, nx), dtype=np.float32)
    for t in range(nt):
        rng.random((ny, nx), dtype=np.float32, out=field[t])
        field[t] *= 50.0
        field[t] += 255.0
    m = sp.csr_matrix(syn.make_shapes(nx, ny, 300), dtype=np.float64)
    op = engine.PointwiseOp(ny=ny, nx=nx, shift=-273.15)
    plan = engine.get_plan(m, ny, nx)
    try:
        secs = []
        for _ in range(2):  # the first call also allocates the pinned staging buffers
            t = time.perf_counter()
            got = op.reduce(plan, field)
            secs.append(time.perf_counter() - t)
        print(f"\nhost-streamed temperature reduce, 1440x720x100 pageable -> 300 shapes: "
              f"{secs[0] * 1e3:.1f} ms first call, {secs[1] * 1e3:.1f} ms with the staging pool warm")
    finally:
        ab.release_host_staging()
    d = torch.from_numpy(field).cuda()
    ref = op.reduce(plan, d).cpu().numpy()
    del d
    _same_bits(got, ref, "full scale")
    want = np.empty((nt, m.shape[0]), dtype=np.float64)
    for t0 in range(0, nt, 10):
        blk = field[t0:t0 + 10].reshape(-1, nx * ny).astype(np.float64) - 273.15
        want[t0:t0 + 10] = (m @ blk.T).T
    assert_parity(got, want, cap_of(m) * 300.0, what="stream-pointwise full scale", additive=True)


# ---------------------------------------------------------------------------------- 7. the public API


@pytest.fixture(scope="module")
def ds_api():
    return syn.make_dataset(NX, NY, NT, x0=-10.0, y0=-20.0, dx=0.5, dy=1.0, extra=("runoff",))


CONVERTERS = {
    "pv": lambda c, m: c.pv("CSi", "latitude_optimal", matrix=m, aggregate_time=None),
    "wind": lambda c, m: c.wind("Vestas_V112_3MW", matrix=m, aggregate_time=None),
    "csp": lambda c, m: c.csp(CSP, matrix=m, aggregate_time=None),
    "temperature": lambda c, m: c.temperature(matrix=m, aggregate_time=None),
    "cop": lambda c, m: c.coefficient_of_performance(matrix=m, aggregate_time=None),
    "runoff": lambda c, m: c.runoff(matrix=m, aggregate_time=None),
    "heat_demand": lambda c, m: c.heat_demand(matrix=m, aggregate_time=None, hour_shift=3.0),
    "cooling_demand": lambda c, m: c.cooling_demand(matrix=m, aggregate_time=None, hour_shift=-5.5),
}
PINNED_SUBSET = ["influx_toa", "albedo", "roughness", "temperature", "height"]


@pytest.mark.parametrize("name", list(CONVERTERS))
def test_public_converters_on_every_host_residency(ds_api, shapes, deterministic, name):
    """Host cutout, its pin_host() copy and a cutout whose variables are partly pinned
    (pin_host(variables=...)) and partly pageable: bitwise the unpadded device-resident cutout."""
    host = ab.Cutout(data=ds_api)
    pinned = host.pin_host()
    part = host.pin_host(variables=PINNED_SUBSET)
    mixed = ab.Cutout(data=_with_vars(ds_api, **{k: part.data.raw(k) for k in PINNED_SUBSET}))
    ref = np.asarray(CONVERTERS[name](host.to_device(pad=False), shapes).values)
    for what, cut in (("host", host), ("pinned", pinned), ("mixed", mixed)):
        _same_bits(np.asarray(CONVERTERS[name](cut, shapes).values), ref, f"{name} {what}")


@pytest.mark.parametrize("alt,az", [(np.float32, np.float64), (np.float64, np.float32)],
                         ids=["f32alt_f64az", "f64alt_f32az"])
def test_mixed_solar_position_dtypes(alt, az):
    """A stored solar position whose altitude and azimuth differ in dtype: both are read as float32,
    on the host and on the device, for pv, csp and line_rating."""
    ds = _with_solar(syn.make_dataset(40, 21, 24, x0=5.0, y0=35.0, kinds=("pv",)), alt, az)
    m = syn.make_shapes(40, 21, 9)
    od = oracle_ds(ds)
    cfg = ab.get_cspinstallationconfig(CSP)
    want_pv = _oracle_pv(od, m)
    want_csp = O.convert_and_aggregate(od, O.convert_csp, matrix=m, aggregate_time=None, installation=cfg)
    assert want_pv.sum() > 0 and want_csp.sum() > 0
    lds = _with_solar(syn.make_line_rating_dataset(36, 20, 24, x0=6.0, y0=47.0), alt, az)
    lx, ly = np.asarray(lds.coords["x"]), np.asarray(lds.coords["y"])
    lines = syn.make_line_network(lx, ly, 10)
    lod = oracle_ds(lds)
    assert lod["solar_altitude"].dtype == alt and lod["solar_azimuth"].dtype == az
    want_lr = LO.line_rating(lod, gis.compute_intersectionmatrix(lx, ly, lines),
                             pd.Series([LO.line_azimuth(s["coordinates"]) for s in lines]), 1e-4)
    for residency in ("host", "device"):
        c, lc = ab.Cutout(data=ds), ab.Cutout(data=lds)
        if residency == "device":
            c, lc = c.to_device(), lc.to_device()
        assert_parity(bt(CONVERTERS["pv"](c, m)), want_pv, cap_of(m), what=f"mixed-solar-pv {residency}")
        assert_parity(bt(CONVERTERS["csp"](c, m)), want_csp, cap_of(m), what=f"mixed-solar-csp {residency}")
        assert_parity(np.asarray(lc.line_rating(lines, 1e-4).values), want_lr, what=f"mixed-solar-dlr {residency}")


def test_bad_fields_raise_before_any_launch(ds_full, plan):
    """Fields with fewer steps than a call reads, a day table that ends past the temperature's last
    step, and a device solar position whose width is not the operator's: each call raises in Python,
    before a pointer reaches the library."""
    import torch

    pv = _pv_spec(ds_full)
    wind = convert._WindSpec(ds_full, _turbine(80), "logarithmic")
    heat = convert._HeatSpec(ds_full, 17.0, 1.3, 0.2, 3.0)
    pv64 = _pv_spec(_with_solar(ds_full, np.float64, np.float64))
    pv32 = _pv_spec(_with_solar(ds_full, np.float32, np.float32))
    csp64 = convert._CspSpec(_with_solar(ds_full, np.float64, np.float64), ab.get_cspinstallationconfig(CSP))
    lds = _with_solar(syn.make_line_rating_dataset(36, 20, 24, x0=6.0, y0=47.0), np.float64, np.float64)
    lr = convert._LineRatingSpec(ab.Cutout(data=lds).to_device(pad=False).data,
                                 {k: np.ones(2) for k in _lib.LINE_PARAMS})
    lr_plan = engine.get_plan(sp.csr_matrix(np.ones((2, 36 * 20))), 20, 36, entries=True)
    short = dict(pv.fields, albedo=pv.fields["albedo"][:-1])
    late = heat.day_start.copy()
    late[-1] += 1
    cases = {
        "pv short field": (ValueError, "'albedo' has 36 steps", lambda f: pv.op.reduce(plan, f), short),
        "pv cells short field": (ValueError, "'albedo' has 36 steps", lambda f: pv.op.cells(f), _dev(short)),
        "pv nt past the fields": (ValueError, "reads 38", lambda f: pv.op.reduce(plan, f, nt=NT + 1), pv.fields),
        "wind short aux": (ValueError, "'aux' has 36 steps", lambda f: wind.op.reduce(plan, f["wnd"], f["aux"]),
                           {"wnd": wind.wnd, "aux": wind.aux[:-1]}),
        "heat table past the end": (ValueError, "reads 38", lambda f: heat.op.reduce(plan, f, late), heat.temp),
        "heat cells table past the end": (ValueError, "reads 38", lambda f: heat.op.cells(f, late), _dev(heat.temp)),
    }
    d64, d32, dc64 = _dev(pv64.fields), _dev(pv32.fields), _dev(csp64.fields)
    cases.update({
        "pv f64 op, f32 azimuth": (TypeError, "float64", lambda f: pv64.op.reduce(plan, f),
                                   dict(d64, solar_azimuth=d64["solar_azimuth"].float())),
        "pv f32 op, f64 altitude": (TypeError, "float32", lambda f: pv32.op.reduce(plan, f),
                                    dict(d32, solar_altitude=d32["solar_altitude"].double())),
        "pv cells f32 op, f64 azimuth": (TypeError, "float32", lambda f: pv32.op.cells(f),
                                         dict(d32, solar_azimuth=d32["solar_azimuth"].double())),
        "csp f64 op, f32 altitude": (TypeError, "float64", lambda f: csp64.op.reduce(plan, f),
                                     dict(dc64, solar_altitude=dc64["solar_altitude"].float())),
        "line rating f64 op, f32 azimuth": (TypeError, "float64", lambda f: lr.op.reduce(lr_plan, f),
                                            dict(lr.fields, solar_azimuth=lr.fields["solar_azimuth"].to(torch.float32))),
    })
    n0 = _lib.launch_count()
    for what, (exc, match, call, fields) in cases.items():
        with pytest.raises(exc, match=match):
            call(fields)
        assert _lib.launch_count() == n0, f"{what}: launched a kernel"
    # host solar fields are converted to the operator's width, so these calls are fine
    host = dict(pv64.fields, solar_azimuth=pv64.fields["solar_azimuth"].astype(np.float32))
    assert np.isfinite(pv64.op.reduce(plan, host)).all()
