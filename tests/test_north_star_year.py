"""The graded workloads over the whole year, on every bus and every step: PV, wind and heat
demand on the bench's 1440 x 720 x 8760 cutout -> 3000 shapes, against ``oracle/torch_f64.py``,
a float64 restatement of ``atlite_oracle`` that runs on the GPU next to the kernels.

CPU tests pin the restatement to ``atlite_oracle`` (1e-12 relative, identical zero and NaN
positions) on a coarse global grid with the rows where the sky and the panel tilt change: the
poles, |lat| = 25 and 50 (the bands of latitude_optimal), the equator; steps at both solstices
and both equinoxes; wind speeds at every knot of the power curve; heat with an hour shift.

GPU tests walk the year in parts that fit the free device memory and check, per operator, the
public call against the restatement reduced with the shapes' float64 CSR on the device.  A
(bus, step) entry whose cells sit at a discontinuity (the sun's altitude threshold, the cut-out
speed) may differ by the flip allowance of those cells; every other entry meets the parity bar
of ``conftest.assert_parity``, and a night entry is exactly 0.
"""

import time
import warnings

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp
from conftest import assert_parity

import atlite_oracle as O
import atlite_b200 as ab
from atlite_b200 import synthetic as syn

torch = pytest.importorskip("torch")
import torch_f64 as tf  # noqa: E402

from bench import NBUS, NT, NX, NY, ORIENT, PANEL, TURBINE, X0, Y0  # noqa: E402

warnings.filterwarnings("ignore", category=DeprecationWarning)

# ------------------------------------------------------------------ CPU: the restatement is the oracle

# rows: the south pole, the Antarctic circle, the band edges of latitude_optimal at +-25 and +-50,
# the equator and the north-most row of the bench's grid; columns every 7.5 degrees
PIN_LAT = np.array([-90.0, -75.0, -66.5, -50.0, -37.75, -25.0, -12.25, 0.0, 12.5, 25.0, 37.5, 50.0, 66.5, 80.0,
                    89.75])
PIN_LON = np.arange(-180.0, 180.0, 7.5)
# whole days at both equinoxes and both solstices, and 24 steps spread over the year
PIN_TIME = pd.DatetimeIndex(np.concatenate([
    pd.date_range(d, periods=24, freq="h").values for d in ("2013-03-20", "2013-06-21", "2013-09-22", "2013-12-21")
] + [pd.date_range("2013-01-01 05:00", periods=24, freq="365h").values]))


def _pin(got, want, what, rtol=1e-12, atol=0.0):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    assert np.array_equal(np.isnan(got), np.isnan(want)), f"{what}: NaN positions differ"
    assert np.array_equal(got == 0, want == 0), f"{what}: zero positions differ"
    ok = np.isfinite(want) & (want != 0)
    err = np.abs(got[ok] - want[ok]) / (np.abs(want[ok]) + atol / rtol)
    assert err.size == 0 or err.max() <= rtol, f"{what}: max relative difference {err.max():.3e}"


@pytest.fixture(scope="module")
def pin_fields():
    f = syn.make_fields(PIN_TIME, PIN_LON, PIN_LAT, kinds=("pv", "wind", "temperature"))
    f["influx_direct"][30, 7, 3] = np.nan  # NaN inputs: the oracle's fillna rules
    f["albedo"][40, 9, 20] = np.nan
    f["temperature"][35, 3, 11] = np.nan
    return f


def _oracle_ds(f, time, lon, lat, names):
    d = {k: f[k] for k in names}
    d.update(time=time, lon=lon, lat=lat)
    return d


PV_NAMES = ("influx_toa", "influx_direct", "influx_diffuse", "albedo", "temperature")


@pytest.mark.parametrize("orientation", ["latitude_optimal", {"slope": 30.0, "azimuth": 180.0}],
                         ids=["latitude_optimal", "constant"])
def test_pv_restatement_is_the_oracle(pin_fields, orientation):
    panel = ab.get_solarpanelconfig(PANEL)
    want = O.convert_pv(_oracle_ds(pin_fields, PIN_TIME, PIN_LON, PIN_LAT, PV_NAMES), panel,
                        O.get_orientation(orientation))
    got, _ = tf.pv({k: torch.from_numpy(pin_fields[k]) for k in PV_NAMES}, PIN_TIME, PIN_LON, PIN_LAT, panel,
                   orientation)
    assert got.dtype == torch.float64
    assert (want > 0).sum() > 0.2 * want.size and (want == 0).sum() > 0.2 * want.size  # day and night
    for i in (0, 5, 9, 14):  # lat -90, -25, 25 and 89.75 see daylight
        assert (want[:, i] > 0).any(), PIN_LAT[i]
    _pin(got.numpy(), want, f"pv {orientation}")
    # the solar position itself, where the sun is up
    sp_o = O.solar_position(_oracle_ds(pin_fields, PIN_TIME, PIN_LON, PIN_LAT, ()))
    sp_t = tf.solar_position(PIN_TIME, PIN_LON, PIN_LAT, "cpu")
    np.testing.assert_allclose(sp_t["altitude"].numpy(), sp_o["altitude"], rtol=0, atol=1e-13)
    up = sp_o["altitude"] > 0.01
    np.testing.assert_allclose(sp_t["azimuth"].numpy()[up], sp_o["azimuth"][up], rtol=0, atol=1e-9)


def _knot_speeds(turbine):
    """Every knot and one and two float32 ulps either side, as float32."""
    v = np.unique(np.asarray(turbine["V"], dtype=np.float32))
    out = [v]
    for k in (1, 2):
        up, dn = v, v
        for _ in range(k):
            up, dn = np.nextafter(up, np.float32(np.inf)), np.nextafter(dn, np.float32(-np.inf))
        out += [up, dn]
    return np.concatenate(out)


@pytest.mark.parametrize("hub", [None, 100.0], ids=["hub80_log_law", "hub100"])
def test_wind_restatement_is_the_oracle(pin_fields, hub):
    turbine = ab.get_windturbineconfig(TURBINE)
    if hub is not None:
        turbine = dict(turbine, hub_height=hub)
    f = {k: pin_fields[k].copy() for k in ("wnd100m", "roughness")}
    r = f["roughness"]
    # hub speeds at the knots: the 100 m speed itself for a hub at 100 m; for the log law the 100 m
    # speed that lands nearest each knot, and its float32 neighbours
    speeds = _knot_speeds(turbine)
    cells = np.arange(len(speeds) * 3)
    flat_w, flat_r = f["wnd100m"].reshape(-1), r.reshape(-1)
    if hub is None:
        ratio = (O.extrapolate_wind_speed({"wnd100m": np.ones_like(flat_r[cells]), "roughness": flat_r[cells]},
                                          turbine["hub_height"]))
        base = np.repeat(speeds, 3)
        planted = (base / ratio).astype(np.float32)
        planted = np.where(cells % 3 == 1, np.nextafter(planted, np.float32(np.inf)), planted)
        planted = np.where(cells % 3 == 2, np.nextafter(planted, np.float32(-np.inf)), planted)
    else:
        planted = np.repeat(speeds, 3)
    flat_w[cells] = planted
    flat_w[cells[-1] + 1] = np.nan
    ds = _oracle_ds(f, PIN_TIME, PIN_LON, PIN_LAT, ("wnd100m", "roughness"))
    want = O.convert_wind(ds, turbine)
    want_hub = np.asarray(O.extrapolate_wind_speed(ds, turbine["hub_height"]), dtype=np.float64)
    got_hub = tf.wind_speed(torch.from_numpy(f["wnd100m"]), torch.from_numpy(r), turbine["hub_height"])
    got, _ = tf.wind(torch.from_numpy(f["wnd100m"]), torch.from_numpy(r), turbine)
    assert got.dtype == got_hub.dtype == torch.float64
    got, got_hub = got.numpy(), got_hub.numpy()
    # the interpolation alone, on the oracle's own hub speeds
    _pin(tf.interp(torch.from_numpy(want_hub), turbine["V"], np.asarray(turbine["POW"]) / turbine["P"]).numpy(),
         want, f"wind interp {hub}", atol=1e-15)
    if hub is not None:
        _pin(got, want, "wind hub 100", atol=1e-15)
        return
    # NumPy's float32 log (SIMD) is one ulp off the correctly rounded one for a few per cent of
    # arguments (which ones also depends on the array's alignment); the restatement rounds the
    # float64 log.  So the hub speeds are the oracle's to 1e-12 on most cells, and within that ulp
    # (2**-23 relative) on the others.  Where they agree, so do the capacity factors: to 1e-12, or
    # 1e-15 absolute just above a knot, where slope * (v - knot) cancels.
    ok = ~np.isnan(want_hub)
    assert np.array_equal(np.isnan(got_hub), ~ok)
    same = ok & (np.abs(np.nan_to_num(got_hub - want_hub)) <= 1e-12 * np.abs(np.nan_to_num(want_hub)))
    assert same.mean() > 0.9
    assert same.reshape(-1)[cells].mean() > 0.8  # most planted knot speeds are pinned
    _pin(got[same], want[same], "wind log law", atol=1e-15)
    assert (np.abs(got_hub[ok] - want_hub[ok]) <= 2.4e-7 * np.abs(want_hub[ok])).all()


@pytest.mark.parametrize("hour_shift", [0.0, -5.0])
@pytest.mark.parametrize("params", [(15.0, 1.0, 0.0), (17.0, 1.3, 0.2)], ids=["graded", "other"])
def test_heat_restatement_is_the_oracle(hour_shift, params):
    tm = pd.date_range("2013-12-20", periods=4 * 24 + 7, freq="h")
    f = syn.make_fields(tm, PIN_LON, PIN_LAT, kinds=("temperature",))
    T = f["temperature"]
    T[3, 2, 5] = np.nan  # one NaN step of a day
    T[0:24, 4, 6] = np.nan  # a whole (unshifted) day
    want, _ = O.convert_heat_demand(_oracle_ds(f, tm, PIN_LON, PIN_LAT, ("temperature",)), *params, hour_shift)
    got, allowance = tf.heat_demand(torch.from_numpy(T), tm, *params, hour_shift)
    assert got.dtype == torch.float32 and want.dtype == np.float32
    assert float(allowance) == 0.0
    assert len(want) == (5 if hour_shift == 0 else 6)
    np.testing.assert_array_equal(got.numpy(), want)  # float32 either side: bit for bit


def _sun_crossing(time, lat, thr=1.0):
    """The longitude where the restatement's altitude at ``time`` and ``lat`` is the threshold
    (morning side), by bisection."""
    lo, hi = -180.0, 180.0
    alt = lambda lon: float(tf.solar_position([time], [lon], [lat], "cpu")["altitude"][0, 0, 0])  # noqa: E731
    grid = np.linspace(lo, hi, 721)
    a = np.array([alt(v) for v in grid]) - np.radians(thr)
    i = int(np.flatnonzero((a[:-1] < 0) & (a[1:] >= 0))[0])
    lo, hi = grid[i], grid[i + 1]
    for _ in range(60):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if alt(mid) < np.radians(thr) else (lo, mid)
    return 0.5 * (lo + hi)


def test_flip_allowances():
    """Zero away from the discontinuities, the size of the jump on cells planted at them."""
    # PV: columns at the 1 degree crossing and at 1e-3 / 1e-2 degree of longitude from it
    t0, lat = pd.Timestamp("2013-06-21 09:00"), np.array([10.0, 25.0])
    lon0 = _sun_crossing(t0, 10.0)
    lon = np.array([lon0, lon0 + 1e-3, lon0 - 1e-2, lon0 + 30.0])
    tm = pd.DatetimeIndex([t0])
    # bright inputs: at the synthetic fields' 24 W/m2 top-of-atmosphere influx the Huld efficiency
    # is already 0 at the threshold
    f = {k: torch.full((1, 2, 4), v, dtype=torch.float32) for k, v in
         (("influx_toa", 1000.0), ("influx_direct", 600.0), ("influx_diffuse", 150.0), ("albedo", 0.2),
          ("temperature", 290.0))}
    value, allowance = tf.pv(f, tm, lon, lat, ab.get_solarpanelconfig(PANEL), ORIENT)
    alt = tf.solar_position(tm, lon, lat, "cpu")["altitude"]
    assert abs(float(alt[0, 0, 0]) - np.radians(1.0)) < 1e-12
    assert float(allowance[0, 0, 0]) > 1e-3  # the sun at the threshold: the whole unmasked value
    assert float(value[0, 0, 0]) in (0.0, float(allowance[0, 0, 0]))
    far = torch.abs(alt - np.radians(1.0)) >= tf.PV_ALTITUDE_WINDOW
    assert bool(far[0, 0, 1:].all()) and bool(far[0, 1].all())
    assert bool((allowance[far] == 0).all())
    # and on the pin grid, a year's sample: nothing is near the threshold
    pf = syn.make_fields(PIN_TIME, PIN_LON, PIN_LAT, kinds=("pv",))
    _, a = tf.pv({k: torch.from_numpy(v) for k, v in pf.items()}, PIN_TIME, PIN_LON, PIN_LAT,
                 ab.get_solarpanelconfig(PANEL), ORIENT)
    near = torch.abs(tf.solar_position(PIN_TIME, PIN_LON, PIN_LAT, "cpu")["altitude"] - np.radians(1.0)) \
        < tf.PV_ALTITUDE_WINDOW
    assert bool((a[~near] == 0).all())
    # wind: hub speeds (a hub at 100 m: the 100 m speed) at and around the 25 m/s cut-out
    turbine = dict(ab.get_windturbineconfig(TURBINE), hub_height=100.0)
    w = torch.tensor([25.0, np.nextafter(np.float32(25), np.float32(0)), 25.0 * (1 + 5e-6), 25.0 * (1 - 2e-5),
                      24.9, 25.1, 12.0, 3.0, 0.0, 30.0], dtype=torch.float32)[None, None, :]
    value, allowance = tf.wind(w, torch.full_like(w, 0.03), turbine)
    np.testing.assert_array_equal(allowance[0, 0].numpy(), [1.0, 1.0, 1.0, 0, 0, 0, 0, 0, 0, 0])
    assert float(value[0, 0, 0]) == 0.0 and float(value[0, 0, 1]) == 1.0  # the jump itself
    # the log law on a Weibull field: only speeds near 25 m/s carry an allowance
    wf = syn.make_fields(PIN_TIME, PIN_LON, PIN_LAT, kinds=("wind",))
    turbine = ab.get_windturbineconfig(TURBINE)
    hub = tf.wind_speed(torch.from_numpy(wf["wnd100m"]), torch.from_numpy(wf["roughness"]), turbine["hub_height"])
    _, a = tf.wind(torch.from_numpy(wf["wnd100m"]), torch.from_numpy(wf["roughness"]), turbine)
    near = torch.abs(hub - 25.0) <= 25.0 * tf.WIND_KNOT_WINDOW
    assert bool((a[~near] == 0).all()) and bool((a[near] == 1.0).all())


# ------------------------------------------------------------------ GPU: the graded year

SUB = 48  # steps per slab of the float64 reference
REF_WORK = 18  # float64 (SUB, ny, nx) arrays the PV reference holds at its peak (with margin)


def _parts(bytes_per_step, align=1):
    """Time parts [(a, b)] of the year whose inputs, plus the reference's working set, stay within
    60 % of the free device memory."""
    free, _ = torch.cuda.mem_get_info()
    budget = 0.6 * free - REF_WORK * SUB * NX * NY * 8
    n = int(budget // bytes_per_step) // align * align
    assert n >= max(SUB, align), f"not enough free device memory ({free / 2**30:.1f} GiB)"
    n = min(n, NT)
    return [(a, min(NT, a + n)) for a in range(0, NT, n)]


@pytest.fixture(scope="module")
def grid():
    from atlite_b200 import engine

    dev = torch.device("cuda", 0)
    x, y = syn.make_coords(NX, NY, X0, Y0)
    shapes = syn.make_shapes(NX, NY, NBUS)  # bench.py's shapes

    def dev_csr(m):
        m = sp.csr_matrix(m, dtype=np.float64)
        return torch.sparse_csr_tensor(torch.as_tensor(m.indptr, dtype=torch.int64, device=dev),
                                       torch.as_tensor(m.indices, dtype=torch.int64, device=dev),
                                       torch.as_tensor(m.data, device=dev), m.shape)

    g = dict(dev=dev, x=x, y=y, time=syn.make_time(NT), shapes=shapes, plan=engine.get_plan(shapes, NY, NX),
             W=dev_csr(shapes), Wabs=dev_csr(abs(shapes)), cap=np.asarray(shapes.sum(-1)).ravel())
    yield g
    del g
    torch.cuda.empty_cache()


def _cutout(fields, g, a, b):
    return ab.Cutout(data=ab.Dataset(fields, coords=dict(time=g["time"][a:b], x=g["x"], y=g["y"], lon=g["x"],
                                                        lat=g["y"])))


def _bus_sums(g, cube, weights="W"):
    """(t, ny, nx) float64 on the device -> (bus, t) float64 on the host, with the shapes' CSR
    (or its absolute values, for the allowances)."""
    return torch.sparse.mm(g[weights], cube.reshape(len(cube), -1).T.contiguous()).cpu().numpy()


def _check_year(label, got, want, allowance, capacity, unit=1.0):
    """Every (bus, step) entry: the parity bar, plus the reduced allowance where it is non-zero;
    exact zeros at night.  Returns the number of entries that needed an allowance."""
    capb = np.broadcast_to(np.asarray(capacity, dtype=np.float64)[:, None], got.shape)
    flag = allowance > 0
    n_flag = int(flag.sum())
    assert n_flag < 0.01 * flag.size, f"{label}: {n_flag} of {flag.size} entries need an allowance"
    assert_parity(got[~flag], want[~flag], capb[~flag], what=f"{label} every bus and step", unit=unit)
    if n_flag:
        # assert_parity's tolerance (conftest) plus the reduced flip allowance
        tol = 1e-4 * np.maximum(np.abs(want[flag]), 1e-6 * capb[flag]) + 1.2e-7 * unit + allowance[flag]
        err = np.abs(got[flag] - want[flag])
        assert (err <= tol).all(), f"{label}: {(err > tol).sum()} of {n_flag} allowance entries outside"
    night = (want == 0) & ~flag
    assert (got[night] == 0).all(), f"{label}: {(got[night] != 0).sum()} night entries are not exactly 0"
    print(f"{label}: {got.size} entries, {n_flag} with an allowance, {int(night.sum())} exact night zeros, "
          f"max |err| {np.abs(got - want).max():.3e}")
    return n_flag


def _same_bits(public, spec_result):
    """The public call's (bus, t) float64 result == the spec-level (t, bus) float32 result, bit for bit."""
    s = spec_result.cpu().numpy()
    assert s.dtype == np.float32
    np.testing.assert_array_equal(public.T, s.astype(np.float64))


def _year(g, make_fields, bytes_per_step, convert, reference, spec_reduce, align=1, annual=True):
    """Walk the year for one operator.  Returns (got, want, allowance) of the bus results (bus, t)
    and of the per-cell annual sums (y, x)."""
    got_l, want_l, allow_l = [], [], []
    cells_got = np.zeros((NY, NX))
    cells_want = torch.zeros((NY, NX), dtype=torch.float64, device=g["dev"])
    cells_allow = torch.zeros_like(cells_want)
    for p, (a, b) in enumerate(_parts(bytes_per_step, align)):
        f = make_fields(a, b)
        cut = _cutout(f, g, a, b)
        got = np.asarray(convert(cut, matrix=g["shapes"], aggregate_time=None).values)
        assert got.shape[0] == NBUS
        if p == 0:  # the bench's spec-level call computes the public call's float32 values
            prev = ab.set_deterministic(True)  # a fixed summation order: bitwise comparable
            try:
                _same_bits(np.asarray(convert(cut, matrix=g["shapes"], aggregate_time=None).values),
                           spec_reduce(f, a, b))
            finally:
                ab.set_deterministic(prev)
        if annual:
            cells_got += np.asarray(convert(cut, aggregate_time="sum").values, dtype=np.float64)
        want = np.empty_like(got)
        allow = np.zeros_like(got)
        for s in range(a, b, align * max(1, SUB // align)):
            e = min(b, s + align * max(1, SUB // align))
            v, al = reference(f, s - a, e - a, g["time"][s:e])
            i, j = (s - a) // align, (e - a) // align
            want[:, i:j] = _bus_sums(g, v.to(torch.float64))
            if al.dim():
                allow[:, i:j] = _bus_sums(g, al, "Wabs")
                cells_allow += al.sum(0)
            if annual:
                cells_want += v.sum(0)
            del v, al
        got_l.append(got), want_l.append(want), allow_l.append(allow)
        del f, cut
        torch.cuda.empty_cache()
    return ((np.concatenate(got_l, 1), np.concatenate(want_l, 1), np.concatenate(allow_l, 1)),
            (cells_got, cells_want.cpu().numpy(), cells_allow.cpu().numpy()))


def _check_annual(label, got, want, allowance):
    """Per-cell annual sums: a year's sum of capacity factors has capacity NT (one per step)."""
    flag = allowance > 0
    assert_parity(got[~flag], want[~flag], np.full((~flag).sum(), float(NT)), what=f"{label} per-cell annual sums")
    tol = 1e-4 * np.maximum(np.abs(want[flag]), 1e-6 * NT) + 1.2e-7 + allowance[flag]
    assert (np.abs(got[flag] - want[flag]) <= tol).all()
    print(f"{label}: {got.size} cells, {int(flag.sum())} with an allowance, max |err| {np.abs(got - want).max():.3e}")


@pytest.mark.gpu
def test_pv_year_every_bus_and_step(grid):
    from atlite_b200.convert import _PvSpec

    g, t0 = grid, time.perf_counter()
    torch.cuda.reset_peak_memory_stats()
    panel = ab.get_solarpanelconfig(PANEL)

    def fields(a, b):  # bench.py: make_pv_fields_device(seed=0)
        return syn.make_pv_fields_device(g["time"][a:b], g["x"], g["y"], g["dev"], seed=0, t_offset=a)

    def spec_reduce(f, a, b):
        spec = _PvSpec(_cutout(f, g, a, b).data, panel, ab.get_orientation(ORIENT))
        return spec.op.reduce(g["plan"], spec.fields)

    def reference(f, i, j, tm):
        return tf.pv({k: v[i:j] for k, v in f.items()}, tm, g["x"], g["y"], panel, ORIENT)

    bus, cells = _year(g, fields, 20 * NX * NY, lambda c, **kw: c.pv(PANEL, ORIENT, **kw), reference,
                       spec_reduce)
    n = _check_year("pv_year", *bus, g["cap"])
    assert (bus[1] > 0).any(axis=0).sum() == NT  # daylight on some bus at every step
    _check_annual("pv_annual", *cells)
    print(f"pv: {n} allowance entries; wall {time.perf_counter() - t0:.1f} s, "
          f"peak device memory {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")


@pytest.mark.gpu
def test_wind_year_every_bus_and_step(grid):
    from atlite_b200.convert import _WindSpec

    g, t0 = grid, time.perf_counter()
    torch.cuda.reset_peak_memory_stats()
    turbine = ab.get_windturbineconfig(TURBINE)

    def fields(a, b):  # bench.py: make_wind_fields_device(seed=1)
        return syn.make_wind_fields_device(b - a, NY, NX, g["dev"], seed=1, t_offset=a)

    def spec_reduce(f, a, b):
        ws = _WindSpec(_cutout(f, g, a, b).data, turbine)
        return ws.op.reduce(g["plan"], ws.wnd, ws.aux)

    def reference(f, i, j, tm):
        return tf.wind(f["wnd100m"][i:j], f["roughness"][i:j], turbine)

    bus, cells = _year(g, fields, 8 * NX * NY, lambda c, **kw: c.wind(TURBINE, **kw), reference,
                       spec_reduce)
    n = _check_year("wind_year", *bus, g["cap"])
    _check_annual("wind_annual", *cells)
    print(f"wind: {n} allowance entries; wall {time.perf_counter() - t0:.1f} s, "
          f"peak device memory {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")


@pytest.mark.gpu
def test_heat_year_every_bus_and_day(grid):
    from atlite_b200.convert import _HeatSpec

    g, t0 = grid, time.perf_counter()
    torch.cuda.reset_peak_memory_stats()

    def fields(a, b):  # bench.py: make_pv_fields_device(seed=2, names=("temperature",))
        return syn.make_pv_fields_device(g["time"][a:b], g["x"], g["y"], g["dev"], seed=2, names=("temperature",),
                                         t_offset=a)

    def spec_reduce(f, a, b):
        hs = _HeatSpec(_cutout(f, g, a, b).data, 15.0, 1.0, 0.0, 0.0)
        return hs.op.reduce(g["plan"], hs.temp, hs.day_start)

    def reference(f, i, j, tm):
        return tf.heat_demand(f["temperature"][i:j], tm, 15.0, 1.0, 0.0, 0.0)

    def convert(c, **kw):
        return c.heat_demand(threshold=15.0, a=1.0, constant=0.0, hour_shift=0.0, **kw)

    # parts and reference slabs cut on day boundaries (hour_shift 0: every 24 steps)
    bus, _ = _year(g, fields, 4 * NX * NY, convert, reference, spec_reduce, align=24, annual=False)
    assert bus[0].shape == (NBUS, NT // 24)
    assert not bus[2].any()
    _check_year("heat_year", *bus[:2], np.zeros_like(bus[0]), g["cap"] * 50.0)
    print(f"heat: wall {time.perf_counter() - t0:.1f} s, "
          f"peak device memory {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
