"""Power-curve interpolation tables (LUT and binary-search fallback) against np.interp.

atl_wind_curve_eval_host builds the very tables atl_wind_create uploads and evaluates
them with the same fp32 formula the kernels use (one shared __host__ __device__
function), so the np.interp semantics the reference relies on (convert.py:648-649:
clamped ends, duplicate knots = steps, NaN propagation) are pinned without a GPU.
"""

import ctypes as C

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

from atlite_b200 import _lib, resource


def eval_host(V, P, x, mode=-1):
    """mode: -1 what atl_wind_create picks, 0 binary search, 1 general LUT, 2 lattice LUT with
    compares, 3 saturating lattice LUT"""
    lib = _lib.load()
    V = np.ascontiguousarray(V, dtype=np.float64)
    P = np.ascontiguousarray(P, dtype=np.float64)
    x = np.ascontiguousarray(x, dtype=np.float32)
    y = np.empty_like(x)
    used = C.c_int32(-1)
    _lib.check(lib.atl_wind_curve_eval_host(_lib.ptr(V), _lib.ptr(P), len(V), int(mode),
                                            x.ctypes.data, len(x), y.ctypes.data, C.byref(used)))
    return y, used.value


def probe_points(V, rng, n=20000):
    v32 = V.astype(np.float32)
    return np.concatenate([
        rng.uniform(V[0] - 3.0, V[-1] + 10.0, n),
        V, np.nextafter(v32, np.float32(np.inf)), np.nextafter(v32, np.float32(-np.inf)),
        [np.nan, np.inf, -np.inf, 0.0, -0.0],
    ]).astype(np.float32)


def check(V, P, x, y, slope_scale):
    want = np.interp(x.astype(np.float64), V, P)
    assert np.array_equal(np.isnan(y), np.isnan(want))
    ok = ~np.isnan(want)
    # fp32 evaluation: a few ulp of the value, plus the steepest slope times two ulp of
    # the largest speed (a knot that is not a float sits up to one ulp from its fp32
    # stand-in, and x itself is only known to half an ulp)
    tol = 4e-7 * max(1.0, np.abs(P).max()) + 2.0 * float(np.spacing(np.float32(V[-1]))) * slope_scale
    np.testing.assert_allclose(y[ok], want[ok], rtol=0, atol=tol)


def steepest(V, P):
    dv = np.diff(V)
    return float(np.max(np.abs(np.diff(P)[dv > 0] / dv[dv > 0]))) if (dv > 0).any() else 0.0


@pytest.mark.parametrize("name", sorted(resource.windturbines))
def test_shipped_turbines_use_a_lut_and_match_np_interp(name):
    t = resource.get_windturbineconfig(name)
    V, P = t["V"], t["POW"] / t["P"]
    x = probe_points(V, np.random.default_rng(1))
    y, used = eval_host(V, P, x)
    assert used in (1, 2, 3), "every shipped power curve should qualify for a single-load LUT"
    check(V, P, x, y, steepest(V, P))
    for mode in (0, 1, 2, 3):  # every table the curve qualifies for
        ym, used_m = eval_host(V, P, x, mode)
        assert used_m in (0, mode)
        check(V, P, x, ym, steepest(V, P))
    assert eval_host(V, P, x, 1)[1] == 1  # the general LUT takes every shipped curve
    # exactly at float-representable knots: np.interp's value to one ulp of fp32 (steps are
    # stored separately and added back; the lattice table evaluates slope * x + intercept)
    if np.array_equal(V.astype(np.float32).astype(np.float64), V):
        for mode in (1, 2, 3):
            yk, _ = eval_host(V, P, V.astype(np.float32), mode)
            np.testing.assert_allclose(yk, np.interp(V, V, P), rtol=0,
                                       atol=(1.2e-7 if mode == 1 else 5e-7) * np.abs(P).max())


def test_lattice_mode_is_chosen_for_lattice_curves():
    names = {n: eval_host(*(lambda t: (t["V"], t["POW"] / t["P"]))(resource.get_windturbineconfig(n)),
                          np.zeros(1, np.float32))[1] for n in resource.windturbines}
    assert names["Vestas_V112_3MW"] == 2 and names["Enercon_E126_7500kW"] == 2
    assert sum(v == 2 for v in names.values()) >= 20, names
    t = resource.windturbine_smooth(resource.get_windturbineconfig("Vestas_V112_3MW"))
    assert eval_host(t["V"], t["POW"] / t["P"], np.zeros(1, np.float32))[1] == 2  # linspace(0, 35, 72)


def test_smoothed_curve_and_steps():
    t = resource.windturbine_smooth(resource.get_windturbineconfig("Vestas_V112_3MW"))
    V, P = t["V"], t["POW"] / t["P"]
    x = probe_points(V, np.random.default_rng(2))
    y, used = eval_host(V, P, x)
    check(V, P, x, y, steepest(V, P))
    # cut-in step AND cut-out step AND a step at the very first knot
    for V, P, auto, general in [
        ([3, 3, 5, 12, 25, 25], [0, 0.1, 0.3, 1, 1, 0], 2, 1),       # a step at the first knot cannot fold
        ([0, 3, 3, 12, 25, 25], [0, 0, 0.2, 1, 1, 0], 2, 1),
        ([0, 3, 3, 12, 12, 25], [0, 0, 0.2, 0.9, 1, 1], 2, 0),      # two interior steps
        ([0, 3, 3, 12, 12, 25, 25], [0, 0, 0.2, 0.9, 1, 1, 0], 2, 0),  # three steps: folded, else search
        ([2, 2, 2, 10, 25], [0, 0.5, 0.1, 1, 0.2], 2, 1),             # triple knot, no cut-out step
        ([0, 2.37, 9.1, 25.003], [0, 0.1, 0.9, 1.0], 1, 1),           # off-lattice knots
        ([4.0], [0.7], 0, 0),                                         # single knot: constant
    ]:
        V, P = np.array(V, float), np.array(P, float)
        x = probe_points(V, np.random.default_rng(3), 5000)
        y, used = eval_host(V, P, x)
        assert used == auto, (V, P, used)
        check(V, P, x, y, steepest(V, P))
        y, used = eval_host(V, P, x, 1)
        assert used == general, (V, P, used)
        check(V, P, x, y, steepest(V, P))


@settings(max_examples=150, deadline=None)
@given(
    st.lists(st.floats(0.05, 3.0), min_size=1, max_size=40),
    st.lists(st.floats(0.0, 1.0), min_size=41, max_size=41),
    st.lists(st.integers(0, 39), max_size=3),
    st.integers(0, 2**31 - 1),
)
def test_random_curves(steps, pows, dup_at, seed):
    V = np.concatenate([[1.0], 1.0 + np.cumsum(steps)])
    for d in dup_at:  # duplicate some knots (zero-width segments = steps)
        if d + 1 < len(V):
            V[d + 1] = V[d]
    V = np.sort(V)
    P = np.array(pows[: len(V)])
    x = probe_points(V, np.random.default_rng(seed), 2000)
    for mode in (-1, 0, 1, 2, 3):
        y, used = eval_host(V, P, x, mode)
        check(V, P, x, y, steepest(V, P))


def curve_info(V, P, mode=-1):
    V = np.ascontiguousarray(V, dtype=np.float64)
    P = np.ascontiguousarray(P, dtype=np.float64)
    info = np.zeros(4, dtype=np.int32)
    _lib.check(_lib.load().atl_wind_curve_info_host(_lib.ptr(V), _lib.ptr(P), len(V), int(mode), _lib.ptr(info)))
    return dict(table=int(info[0]), compares=int(info[1]), steps=int(info[2]), bytes=int(info[3]))


def test_steps_fold_into_the_lattice_table_exactly():
    """A step on a bucket boundary needs no per-cell compare when the bucket function crosses the
    boundary exactly at the step's float threshold; the table builder verifies that in the
    kernel's float arithmetic.  Every shipped lattice curve folds; the values at the knots and
    one float either side are np.interp's (a step is O(0.1..1), the tolerance 1e-5)."""
    folded = 0
    for name in sorted(resource.windturbines):
        t = resource.get_windturbineconfig(name)
        V, P = t["V"], t["POW"] / t["P"]
        info = curve_info(V, P)
        if info["table"] not in (2, 3):
            continue
        assert info["table"] == 2 and info["compares"] == 0, (name, info)
        assert curve_info(V, P, 3)["table"] == 3  # the saturating variant qualifies too (not the default: slower)
        forced = curve_info(V, P, 2)  # mode 2 keeps the compares: the other code path stays tested
        assert forced["compares"] == info["steps"] <= 2
        folded += info["steps"] > 0
        v32 = V.astype(np.float32)
        x = np.concatenate([v32, np.nextafter(v32, np.float32(np.inf)), np.nextafter(v32, np.float32(-np.inf))])
        y, _ = eval_host(V, P, x)
        y2, _ = eval_host(V, P, x, 2)
        x = np.concatenate([x, np.array([np.inf, -np.inf, 1e30, -1e30, -1.0, 400.0], np.float32)])
        y, y2, y3 = eval_host(V, P, x)[0], eval_host(V, P, x, 2)[0], eval_host(V, P, x, 3)[0]
        np.testing.assert_allclose(y, np.interp(x.astype(np.float64), V, P), rtol=0, atol=1e-5)
        np.testing.assert_allclose(y3, y, rtol=0, atol=1e-5)
        np.testing.assert_allclose(y, y2, rtol=0, atol=1e-5)
    assert folded >= 20
    # a step at the very first knot cannot fold (speeds below it clamp onto it); knots that are
    # not binary fractions fold only if the verification passes -- either way np.interp's values
    assert curve_info([3, 3, 5, 12, 25, 25], [0, 0.1, 0.3, 1, 1, 0])["compares"] == 2
    for V, P in [([0, 3.3, 3.3, 12.1, 25.3, 25.3], [0, 0, 0.2, 1, 1, 0]),
                 ([0.1, 2.9, 2.9, 11.3, 25.3], [0, 0, 0.2, 1, 1])]:
        V, P = np.array(V, float), np.array(P, float)
        x = probe_points(V, np.random.default_rng(5), 4000)
        y, used = eval_host(V, P, x)
        check(V, P, x, y, steepest(V, P))


@pytest.mark.parametrize("mode", [-1, 2, 3])
def test_speeds_below_the_first_knot_give_the_left_end_exactly(mode):
    """np.interp's left clamp, exactly: the lattice tables read a flat guard row for every speed
    below the first knot, down to the float just below it (a sloped first segment evaluated at the
    knot would leave a rounding residue where the reference gives exactly 0)."""
    curves = [(t["V"], t["POW"] / t["P"]) for t in map(resource.get_windturbineconfig, sorted(resource.windturbines))]
    curves += [([3, 3, 5, 12, 25, 25], [0, 0.1, 0.3, 1, 1, 0]), ([3, 5, 12, 25], [0, 0.3, 1, 1]),
               ([2.5, 5, 7.5, 25, 25], [0.05, 0.3, 1, 1, 0]), ([0.1, 2.9, 2.9, 11.3, 25.3], [0, 0, 0.2, 1, 1])]
    lattice = 0
    for V, P in curves:
        V, P = np.asarray(V, float), np.asarray(P, float)
        if curve_info(V, P, mode)["table"] not in (2, 3):
            continue
        lattice += 1
        v0 = np.float32(V[0])
        x = np.array([np.nextafter(v0, np.float32(-np.inf)), v0 - np.float32(1e-3), v0 * np.float32(0.5), -1.0, -np.inf],
                     np.float32)
        y, _ = eval_host(V, P, x, mode)
        assert (y == np.float32(P[0])).all(), (V, y)
    assert lattice >= 20
