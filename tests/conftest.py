import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run on an H100)")


def _cuda_ready():
    """Is a CUDA device visible?  (A missing libatlite_b200.so on a GPU box is NOT a
    reason to skip: there the tests must fail loudly.)"""
    try:
        import torch

        if not torch.cuda.is_available():
            return False, "needs a CUDA device"
    except Exception as e:  # noqa: BLE001
        return False, f"torch unavailable: {e!r}"
    return True, ""


def pytest_collection_modifyitems(config, items):
    """`pytest tests` on a machine without CUDA reports the GPU tests as skipped
    instead of failing in torch; the loud-failure contract of the product itself is
    covered by tests/test_host_logic.py::test_no_gpu_fails_loudly."""
    ok, why = _cuda_ready()
    if ok:
        return
    skip = pytest.mark.skip(reason=why)
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def oracle_ds(ds):
    """atlite_b200 Dataset -> plain dict the oracle consumes."""
    d = {k: np.asarray(ds.raw(k)) for k in ds.keys()}
    d["time"] = ds.coords["time"]
    d["lon"] = np.asarray(ds.coords["lon"])
    d["lat"] = np.asarray(ds.coords["lat"])
    return d


PARITY_STATS = {}  # operator label -> observed maxima (written to test-results/ at session end)


def assert_parity(got, want, capacity=None, rtol=1e-4, atol_cap=1e-6, what="", additive=False, unit=1.0):
    """The parity bar (SURVEY.md section 8c): fp32 kernels vs the float64 oracle,

        |gpu - oracle| <= 1e-4 * max(|oracle|, 1e-6 * capacity_bus)  +  1.2e-7 * unit

    capacity = row sum of the aggregation matrix (times the value scale of the operator
    where the per-cell values are not capacity factors; 1 for per-cell / per-unit
    outputs); identical NaN positions.  The last term is two float32 ulps of ONE cell's
    value scale (`unit`, 1 for capacity factors): a per-cell value such as 4e-8 just above
    the cut-in speed is the difference of O(0.1) float32 quantities (slope * v + intercept)
    and cannot be exact to 1e-4 of itself; for bus sums the term is negligible.  ``additive=True`` (only for signed quantities
    whose bus sums cancel -- the deg C temperature family) uses the looser
    1e-4 * |oracle| + 1e-6 * capacity.  The observed maximum of
    |gpu - oracle| / max(|oracle|, 1e-6 * capacity) is recorded per operator."""
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    cap = 1.0 if capacity is None else np.asarray(capacity, dtype=np.float64)
    nan_g, nan_w = np.isnan(got), np.isnan(want)
    assert np.array_equal(nan_g, nan_w), f"{what}: NaN positions differ ({nan_g.sum()} vs {nan_w.sum()})"
    floor = atol_cap * np.maximum(cap, 1e-30)
    denom = np.maximum(np.abs(want), floor)
    tol = (rtol * np.abs(want) + floor if additive else rtol * denom) + 1.2e-7 * unit
    err = np.abs(got - want)
    if err.size:
        # observed errors, per operator: relative error of every value that is at least 0.1 % of
        # its capacity (what the 1e-4 bar is about), absolute error / capacity of the smaller ones
        capb = np.broadcast_to(np.maximum(cap, 1e-30), err.shape)
        big = (np.abs(want) >= 1e-3 * capb) & ~nan_w
        rel = float((err[big] / np.abs(want)[big]).max()) if big.any() else 0.0
        small = ~big & ~nan_w
        ab = float((err[small] / capb[small]).max()) if small.any() else 0.0
        st = PARITY_STATS.setdefault((what.split() or ["?"])[0],
                                     {"max_rel_err": 0.0, "max_abs_err_over_capacity_small_values": 0.0,
                                      "n_values": 0, "n_calls": 0})
        st["max_rel_err"] = max(st["max_rel_err"], rel)
        st["max_abs_err_over_capacity_small_values"] = max(st["max_abs_err_over_capacity_small_values"], ab)
        st["n_values"] += int(err.size)
        st["n_calls"] += 1
    bad = (err > tol) & ~nan_w
    if bad.any():
        i = np.unravel_index(np.nanargmax(np.where(bad, err / np.maximum(tol, 1e-300), 0)), got.shape)
        raise AssertionError(
            f"{what}: {bad.sum()} of {bad.size} outside tolerance; worst at {i}: "
            f"got {got[i]!r} want {want[i]!r} (err {err[i]:.3e}, tol {np.broadcast_to(tol, got.shape)[i]:.3e})"
        )


def pytest_sessionfinish(session, exitstatus):
    """Write the observed parity errors per operator to test-results/parity_errors.json."""
    if not PARITY_STATS:
        return
    import json

    out = os.path.join(ROOT, "test-results")
    try:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "parity_errors.json"), "w") as fh:
            json.dump({"bar": "|gpu-oracle| <= 1e-4*max(|oracle|, 1e-6*capacity) + 1.2e-7*unit  (SURVEY 8c + 2 float32 ulp)",
                       "columns": "max_rel_err over values >= 0.1% of their capacity; max |err|/capacity over the smaller ones",
                       "observed": {k: PARITY_STATS[k] for k in sorted(PARITY_STATS)}}, fh, indent=1)
    except OSError:
        pass


@pytest.fixture(scope="session")
def have_gpu():
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:  # noqa: BLE001
        return False
