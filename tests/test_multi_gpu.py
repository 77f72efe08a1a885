"""Multi-GPU result check on hardware: the time-sharded path (one process per GPU, NCCL
gather of the (time, bus) result / all-reduce of per-cell time sums) must reproduce the
unsharded computation.  Runs tools/dist_check.py under torchrun when at least two GPUs
are visible (``python -m pytest tests -m gpu`` on a box with two or more GPUs); the gloo world-2
variant of the same logic runs on the CPU in tests/test_host_logic.py."""

import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _n_gpus():
    import torch

    return torch.cuda.device_count()


@pytest.mark.parametrize("days", [7, 1])  # 1 day on >= 2 ranks: some ranks hold an EMPTY shard
def test_time_sharded_results_equal_unsharded_on_nccl(days):
    n = _n_gpus()
    if n < 2:
        pytest.skip("needs >= 2 visible GPUs")
    world = min(n, 8)
    env = dict(os.environ, DIST_CHECK_DAYS=str(days))
    port = 29600 + (os.getpid() + days) % 300
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tools", "dist_check.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0 and f"DIST_CHECK PASS world={world}" in r.stdout, tail


def test_single_process_multi_device_equals_single_device():
    """Cutout(..., devices=...) fans the time axis of a HOST cutout out to several GPUs from
    one process; the result must equal the one-GPU result."""
    n = _n_gpus()
    if n < 2:
        pytest.skip("needs >= 2 visible GPUs")
    import numpy as np

    import atlite_b200 as ab
    from atlite_b200 import synthetic as syn

    nx, ny, nt, nbus = 64, 40, 24 * 5, 9
    ds = syn.make_dataset(nx, ny, nt, x0=0.0, y0=30.0)
    m = syn.make_shapes(nx, ny, nbus)
    one = ab.Cutout(data=ds)
    many = ab.Cutout(data=ds, devices="all")
    for call in (lambda c: c.pv("CSi", "latitude_optimal", matrix=m, aggregate_time=None),
                 lambda c: c.wind("Vestas_V112_3MW", matrix=m, aggregate_time=None),
                 lambda c: c.heat_demand(matrix=m, aggregate_time=None),
                 lambda c: c.wind("Vestas_V112_3MW", matrix=m, aggregate_time="sum")):
        a, b = call(one), call(many)
        assert a.dims == b.dims and a.shape == b.shape
        np.testing.assert_allclose(np.asarray(b.values), np.asarray(a.values), rtol=2e-5, atol=1e-6)
