"""CPU tests of the host-side mirror: resources, orientation, day bins, labelled
containers, argument validation, the C-ABI export table, and the 2-rank gloo
path of the time-shard gather."""

import ctypes
import os
import re

import numpy as np
import pandas as pd
import pytest
from conftest import ROOT

import atlite_oracle as O
import atlite_b200 as ab
from atlite_b200 import _lib, proj, synthetic as syn
from atlite_b200.convert import day_bins
from atlite_b200.dist import shard_bounds


def test_registries_and_turbine_validation():
    assert len(ab.windturbines) == 27 and set(ab.solarpanels) == {"CSi", "CdTe", "KANENA"}
    t = ab.get_windturbineconfig("Vestas_V112_3MW")
    assert t["P"] == 3.06 and t["hub_height"] == 80.0 and t["V"][-1] == t["V"][-2] == 25
    # cut-out padding (reference test/test_resource.py:17-23, resource.py:357-363)
    d = dict(V=[0, 5, 10], POW=[0, 1, 2], P=2, hub_height=100)
    assert ab.get_windturbineconfig(dict(d), add_cutout_windspeed=True)["POW"][-1] == 0
    assert ab.get_windturbineconfig(dict(d), add_cutout_windspeed=True)["V"][-1] == 10
    assert len(ab.get_windturbineconfig(dict(d), add_cutout_windspeed=False)["V"]) == 3
    with pytest.raises(ValueError):
        ab.get_windturbineconfig(dict(V=[0, 5, 3], POW=[0, 1, 2], P=2, hub_height=100))
    with pytest.raises(ValueError):
        ab.get_windturbineconfig(dict(V=[0, 5], POW=[0, 1, 2], P=2, hub_height=100))
    with pytest.raises(ValueError):
        ab.get_windturbineconfig(dict(V=[0, 5], POW=[0, 1]))


def test_smooth_matches_oracle():
    t = ab.get_windturbineconfig("Enercon_E101_3000kW")
    a, b = ab.windturbine_smooth(t), O.windturbine_smooth(t)
    np.testing.assert_allclose(a["POW"], b["POW"], rtol=0, atol=1e-15)
    np.testing.assert_array_equal(a["V"], b["V"])
    assert a["P"] == b["P"]


@pytest.mark.parametrize("name", ["latitude_optimal", "latitude", {"slope": 30.0, "azimuth": 170.0}])
def test_orientation_matches_oracle(name):
    lat = np.radians(np.linspace(-80, 80, 33))
    a = ab.get_orientation(name)(None, lat, None)
    b = O.get_orientation(name)(None, lat, None)
    for k in ("slope", "azimuth"):
        np.testing.assert_array_equal(np.broadcast_to(a[k], lat.shape), np.broadcast_to(b[k], lat.shape))


@pytest.mark.parametrize("shift", [0.0, 4.0, -5.0, 0.5])
def test_day_bins_match_oracle(shift):
    time = pd.date_range("2013-03-30 07:00", periods=100, freq="h")
    labels, offs = day_bins(time, shift)
    olabels, gid = O.day_bins(time, shift)
    assert list(labels) == list(olabels)
    for d in range(len(labels)):
        assert (gid[offs[d]:offs[d + 1]] == d).all()
    assert offs[0] == 0 and offs[-1] == 100


def test_labelled_containers():
    ds = syn.make_dataset(8, 6, 5, kinds=("wind",))
    assert "wnd100m" in ds and "lon" in ds and ds.sizes == {"time": 5, "y": 6, "x": 8}
    da = ds["wnd100m"]
    assert da.dims == ("time", "y", "x")
    np.testing.assert_allclose(da.mean("time").values, ds.raw("wnd100m").mean(0), rtol=1e-6)
    assert da.sum("time").dims == ("y", "x")
    assert da.isel(time=0).dims == ("y", "x")
    assert float(da.sel(time="2013-01-01 02:00").sum()) == pytest.approx(ds.raw("wnd100m")[2].sum(), rel=1e-5)
    assert (da.notnull()).all()
    assert ((da * 2.0).values == ds.raw("wnd100m") * 2).all()
    c = ab.Cutout(data=ds)
    g = c.grid
    assert list(g.columns) == ["x", "y"] and len(g) == 48
    # y-major, x-minor: reference test/test_gis.py:234-238
    np.testing.assert_array_equal(g.x.values[:8], ds.coords["x"])
    assert (g.y.values[:8] == ds.coords["y"][0]).all()


def test_validation_errors_before_any_gpu_work():
    ds = syn.make_dataset(8, 6, 5, kinds=("wind",))
    c = ab.Cutout(data=ds)

    def identity_convert(d, **kw):
        return d["wnd100m"]

    for bad in ("invalid", False, True):
        with pytest.raises(ValueError, match="aggregate_time must be"):
            ab.convert_and_aggregate(c, identity_convert, aggregate_time=bad)
    with pytest.raises(ValueError, match="Cannot use"):
        ab.convert_and_aggregate(c, identity_convert, capacity_factor=True, aggregate_time="mean")
    with pytest.raises(ValueError, match="One of `matrix`"):
        ab.convert_and_aggregate(c, identity_convert, per_unit=True, aggregate_time="sum")
    with pytest.raises(ValueError, match="ambiguous"):
        ab.convert_and_aggregate(c, identity_convert, matrix=np.ones((1, 48)), shapes=[1], aggregate_time=None)
    with pytest.raises(ValueError, match="2-dimensional"):
        ab.convert_and_aggregate(c, identity_convert, matrix=np.ones((48,)), aggregate_time=None)
    # plugin protocol without aggregation never needs the GPU
    with pytest.warns(FutureWarning, match="aggregate_time='legacy'"):
        r = ab.convert_and_aggregate(c, identity_convert)
    np.testing.assert_allclose(r.values, ds.raw("wnd100m").sum(0), rtol=1e-6)
    with pytest.warns(FutureWarning, match="capacity_factor is deprecated"):
        r = ab.convert_and_aggregate(c, identity_convert, capacity_factor=True)
    assert "time" not in r.dims


def test_cabi_exports_every_declared_symbol_at_abi_version_6():
    header = open(os.path.join(ROOT, "include", "atlite_b200.h")).read()
    declared = set(re.findall(r"\b(atl_[a-z0-9_]+)\s*\(", header))
    assert declared, "no declarations found"
    assert os.path.exists(_lib.LIB_PATH), "libatlite_b200.so not built (run __graft_entry__.build())"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    missing = [s for s in sorted(declared) if not hasattr(lib, s)]
    assert not missing, f"not exported: {missing}"
    assert set(_lib.EXPORTED_SYMBOLS) == declared
    assert _lib.load().atl_abi_version() == 6


@pytest.mark.parametrize("side", ["from_", "to"])
def test_unknown_crs_is_refused_before_device_work(side):
    """Every entry point that projects (atl_avail_raster_sample, atl_avail_count, atl_reproject)
    checks its AtlProjection on the host and refuses an unknown CRS kind before touching a device.
    The descriptors are valid otherwise, but for a negative band row that is checked later, so no
    kernel could run even if the CRS went unchecked; the reprojection has an empty batch."""
    lib = _lib.load()
    P = proj.device_projection(3035, 4326)
    getattr(P, side).kind = 7
    L = _lib.Lattice(0.0, 1.0, 0.0, -1.0, 4, 4)
    s = _lib.RasterSample(win=L, ras=L, proj=P, idx=8, idx_bytes=1, lut=8, out=8, win_row0=-1)
    c = _lib.AvailCount(win=L, proj=P, excl=8, gdx=1.0, gdy=1.0, gnx=1, gny=1, counts=8, win_row0=-1)
    r = _lib.Reproject(src=L, dst=L, proj=P, resampling=_lib.RESAMPLING_NEAREST)
    for rc in (lib.atl_avail_raster_sample(0, ctypes.byref(s), None), lib.atl_avail_count(0, ctypes.byref(c), None),
               lib.atl_reproject(0, ctypes.byref(r), 1, 0, None, 4, 16, None, None)):
        assert rc == -1  # ATL_ERR_INVALID
        assert lib.atl_last_error() == b"unknown CRS in the projection"


def test_no_gpu_fails_loudly(have_gpu):
    if have_gpu:
        pytest.skip("GPU present")
    ds = syn.make_dataset(8, 6, 5, kinds=("wind",))
    with pytest.raises(_lib.AtlError):
        ab.Cutout(data=ds).wind("Vestas_V112_3MW", matrix=np.ones((1, 48)), aggregate_time=None)


def test_shard_bounds():
    for nt, world, align in [(8760, 8, 1), (8760, 8, 24), (100, 3, 24), (5, 8, 1), (48, 2, 24)]:
        b = [shard_bounds(nt, world, r, align) for r in range(world)]
        assert b[0][0] == 0 and b[-1][1] == nt
        for (a0, a1), (b0, b1) in zip(b[:-1], b[1:]):
            assert a1 == b0 and a0 <= a1
        for lo, hi in b:
            assert lo % align == 0 or lo == nt


def _gloo_worker(rank, world, port, q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from atlite_b200.dist import TimeShard

        nt, nbus = 50, 7
        full = np.arange(nt * nbus, dtype=np.float32).reshape(nt, nbus)
        time = pd.date_range("2013-01-01", periods=nt, freq="h")
        for align in (1, 24):  # equal and ragged shards
            lo, hi = shard_bounds(nt, world, rank, align)
            sh = TimeShard()
            out, lab = sh.gather_time(full[lo:hi], time[lo:hi])
            assert np.array_equal(out.numpy(), full), (rank, align)
            assert list(lab) == list(time)
        # asynchronous gather of equal shards (what bench.py overlaps with the next pass)
        lo, hi = shard_bounds(nt, world, rank, 1)
        works = []
        for k in range(3):
            out, work = TimeShard().gather_time(full[lo:hi] + k, counts=[nt // world] * world, async_op=True)
            works.append((out, work, k))
        for out, work, k in works:
            work.wait()
            assert np.array_equal(out.numpy(), full + k), (rank, k)
        plane = np.full((3, 4), float(rank + 1), dtype=np.float32)
        tot, n = TimeShard().sum_over_ranks(plane, 10 * (rank + 1))
        assert np.allclose(tot.numpy(), sum(range(1, world + 1))) and n == 10 * sum(range(1, world + 1))
        # (sum, valid-step count) planes of a time-aggregated per-cell output: one all-reduce
        tot, cnt = TimeShard().sum_planes(plane, np.full((3, 4), 5.0 * (rank + 1), dtype=np.float32))
        assert np.allclose(tot.numpy(), sum(range(1, world + 1))) and np.allclose(cnt.numpy(), 5 * sum(range(1, world + 1)))
        q.put((rank, "ok"))
    except Exception as e:  # noqa: BLE001
        q.put((rank, repr(e)))
    finally:
        dist.destroy_process_group()


def test_time_shard_gather_gloo_world2():
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res


def test_run_partitioned_returns_results_in_order_and_releases_part_inputs(monkeypatch):
    """The partitioned runner (convert._run_partitioned) on a fake device layer: results come back in time
    order with the labels the orchestration needs, and a part's input dataset does not outlive the part --
    otherwise a lazily loaded cutout larger than the host memory would pile up in RAM part by part."""
    import gc
    import types
    import weakref

    import numpy as np

    from atlite_b200 import convert, engine

    fake_torch = types.SimpleNamespace(cuda=types.SimpleNamespace(set_device=lambda d: None))
    monkeypatch.setattr(engine, "_torch", lambda: fake_torch)
    alive = []

    class Part:  # what LazyDataset.isel_time hands out: owns the decoded arrays of one part
        def __init__(self, lo, hi):
            self.lo, self.hi, self.payload = lo, hi, np.zeros(1000)

    class Source:
        lazy = True

        def isel_time(self, lo, hi):
            p = Part(lo, hi)
            alive.append(weakref.ref(p))
            return p

    peak = []

    class Spec:
        name, units = "thing", "MW"

        def __init__(self, part, scale=1.0):
            self.part, self.scale = part, scale
            self.time_labels = np.arange(part.lo, part.hi)

    def run(spec, dev):
        gc.collect()
        peak.append(sum(r() is not None for r in alive))
        return np.full((spec.part.hi - spec.part.lo, 2), dev * 100.0 + spec.part.lo) * spec.scale

    parts = [(0, 3, 0), (3, 5, 1), (5, 9, 0), (9, 10, 1)]
    out = convert._run_partitioned(Source(), Spec, dict(scale=2.0), parts, run, 1)
    assert [v.shape[0] for v, _ in out] == [3, 2, 4, 1]
    assert [float(v[0, 0]) for v, _ in out] == [0.0, 206.0, 10.0, 218.0]
    assert np.array_equal(np.concatenate([m.time_labels for _, m in out]), np.arange(10))
    assert out[0][1].name == "thing" and out[0][1].units == "MW"
    gc.collect()
    assert not any(r() is not None for r in alive), "part inputs must be released"
    assert max(peak) <= 2  # one part per device thread at a time (two devices here)


def test_matrix_digest_is_a_content_key():
    """The plan-cache key (engine.matrix_digest over atl_hash128): equal for equal matrices, different
    for any changed value, index, dtype or shape, and for every one-bit / one-byte-length change of
    the hashed bytes."""
    import ctypes as C

    import numpy as np
    import scipy.sparse as sp

    from atlite_b200 import _lib, engine

    m = sp.random(40, 900, density=0.05, random_state=3, format="csr")
    d = engine.matrix_digest(m)
    assert engine.matrix_digest(m.copy()) == d and engine.matrix_digest(sp.csr_matrix(m.toarray())) == d
    for change in ("data", "indices", "dtype", "shape"):
        m2 = m.copy()
        if change == "data":
            m2.data[17] = np.nextafter(m2.data[17], 2.0)
        elif change == "indices":
            m2.indices[5], m2.indices[6] = m2.indices[6], m2.indices[5]
        elif change == "dtype":
            m2.data = m2.data.astype(np.float32)
        else:
            m2 = sp.csr_matrix((m.data, m.indices, m.indptr), shape=(40, 901))
        assert engine.matrix_digest(m2) != d, change

    def h(x, seed=0):
        out = (C.c_uint64 * 2)()
        _lib.check(_lib.load().atl_hash128(x.ctypes.data_as(C.c_void_p), x.nbytes, seed, out))
        return out[0], out[1]

    b = np.random.default_rng(0).integers(0, 255, 777, dtype=np.uint8)
    seen = {h(b)}
    for i in range(777):
        c = b.copy()
        c[i] ^= 1 << (i % 8)
        seen.add(h(c))
    for n in range(64):
        seen.add(h(b[:n]))
    assert len(seen) == 1 + 777 + 64 and h(b, 1) != h(b, 0)


def test_finish_results_device_path_equals_the_numpy_path():
    """convert._finish_results: the tail of convert_and_aggregate (float64, per-unit with zero-capacity
    buses, NaN -> 0 but inf kept, NaN-skipping time aggregation, (bus, time) layout) computed with torch
    ops -- what runs on the GPU for device results -- against the NumPy statement of the same lines."""
    import numpy as np
    import torch

    from atlite_b200 import convert

    rng = np.random.default_rng(0)
    res = rng.uniform(0, 5, (37, 11)).astype(np.float32)
    res[3, 2] = np.nan
    res[5, 4] = np.inf
    res[:, 7] = np.nan          # a bus that is NaN throughout: nanmean -> NaN, nansum -> 0
    caps = rng.uniform(1, 3, 11)
    caps[1] = 0.0               # zero capacity: x / NaN -> NaN -> 0
    for c in (None, caps):
        for agg in (None, "sum", "mean"):
            for bus_major in (False, True):
                want = convert._finish_results(res, c, agg, bus_major)
                got = convert._finish_results(torch.from_numpy(res), c, agg, bus_major)
                assert got.dtype == np.float64 and got.shape == want.shape and got.flags["C_CONTIGUOUS"]
                np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
                np.testing.assert_allclose(got, want, rtol=1e-15, atol=0)
    w = convert._finish_results(res, caps, None, True)
    assert w.shape == (11, 37) and w[1].tolist() == [0.0] * 37 and np.isinf(w[4, 5]) and w[2, 3] == 0.0


def test_layout_product_stores_what_the_sparse_product_stores():
    """convert.scale_columns is csr_matrix(matrix) * spdiag(layout) entry by entry: the same
    indptr, indices and data.  The sparse product stores no 0 -- neither a layout 0 nor a stored
    0 of the matrix (explicit, or duplicates that cancel) -- and a CSR reduce multiplies every
    stored entry, so a kept 0 on a NaN cell would turn its bus NaN."""
    import scipy.sparse as sp

    from atlite_b200.convert import scale_columns

    rng = np.random.default_rng(3)
    n_bus, S = 7, 60
    rows = list(rng.integers(0, n_bus, 150)) + [0, 1, 2, 2, 3, 3]
    cols = list(rng.integers(21, S, 150)) + [4, 9, 11, 11, 20, 20]
    vals = list(rng.uniform(-1, 2, 150)) + [0.0, 0.0, 0.7, -0.7, 0.25, 0.5]  # stored zeros, duplicates
    m = sp.csr_matrix((vals, (rows, cols)), shape=(n_bus, S))
    lay = rng.uniform(0, 3, S)
    lay[[1, 4, 20, 33, 59]] = 0.0  # layout zeros, on stored and on unstored cells
    lay[7] = np.nan
    assert (m.data == 0).sum() >= 3 and (lay[m.indices] == 0).any()
    snapshot = (m.indptr.copy(), m.indices.copy(), m.data.copy())
    want = sp.csr_matrix(m) * sp.diags(lay).tocsr()
    want.sort_indices()
    got = scale_columns(m, lay)
    assert got.has_sorted_indices
    np.testing.assert_array_equal(got.indptr, want.indptr)
    np.testing.assert_array_equal(got.indices, want.indices)
    np.testing.assert_array_equal(got.data, want.data)  # NaN layout entries included
    for a, b in zip((m.indptr, m.indices, m.data), snapshot):
        np.testing.assert_array_equal(a, b)  # the caller's matrix is left alone
    # a raw CSR with unsummed duplicates: the product sums them first
    raw = sp.csr_matrix((np.array([0.5, -0.5, 1.0]), np.array([3, 3, 5]), np.array([0, 3])), shape=(1, S))
    got = scale_columns(raw, np.ones(S))
    assert got.indices.tolist() == [5] and got.data.tolist() == [1.0]
    assert raw.nnz == 3
