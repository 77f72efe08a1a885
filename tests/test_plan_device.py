"""Aggregation plans built on the device, and aggregation matrices that live there.

Plan bytes: every array of a plan built by atl_plan_create_device (from device CSR) and by the
host-array entry points (which upload and call the same builder) is compared, as raw bytes, with
what the host tiling (atl_plan_tiling_host / atl_plan_pairs_host, the CPU reference) gives.  Raw
bytes make -0.0 and +0.0, and NaN payloads, count.  Errors: the host builder's codes and messages.
Results: CUDA sparse CSR, CUDA dense and scipy matrices give bitwise equal conversions under
ATL_DETERMINISTIC semantics (``set_deterministic``), capacities included.
"""

import ctypes as C
import warnings

import numpy as np
import pytest
import scipy.sparse as sp

import atlite_b200 as ab
from atlite_b200 import _lib, engine, synthetic as syn

pytestmark = pytest.mark.gpu

ARRAYS = _lib.PLAN_ARRAYS


# ------------------------------------------------------------------ the host reference


def _host_layout_perm(nx, pitch):
    """local index in the host tiling (lane layout of nx) -> local index in the layout of pitch."""
    vec_h, vec_t = nx % 4 == 0, pitch % 4 == 0
    perm = np.arange(128)
    if vec_h == vec_t:
        return perm
    for loc in range(128):
        if vec_h:
            ly, rest = divmod(loc, 32)
            lx = (rest // 4) * 4 + (rest & 3)
        else:
            lx, ly = divmod(loc, 4)
        perm[loc] = ((ly * 8 + lx // 4) * 4 + (lx & 3)) if vec_t else (lx * 4 + ly)
    return perm


def _stage(local):
    return 32 * (local & 3) + (local >> 2)


def _local(stage):
    return 4 * (stage & 31) + (stage >> 5)


def reference(indptr, indices, data, n_bus, ny, nx, pitch, entries):
    """name -> expected bytes of every plan array (b"" where the plan has none), and the info."""
    lib = _lib.load()
    args = (ny, nx, n_bus, _lib.ptr(indptr), _lib.ptr(indices), _lib.ptr(data))
    info = _lib.PlanInfo()
    _lib.check(lib.atl_plan_tiling_host(*args, C.byref(info), None, None, None, 0))
    ns = int(info.n_slots)
    tsp = np.zeros(info.n_tiles + 1, np.int32)
    row = np.zeros(max(ns, 1), np.int32)
    w = np.zeros(max(ns, 1) * 128, np.float32)
    _lib.check(lib.atl_plan_tiling_host(*args, C.byref(info), _lib.ptr(tsp), _lib.ptr(row), _lib.ptr(w), max(ns, 1)))
    row, w = row[:ns], w[: ns * 128].reshape(ns, 128)
    n = C.c_int64(0)
    _lib.check(lib.atl_plan_pairs_host(*args, C.byref(n), None, None, None, 0, 0))
    ptr = np.zeros(ns + 1, np.int32)
    cell = np.zeros(max(n.value, 1), np.int32)
    pw = np.zeros(max(n.value, 1), np.float32)
    _lib.check(lib.atl_plan_pairs_host(*args, C.byref(n), _lib.ptr(ptr), _lib.ptr(cell), _lib.ptr(pw), ns,
                                       max(n.value, 1)))
    # the host tiling lays weights out for pitch == nx; move them to the lane layout of `pitch`
    perm = _host_layout_perm(nx, pitch)
    wt = np.zeros_like(w)
    wt[:, perm] = w
    spt = perm[_local(cell[: n.value])]
    fused = bool(info.fused)
    out = {k: b"" for k in ARRAYS}
    if fused or entries:
        pairs, rec = [], np.zeros((ns, 2), np.int32)
        for s in range(ns):
            st = _stage(spt[ptr[s]:ptr[s + 1]])
            order = np.argsort(st, kind="stable")
            e = np.zeros((-(-len(st) // 8) * 8,), dtype=[("off", "<u4"), ("w", "<f4")])
            e["off"], e["w"] = 128 * 8, 0.0
            e["off"][: len(st)] = st[order] * 8
            e["w"][: len(st)] = pw[ptr[s]:ptr[s + 1]][order]
            rec[s] = (sum(len(p) for p in pairs), len(e) // 8)
            pairs.append(e)
        out.update(tile_slot_ptr=tsp.tobytes(), slot_row=row.tobytes(), slot_rec=rec.tobytes(),
                   pairs=b"".join(p.tobytes() for p in pairs),
                   active=np.flatnonzero(np.diff(tsp)).astype(np.int32).tobytes())
    if fused:
        out.update(slot_w4=np.concatenate([wt.ravel(), np.zeros(3 * 128, np.float32)]).tobytes(),
                   slot_ident=np.arange(ns, dtype=np.int32).tobytes(),
                   row_slot_ptr=np.concatenate([[0], np.cumsum(np.bincount(row, minlength=n_bus))]).astype(np.int32).tobytes(),
                   row_slots=np.argsort(row, kind="stable").astype(np.int32).tobytes())
    nnz = int(indptr[-1])
    out.update(indptr=indptr.tobytes(), indices=indices[:nnz].tobytes(), vals=data[:nnz].astype(np.float32).tobytes())
    return out, info


def export(handle):
    lib = _lib.load()
    out = {}
    for i, name in enumerate(ARRAYS):
        n = C.c_int64(0)
        _lib.check(lib.atl_plan_export(handle, i, None, 0, C.byref(n)))
        buf = np.zeros(n.value, np.uint8)
        _lib.check(lib.atl_plan_export(handle, i, _lib.ptr(buf), n.value, C.byref(n)))
        out[name] = buf.tobytes()
    return out


def _arrays(m):
    m = sp.csr_matrix(m)
    return (np.ascontiguousarray(m.indptr, np.int64), np.ascontiguousarray(m.indices, np.int32),
            np.ascontiguousarray(m.data, np.float64))


def build_device(indptr, indices, data, n_bus, ny, nx, pitch, entries):
    import torch

    lib = _lib.load()
    d = [torch.from_numpy(a).cuda() for a in (indptr, indices, data)]
    h = C.c_void_p()
    rc = lib.atl_plan_create_device(0, ny, nx, pitch, n_bus, len(data), *(C.c_void_p(t.data_ptr() or None) for t in d),
                                    int(entries), C.c_void_p(torch.cuda.current_stream().cuda_stream), C.byref(h))
    return rc, h


def build_host(indptr, indices, data, n_bus, ny, nx, pitch, entries):
    lib = _lib.load()
    create = lib.atl_plan_create_entries if entries else lib.atl_plan_create_pitched
    h = C.c_void_p()
    rc = create(0, ny, nx, pitch, n_bus, _lib.ptr(indptr), _lib.ptr(indices), _lib.ptr(data), C.byref(h))
    return rc, h


def check_plan(arrays, n_bus, ny, nx, pitch, entries, builders=(build_device, build_host)):
    lib = _lib.load()
    want, winfo = reference(*arrays, n_bus, ny, nx, pitch, entries)
    for build in builders:
        rc, h = build(*arrays, n_bus, ny, nx, pitch, entries)
        _lib.check(rc)
        try:
            got = export(h)
            info = _lib.PlanInfo()
            _lib.check(lib.atl_plan_info(h, C.byref(info)))
        finally:
            lib.atl_plan_destroy(h)
        what = f"{build.__name__} {ny}x{nx} pitch {pitch} entries={entries}"
        for name in ARRAYS:
            assert got[name] == want[name], f"{what}: {name} differs ({len(got[name])} vs {len(want[name])} bytes)"
        for f in ("n_tiles", "n_active_tiles", "n_slots", "fused", "nnz"):
            assert getattr(info, f) == getattr(winfo, f), (what, f)
        assert info.vec == (pitch % 4 == 0) and info.pitch == pitch
        assert info.n_pairs == (winfo.n_pairs if (winfo.fused or entries) else 0), what
    return winfo


# ------------------------------------------------------------------ plan bytes


def test_zoo_plans_are_the_host_plans():
    from test_reduce_semantics import NX, NY, zoo

    for name, m in zoo().items():
        for pitch in (NX, NX + 2):  # scalar and 128-bit lane layouts
            for entries in (False, True):
                info = check_plan(_arrays(m), m.shape[0], NY, NX, pitch, entries)
                assert info.fused == (name != "identity"), name


@pytest.mark.parametrize("ny,nx,pitch", [(11, 70, 70), (9, 70, 72), (7, 33, 40), (13, 64, 64), (5, 65, 67),
                                         (37, 261, 264), (4, 32, 32), (1, 1, 4)])
def test_random_plans_are_the_host_plans(ny, nx, pitch):
    rng = np.random.default_rng(ny * 1000 + nx)
    for n_bus, density in ((1, 0.9), (6, 0.2), (40, 0.05)):
        m = sp.random(n_bus, ny * nx, density=density, random_state=rng, format="csr",
                      data_rvs=lambda k: rng.uniform(-2, 2, k))
        for entries in (False, True):
            check_plan(_arrays(m), n_bus, ny, nx, pitch, entries)


def test_empty_matrix_plan():
    for n_bus in (0, 3):
        for entries in (False, True):
            info = check_plan(_arrays(sp.csr_matrix((n_bus, 9 * 70))), n_bus, 9, 70, 72, entries)
            assert info.n_slots == 0 and info.fused == 1


def test_layout_row_at_full_resolution():
    ny, nx = 720, 1440
    lay = syn.make_layout(nx, ny).reshape(-1)
    lay[np.random.default_rng(3).uniform(size=lay.size) < 0.3] = 0.0  # unstored cells
    m = sp.csr_matrix(lay[None, :])
    for pitch in (nx, nx + 4):
        check_plan(_arrays(m), 1, ny, nx, pitch, False)


def test_one_bus_per_cell_keeps_its_entries():
    ny, nx = 24, 70
    m = sp.identity(ny * nx, format="csr") * 0.5
    for pitch in (nx, 72):
        info = check_plan(_arrays(m), ny * nx, ny, nx, pitch, True)
        assert info.fused == 0


def test_weights_that_round_to_zero_subnormals_signed_zeros_and_nan():
    ny, nx = 9, 70
    S = ny * nx
    vals = np.array([0.0, -0.0, 1e-50, -1e-50, 1e-40, -3e-39, 1.4e-45, 7e-46, 1.0 + 2 ** -30, 1e39, -1e39,
                     np.nan, -np.nan, np.inf, -np.inf, 2.5, -0.75])
    vals[12] = np.frombuffer(np.uint64(0xFFF0000000000123).tobytes(), np.float64)[0]  # a signalling NaN
    rng = np.random.default_rng(4)
    cols = np.sort(rng.choice(S, len(vals), replace=False))
    m = sp.csr_matrix((vals, cols, [0, 6, 6, len(vals)]), shape=(3, S))
    assert m.has_canonical_format
    for pitch in (70, 72):
        for entries in (False, True):
            check_plan(_arrays(m), 3, ny, nx, pitch, entries)


def test_duplicates_through_the_host_entry_points_are_summed_as_before():
    """A raw CSR with shuffled columns and duplicates, the input build_tiling sums in CSR order."""
    rng = np.random.default_rng(5)
    ny, nx, nb = 37, 261, 9
    indptr, idx, dat = [0], [], []
    for r in range(nb):
        c = rng.integers(0, ny * nx, 400)
        c[::7] = c[0]  # the same cell many times
        idx += list(c)
        dat += list(rng.uniform(-1, 1, 400))
        indptr.append(len(idx))
    arrays = (np.array(indptr, np.int64), np.array(idx, np.int32), np.array(dat, np.float64))
    for pitch in (nx, 264):
        check_plan(arrays, nb, ny, nx, pitch, False)
        check_plan(arrays, nb, ny, nx, pitch, True)


def test_shapes_3000_at_full_resolution():
    ny, nx = 720, 1440
    m = syn.make_shapes(nx, ny, 3000)
    info = check_plan(_arrays(m), 3000, ny, nx, nx, False)
    assert info.fused == 1 and info.nnz == m.nnz


# ------------------------------------------------------------------ errors


@pytest.mark.parametrize("build", [build_device, build_host])
def test_bad_input_gives_the_host_builders_errors(build):
    lib = _lib.load()
    idx = np.array([1, 2, 3], np.int32)
    dat = np.ones(3)
    cases = [
        ((np.array([0, 2, 1, 3], np.int64), idx, dat, 3, 2, 4, 4), b"indptr not monotone"),
        ((np.array([0, 1, 3], np.int64), np.array([1, 8, 2], np.int32), dat, 2, 2, 4, 4), b"column index out of range"),
        ((np.array([0, 1, 3], np.int64), np.array([1, -1, 2], np.int32), dat, 2, 2, 4, 4), b"column index out of range"),
        ((np.array([0, 1, 3], np.int64), idx, dat, 2, 1 << 15, 1 << 14, 1 << 14), b"grid too large"),
    ]
    for (indptr, i, d, n_bus, ny, nx, pitch), msg in cases:
        rc, h = build(indptr, i, d, n_bus, ny, nx, pitch, False)
        assert rc == -1 and not h, msg
        assert msg in lib.atl_last_error()
        rc_host = lib.atl_plan_tiling_host(ny, nx, n_bus, _lib.ptr(indptr), _lib.ptr(i), _lib.ptr(d),
                                           C.byref(_lib.PlanInfo()), None, None, None, 0)
        assert rc_host == -1 and msg in lib.atl_last_error()


def test_non_canonical_sparse_tensors_are_refused():
    import torch

    S = 4 * 40
    crow = torch.tensor([0, 2, 3], device="cuda")
    for col in ([7, 5, 9], [5, 5, 9]):  # unsorted, duplicate
        m = torch.sparse_csr_tensor(crow, torch.tensor(col, device="cuda"), torch.ones(3, dtype=torch.float64,
                                    device="cuda"), (2, S))
        with pytest.raises(ValueError, match="to_sparse_coo"):
            engine.Plan(m, 4, 40)
    # the first entry of a row may be below the last of the previous one
    ok = torch.sparse_csr_tensor(crow, torch.tensor([5, 9, 1], device="cuda"), torch.ones(3, dtype=torch.float64,
                                 device="cuda"), (2, S))
    assert engine.Plan(ok, 4, 40).info["nnz"] == 3
    with pytest.raises(ValueError, match="columns"):
        engine.Plan(ok, 4, 41)


# ------------------------------------------------------------------ results

NX, NY, NT = 70, 45, 53


@pytest.fixture(scope="module")
def cutouts():
    ds = syn.make_dataset(NX, NY, NT, x0=-180.0, y0=-88.0, dx=360.0 / NX, dy=4.0, start="2013-03-18 05:00")
    heat = syn.make_dataset(NX, NY, 6 * 24, x0=-180.0, y0=-88.0, dx=360.0 / NX, dy=4.0, start="2013-03-01",
                            kinds=("temperature",))
    return {"main": ab.Cutout(data=ds), "main-device": ab.Cutout(data=ds).to_device(),
            "heat": ab.Cutout(data=heat).to_device()}


def _scaled_temperature(ds, scale):
    return ds.raw("temperature") * scale


CALLS = {
    "pv": ("main-device", lambda c, **kw: c.pv(panel="CSi", orientation="latitude_optimal", **kw)),
    "wind": ("main-device", lambda c, **kw: c.wind("Vestas_V112_3MW", **kw)),
    "heat": ("heat", lambda c, **kw: c.heat_demand(threshold=17.0, a=1.3, hour_shift=5.0, **kw)),
    "custom": ("main-device", lambda c, **kw: c.convert_and_aggregate(_scaled_temperature, scale=0.5, **kw)),
    "pv-host-cutout": ("main", lambda c, **kw: c.pv(panel="CSi", orientation="latitude_optimal", **kw)),
}


def _matrices():
    shapes = syn.make_shapes(NX, NY, 23)
    rng = np.random.default_rng(8)
    signed = shapes.copy()
    signed.data = signed.data * rng.uniform(-1.0, 1.0, signed.nnz)
    signed.data[::17] = 0.0  # stored zeros: kept by scipy and the CUDA CSR, dropped by a dense matrix
    return {"shapes": shapes, "signed": signed, "identity": sp.identity(NX * NY, format="csr")}


def _layout(cutout):
    lay = syn.make_layout(NX, NY)
    lay[::5, ::3] = 0.0
    return ab.DataArray(lay, {"y": cutout.data.coords["y"], "x": cutout.data.coords["x"]}, ("y", "x"))


def _bytes(r):
    if isinstance(r, tuple):
        return tuple(_bytes(x) for x in r)
    return np.ascontiguousarray(np.asarray(r.values)).tobytes(), tuple(r.dims), tuple(map(str, r.coords))


@pytest.fixture
def deterministic():
    prev = ab.set_deterministic(True)
    try:
        yield
    finally:
        ab.set_deterministic(prev)


@pytest.mark.parametrize("opts", ["plain", "layout", "per_unit", "capacity", "layout-per_unit-capacity", "sum"])
@pytest.mark.parametrize("call", list(CALLS))
def test_cuda_matrices_give_the_scipy_results(call, opts, cutouts, deterministic):
    import torch

    name, fn = CALLS[call]
    c = cutouts[name]
    kw = dict(aggregate_time="sum" if opts == "sum" else None)
    if "layout" in opts:
        kw["layout"] = _layout(c)
    if "per_unit" in opts:
        kw["per_unit"] = True
    if "capacity" in opts:
        kw["return_capacity"] = True
    mats = _matrices()
    for mname, m in mats.items():
        if mname == "identity" and call not in ("custom", "wind"):
            continue
        csr = torch.sparse_csr_tensor(torch.from_numpy(m.indptr.astype(np.int64)),
                                      torch.from_numpy(m.indices.astype(np.int64)),
                                      torch.from_numpy(m.data), m.shape).cuda()
        dense = torch.from_numpy(m.toarray()).cuda()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            want = _bytes(fn(c, matrix=m, **kw))
            want_dense = _bytes(fn(c, matrix=sp.csr_matrix(m.toarray()), **kw))
            got = _bytes(fn(c, matrix=csr, **kw))
            got_dense = _bytes(fn(c, matrix=dense, **kw))
        assert got == want, f"{call} {opts} {mname}: CUDA sparse CSR differs from scipy"
        assert got_dense == want_dense, f"{call} {opts} {mname}: CUDA dense differs from scipy"


def test_several_devices(deterministic):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ds = syn.make_dataset(NX, NY, NT, x0=-180.0, y0=-88.0, dx=360.0 / NX, dy=4.0, start="2013-03-18 05:00")
    many = ab.Cutout(data=ds, devices="all")
    m = _matrices()["shapes"]
    csr = torch.from_numpy(m.toarray()).cuda().to_sparse_csr()
    for kw in (dict(), dict(layout=_layout(many), per_unit=True, return_capacity=True)):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            want = _bytes(many.pv(panel="CSi", orientation="latitude_optimal", matrix=m, aggregate_time=None, **kw))
            got = _bytes(many.pv(panel="CSi", orientation="latitude_optimal", matrix=csr, aggregate_time=None, **kw))
        assert got == want
