"""CPU tests of the aggregation-plan tiling (atl_plan_tiling_host, no GPU): the
(tile, bus) slots with their 128-entry weight vectors must reproduce the CSR
matrix EXACTLY (float32 weights), for both lane layouts, ragged grids,
duplicates, explicit zeros and empty rows."""

import ctypes as C

import numpy as np
import scipy.sparse as sp
from hypothesis import given, settings, strategies as st

from atlite_b200 import _lib, synthetic as syn


def tiling(m, ny, nx):
    lib = _lib.load()
    m = sp.csr_matrix(m)
    indptr = np.ascontiguousarray(m.indptr, dtype=np.int64)
    idx = np.ascontiguousarray(m.indices, dtype=np.int32)
    dat = np.ascontiguousarray(m.data, dtype=np.float64)
    info = _lib.PlanInfo()
    _lib.check(lib.atl_plan_tiling_host(ny, nx, m.shape[0], _lib.ptr(indptr), _lib.ptr(idx), _lib.ptr(dat),
                                        C.byref(info), None, None, None, 0))
    ns = max(int(info.n_slots), 1)
    tsp = np.zeros(info.n_tiles + 1, dtype=np.int32)
    row = np.zeros(ns, dtype=np.int32)
    w = np.zeros(ns * 128, dtype=np.float32)
    _lib.check(lib.atl_plan_tiling_host(ny, nx, m.shape[0], _lib.ptr(indptr), _lib.ptr(idx), _lib.ptr(dat),
                                        C.byref(info), _lib.ptr(tsp), _lib.ptr(row), _lib.ptr(w), ns))
    return info, tsp, row[: info.n_slots], w[: info.n_slots * 128].reshape(-1, 128)


def dense_from_tiling(info, tsp, row, w, n_bus, ny, nx):
    """Invert the lane layout documented in include/atlite_b200.h."""
    vec = nx % 4 == 0
    n_tx = -(-nx // 32)
    out = np.zeros((n_bus, ny * nx), dtype=np.float64)
    for tile in range(info.n_tiles):
        ty, tx = divmod(tile, n_tx)
        for s in range(tsp[tile], tsp[tile + 1]):
            for ly in range(4):
                for lx in range(32):
                    iy, ix = ty * 4 + ly, tx * 32 + lx
                    loc = ((ly * 8 + lx // 4) * 4 + (lx & 3)) if vec else (lx * 4 + ly)
                    if iy < ny and ix < nx:
                        out[row[s], iy * nx + ix] += w[s, loc]
                    else:
                        assert w[s, loc] == 0.0, "weight on an out-of-grid cell"
    return out


@settings(max_examples=40, deadline=None)
@given(ny=st.integers(1, 11), nx=st.integers(1, 70), n_bus=st.integers(1, 6),
       density=st.floats(0.01, 0.6), seed=st.integers(0, 10_000))
def test_tiling_reproduces_csr(ny, nx, n_bus, density, seed):
    rng = np.random.default_rng(seed)
    S = ny * nx
    m = sp.random(n_bus, S, density=density, random_state=seed, format="csr",
                  data_rvs=lambda k: rng.uniform(-2, 2, k))
    info, tsp, row, w = tiling(m, ny, nx)
    want = np.asarray(m.astype(np.float32).todense(), dtype=np.float64)
    got = dense_from_tiling(info, tsp, row, w, n_bus, ny, nx)
    np.testing.assert_array_equal(got, want)
    assert info.nnz == m.nnz and tsp[-1] == info.n_slots
    assert (np.diff(tsp) >= 0).all()
    # slots of a tile are distinct buses in ascending order
    for t in range(info.n_tiles):
        r = row[tsp[t]:tsp[t + 1]]
        assert (np.diff(r) > 0).all()


def pair_lists(m, ny, nx, n_slots):
    lib = _lib.load()
    m = sp.csr_matrix(m)
    indptr = np.ascontiguousarray(m.indptr, dtype=np.int64)
    idx = np.ascontiguousarray(m.indices, dtype=np.int32)
    dat = np.ascontiguousarray(m.data, dtype=np.float64)
    n = C.c_int64(0)
    args = (ny, nx, m.shape[0], _lib.ptr(indptr), _lib.ptr(idx), _lib.ptr(dat))
    _lib.check(lib.atl_plan_pairs_host(*args, C.byref(n), None, None, None, 0, 0))
    ptr = np.zeros(n_slots + 1, dtype=np.int32)
    cell = np.zeros(max(n.value, 1), dtype=np.int32)
    w = np.zeros(max(n.value, 1), dtype=np.float32)
    _lib.check(lib.atl_plan_pairs_host(*args, C.byref(n), _lib.ptr(ptr), _lib.ptr(cell), _lib.ptr(w),
                                       n_slots, max(n.value, 1)))
    return n.value, ptr, cell[: n.value], w[: n.value]


def dense_from_pairs(info, tsp, row, ptr, cell, w, n_bus, ny, nx):
    """The staged reduce on paper: entry {c, w} of a slot of tile (ty, tx) multiplies the value
    the lane c % 32 parked as its (c // 32)-th cell (include/atlite_b200.h, atl_plan_pairs_host)."""
    vec = nx % 4 == 0
    n_tx = -(-nx // 32)
    out = np.zeros((n_bus, ny * nx), dtype=np.float64)
    for tile in range(info.n_tiles):
        ty, tx = divmod(tile, n_tx)
        for s in range(tsp[tile], tsp[tile + 1]):
            cs = cell[ptr[s]:ptr[s + 1]]
            assert (np.diff(cs) > 0).all(), "entries of a slot are sorted by staging index, no duplicates"
            for c, wt in zip(cs, w[ptr[s]:ptr[s + 1]]):
                lane, i = c % 32, c // 32
                ly, lx = (lane // 8, 4 * (lane % 8) + i) if vec else (i, lane)
                iy, ix = ty * 4 + ly, tx * 32 + lx
                assert iy < ny and ix < nx, "entry on an out-of-grid cell"
                out[row[s], iy * nx + ix] += wt
    return out


@settings(max_examples=40, deadline=None)
@given(ny=st.integers(1, 11), nx=st.integers(1, 70), n_bus=st.integers(1, 6),
       density=st.floats(0.01, 0.6), seed=st.integers(0, 10_000))
def test_pair_lists_reproduce_csr(ny, nx, n_bus, density, seed):
    """The entry lists the staged reduce kernel walks hold exactly the stored entries."""
    rng = np.random.default_rng(seed)
    m = sp.random(n_bus, ny * nx, density=density, random_state=seed, format="csr",
                  data_rvs=lambda k: rng.uniform(-2, 2, k))
    info, tsp, row, _ = tiling(m, ny, nx)
    n, ptr, cell, w = pair_lists(m, ny, nx, int(info.n_slots))
    assert n == m.nnz == info.n_pairs and ptr[-1] == n
    got = dense_from_pairs(info, tsp, row, ptr, cell, w, n_bus, ny, nx)
    np.testing.assert_array_equal(got, np.asarray(m.astype(np.float32).todense(), dtype=np.float64))


def test_pair_lists_keep_explicit_zeros_and_sum_duplicates():
    ny, nx = 6, 40
    S = ny * nx
    indptr = np.array([0, 2, 3, 3, 5], dtype=np.int64)  # raw CSR with a duplicate column and a stored 0.0
    idx = np.array([5, 5, 7, S - 1, S - 1], dtype=np.int32)
    dat = np.array([1.0, 2.0, 0.0, -3.0, 0.5])
    lib = _lib.load()
    n = C.c_int64(0)
    _lib.check(lib.atl_plan_pairs_host(ny, nx, 4, _lib.ptr(indptr), _lib.ptr(idx), _lib.ptr(dat), C.byref(n),
                                       None, None, None, 0, 0))
    assert n.value == 3  # (0,5) summed to 3.0, the stored zero (1,7) kept (scipy multiplies it), (3,S-1) summed
    ptr, cell, w = np.zeros(4, np.int32), np.zeros(3, np.int32), np.zeros(3, np.float32)
    _lib.check(lib.atl_plan_pairs_host(ny, nx, 4, _lib.ptr(indptr), _lib.ptr(idx), _lib.ptr(dat), C.byref(n),
                                       _lib.ptr(ptr), _lib.ptr(cell), _lib.ptr(w), 3, 3))
    assert sorted(w.tolist()) == [-2.5, 0.0, 3.0]


def test_duplicates_zeros_and_empty_rows():
    ny, nx = 6, 40
    S = ny * nx
    m = sp.csr_matrix((np.array([1.0, 2.0, 0.0, -3.0, 0.5]), (np.array([0, 0, 1, 3, 3]), np.array([5, 5, 7, S - 1, S - 1]))),
                      shape=(4, S))  # COO duplicates are summed by csr_matrix
    info, tsp, row, w = tiling(m, ny, nx)
    got = dense_from_tiling(info, tsp, row, w, 4, ny, nx)
    np.testing.assert_array_equal(got, np.asarray(m.todense()))
    assert got[0, 5] == 3.0 and got[3, S - 1] == -2.5 and not got[2].any()


def test_shape_like_matrices_fuse_and_identity_does_not():
    info, *_ = tiling(syn.make_shapes(200, 200, 100), 200, 200)
    assert info.fused == 1 and 2.0 < info.slots_per_active_tile < 5.0
    assert info.n_active_tiles == info.n_tiles == 7 * 50
    info, *_ = tiling(sp.identity(64 * 8, format="csr"), 8, 64)
    assert info.fused == 0  # one bus per cell: two-pass CSR path
    info, *_ = tiling(sp.csr_matrix((3, 64 * 8)), 8, 64)
    assert info.n_active_tiles == 0 and info.n_slots == 0
    # land mask: tiles without any entry are inactive (their inputs are never read)
    m = syn.make_shapes(128, 64, 10).tolil()
    m[:, : 64 * 128 // 2] = 0
    info, *_ = tiling(m.tocsr(), 64, 128)
    assert info.n_active_tiles == info.n_tiles // 2


def test_bad_input_is_rejected():
    lib = _lib.load()
    info = _lib.PlanInfo()
    indptr = np.array([0, 1], dtype=np.int64)
    idx = np.array([99], dtype=np.int32)
    dat = np.array([1.0])
    rc = lib.atl_plan_tiling_host(2, 4, 1, _lib.ptr(indptr), _lib.ptr(idx), _lib.ptr(dat), C.byref(info), None, None, None, 0)
    assert rc == -1 and b"out of range" in lib.atl_last_error()


def test_unsorted_columns_and_duplicates_take_the_general_ordering_path():
    """build_tiling orders a bus's entries of a tile by a 4-way de-interleave when the CSR row has
    ascending columns (scipy's canonical form) and by an insertion sort otherwise; a hand-made CSR
    with shuffled columns and duplicates must give the plan of its canonical form."""
    rng = np.random.default_rng(5)
    ny, nx, nb = 37, 261, 9
    rows, cols, vals = [], [], []
    for r in range(nb):
        c = rng.integers(0, ny * nx, 400)
        rows += [r] * 400
        cols += list(c)
        vals += list(rng.uniform(0, 1, 400))
    canonical = sp.csr_matrix((vals, (rows, cols)), shape=(nb, ny * nx))
    indptr, idx, dat = [0], [], []
    for r in range(nb):
        sel = [i for i, rr in enumerate(rows) if rr == r]
        rng.shuffle(sel)
        idx += [cols[i] for i in sel]
        dat += [vals[i] for i in sel]
        indptr.append(len(idx))
    raw = sp.csr_matrix((np.array(dat), np.array(idx, dtype=np.int32), np.array(indptr)), shape=(nb, ny * nx))
    assert not raw.has_sorted_indices
    info, tsp, row, w = tiling(raw, ny, nx)
    info_c, tsp_c, row_c, w_c = tiling(canonical, ny, nx)
    assert np.array_equal(tsp, tsp_c) and np.array_equal(row, row_c)
    np.testing.assert_allclose(w, w_c, rtol=0, atol=5e-7)  # duplicates summed in another order, in fp32
    np.testing.assert_allclose(dense_from_tiling(info, tsp, row, w, nb, ny, nx), canonical.toarray(), atol=5e-7)
    n_raw, n_can = len(row), len(row_c)
    assert n_raw == n_can
    p1, c1, w1 = pair_lists(raw, ny, nx, n_raw)[:3]
    p2, c2, w2 = pair_lists(canonical, ny, nx, n_can)[:3]
    assert np.array_equal(p1, p2) and np.array_equal(c1, c2)
    np.testing.assert_allclose(w1, w2, rtol=0, atol=5e-7)


def test_stored_zero_weights_are_negative_zero():
    """A stored entry whose float32 weight is 0 -- an explicit 0.0, duplicates that cancel, a
    float64 weight below float32's range -- is -0.0f in the slot's weight vector, every unstored
    cell +0.0f: the exact path multiplies stored entries only, as scipy does (0 * NaN = NaN)."""
    ny = 9
    for nx in (70, 72):  # scalar and 128-bit lane layouts
        S = ny * nx
        rng = np.random.default_rng(2)
        rows = list(rng.integers(0, 5, 300)) + [0, 1, 2, 2, 3, 4, 4]
        cols = list(rng.integers(0, S, 300)) + [3, 64, 100, 100, S - 1, 200, 200]
        vals = list(rng.uniform(-2.0, 2.0, 300)) + [0.0, -0.0, 0.7, -0.7, 1e-50, 0.25, -0.25]
        m = sp.csr_matrix((vals, (rows, cols)), shape=(5, S))  # duplicates summed, zero sums stored
        info, tsp, row, w = tiling(m, ny, nx)
        assert info.vec == (nx % 4 == 0)
        # sign bits mapped back onto (bus, cell); dense_from_tiling also checks that no
        # out-of-grid position of a weight vector carries one
        neg = dense_from_tiling(info, tsp, row, (np.signbit(w) & (w == 0)).astype(np.float32), 5, ny, nx)
        stored_zero = sp.csr_matrix(((m.data.astype(np.float32) == 0).astype(np.float64), m.indices, m.indptr),
                                    shape=m.shape).toarray()
        assert stored_zero.sum() == 5
        np.testing.assert_array_equal(neg, stored_zero)
        np.testing.assert_array_equal(dense_from_tiling(info, tsp, row, w, 5, ny, nx),
                                      np.asarray(m.astype(np.float32).todense(), dtype=np.float64))


def test_reduce_zoo_reaches_the_branches_it_names():
    """The matrices of tests/test_reduce_semantics.py hit what they claim: tiles with 1..9 and
    more than 24 slots, a last active tile with one slot, tiles of exactly 256 and of more than
    256 padded entries (heat's entry cache and its global-memory path), a fused plan for every
    matrix but `identity`."""
    from test_reduce_semantics import NX, NY, Z_FREE, Z_PAIR, Z_TINY, Z_ZERO, zoo

    mats = zoo()
    padded = {}
    for name, m in mats.items():
        info, tsp, row, w = tiling(m, NY, NX)
        assert info.fused == (name != "identity"), name
        if not info.fused:
            continue
        n, ptr, _, _ = pair_lists(m, NY, NX, int(info.n_slots))
        per_slot = -(-np.diff(ptr) // 8) * 8  # entries padded to PAIR_PAD
        padded[name] = np.add.reduceat(per_slot, tsp[:-1][np.diff(tsp) > 0]) if info.n_slots else np.array([])
        if name == "slot_ladder":
            counts = np.diff(tsp)
            assert set(range(1, 10)) <= set(counts.tolist()) and counts.max() > 24
            assert info.slots_per_active_tile <= 24.0
            active = np.flatnonzero(counts)
            assert counts[active[-1]] == 1 and active[-1] == info.n_tiles - 1
            assert (np.diff(np.concatenate([[0], m.indptr]))[1:] == 0).any()  # an empty bus
        if name == "land_mask":
            assert info.n_active_tiles == info.n_tiles // 2
            assert (np.diff(m.indptr) == 0).any()
    assert 256 in padded["entry_cap"].tolist() and padded["entry_cap"].max() > 256
    assert padded["dense_rows"].max() == 640  # 5 x 128 on every full tile
    assert padded["shapes"].max() <= 256  # the baseline is cached everywhere
    # the stored zeros really are stored, and their cells are stored nowhere else
    sz = mats["stored_zeros"].tocsc()
    for cell, bus in ((Z_ZERO, 3), (Z_PAIR, 5), (Z_TINY, 7)):
        col = sz.indices[sz.indptr[cell]:sz.indptr[cell + 1]]
        assert col.tolist() == [bus], (cell, col)
        assert np.float32(sz.data[sz.indptr[cell]]) == 0
    assert sz.indptr[Z_FREE + 1] == sz.indptr[Z_FREE]
