"""The PV sun gate: kernels that compute the solar position in-kernel skip the input loads of
lane-steps (and whole warp batches) whose cells all have the sun below the altitude threshold,
where the result is exactly 0 whatever the inputs hold.  Checked against the float64 oracle on a
global grid (polar rows, the terminator crossing inside lanes and tiles) at a solstice and an
equinox, with NaN / Inf planted in sun-down cells next to lit ones and in lit cells, through the
fused reduce, the per-cell cube and the per-cell time mean, for both lane layouts.
"""

import warnings

import numpy as np
import pytest
import scipy.sparse as sp
from conftest import assert_parity, oracle_ds

import atlite_oracle as O
import atlite_b200 as ab
from atlite_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

NX, NY = 70, 45  # 360 deg x 176 deg: 5.14 deg columns (4 per 128-bit lane), 4 deg rows up to 88 deg
THR = np.radians(1.0)  # the default altitude threshold
# (start, steps): odd lengths, not a multiple of the 16-step time blocks; lit runs of every length
DAYS = [("2013-06-21 00:00", 41), ("2013-03-20 03:00", 37)]
CASES = [  # PvPhys MODE 1, 4 (Bofinger), 4 (tracking + Hay-Davies), 0 (outflux albedo)
    ("era5", dict(panel="CSi", orientation="latitude_optimal")),
    ("era5", dict(panel="KANENA", orientation="latitude_optimal")),
    ("era5", dict(panel="CSi", orientation={"slope": 25.0, "azimuth": 200.0}, tracking="horizontal",
                  trigon_model="other")),
    ("outflux", dict(panel="CSi", orientation="latitude_optimal")),
]


def _dataset(start, nt, kind):
    ds = syn.make_dataset(NX, NY, nt, x0=-180.0, y0=-88.0, dx=360.0 / NX, dy=4.0, start=start, kinds=("pv",),
                          extra=("outflux",) if kind == "outflux" else ())
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        alt = O.solar_position(oracle_ds(ds))["altitude"]
    rng = np.random.default_rng(5)
    names = sorted(ds.keys())
    dark = alt < THR - 0.01
    lit = alt > THR + 0.01
    # sun-down cells whose neighbour in x or in y is lit at the same step
    edge = np.zeros_like(dark)
    edge[:, :, :-1] |= dark[:, :, :-1] & lit[:, :, 1:]
    edge[:, :, 1:] |= dark[:, :, 1:] & lit[:, :, :-1]
    edge[:, :-1, :] |= dark[:, :-1, :] & lit[:, 1:, :]
    edge[:, 1:, :] |= dark[:, 1:, :] & lit[:, :-1, :]
    e_idx = np.argwhere(edge)
    for k, (t, y, x) in enumerate(e_idx[rng.choice(len(e_idx), 60, replace=False)]):
        ds.raw(names[k % len(names)])[t, y, x] = (np.nan, np.inf, -np.inf)[k % 3]
    l_idx = np.argwhere(lit)
    for k, (t, y, x) in enumerate(l_idx[rng.choice(len(l_idx), 8, replace=False)]):
        ds.raw(names[k % len(names)])[t, y, x] = np.nan
    t, y, x = l_idx[rng.choice(len(l_idx))]
    ds.raw("influx_direct")[t, y, x] = np.inf  # clipped to influx_toa: a finite result
    near = np.abs(alt - THR) < 1e-3  # float32 vs float64 solar position may decide either way here
    return ds, dark, edge, near


@pytest.fixture(scope="module")
def shapes():
    return syn.make_shapes(NX, NY, 17)


@pytest.mark.parametrize("start,nt", DAYS, ids=["solstice", "equinox"])
@pytest.mark.parametrize("kind,case", CASES, ids=["mode1", "mode4-bofinger", "mode4-tracking", "mode0-outflux"])
def test_sun_gate_matches_the_oracle_with_exact_zeros(shapes, start, nt, kind, case):
    ds, dark, edge, near = _dataset(start, nt, kind)
    assert dark.any() and (~dark).any() and edge.sum() >= 60
    od = oracle_ds(ds)
    pv_kw = dict(case)
    case = dict(case)
    panel = ab.get_solarpanelconfig(case.pop("panel"))
    orient = O.get_orientation(case.pop("orientation"))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        cube = O.convert_pv(od, panel, orient, **case)  # (time, y, x)
        mean = np.nanmean(cube, axis=0)
    # (NaN in a lit cell reaches the result only with the Hay-Davies model: the simple one and the
    # panel models fill it with 0 -- on the GPU both go through the exact path)
    assert (cube[dark] == 0).all(), "the oracle masks every sun-down cell to 0"
    flat = cube.reshape(nt, -1)
    want = (shapes @ flat.T).T  # scipy: NaN only where a stored entry meets it
    pattern = sp.csr_matrix((np.ones(shapes.nnz), shapes.indices, shapes.indptr), shape=shapes.shape)
    near_bus = (pattern @ near.reshape(nt, -1).T).T > 0
    cap = np.asarray(shapes.sum(-1)).flatten()
    for c in (ab.Cutout(data=ds), ab.Cutout(data=ds).to_device()):  # scalar lanes / padded 128-bit lanes
        got = np.asarray(c.pv(matrix=shapes, aggregate_time=None, **pv_kw).values).T
        assert_parity(got, want, cap, what=f"sun gate reduce {kind} {case}")
        z = (want == 0) & ~near_bus
        assert z.any() and (got[z] == 0).all(), "oracle-zero bus sums must be exactly zero"
        gc = np.asarray(c.pv(aggregate_time=None, **pv_kw).values)
        assert_parity(gc, cube, what=f"sun gate cells {kind} {case}")
        assert (gc[dark] == 0).all(), "sun-down cells must be exactly zero whatever their inputs"
        gm = np.asarray(c.pv(aggregate_time="mean", **pv_kw).values)
        assert_parity(gm, mean, what=f"sun gate mean {kind} {case}")
        night = dark.all(0)  # polar night: every step dark, inputs with NaN / Inf included
        assert (gm[night] == 0).all()
