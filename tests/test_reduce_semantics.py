"""Every shape-reduce path against scipy's sparse product.

The per-cell values of every operator are reduced into buses by the aggregation matrix; the
reference does this with a scipy CSR product, which multiplies every STORED entry (a stored 0 on a
NaN cell gives NaN) and never an unstored one.  Here that step has several implementations, and
which one runs depends on the operator, the lane layout, the plan and the deterministic switch:
the shuffle reduce (4 slots x 2 steps per butterfly, with or without the first slot group's
weights in registers), the per-step reduce of odd batches and time-block tails, the cold exact
path, heat's staged reduce (tile entries cached in shared memory or read from global memory), the
two-pass fallback (per-cell cube, then a CSR gather) and the deterministic per-slot partials.

This module runs a conformance grid -- operator x matrix x lane layout x deterministic switch --
against the float64 oracle on a 70 x 45 global cutout (3 x 12 tiles, a 6-wide last tile column
and a 1-tall last tile row).  The matrix zoo (`zoo()`) aims each matrix at a branch of those
paths; tests/test_plan_tiling.py checks on the CPU that the zoo still reaches them.  NaNs are
planted where the physics lets them reach the per-cell result, on cells stored with weight 0,
stored by two buses, or not stored at all.
"""

import warnings

import numpy as np
import pytest
import scipy.sparse as sp
from conftest import assert_parity, oracle_ds

import atlite_oracle as O
import era5_oracle as EO
import atlite_b200 as ab
from atlite_b200 import _lib, convert, engine, synthetic as syn

pytestmark = pytest.mark.gpu

NX, NY = 70, 45  # 3 x 12 tiles of 32 x 4: last tile column 6 cells wide, last tile row 1 cell tall
S = NX * NY
NT = 53  # per-step operators: three 16-step time blocks and a short fourth one
START = "2013-03-18 05:00"
HEAT_STEPS, HOUR_SHIFT = 18 * 24, 5.0  # 19 day bins, partial first and last: 8-day chunks 8, 8, 3
SUN_THRESHOLDS = np.radians([0.0, 1.0, 3.75])  # altitude tests of the PV gate and of CSP's DNI


def tile_cells(ty, tx):
    return np.array([y * NX + x for y in range(4 * ty, min(4 * ty + 4, NY))
                     for x in range(32 * tx, min(32 * tx + 32, NX))])


def _shapes():
    return syn.make_shapes(NX, NY, 23)


def _shared_cell(m):
    """A cell that two buses store (a region border of the Voronoi shapes)."""
    counts = np.diff(m.tocsc().indptr)
    return int(np.flatnonzero(counts == 2)[40])


# Cells that carry NaN in some steps.  The first four are special in the `stored_zeros` matrix:
Z_ZERO = 13 * NX + 40   # stored only as an explicit 0.0 of bus 3
Z_PAIR = 21 * NX + 10   # stored only as a +0.7 / -0.7 duplicate pair of bus 5 (sums to a stored 0)
Z_TINY = 30 * NX + 50   # stored only with weight 1e-50 (bus 7), which is 0 in float32
Z_FREE = 6 * NX + 66    # stored by no bus
Z_SHARED = _shared_cell(_shapes())  # stored by two buses
# ... and more NaN cells in the tiles the slot ladder fills (1, 2, 3 slots, the 32-slot tile, the
# 6-wide tile column and the polar last row)
NAN_CELLS = [Z_ZERO, Z_PAIR, Z_TINY, Z_FREE, Z_SHARED,
             2 * NX + 5, 1 * NX + 40, 3 * NX + 66, 22 * NX + 45, 44 * NX + 67]


def _csr(rows, cols, vals, n_bus):
    """COO -> CSR as scipy does it: duplicates summed, a sum of 0 stays a stored entry."""
    return sp.csr_matrix((np.asarray(vals, dtype=np.float64), (np.asarray(rows), np.asarray(cols))),
                         shape=(n_bus, S))


def zoo():
    """name -> (n_bus, ny*nx) float64 CSR matrix; each one aims at a branch of the reduce."""
    rng = np.random.default_rng(11)
    shapes = _shapes()
    mats = {"shapes": shapes}

    # slot_ladder: tiles 0..8 with exactly 1..9 slots (bus i % k for the i-th cell of the tile), tile
    # 16 with 32 (more than heat's SLOT_CAP; the plan still fuses: 78 slots over 11 tiles), and the
    # LAST active tile with 1 slot: the grouped reduce reads the 3 zero slots behind the plan's end.
    # Bus 0 has a slot in every active tile, buses 9..31 only in tile 16, bus 32 none.
    rows, cols = [], []
    for k, tile in zip(range(1, 10), range(9)):
        c = tile_cells(*divmod(tile, 3))
        rows += list(np.arange(len(c)) % k)
        cols += list(c)
    c = tile_cells(*divmod(16, 3))
    rows += list(np.arange(len(c)) % 32)
    cols += list(c)
    c = tile_cells(*divmod(35, 3))
    rows += [0] * len(c)
    cols += list(c)
    mats["slot_ladder"] = _csr(rows, cols, rng.uniform(0.2, 1.0, len(rows)), 33)

    # entry_cap: tile 4 = 2 buses over all 128 cells = 256 padded entries (heat caches the tile);
    # tile 13 = 3 buses over 128 + 128 + 1 cells = 264 padded entries (heat reads global memory).
    # Bus 5 covers every other cell.
    rows, cols = [], []
    t4, t13 = tile_cells(1, 1), tile_cells(4, 1)
    for b, c in ((0, t4), (1, t4), (2, t13), (3, t13), (4, t13[:1])):
        rows += [b] * len(c)
        cols += list(c)
    rest = np.setdiff1d(np.arange(S), np.concatenate([t4, t13]))
    rows += [5] * len(rest)
    cols += list(rest)
    mats["entry_cap"] = _csr(rows, cols, rng.uniform(0.2, 1.0, len(rows)), 6)

    # dense_rows: 5 buses over every cell (640 entries per tile)
    mats["dense_rows"] = sp.csr_matrix(rng.uniform(0.0, 1.0, (5, S)))

    # land_mask: the shapes on every other tile only (the rest inactive), plus an empty bus 10
    ty, tx = np.divmod(np.arange(S), NX)
    keep = ((ty // 4) * 3 + tx // 32) % 2 == 0
    m = shapes.multiply(keep[None, :].astype(np.float64)).tocsr()
    m.eliminate_zeros()
    mats["land_mask"] = sp.vstack([m[:10], sp.csr_matrix((1, S)), m[10:]]).tocsr()

    # signed: every entry w of 12 shapes has a partner -u*w on the next cell of the row (bus sums
    # cancel to about 0), and a third of the entries come as two COO halves (duplicates)
    base = syn.make_shapes(NX, NY, 12).tocoo()
    r, c, w = base.row, base.col, base.data
    nxt = (c % NX) < NX - 1
    u = rng.uniform(0.9, 1.1, nxt.sum())
    half = rng.uniform(size=len(w)) < 1 / 3
    rows = np.concatenate([r[~half], r[half], r[half], r[nxt]])
    cols = np.concatenate([c[~half], c[half], c[half], c[nxt] + 1])
    vals = np.concatenate([w[~half], w[half] / 2, w[half] / 2, -u * w[nxt]])
    mats["signed"] = _csr(rows, cols, vals, 12)

    # stored_zeros: the shapes without Z_ZERO / Z_PAIR / Z_TINY / Z_FREE, plus an explicit 0.0, a
    # +w / -w duplicate pair and a 1e-50 weight on three of them (Z_SHARED keeps its two buses)
    coo = shapes.tocoo()
    drop = np.isin(coo.col, [Z_ZERO, Z_PAIR, Z_TINY, Z_FREE])
    rows = list(coo.row[~drop]) + [3, 5, 5, 7]
    cols = list(coo.col[~drop]) + [Z_ZERO, Z_PAIR, Z_PAIR, Z_TINY]
    vals = list(coo.data[~drop]) + [0.0, 0.7, -0.7, 1e-50]
    mats["stored_zeros"] = _csr(rows, cols, vals, 23)

    # identity: one bus per cell -- every operator takes the two-pass path
    mats["identity"] = sp.identity(S, format="csr")
    return mats


def layout_values():
    """A layout that is 0 exactly on the NaN cells (as real layouts are 0 over the sea)."""
    lay = syn.make_layout(NX, NY)
    lay.reshape(-1)[NAN_CELLS] = 0.0
    return lay


# (matrix, layout?, per_unit?) cases of the grid
CASES = [(name, False, False) for name in ("shapes", "slot_ladder", "entry_cap", "dense_rows", "land_mask",
                                           "signed", "stored_zeros", "identity")]
CASES += [(name, True, pu) for name in ("shapes", "identity") for pu in (False, True)]
CASE_IDS = [n + ("-layout" if lay else "") + ("-per_unit" if pu else "") for n, lay, pu in CASES]


# ------------------------------------------------------------------ datasets


def _raw_era5(ds):
    """Raw ERA5 variables that derive back to the prepared fields of `ds`: accumulated J m-2
    irradiation and wind components along a seeded azimuth.  The 10 m components follow a seeded
    shear exponent in 0.05 .. 0.4, not the dataset's own `wnd_shear_exp` (the main dataset has none;
    the oracle derives every field from the raw ones)."""
    rng = np.random.default_rng(17)
    f = {k: np.asarray(ds.raw(k), dtype=np.float64) for k in ds.keys()}
    ssrd = (f["influx_direct"] + f["influx_diffuse"]) * 3600.0
    az = rng.uniform(0.0, 2.0 * np.pi, ssrd.shape)
    alpha = rng.uniform(0.05, 0.4, ssrd.shape)
    w100, w10 = f["wnd100m"], f["wnd100m"] * 0.1 ** alpha
    az10 = az + rng.uniform(-0.3, 0.3, ssrd.shape)
    raw = dict(ssrd=ssrd, fdir=f["influx_direct"] * 3600.0, ssr=ssrd * (1.0 - f["albedo"]),
               tisr=f["influx_toa"] * 3600.0, t2m=f["temperature"], u100=w100 * np.sin(az), v100=w100 * np.cos(az),
               u10=w10 * np.sin(az10), v10=w10 * np.cos(az10), fsr=f["roughness"])
    return ab.Dataset({k: (("time", "y", "x"), v.astype(np.float32)) for k, v in raw.items()},
                      coords=dict(ds.coords))


def _step_dataset(kind):
    """53 hourly steps from a March start, longitudes -180..180: the terminator crosses tiles, so
    sun-gated batches are skipped in some tiles and run in others.  Every input field is NaN at the
    3 steps of highest solar altitude of each NaN cell (lit cells: NaN reaches the PV result under
    Hay-Davies; wind, temperature and the custom function propagate it at any step).  `raw` holds
    raw ERA5 variables instead, whose solar position is taken at -30 min (ERA5's accumulations)."""
    extra = {"outflux": ("outflux",), "soil": ("soil temperature",)}.get(kind, ())
    kinds = ("pv",) if kind == "outflux" else ("pv", "wind", "temperature")
    ds = syn.make_dataset(NX, NY, NT, x0=-180.0, y0=-88.0, dx=360.0 / NX, dy=4.0, start=START,
                          kinds=kinds, extra=extra)
    if kind == "soil":  # the sea is exactly the NaN cells (all steps)
        st = ds.raw("soil temperature")
        st[...] = np.where(np.isnan(st), ds.raw("temperature") - 5.0, st)
    if kind == "raw":
        ds = _raw_era5(ds)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        alt = O.solar_position(oracle_ds(ds), time_shift="-30min" if kind == "raw" else "0h")["altitude"]
    alt = np.broadcast_to(alt, (NT, NY, NX))
    for cell in NAN_CELLS:
        y, x = divmod(cell, NX)
        steps = np.argsort(alt[:, y, x])[-3:]
        for name in ds.keys():
            ds.raw(name)[steps, y, x] = np.nan
    if kind == "soil":
        ds.raw("soil temperature")[:, np.array(NAN_CELLS) // NX, np.array(NAN_CELLS) % NX] = np.nan
    if kind in ("stored", "stored64"):  # the oracle's solar position in float32 (PV MODE 3) or float64
        with warnings.catch_warnings():  # (MODE 2, what era5.prepare stores); neither has a sun gate
            warnings.simplefilter("ignore")
            sp_ = O.solar_position(oracle_ds(ds))
        dt = np.float32 if kind == "stored" else np.float64
        ds["solar_altitude"] = np.broadcast_to(sp_["altitude"], (NT, NY, NX)).astype(dt)
        ds["solar_azimuth"] = np.broadcast_to(sp_["azimuth"], (NT, NY, NX)).astype(dt)
    near = np.zeros((NT, NY, NX), bool)  # float32 vs float64 solar position may decide either way
    for thr in SUN_THRESHOLDS:
        near |= np.abs(alt - thr) < 1e-3
    return ds, near


def _oracle_raw_ds(ds):
    """The oracle's view of a raw ERA5 dataset: EO.get_data_* of its fields and the solar position
    at -30 min, as era5.prepare would store them."""
    d = oracle_ds(ds)
    ow = EO.get_data_wind(d["u100"], d["v100"], d["u10"], d["v10"], d["fsr"])
    oi = EO.get_data_influx(d["ssrd"], d["ssr"], d["tisr"], d["fdir"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sol = O.solar_position(d, time_shift="-30min")
    od = {k: d[k] for k in ("time", "lon", "lat")}
    od.update(solar_altitude=np.broadcast_to(sol["altitude"], (NT, NY, NX)),
              solar_azimuth=np.broadcast_to(sol["azimuth"], (NT, NY, NX)), temperature=d["t2m"])
    od.update({k: ow[k] for k in ("wnd100m", "roughness", "wnd_shear_exp")})
    od.update({k: oi[k] for k in ("influx_toa", "influx_direct", "influx_diffuse", "albedo")})
    return od


def _heat_dataset():
    """18 days of hours, binned by (time + 5 h): 19 day bins, the first and the last partial.  Each
    NaN cell is NaN for a whole day (its daily mean is NaN), for the partial last day, and at one
    step of another day (skipped by the daily mean)."""
    ds = syn.make_dataset(NX, NY, HEAT_STEPS, x0=-180.0, y0=-88.0, dx=360.0 / NX, dy=4.0,
                          start="2013-03-01 00:00", kinds=("temperature",))
    _, gid = O.day_bins(ds.coords["time"], HOUR_SHIFT)
    assert gid[-1] == 18 and (gid == 0).sum() == 19 and (gid == 18).sum() == 5
    t = ds.raw("temperature")
    for k, cell in enumerate(NAN_CELLS):
        y, x = divmod(cell, NX)
        t[gid == 3 + k, y, x] = np.nan
        t[gid == 18, y, x] = np.nan
        t[np.flatnonzero(gid == 14)[k], y, x] = np.nan
    return ds, None


def _convert_scaled_temperature(ds, scale):
    return ds.raw("temperature") * scale  # a NumPy array, or a (row-padded) CUDA tensor of a device cutout


def _oracle_scaled_temperature(ds, scale):
    return np.asarray(ds["temperature"], dtype=np.float64) * scale


_CURVE = dict(V=[0.0, 1.0, 1.0001, 3.0, 3.0, 7.5, 12.0, 25.0, 25.0],  # knots too close for a LUT
              POW=[0.0, 0.0, 0.1, 0.4, 0.5, 1.5, 2.0, 2.0, 0.0], P=2.0, hub_height=80)
_HEAT = dict(threshold=17.0, a=1.3, constant=0.2, hour_shift=HOUR_SHIFT)
_COOL = dict(threshold=-5.0, a=1.7, constant=0.3, hour_shift=HOUR_SHIFT)
_PV1 = dict(panel="CSi", orientation="latitude_optimal")
_PV4 = dict(panel="CSi", orientation={"slope": 25.0, "azimuth": 200.0}, tracking="horizontal", trigon_model="other")


def _pv_oracle(case):
    case = dict(case)
    return O.convert_pv, dict(panel=ab.get_solarpanelconfig(case.pop("panel")),
                              orientation=O.get_orientation(case.pop("orientation")), **case)


# name -> (dataset, call(cutout, **kw), (oracle function, its keywords), value scale, additive, unit).
# `unit` (conftest.assert_parity) is the magnitude of the float32 quantities whose difference is ONE
# cell's value: the daily mean of ~290 K temperatures times `a` for heat and cooling, slope * speed
# of the 500 / (m/s) segment between the 1.0 and 1.0001 m/s knots for the binary-search curve.  It
# matters where a bus is one cell (identity, with or without a layout); for bus sums it is negligible.
OPS = {
    "pv-mode1": ("main", lambda c, **kw: c.pv(**_PV1, **kw), _pv_oracle(_PV1), 1.0, False, 1.0),
    "pv-mode4": ("main", lambda c, **kw: c.pv(**_PV4, **kw), _pv_oracle(_PV4), 1.0, False, 1.0),
    "pv-mode0-outflux": ("outflux", lambda c, **kw: c.pv(**_PV1, **kw), _pv_oracle(_PV1), 1.0, False, 1.0),
    "pv-mode3-stored": ("stored", lambda c, **kw: c.pv(**_PV1, **kw), _pv_oracle(_PV1), 1.0, False, 1.0),
    "pv-mode5-raw": ("raw", lambda c, **kw: c.pv(**_PV1, **kw), _pv_oracle(_PV1), 1.0, False, 1.0),
    "pv-mode6-raw": ("raw", lambda c, **kw: c.pv(**_PV4, **kw), _pv_oracle(_PV4), 1.0, False, 1.0),
    "pv-mode2-stored-f64": ("stored64", lambda c, **kw: c.pv(**_PV1, **kw), _pv_oracle(_PV1), 1.0, False, 1.0),
    "wind": ("main", lambda c, **kw: c.wind("Vestas_V112_3MW", **kw),
             (O.convert_wind, dict(turbine=ab.get_windturbineconfig("Vestas_V112_3MW"))), 1.0, False, 1.0),
    "wind-bsearch": ("main", lambda c, **kw: c.wind(dict(_CURVE), **kw),
                     (O.convert_wind, dict(turbine=ab.get_windturbineconfig(dict(_CURVE)))), 1.0, False, 500.0),
    "wind-raw-log": ("raw", lambda c, **kw: c.wind("Vestas_V112_3MW", **kw),
                     (O.convert_wind, dict(turbine=ab.get_windturbineconfig("Vestas_V112_3MW"))), 1.0, False, 1.0),
    "wind-raw-power": ("raw", lambda c, **kw: c.wind("Vestas_V112_3MW", interpolation_method="power", **kw),
                       (O.convert_wind, dict(turbine=ab.get_windturbineconfig("Vestas_V112_3MW"),
                                             interpolation_method="power")), 1.0, False, 1.0),
    "wind-raw-bsearch": ("raw", lambda c, **kw: c.wind(dict(_CURVE), **kw),
                         (O.convert_wind, dict(turbine=ab.get_windturbineconfig(dict(_CURVE)))), 1.0, False, 500.0),
    "heat": ("heat", lambda c, **kw: c.heat_demand(**_HEAT, **kw), (O.convert_heat_demand, _HEAT), 50.0, False,
             300.0 * _HEAT["a"]),
    "cooling": ("heat", lambda c, **kw: c.cooling_demand(**_COOL, **kw), (O.convert_cooling_demand, _COOL),
                50.0, False, 300.0 * _COOL["a"]),
    "soil": ("soil", lambda c, **kw: c.soil_temperature(**kw), (O.convert_soil_temperature, {}), 300.0, True, 1.0),
    # soil_temperature fills NaN with 0; temperature lets NaN reach the pointwise reduce
    "temperature": ("main", lambda c, **kw: c.temperature(**kw), (O.convert_temperature, {}), 300.0, True, 1.0),
    "csp": ("main", lambda c, **kw: c.csp("SAM_solar_tower", **kw),
            (O.convert_csp, dict(installation=ab.get_cspinstallationconfig("SAM_solar_tower"))), 1.0, False, 1.0),
    "spmm-custom": ("main", lambda c, **kw: c.convert_and_aggregate(_convert_scaled_temperature, scale=0.5, **kw),
                    (_oracle_scaled_temperature, dict(scale=0.5)), 300.0, False, 1.0),
}
SUN_OPS = {"pv-mode1", "pv-mode4", "pv-mode0-outflux", "pv-mode3-stored", "csp", "pv-mode5-raw", "pv-mode6-raw",
           "pv-mode2-stored-f64"}
LAYOUTS = ["host", "device-scalar", "device-vec"]


@pytest.fixture(scope="module")
def data():
    """dataset name -> (oracle dict, near-threshold cube, {lane layout: Cutout}); built lazily."""
    made = {}

    def get(name):
        if name not in made:
            ds, near = _heat_dataset() if name == "heat" else _step_dataset(name)
            host = ab.Cutout(data=ds)
            padded = host.to_device()
            for n in padded.data.data_vars:
                assert padded.data.raw(n).shape[-1] == 72
                padded.data.raw(n)[..., NX:] = float("nan")
            od = _oracle_raw_ds(ds) if name == "raw" else oracle_ds(ds)
            made[name] = (od, near, {"host": host, "device-scalar": host.to_device(pad=False), "device-vec": padded})
        return made[name]

    return get


@pytest.fixture(scope="module")
def cubes(data):
    """operator -> float64 oracle cube (time, ny, nx), computed once per operator."""
    made = {}

    def get(op):
        if op not in made:
            fn, kw = OPS[op][2]
            with warnings.catch_warnings(), np.errstate(all="ignore"):
                warnings.simplefilter("ignore")
                r = fn(data(OPS[op][0])[0], **kw)
            made[op] = np.asarray(r[0] if isinstance(r, tuple) else r, dtype=np.float64)
        return made[op]

    return get


@pytest.fixture(scope="module")
def mats():
    return zoo()


@pytest.fixture
def deterministic():
    prev = ab.set_deterministic(True)
    try:
        yield
    finally:
        ab.set_deterministic(prev)


def _layout_da(ds_coords):
    return ab.DataArray(layout_values(), {"y": ds_coords["y"], "x": ds_coords["x"]}, ("y", "x"))


def _time_bus(res):
    v = np.asarray(res.values)
    return v if res.dims[0] == "time" else v.T


def _expected(op, case, data, cubes, mats):
    """(want (time, bus), capacity for the parity bar, the matrix the values were reduced with)."""
    name, lay, pu = case
    od, _, _ = data(OPS[op][0])
    m = mats[name]
    scale = OPS[op][3]
    if not lay:
        cube = cubes(op)
        want = np.asarray((m @ cube.reshape(cube.shape[0], -1).T).T)  # O.aggregate_matrix
        return want, np.asarray(abs(m).sum(-1)).flatten() * scale, m
    fn, kw = OPS[op][2]
    lv = layout_values()
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore")
        want = O.convert_and_aggregate(od, fn, matrix=m, layout=lv, per_unit=pu, aggregate_time=None, **kw)
    ml = sp.csr_matrix(m) * sp.diags(lv.reshape(-1)).tocsr()
    cap = 1.0 if pu else np.asarray(abs(ml).sum(-1)).flatten() * scale
    return want, cap, ml


def _call(op, case, cutout, mats):
    name, lay, pu = case
    kw = dict(matrix=mats[name], aggregate_time=None)
    if lay:
        kw.update(layout=_layout_da(cutout.data.coords), per_unit=pu)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return _time_bus(OPS[op][1](cutout, **kw))


def _check(op, case, got, want, cap, m, near, what):
    additive = OPS[op][4] or case[0] == "signed"
    # two ulps of the largest single-cell contribution to each bus: unit x the bus's largest weight
    # (divided by its capacity for per-unit results)
    wmax = abs(m).max(axis=1).toarray().ravel()
    if case[2]:
        rowsum = np.asarray(m.sum(-1)).ravel()
        wmax = np.divide(wmax, rowsum, out=np.zeros_like(wmax), where=rowsum != 0)
    assert_parity(got, want, cap, what=what, additive=additive, unit=OPS[op][5] * wmax)
    # exact zeros where the oracle is exactly 0, unless a stored entry meets a cell whose sun
    # altitude is within float32 reach of a threshold
    z = want == 0
    if near is not None and op in SUN_OPS:
        pattern = sp.csr_matrix((np.ones(m.nnz), m.indices, m.indptr), shape=m.shape)
        z &= ~((pattern @ near.reshape(near.shape[0], -1).T).T > 0)
    assert (got[z] == 0).all(), f"{what}: {int((got[z] != 0).sum())} oracle-zero bus sums are not exactly 0"


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
@pytest.mark.parametrize("op", list(OPS))
def test_reduce_matches_scipy(op, case, data, cubes, mats):
    want, cap, m = _expected(op, case, data, cubes, mats)
    _, near, cutouts = data(OPS[op][0])
    for lname in LAYOUTS:
        got = _call(op, case, cutouts[lname], mats)
        _check(op, case, got, want, cap, m, near, f"{op} {'-'.join(map(str, case))} {lname}")


@pytest.mark.parametrize("case", [c for c in CASES if c[0] != "identity"],
                         ids=[i for i, c in zip(CASE_IDS, CASES) if c[0] != "identity"])
@pytest.mark.parametrize("op", list(OPS))
def test_deterministic_reduce_is_repeatable_and_matches_scipy(op, case, data, cubes, mats, deterministic):
    """Per-slot partials and a fixed-order gather (heat's det_acc, k_gather_slots on buses with
    0, 1 and many slots): bitwise repeatable, on the parity bar, and equal to the atomics run."""
    want, cap, m = _expected(op, case, data, cubes, mats)
    _, near, cutouts = data(OPS[op][0])
    for lname in LAYOUTS:
        what = f"{op} {'-'.join(map(str, case))} {lname} deterministic"
        a = _call(op, case, cutouts[lname], mats)
        b = _call(op, case, cutouts[lname], mats)
        assert a.dtype == b.dtype and a.tobytes() == b.tobytes(), f"{what}: two runs differ"
        _check(op, case, a, want, cap, m, near, what)
        ab.set_deterministic(False)
        try:
            free = _call(op, case, cutouts[lname], mats)
        finally:
            ab.set_deterministic(True)
        np.testing.assert_allclose(a, free, rtol=2e-5, atol=2e-5 * np.nanmax(np.abs(free), initial=0.0),
                                   err_msg=what)


def test_zoo_plans_fuse_and_walk_several_time_blocks(mats):
    """The per-step grid runs several 16-step time blocks per tile and a short last one (batch
    loop and per-step tail), by pick_tb's rule in kernels.cuh; identity takes the two-pass path."""
    import torch

    sm = torch.cuda.get_device_properties(0).multi_processor_count
    for name, m in mats.items():
        info = engine.get_plan(m, NY, NX).info
        assert info["fused"] == (name != "identity"), name
        if not info["fused"]:
            continue
        gx = -(-info["n_active_tiles"] // 4)
        tb = min(max(-(-NT * gx // (sm * 5 * 24)), 16), 128)
        tb = min(tb + (tb & 1), NT)
        assert tb == 16 and NT % tb and NT // tb >= 3, (name, tb)


class _Recorder:
    """Stands in for an engine operator: records what the spec asks for."""

    def __init__(self, **kw):
        self.kw = kw


@pytest.mark.parametrize("op", ["pv-mode5-raw", "pv-mode6-raw", "pv-mode2-stored-f64"])
def test_pv_operators_take_the_branch_they_name(op, monkeypatch):
    """Raw ERA5 fields with the solar position computed at -30 min, or a stored float64 solar position."""
    monkeypatch.setattr(convert.engine, "PvOp", _Recorder)
    ds, _ = _step_dataset(OPS[op][0])
    case = dict(_PV1 if op != "pv-mode6-raw" else _PV4)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        spec = convert._PvSpec(ds, ab.get_solarpanelconfig(case.pop("panel")), ab.get_orientation(case.pop("orientation")),
                               **case)
    kw = spec.op.kw
    if op == "pv-mode2-stored-f64":
        assert kw["irr_branch"] == _lib.IRR_DIRECT_DIFFUSE and kw["solar_src"] == _lib.SOLAR_STORED_F64
        assert ds.raw("solar_altitude").dtype == np.float64
    else:
        assert kw["irr_branch"] == _lib.IRR_ERA5_RAW and kw["solar_src"] == _lib.SOLAR_COMPUTED
        assert kw["time_shift"] == "-30min"
        for slot, var in dict(influx="ssrd", outflux="ssr", influx_toa="tisr", influx_direct="fdir",
                              temperature="t2m").items():
            assert spec.fields[slot] is ds.raw(var), slot


@pytest.mark.parametrize("op,method,fields", [("wind-raw-log", _lib.WIND_LOG, {"u100", "v100", "fsr"}),
                                              ("wind-raw-power", _lib.WIND_POWER, {"u100", "v100", "u10", "v10"}),
                                              ("wind-raw-bsearch", _lib.WIND_LOG, {"u100", "v100", "fsr"})])
def test_wind_operators_read_the_raw_fields(op, method, fields, monkeypatch):
    monkeypatch.setattr(convert.engine, "WindOp", _Recorder)
    ds, _ = _step_dataset("raw")
    turb = dict(_CURVE) if op == "wind-raw-bsearch" else "Vestas_V112_3MW"
    spec = convert._WindSpec(ds, ab.get_windturbineconfig(turb), "power" if op == "wind-raw-power" else "logarithmic")
    assert spec.op.kw["method"] == method and set(spec.raw) == fields
    if op == "wind-raw-bsearch":  # knots too close for any table: LMODE 0, the binary search
        from test_wind_curve import curve_info

        t = ab.get_windturbineconfig(dict(_CURVE))
        assert curve_info(t["V"], np.asarray(t["POW"]) / t["P"])["table"] == 0
