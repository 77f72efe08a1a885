"""Cutout.hydro: basin-routed inflow per plant.

CPU: the oracle (oracle/hydro_oracle.py) against the reference's own hydro path
(tests/golden/reference_hydro.npz), the host logic of atlite_b200/hydro.py against the reference's
walk and against exact point location and analytic equal-area areas, and the argument checks.
GPU: the shift-and-sum kernel against a NumPy ``np.roll`` sum, and ``Cutout.hydro`` end to end
against the oracle on host- and device-resident, prepared and raw ERA5 cutouts.
"""

import logging
import os
import sys
import types

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

import atlite_b200 as ab
import era5_runoff_height_oracle as ERH
import hydro_oracle as HO
from atlite_b200 import engine, gis, hydro, synthetic as syn

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "reference_hydro.npz")


def _golden():
    return np.load(GOLDEN)


def _split(ptr, flat):
    return [list(flat[ptr[i]:ptr[i + 1]]) for i in range(len(ptr) - 1)]


# --------------------------------------------------------------------------------------------
# CPU: the oracle against the reference's own functions
# --------------------------------------------------------------------------------------------


def test_oracle_walk_and_unique_basins_match_the_reference():
    g = _golden()
    ups, unique = HO.determine_basins(g["ids"], g["next_down"], g["plant_hids"])
    assert ups == _split(g["upstream_ptr"], g["upstream"])
    assert unique == list(g["unique"])


def test_oracle_matches_the_reference_hydro():
    g = _golden()
    pos = {b: i for i, b in enumerate(g["ids"])}
    ups, unique = HO.determine_basins(g["ids"], g["next_down"], g["plant_hids"])
    m = HO.normalise(g["rows"][[pos[b] for b in unique]])
    np.testing.assert_allclose(m, g["normalised"], rtol=1e-14, atol=0)
    assert np.count_nonzero(m) == int(g["normalised_nnz"])
    R = m @ g["cells"].T
    dist = {b: g["dist_main"][pos[b]] for b in g["ids"]}
    for k, fs in enumerate(g["flowspeeds"]):
        scaled = {b: R[i] * g["area"][pos[b]] for i, b in enumerate(unique)}
        got = HO.shift_and_aggregate(ups, list(g["plant_hids"]), dist, scaled, fs)
        want = g[f"inflow_{k}"]
        np.testing.assert_allclose(got, want, rtol=1e-9, atol=0)


def test_golden_tree_has_the_cases_it_claims():
    g = _golden()
    pos = {b: i for i, b in enumerate(g["ids"])}
    ups = _split(g["upstream_ptr"], g["upstream"])
    shifts = [HO.travel_steps(g["dist_main"][pos[b]] - g["dist_main"][pos[h]], 1.0)
              for u, h in zip(ups, g["plant_hids"]) for b in u]
    T = len(g["time_ns"])
    assert min(shifts) < 0 and max(shifts) >= T
    assert set(ups[0]) < set(ups[2]) and set(ups[1]) < set(ups[2])  # a plant downstream of two others
    assert not set(g["ids"]) <= set(g["unique"])  # a basin no plant drains
    assert (g["normalised"][list(g["unique"]).index(133)] == 0).all()  # the off-grid basin


# --------------------------------------------------------------------------------------------
# CPU: host logic of atlite_b200/hydro.py
# --------------------------------------------------------------------------------------------


def _golden_frame(g):
    return pd.DataFrame({"HYBAS_ID": g["ids"], "DIST_MAIN": g["dist_main"], "NEXT_DOWN": g["next_down"]})


def test_upstream_walk_matches_the_reference():
    g = _golden()
    f = _golden_frame(g)
    idx = pd.Index(f["HYBAS_ID"])
    roots = idx.get_indexer(g["plant_hids"])
    ptr, up = hydro.upstream_basins(idx.get_indexer(f["NEXT_DOWN"]), roots)
    np.testing.assert_array_equal(ptr, g["upstream_ptr"])
    np.testing.assert_array_equal(g["ids"][up], g["upstream"])


def test_route_on_the_golden_tree():
    """determine_basins with point location: one unit square per basin on a row, plants at centres."""
    g = _golden()
    f = _golden_frame(g)
    f["geometry"] = [np.array([[i, 0.0], [i + 1, 0.0], [i + 1, 1.0], [i, 1.0]]) for i in range(len(f))]
    col = {b: i for i, b in enumerate(g["ids"])}
    plants = pd.DataFrame({"lon": [col[h] + 0.5 for h in g["plant_hids"]], "lat": 0.5},
                          index=pd.Index(g["plant_names"], name="name"))
    r = hydro.route(plants, f)
    b = r.basins
    assert list(b.plants["hid"]) == list(g["plant_hids"])
    assert [list(u) for u in b.plants["upstream"]] == _split(g["upstream_ptr"], g["upstream"])
    assert list(b.shapes.index) == list(g["unique"]) and b.shapes.index.name == "hid"
    assert list(b.meta.index) == list(g["unique"]) and "geometry" not in b.meta.columns
    np.testing.assert_array_equal(b.meta.index.to_numpy()[r.rows], g["upstream"])
    np.testing.assert_array_equal(r.ptr, g["upstream_ptr"])
    assert list(hydro.determine_basins(plants, f).shapes.index) == list(g["unique"])


def test_travel_steps_truncate_toward_zero():
    d = np.array([-18.0, -1.9, 0.0, 1.7, 1.8, 259.9, 260.0, 1e4])
    got = hydro.travel_steps(d, 0.0, 1.0)
    want = np.array([int(v / 3.6 + 0.5) for v in d])
    np.testing.assert_array_equal(got, want)
    assert got[0] == -4 and got[1] == 0
    np.testing.assert_array_equal(hydro.travel_steps(d + 5.0, 5.0, 0.3), [int(v / (0.3 * 3.6) + 0.5) for v in d])
    with pytest.raises(ValueError):
        hydro.travel_steps(np.array([np.nan]), 0.0, 1.0)


def test_upstream_cycle_is_an_error():
    with pytest.raises(ValueError, match="cycle"):
        hydro.upstream_basins(np.array([1, 2, 0]), np.array([0]))


def test_normalised_matrix_stores_no_zeros():
    g = _golden()
    pos = {b: i for i, b in enumerate(g["ids"])}
    rows = g["rows"][[pos[b] for b in g["unique"]]]
    m = hydro.normalise_rows(sp.csr_matrix(rows))
    np.testing.assert_allclose(m.toarray(), g["normalised"], rtol=1e-14, atol=0)
    assert m.nnz == int(g["normalised_nnz"])
    # explicitly stored zeros, an all-zero row (a basin off the grid) and duplicates
    a = sp.csr_matrix((np.array([0.0, 0.5, 0.0, 0.25, 0.25, 0.0]), np.array([0, 1, 2, 3, 3, 0]),
                       np.array([0, 2, 3, 5, 6])), shape=(4, 5))
    m = hydro.normalise_rows(a)
    assert (m.data != 0).all() and m.nnz == 2
    np.testing.assert_array_equal(m.toarray(), [[0, 1, 0, 0, 0], [0] * 5, [0, 0, 0, 1, 0], [0] * 5])
    assert a.nnz == 6  # the argument is left as it was


# point location: shapely ``intersects`` semantics against exact rational arithmetic

_SQUARE_WITH_HOLE = {"type": "Polygon", "coordinates": [[[0, 0], [4, 0], [4, 4], [0, 4], [0, 0]],
                                                        [[1, 1], [1, 3], [3, 3], [3, 1], [1, 1]]]}
_MULTI = {"type": "MultiPolygon", "coordinates": [[[[10, 0], [12, 0], [11, 2]]],
                                                  [[[13, 0.1], [15.3, 0.1], [15.3, 0.7], [13, 0.7]]]]}
_SKEW = np.array([[20.1, 0.3], [23.7, 0.1], [22.9, 3.3], [20.3, 2.9]])  # no dyadic coordinates


def _locate(shapes, pts):
    f = pd.DataFrame({"HYBAS_ID": np.arange(len(shapes)) + 1, "DIST_MAIN": 0.0, "NEXT_DOWN": 0,
                      "geometry": shapes}).set_index("HYBAS_ID")
    plants = pd.DataFrame({"lon": [p[0] for p in pts], "lat": [p[1] for p in pts]},
                          index=[f"p{i}" for i in range(len(pts))])
    return hydro.find_basins(plants, f["geometry"])


@pytest.mark.parametrize("pt, inside", [
    ((2.0, 0.5), True),    # interior
    ((4.0, 2.5), True),    # on an exterior edge
    ((4.0, 4.0), True),    # on a vertex
    ((2.0, 2.0), False),   # in the hole
    ((1.0, 2.0), True),    # on the hole's boundary
    ((3.0, 3.0), True),    # on a hole vertex
    ((2.0, 4.0 + 1e-12), False),
])
def test_point_in_polygon_with_hole(pt, inside):
    parts = gis.geometry_parts(_SQUARE_WITH_HOLE, polygonal=True)
    assert bool(HO.find_basin([parts], *pt)) is inside
    shapes = [_SQUARE_WITH_HOLE, {"type": "Polygon", "coordinates": [[[-9, -9], [9, -9], [9, 9], [-9, 9]]]}]
    assert _locate(shapes, [pt])[0] == (0 if inside else 1)


def test_point_location_matches_exact_arithmetic():
    shapes = [_SQUARE_WITH_HOLE, _MULTI, _SKEW]
    parts = [gis.geometry_parts(s, polygonal=True) for s in shapes]
    rng = np.random.default_rng(3)
    pts = [tuple(p) for p in np.c_[rng.uniform(-1, 24, 400), rng.uniform(-1, 5, 400)]]
    # points on edges and vertices, also where the coordinates are not dyadic
    for _, ring in [p for ps in parts for p in ps]:
        for a, b in zip(ring, np.roll(ring, -1, axis=0)):
            pts += [tuple(a), tuple((a + b) / 2), tuple(a + (b - a) / 3)]
    pts += [(14.0, 0.1), (15.3, 0.4), (11.0, 2.0), (13.0, 0.7 + 1e-15)]
    want = [(HO.find_basin(parts, *p) or [-1])[0] for p in pts]
    outside = np.array(want) < 0
    got = np.full(len(pts), -1)
    inside_pts = [p for p, o in zip(pts, outside) if not o]
    got[~outside] = _locate(shapes, inside_pts)
    np.testing.assert_array_equal(got, want)
    assert (~outside).sum() > 100 and outside.sum() > 50
    for p in [p for p, o in zip(pts, outside) if o][:20]:
        with pytest.raises(IndexError):
            _locate(shapes, [p])


def test_several_basins_warn_and_take_the_first(caplog):
    a = np.array([[0.0, 0.0], [2.0, 0.0], [2.0, 2.0], [0.0, 2.0]])
    shapes = [np.array([[5.0, 5.0], [6.0, 5.0], [6.0, 6.0]]), a + 1.0, a]
    with caplog.at_level(logging.WARNING, logger="atlite_b200.hydro"):
        assert list(_locate(shapes, [(1.5, 1.5)])) == [1]
    assert "is in several basins" in caplog.text and "Assuming the first one" in caplog.text


def test_no_basin_is_an_index_error_naming_the_plant():
    with pytest.raises(IndexError, match="p0"):
        _locate([_SKEW], [(0.0, 0.0)])


# areas: ellipsoidal cylindrical equal-area (GRS80) then planar


def test_cea_area_of_a_lonlat_rectangle_and_of_the_globe():
    a = hydro.GRS80_A
    rect = np.array([[5.0, 40.0], [12.5, 40.0], [12.5, 47.25], [5.0, 47.25]])
    want = a * a * np.radians(7.5) * (hydro.authalic_q(47.25) - hydro.authalic_q(40.0)) / 2
    np.testing.assert_allclose(hydro.basin_areas([rect]), [want], rtol=1e-12)
    np.testing.assert_allclose(HO.cea_area(gis.geometry_parts(rect, polygonal=True)), want, rtol=1e-12)
    globe = np.array([[-180.0, -90.0], [180.0, -90.0], [180.0, 90.0], [-180.0, 90.0]])
    np.testing.assert_allclose(hydro.basin_areas([globe]), [5.10066e14], rtol=1e-6)
    # the authalic sphere of GRS80 (radius 6371007.181 m) has the same area
    np.testing.assert_allclose(hydro.basin_areas([globe]), [4 * np.pi * 6371007.181 ** 2], rtol=1e-9)


def test_cea_area_subtracts_holes_and_sums_parts():
    outer = [[0.0, 0.0], [4.0, 0.0], [4.0, 4.0], [0.0, 4.0], [0.0, 0.0]]
    hole = [[1.0, 1.0], [1.0, 3.0], [3.0, 3.0], [3.0, 1.0], [1.0, 1.0]]
    full, cut = hydro.basin_areas([{"type": "Polygon", "coordinates": [outer]},
                                   {"type": "Polygon", "coordinates": [outer, hole]}])
    inner = hydro.basin_areas([{"type": "Polygon", "coordinates": [hole]}])[0]
    np.testing.assert_allclose(cut, full - inner, rtol=1e-12)
    multi = hydro.basin_areas([_MULTI])[0]
    parts = hydro.basin_areas([{"type": "Polygon", "coordinates": c} for c in _MULTI["coordinates"]])
    np.testing.assert_allclose(multi, parts.sum(), rtol=1e-12)


def test_cea_area_matches_the_oracle_on_voronoi_basins():
    x, y = syn.make_coords(20, 12, 5.0, 44.0)
    f = syn.make_basins(x, y, 25, seed=4)
    got = hydro.basin_areas(f["geometry"])
    want = [HO.cea_area(gis.geometry_parts(gm, polygonal=True)) for gm in f["geometry"]]
    np.testing.assert_allclose(got, want, rtol=1e-10)


def test_make_basins_is_one_tree_partly_off_the_grid():
    x, y = syn.make_coords(20, 12, 5.0, 44.0)
    f = syn.make_basins(x, y, 30, seed=2)
    ids = pd.Index(f["HYBAS_ID"])
    assert ids.is_unique and not ids.is_monotonic_increasing
    nd = ids.get_indexer(f["NEXT_DOWN"])
    assert (nd < 0).sum() == 1
    ptr, up = hydro.upstream_basins(nd, np.flatnonzero(nd < 0))
    assert sorted(up) == list(range(len(f)))  # every basin drains to the outlet
    assert (f["DIST_MAIN"].to_numpy()[nd >= 0] > f["DIST_MAIN"].to_numpy()[nd[nd >= 0]]).all()
    xr_, yr_ = x[-1] + 0.125, y[-1] + 0.125  # the grid's north-east corner
    west = np.array([min(r[0] for r in gm["coordinates"][0]) for gm in f["geometry"]])
    south = np.array([min(r[1] for r in gm["coordinates"][0]) for gm in f["geometry"]])
    east = np.array([max(r[0] for r in gm["coordinates"][0]) for gm in f["geometry"]])
    assert ((west >= xr_) | (south >= yr_)).any()  # wholly off the grid
    assert ((west < xr_) & (east > xr_)).any()  # partly
    hit = hydro.find_basins(f.rename(columns={"site_lon": "lon", "site_lat": "lat"}).set_index("HYBAS_ID"),
                            f.set_index("HYBAS_ID")["geometry"])
    np.testing.assert_array_equal(hit, np.arange(len(f)))  # each site lies in its own basin


# argument checks


def test_hydrobasins_missing_column_and_wrong_type():
    f = pd.DataFrame({"HYBAS_ID": [1], "NEXT_DOWN": [0], "geometry": [_SKEW]})
    with pytest.raises(AssertionError, match=r"Couldn't find the column\(s\) DIST_MAIN in the hydrobasins dataset"):
        hydro.read_hydrobasins(f)
    with pytest.raises(AssertionError, match="hydrobasins should be passed as a filename or a GeoDataFrame"):
        hydro.read_hydrobasins([1, 2])


def test_hydrobasins_path_without_geopandas(monkeypatch, tmp_path):
    monkeypatch.setitem(sys.modules, "geopandas", None)  # import geopandas -> ImportError
    for p in (str(tmp_path / "basins.shp"), tmp_path / "basins.shp"):
        with pytest.raises(ImportError, match="geopandas"):
            hydro.read_hydrobasins(p)


def test_hydro_is_bound_to_the_cutout():
    assert ab.Cutout.hydro is ab.convert.hydro
    assert hydro.__name__ == "atlite_b200.hydro"  # the module, as atlite.hydro is


def test_hydro_on_a_time_sharded_cutout_is_not_implemented():
    cut = types.SimpleNamespace(time_shard=object())
    with pytest.raises(NotImplementedError, match="time-sharded"):
        ab.convert.hydro(cut, pd.DataFrame({"lon": [0.0], "lat": [0.0]}), pd.DataFrame())


# --------------------------------------------------------------------------------------------
# GPU: the shift-and-sum kernel
# --------------------------------------------------------------------------------------------


def _roll_sum(R, ptr, rows, shifts, w):
    out = np.zeros((len(ptr) - 1, R.shape[1]))
    for p in range(len(ptr) - 1):
        for e in range(ptr[p], ptr[p + 1]):
            out[p] += np.roll(R[rows[e]] * w[e], shifts[e])
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("T", [700, 256, 1])
def test_kernel_matches_a_numpy_roll_sum(T):
    rng = np.random.default_rng(T)
    B, P = 37, 23
    R = rng.exponential(1.0, (B, T)) * 1e-3
    counts = rng.integers(0, 40, P)
    counts[3] = 0  # a plant without entries
    ptr = np.concatenate([[0], np.cumsum(counts)])
    n = int(ptr[-1])
    rows = rng.integers(0, B, n)
    shifts = rng.integers(-3 * T - 5, 3 * T + 5, n)  # negative and >= T
    shifts[:4] = [0, T, -T, 2 * T + 1]
    w = rng.uniform(1e8, 5e9, n)
    got = engine.hydro_shift_sum(R, ptr, rows, shifts, w).cpu().numpy()
    again = engine.hydro_shift_sum(R, ptr, rows, shifts, w).cpu().numpy()
    want = _roll_sum(R, ptr, rows, shifts, w)
    assert got.shape == (P, T) and got.dtype == np.float64
    assert np.array_equal(got, again)  # bitwise repeatable
    assert np.array_equal(got[3], np.zeros(T))
    # the same products and sums in the same order: equal to the NumPy sum, not just close
    np.testing.assert_array_equal(got, want)


@pytest.mark.gpu
def test_kernel_rejects_rows_outside_the_runoff():
    with pytest.raises(ValueError, match="rows"):
        engine.hydro_shift_sum(np.zeros((2, 5)), [0, 1], [2], [0], [1.0])


# --------------------------------------------------------------------------------------------
# GPU: Cutout.hydro end to end against the oracle
# --------------------------------------------------------------------------------------------


NX, NY, NT = 24, 16, 60


def _case():
    x, y = syn.make_coords(NX, NY, 5.0, 44.0)
    f = syn.make_basins(x, y, 40, seed=5)
    nd = pd.Index(f["HYBAS_ID"]).get_indexer(f["NEXT_DOWN"])
    # a leaf basin with NaN runoff under it: no plant may drain it, so none sits on its way down
    children = np.bincount(nd[nd >= 0], minlength=len(f))
    ancestors = {}
    for b in range(len(f)):
        a, k = [], b
        while nd[k] >= 0:
            k = nd[k]
            a.append(k)
        ancestors[b] = a
    on_grid = (f["site_lon"] < x[-1]) & (f["site_lat"] < y[-1])
    leaf = int(next(b for b in np.argsort(-f["DIST_MAIN"].to_numpy()) if children[b] == 0 and on_grid[b]))
    banned = set(ancestors[leaf]) | {leaf}
    # plants: the busiest basins that are not banned (nested ones among them), plus one leaf
    sizes = np.array([sum(b in ancestors[c] or b == c for c in range(len(f))) for b in range(len(f))])
    pick = [b for b in np.argsort(-sizes, kind="stable") if b not in banned and on_grid[b]][:7]
    plants = pd.DataFrame({"lon": f["site_lon"].to_numpy()[pick], "lat": f["site_lat"].to_numpy()[pick]},
                          index=pd.Index([f"plant{i}" for i in range(len(pick))], name="name"))
    # inconsistent: further from the outlet than any basin, so its upstream basins get negative shifts
    f.loc[f.index[pick[2]], "DIST_MAIN"] = f["DIST_MAIN"].max() + 100.0
    return x, y, f, plants, leaf


def _fields(x, y, leaf_ring):
    rng = np.random.default_rng(9)
    ro = rng.exponential(2e-4, (NT, NY, NX)).astype(np.float32)
    ro[:, 0, :3] = -1e-5  # clipped at 0 on a raw cutout
    height = rng.uniform(0.0, 2000.0, (NY, NX)).astype(np.float32)
    # NaN in the cells wholly inside the leaf basin no plant drains
    full = gis.compute_indicatormatrix(x, y, [leaf_ring]).toarray()[0].reshape(NY, NX) > 1 - 1e-9
    assert full.any()
    ro[:, full] = np.nan
    return ro, height


def _cutouts(raw):
    x, y, f, plants, leaf = _case()
    ro, height = _fields(x, y, f["geometry"].iloc[leaf])
    co = dict(time=syn.make_time(NT), x=x, y=y, lon=x, lat=y)
    if raw:
        z = np.broadcast_to(height * np.float32(9.80665), (NT, NY, NX)).astype(np.float32)
        ds = ab.Dataset({"ro": (("time", "y", "x"), ro), "z": (("time", "y", "x"), z)}, coords=co)
        od = dict(runoff=ERH.get_data_runoff(ro)["runoff"], height=ERH.get_data_height(z[0])["height"])
    else:
        ds = ab.Dataset({"runoff": (("time", "y", "x"), ro), "height": (("y", "x"), height)}, coords=co)
        od = dict(runoff=ro, height=height)
    od.update(time=co["time"], lon=x, lat=y)
    return ds, od, x, y, f, plants


def _oracle(od, x, y, f, plants, **kw):
    table = dict(HYBAS_ID=list(f["HYBAS_ID"]), NEXT_DOWN=list(f["NEXT_DOWN"]), DIST_MAIN=list(f["DIST_MAIN"]),
                 parts=[gis.geometry_parts(g, polygonal=True) for g in f["geometry"]])
    return HO.hydro(od, x, y, plants[["lon", "lat"]].to_numpy(), table, **kw)


def _check(got, want, info, plants, time):
    assert got.dims == ("plant", "time")
    assert list(got.indexes["plant"]) == list(plants.index)
    np.testing.assert_array_equal(np.asarray(got.indexes["time"]), np.asarray(time))
    v = np.asarray(got.values)
    assert v.dtype == np.float64 and np.isfinite(v).all()
    up_area = np.array([sum(info["area"][info["unique"].index(b)] for b in u) for u in info["ups"]])
    err = np.abs(v - want)
    tol = 1e-4 * np.abs(want) + 1e-6 * up_area[:, None]
    assert (err <= tol).all(), f"max err / tol {np.max(err / tol):.3g}"


@pytest.mark.gpu
@pytest.mark.parametrize("raw", [False, True], ids=["prepared", "raw"])
@pytest.mark.parametrize("residency", ["host", "device"])
def test_cutout_hydro_matches_the_oracle(raw, residency):
    ds, od, x, y, f, plants = _cutouts(raw)
    cut = ab.Cutout(data=ds)
    if residency == "device":
        cut = cut.to_device()
    for wh, fs in ((False, 1), (True, 0.7)):
        with pytest.warns(FutureWarning, match="aggregate_time='legacy'"):
            got = cut.hydro(plants, f, flowspeed=fs, weight_with_height=wh)
        want, info = _oracle(od, x, y, f, plants, flowspeed=fs, weight_with_height=wh)
        shifts = [HO.travel_steps(f["DIST_MAIN"][f["HYBAS_ID"] == b].item() - f["DIST_MAIN"][f["HYBAS_ID"] == h].item(), fs)
                  for u, h in zip(info["ups"], info["plant_hids"]) for b in u]
        assert min(shifts) < 0 and max(shifts) >= NT
        assert any(set(u) < set(v) for u in info["ups"] for v in info["ups"])  # nested plants
        _check(got, want, info, plants, od["time"])


@pytest.mark.gpu
def test_cutout_hydro_passes_smoothing_and_quantile_cut_to_runoff():
    ds, od, x, y, f, plants = _cutouts(False)
    got = ab.Cutout(data=ds).hydro(plants, f, smooth=5, lower_threshold_quantile=0.1, aggregate_time=None)

    def post(R):
        roll = pd.DataFrame(R).rolling(5, min_periods=1).mean().values
        thr = pd.Series(roll.T.ravel()).quantile(0.1)
        return np.where(roll >= thr, roll, 0.0)

    want, info = _oracle(od, x, y, f, plants, post=post)
    _check(got, want, info, plants, od["time"])
