"""Synthetic ERA5-shaped cutouts and NUTS-like shape matrices (SURVEY.md section 8d).

Used by tests, ``bench.py`` and ``__graft_entry__.smoke``; there is no network
and no real cutout in the build environment.  Variable names, units and dtypes
follow the reference's ERA5 schema (datasets/era5.py:47-60): float32
``(time, y, x)`` fields on a regular lon/lat grid, hourly UTC time axis.

Fields (seed per variable, independent of how the time axis is chunked):
  influx_toa      1361 W/m2 * max(sin(solar altitude), 0)   (keeps direct+diffuse <= toa)
  influx_direct   toa * kt * (1 - fd),  kt ~ U(0.1, 0.8), fd ~ U(0.2, 0.9)
  influx_diffuse  toa * kt * fd
  albedo          U(0.05, 0.4)
  temperature     U(255, 305) K
  wnd100m         8 * Weibull(k=2) m/s
  roughness       exp(U(ln 1e-4, ln 2)) m
"""

from __future__ import annotations

from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pandas as pd
import scipy.sparse as sp

from .labelled import Dataset

SEEDS = dict(kt=1, fd=2, albedo=3, temperature=4, wnd100m=5, roughness=6, layout=7, shapes=8,
             wnd_shear_exp=9, humidity=10, outflux=11, soil=12, dewpoint=13, runoff=14, height=15)
_BLOCK = 24  # RNG block length in time steps


def make_time(nt, start="2013-01-01"):
    return pd.date_range(start, periods=nt, freq="h")


def make_coords(nx, ny, x0=0.0, y0=30.0, dx=0.25, dy=0.25):
    x = np.round(x0 + dx * np.arange(nx), 9)
    y = np.round(y0 + dy * np.arange(ny), 9)
    return x, y


def solar_tables(time, time_shift="0h"):
    """Time-only part of the Michalsky almanac the reference evaluates in
    pv/solar_position.py:71-97: sin/cos of the declination and of
    H0 = radians(local mean sidereal time at lon=0) - right ascension."""
    t = pd.DatetimeIndex(time) + pd.to_timedelta(time_shift)
    n = np.asarray(t.to_julian_date(), dtype=np.float64) - 2451545.0
    hour, minute = np.asarray(t.hour), np.asarray(t.minute)
    L = 280.460 + 0.9856474 * n
    g = np.radians(357.528 + 0.9856003 * n)
    l = np.radians(L + 1.915 * np.sin(g) + 0.020 * np.sin(2 * g))
    ep = np.radians(23.439 - 4e-7 * n)
    ra = np.arctan2(np.cos(ep) * np.sin(l), np.cos(l))
    h0 = np.radians((6.697375 + (hour + minute / 60.0) + 0.0657098242 * n) * 15.0) - ra
    dec = np.arcsin(np.sin(ep) * np.sin(l))
    return np.sin(dec), np.cos(dec), np.cos(h0), np.sin(h0)


def lit_lane_steps(time, lon, lat, altitude_threshold=1.0, vec=True, time_shift="0h"):
    """(lit, total) (lane, step) pairs of the PV kernels' sun gate with the solar position
    computed in-kernel: a lane -- 4 cells, 4 consecutive columns of one row with 128-bit lanes
    (``vec``), 4 rows of one column otherwise -- loads its inputs at a step iff one of its cells
    has sin(altitude) >= sin(threshold).  Evaluated from the float32 tables the kernel gets
    ({sin, cos} declination, {cos, sin} H0, {cos, sin} lon, {sin, cos} lat) with its operation
    order; each fused multiply-add is emulated in float64, so a cell within an ulp of the
    threshold may be counted the other way.  Bytes the kernels read = lit * 4 cells * the
    bytes per cell-step (20 for the ERA5 inputs)."""
    sd, cd, ch0, sh0 = (np.asarray(a, dtype=np.float32) for a in solar_tables(time, time_shift))
    lon_r, lat_r = np.radians(np.asarray(lon, dtype=np.float64)), np.radians(np.asarray(lat, dtype=np.float64))
    clon, slon = np.cos(lon_r).astype(np.float32), np.sin(lon_r).astype(np.float32)
    sl, cl = np.sin(lat_r).astype(np.float32), np.cos(lat_r).astype(np.float32)
    thr = np.float32(np.sin(np.radians(altitude_threshold)))
    nx, ny = len(clon), len(sl)
    # out-of-grid cells of a lane are border copies (the kernels clamp their indices)
    if vec:
        cols, rows = np.minimum(np.arange(-(-nx // 4) * 4), nx - 1), np.arange(ny)
    else:
        cols, rows = np.arange(nx), np.minimum(np.arange(-(-ny // 4) * 4), ny - 1)
    clon, slon, sl, cl = clon[cols], slon[cols], sl[rows], cl[rows]
    f64 = np.float64
    lit = 0
    for t in range(len(sd)):
        m = slon * np.float32(-sh0[t])  # cos h = fma(cos lon, cos H0, sin lon * -sin H0)
        ch = (clon.astype(f64) * f64(ch0[t]) + m).astype(np.float32)
        a1, a0 = cd[t] * cl, sd[t] * sl  # sin alt = fma(cos h, cos dec cos lat, sin dec sin lat)
        s = (ch[None, :].astype(f64) * a1[:, None] + a0[:, None]).astype(np.float32)
        up = ~(s < thr)
        up = up.reshape(len(rows), -1, 4).any(-1) if vec else up.reshape(-1, 4, len(cols)).any(1)
        lit += int(up.sum())
    total = len(sd) * (len(rows) * len(cols) // 4)
    return lit, total


def sin_altitude(time, lon_deg, lat_deg):
    sd, cd, ch0, sh0 = solar_tables(time)
    lon, lat = np.radians(lon_deg), np.radians(lat_deg)
    cosh = ch0[:, None] * np.cos(lon)[None, :] - sh0[:, None] * np.sin(lon)[None, :]  # (T, nx)
    s = (sd[:, None] * np.sin(lat)[None, :])[:, :, None] + (cd[:, None] * np.cos(lat)[None, :])[
        :, :, None
    ] * cosh[:, None, :]
    return np.clip(s, -1.0, 1.0)


def _rng(var, block):
    return np.random.default_rng([SEEDS[var], block])


def _uniform_block(var, block, shape, lo, hi):
    return _rng(var, block).uniform(lo, hi, size=shape).astype(np.float32)


def _gen_var(var, nt, ny, nx, t_offset, fn, workers=8):
    """Fill (nt, ny, nx) float32 from per-block generators (absolute block ids
    so shards of a longer axis see the same numbers)."""
    out = np.empty((nt, ny, nx), dtype=np.float32)
    first, last = t_offset // _BLOCK, (t_offset + nt - 1) // _BLOCK

    def work(b):
        lo, hi = max(b * _BLOCK, t_offset), min((b + 1) * _BLOCK, t_offset + nt)
        blk = fn(var, b, (_BLOCK, ny, nx))
        out[lo - t_offset : hi - t_offset] = blk[lo - b * _BLOCK : hi - b * _BLOCK]

    blocks = range(first, last + 1)
    if nt * ny * nx > 4_000_000 and workers > 1:
        with ThreadPoolExecutor(workers) as ex:
            list(ex.map(work, blocks))
    else:
        for b in blocks:
            work(b)
    return out


def make_fields(time, x, y, kinds=("pv", "wind", "temperature"), t_offset=0, extra=()):
    """Dict of float32 (time, y, x) fields.  ``t_offset``: index of ``time[0]``
    in the full axis (for time shards).  ``extra``: additional variables among
    'wnd_shear_exp', 'humidity', 'influx', 'outflux', 'soil temperature',
    'dewpoint temperature', 'runoff' (adds the static (y, x) field 'height')."""
    nt, ny, nx = len(time), len(y), len(x)
    f = {}
    if "pv" in kinds:
        toa = np.empty((nt, ny, nx), dtype=np.float32)
        step = max(1, 4_000_000 // (ny * nx))
        for i in range(0, nt, step):
            s = sin_altitude(time[i : i + step], x, y)
            toa[i : i + step] = (1361.0 * np.maximum(s, 0.0)).astype(np.float32)
        kt = _gen_var("kt", nt, ny, nx, t_offset, lambda v, b, sh: _uniform_block(v, b, sh, 0.1, 0.8))
        fd = _gen_var("fd", nt, ny, nx, t_offset, lambda v, b, sh: _uniform_block(v, b, sh, 0.2, 0.9))
        f["influx_toa"] = toa
        f["influx_direct"] = toa * kt * (np.float32(1.0) - fd)
        f["influx_diffuse"] = toa * kt * fd
        del kt, fd
        f["albedo"] = _gen_var("albedo", nt, ny, nx, t_offset,
                               lambda v, b, sh: _uniform_block(v, b, sh, 0.05, 0.4))
    if "pv" in kinds or "temperature" in kinds:
        f["temperature"] = _gen_var("temperature", nt, ny, nx, t_offset,
                                    lambda v, b, sh: _uniform_block(v, b, sh, 255.0, 305.0))
    if "wind" in kinds:
        f["wnd100m"] = _gen_var(
            "wnd100m", nt, ny, nx, t_offset,
            lambda v, b, sh: (8.0 * _rng(v, b).weibull(2.0, size=sh)).astype(np.float32))
        f["roughness"] = _gen_var(
            "roughness", nt, ny, nx, t_offset,
            lambda v, b, sh: np.exp(_rng(v, b).uniform(np.log(1e-4), np.log(2.0), size=sh)).astype(np.float32))
    if "wnd_shear_exp" in extra:
        f["wnd_shear_exp"] = _gen_var("wnd_shear_exp", nt, ny, nx, t_offset,
                                      lambda v, b, sh: _uniform_block(v, b, sh, 0.05, 0.4))
    if "humidity" in extra:
        f["humidity"] = _gen_var("humidity", nt, ny, nx, t_offset,
                                 lambda v, b, sh: _uniform_block(v, b, sh, 0.2, 1.0))
    if "soil temperature" in extra:  # NaN over "sea" like ERA5 stl4 (convert.py:311-314)
        st = _gen_var("soil", nt, ny, nx, t_offset, lambda v, b, sh: _uniform_block(v, b, sh, 270.0, 300.0))
        sea = np.random.default_rng(SEEDS["soil"]).uniform(size=(ny, nx)) < 0.3
        st[:, sea] = np.nan
        f["soil temperature"] = st
    if "dewpoint temperature" in extra:
        f["dewpoint temperature"] = _gen_var("dewpoint", nt, ny, nx, t_offset,
                                             lambda v, b, sh: _uniform_block(v, b, sh, 250.0, 295.0))
    if "runoff" in extra:
        f["runoff"] = _gen_var("runoff", nt, ny, nx, t_offset,
                               lambda v, b, sh: _rng(v, b).exponential(2e-4, size=sh).astype(np.float32))
        f["height"] = np.random.default_rng(SEEDS["height"]).uniform(0.0, 2000.0, size=(ny, nx)).astype(np.float32)
    if "influx" in extra:  # total influx instead of the direct/diffuse pair
        f["influx"] = f.pop("influx_direct") + f.pop("influx_diffuse")
    if "outflux" in extra:
        tot = f["influx"] if "influx" in f else f["influx_direct"] + f["influx_diffuse"]
        f["outflux"] = tot * f.pop("albedo")
    return f


def make_dataset(nx, ny, nt, x0=0.0, y0=30.0, dx=0.25, dy=0.25, start="2013-01-01",
                 kinds=("pv", "wind", "temperature"), t_offset=0, extra=()):
    """A ``Dataset`` ready for ``Cutout(data=...)``; ``t_offset`` selects a
    time shard [t_offset, t_offset+nt) of the axis starting at ``start``."""
    x, y = make_coords(nx, ny, x0, y0, dx, dy)
    time = make_time(t_offset + nt, start)[t_offset:]
    fields = make_fields(time, x, y, kinds, t_offset, extra)
    ds = Dataset(fields, coords=dict(time=time, x=x, y=y, lon=x, lat=y), attrs={"module": "era5"})
    return ds


def make_shapes(nx, ny, n_bus, seed=SEEDS["shapes"], border=True):
    """NUTS-like aggregation matrix (n_bus, ny*nx) CSR float64: Voronoi regions of
    ``n_bus`` random seeds on the index grid (weight 1); cells on a region
    border get a second entry for the neighbouring region with weights
    (w, 1 - w), w ~ U(0.3, 0.7), like area-overlap fractions of real shapes.
    100 % coverage, nnz ~ 1.1-1.3 S."""
    from scipy.spatial import cKDTree

    S = nx * ny
    if n_bus == 1:
        return sp.csr_matrix(np.ones((1, S)))
    rng = np.random.default_rng(seed)
    pts = np.c_[rng.uniform(0, nx, n_bus), rng.uniform(0, ny, n_bus)]
    gx, gy = np.meshgrid(np.arange(nx) + 0.5, np.arange(ny) + 0.5)
    _, lab = cKDTree(pts).query(np.c_[gx.ravel(), gy.ravel()])
    lab = lab.reshape(ny, nx)
    rows = [lab.ravel()]
    cols = [np.arange(S)]
    data = [np.ones(S)]
    if border:
        other = np.full((ny, nx), -1, dtype=np.int64)
        for sy, sx in ((0, 1), (0, -1), (1, 0), (-1, 0)):
            nb = np.roll(lab, (sy, sx), axis=(0, 1))
            ok = np.ones((ny, nx), bool)
            if sx == 1:
                ok[:, 0] = False
            if sx == -1:
                ok[:, -1] = False
            if sy == 1:
                ok[0, :] = False
            if sy == -1:
                ok[-1, :] = False
            pick = ok & (nb != lab) & (other < 0)
            other[pick] = nb[pick]
        bc = np.flatnonzero(other.ravel() >= 0)
        w = rng.uniform(0.3, 0.7, size=len(bc))
        data[0][bc] = w
        rows.append(other.ravel()[bc])
        cols.append(bc)
        data.append(1.0 - w)
    m = sp.csr_matrix(
        (np.concatenate(data), (np.concatenate(rows), np.concatenate(cols))), shape=(n_bus, S)
    )
    m.sum_duplicates()
    return m


def make_layout(nx, ny, seed=SEEDS["layout"]):
    return np.random.default_rng(seed).uniform(0.0, 10.0, size=(ny, nx))


# ----------------------------------------------------------------------
# device-side generator (bench.py: HBM-resident workloads too large to build on
# the host within the time budget).  Same distributions, torch RNG.
# ----------------------------------------------------------------------


DEVICE_BLOCK = 73  # RNG block (time steps) of the device generators: 8760 = 120 * 73, so the
                   # 1/2/4/8-way time shards of a year start on block boundaries


def _device_blocks(nt, t_offset, block):
    """(absolute block id, [lo, hi) inside the block, [dst_lo, dst_hi) in the shard)."""
    first, last = t_offset // block, (t_offset + nt - 1) // block
    for b in range(first, last + 1):
        lo, hi = max(b * block, t_offset), min((b + 1) * block, t_offset + nt)
        yield b, lo - b * block, hi - b * block, lo - t_offset, hi - t_offset


def make_pv_fields_device(time, x, y, device, seed=0, names=None, t_offset=0, block=DEVICE_BLOCK):
    """The five PV fields as float32 CUDA tensors (time, y, x), generated block by block
    straight into the final tensors (temporaries stay below ~1.5 GB, so a cutout that
    nearly fills the HBM can be built: 1440 x 720 x 8760 x 5 fields = 169 GiB).
    The random numbers of a time block depend only on (seed, absolute block id):
    ``time`` = steps [t_offset, t_offset + nt) of the full axis gives exactly the rows
    the unsharded generator produces (the time shards of a multi-GPU run ARE the single
    GPU's cutout).  ``names`` restricts the variables (default: all five)."""
    import torch

    nt, ny, nx = len(time), len(y), len(x)
    names = ("influx_toa", "influx_direct", "influx_diffuse", "albedo", "temperature") if names is None else tuple(names)
    f = {n: torch.empty((nt, ny, nx), dtype=torch.float32, device=device) for n in names}
    if nt == 0:
        return f
    need_toa = any(n.startswith("influx") for n in names)
    if need_toa:
        sd, cd, ch0, sh0 = (torch.from_numpy(a).to(device) for a in solar_tables(time))
        lon = torch.from_numpy(np.radians(x)).to(device)
        lat = torch.from_numpy(np.radians(y)).to(device)
        cosh = ch0[:, None] * torch.cos(lon)[None, :] - sh0[:, None] * torch.sin(lon)[None, :]
        slat, clat = torch.sin(lat), torch.cos(lat)
    g = torch.Generator(device=device)

    def u(lo, hi):
        return torch.rand((block, ny, nx), dtype=torch.float32, device=device, generator=g) * (hi - lo) + lo

    for b, blo, bhi, i, j in _device_blocks(nt, t_offset, block):
        g.manual_seed(1234 + 100_003 * seed + b)
        kt, fd, alb, tmp = u(0.1, 0.8), u(0.2, 0.9), u(0.05, 0.4), u(255.0, 305.0)
        if need_toa:
            s = (sd[i:j, None] * slat[None, :])[:, :, None] + (cd[i:j, None] * clat[None, :])[:, :, None] * cosh[i:j, None, :]
            toa = (1361.0 * s.clamp(min=0.0, max=1.0)).to(torch.float32)
            del s
            if "influx_toa" in f:
                f["influx_toa"][i:j] = toa
            if "influx_direct" in f:
                f["influx_direct"][i:j] = toa * kt[blo:bhi] * (1.0 - fd[blo:bhi])
            if "influx_diffuse" in f:
                f["influx_diffuse"][i:j] = toa * kt[blo:bhi] * fd[blo:bhi]
            del toa
        if "albedo" in f:
            f["albedo"][i:j] = alb[blo:bhi]
        if "temperature" in f:
            f["temperature"][i:j] = tmp[blo:bhi]
        del kt, fd, alb, tmp
    return f


def make_wind_fields_device(nt, ny, nx, device, seed=0, t_offset=0, block=DEVICE_BLOCK):
    """wnd100m = 8 * Weibull(k=2) m/s and roughness = exp(U(ln 1e-4, ln 2)) m as float32
    CUDA tensors (time, y, x); same distributions as ``make_fields``, torch RNG seeded per
    absolute time block like ``make_pv_fields_device``."""
    import torch

    w = torch.empty((nt, ny, nx), dtype=torch.float32, device=device)
    r = torch.empty_like(w)
    g = torch.Generator(device=device)
    lo, hi = float(np.log(1e-4)), float(np.log(2.0))
    for b, blo, bhi, i, j in _device_blocks(nt, t_offset, block) if nt else ():
        g.manual_seed(4321 + 100_003 * seed + b)
        un = torch.rand((block, ny, nx), dtype=torch.float32, device=device, generator=g)
        w[i:j] = (8.0 * torch.sqrt(-torch.log1p(-un)))[blo:bhi]  # Weibull(k=2) by inversion
        un = torch.rand((block, ny, nx), dtype=torch.float32, device=device, generator=g)
        r[i:j] = torch.exp(un * (hi - lo) + lo)[blo:bhi]
        del un
    return {"wnd100m": w, "roughness": r}


def make_voronoi_shapes(x, y, n_shapes, seed=8, margin=0.0):
    """``n_shapes`` convex polygons that PARTITION the cutout extent (cell boxes
    included) -- NUTS-like regions for the indicator-matrix tests and benchmarks.
    Voronoi cells of random seeds, bounded by mirroring the seeds across the four
    sides of the extent.  Returns a list of (N, 2) float64 rings (counter-clockwise,
    not closed); ``margin`` > 0 shrinks the partitioned box inside the extent."""
    from scipy.spatial import Voronoi

    pts, (xlo, xhi, ylo, yhi) = _voronoi_sites(x, y, n_shapes, seed, margin)
    mirrored = [pts]
    for axis, bound in ((0, xlo), (0, xhi), (1, ylo), (1, yhi)):
        m = pts.copy()
        m[:, axis] = 2 * bound - m[:, axis]
        mirrored.append(m)
    vor = Voronoi(np.concatenate(mirrored))
    rings = []
    for k in range(n_shapes):
        region = vor.regions[vor.point_region[k]]
        assert -1 not in region and len(region) >= 3
        ring = vor.vertices[region]
        ring[:, 0] = np.clip(ring[:, 0], xlo, xhi)  # snap round-off on the box sides
        ring[:, 1] = np.clip(ring[:, 1], ylo, yhi)
        c = ring.mean(0)
        order = np.argsort(np.arctan2(ring[:, 1] - c[1], ring[:, 0] - c[0]))
        rings.append(np.ascontiguousarray(ring[order]))
    return rings


def _voronoi_sites(x, y, n, seed, margin):
    """The random sites of ``make_voronoi_shapes`` and the extent they lie in."""
    x, y = np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)
    dx, dy = (x[-1] - x[0]) / (len(x) - 1), (y[-1] - y[0]) / (len(y) - 1)
    xlo, xhi = x[0] - dx / 2 + margin, x[-1] + dx / 2 - margin
    ylo, yhi = y[0] - dy / 2 + margin, y[-1] + dy / 2 - margin
    rng = np.random.default_rng(seed)
    pts = np.c_[rng.uniform(xlo, xhi, n), rng.uniform(ylo, yhi, n)]
    return pts, (xlo, xhi, ylo, yhi)


def make_line_network(x, y, n_sites, seed=8, line_seed=16):
    """A transmission-grid-like line network for the intersection-matrix tests and
    timings: one polyline per pair of neighbouring sites of ``make_voronoi_shapes(x, y,
    n_sites, seed)`` (the edges of their Delaunay triangulation, about 3 per site).
    A line has 2-50 vertices (``line_seed``): the straight connection, its inner
    vertices displaced sideways by up to 10 % of its length.  Returns a list of GeoJSON
    LineString dicts with (N, 2) float64 coordinate arrays (a bare array would be read
    as a polygon ring)."""
    from scipy.spatial import Delaunay

    pts, _ = _voronoi_sites(x, y, n_sites, seed, 0.0)
    tri = Delaunay(pts)
    ind, nb = tri.vertex_neighbor_vertices
    pairs = [(a, b) for a in range(n_sites) for b in nb[ind[a]:ind[a + 1]] if a < b]
    rng = np.random.default_rng(line_seed)
    lines = []
    for a, b in pairs:
        n = int(rng.integers(2, 51))
        t = np.linspace(0.0, 1.0, n)
        d = pts[b] - pts[a]
        side = rng.uniform(-0.1, 0.1, n) * np.sin(np.pi * t)  # the end points stay on the sites
        xy = pts[a] + t[:, None] * d + side[:, None] * np.array([-d[1], d[0]])
        lines.append({"type": "LineString", "coordinates": np.ascontiguousarray(xy)})
    return lines


def make_basins(x, y, n, seed=8, overhang=0.25):
    """A HydroBASINS-like table for ``hydro``: the Voronoi basins of ``make_voronoi_shapes`` over
    the cutout extent stretched by ``overhang`` of its width and height beyond its east and north
    sides, so that some basins lie partly or wholly off the grid.  The basins drain into one tree:
    the outlet is the basin whose site is nearest the south-west corner, and every other basin
    drains into the neighbour (shared Voronoi edge) through which a breadth-first walk from the
    outlet first reached it.  ``DIST_MAIN`` is the distance to the outlet along the tree in km
    (111.2 km per degree between sites), ``NEXT_DOWN`` 0 at the outlet, ``HYBAS_ID`` a shuffled set
    of ids (frame order is not id order).  Returns a DataFrame with ``HYBAS_ID, DIST_MAIN,
    NEXT_DOWN, geometry`` (GeoJSON Polygon dicts) and the basins' sites ``site_lon, site_lat``
    (strictly inside their basins)."""
    from scipy.spatial import Delaunay

    x, y = np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)
    dx, dy = (x[-1] - x[0]) / (len(x) - 1), (y[-1] - y[0]) / (len(y) - 1)
    kx, ky = max(1, int(round(overhang * len(x)))), max(1, int(round(overhang * len(y))))
    xe = np.concatenate([x, x[-1] + dx * np.arange(1, kx + 1)])
    ye = np.concatenate([y, y[-1] + dy * np.arange(1, ky + 1)])
    rings = make_voronoi_shapes(xe, ye, n, seed)
    pts, (xlo, _, ylo, _) = _voronoi_sites(xe, ye, n, seed, 0.0)
    ind, nb = Delaunay(pts).vertex_neighbor_vertices
    outlet = int(np.argmin(np.hypot(pts[:, 0] - xlo, pts[:, 1] - ylo)))
    parent = np.full(n, -1)
    dist = np.zeros(n)
    parent[outlet] = outlet
    queue = [outlet]
    for b in queue:
        for c in nb[ind[b]:ind[b + 1]]:
            if parent[c] < 0:
                parent[c] = b
                dist[c] = dist[b] + 111.2 * np.hypot(*(pts[c] - pts[b]))
                queue.append(c)
    ids = 1000 + np.random.default_rng(seed + 1).permutation(n) * 7
    next_down = np.where(np.arange(n) == outlet, 0, ids[parent])
    return pd.DataFrame({"HYBAS_ID": ids, "DIST_MAIN": dist, "NEXT_DOWN": next_down,
                         "geometry": [{"type": "Polygon", "coordinates": [r]} for r in rings],
                         "site_lon": pts[:, 0], "site_lat": pts[:, 1]})


def make_line_rating_dataset(nx, ny, nt, x0=0.0, y0=30.0, dx=0.25, dy=0.25, start="2013-01-01", seed=41):
    """A ``Dataset`` with the inputs of ``line_rating``: temperature (255-305 K), wnd100m
    (Weibull, mean ~7 m/s), wnd_azimuth ([0, 2 pi)), influx_direct (0-900 W/m2) and the static
    height (0-2000 m), float32.  The ranges keep the heat balance ``qc + qr - qs`` of the
    default conductor far from 0 (natural convection alone exceeds the largest solar gain)."""
    x, y = make_coords(nx, ny, x0, y0, dx, dy)
    time = make_time(nt, start)
    rng = np.random.default_rng(seed)
    sh = (nt, ny, nx)
    f = {
        "temperature": rng.uniform(255.0, 305.0, sh).astype(np.float32),
        "wnd100m": (8.0 * rng.weibull(2.0, sh)).astype(np.float32),
        "wnd_azimuth": rng.uniform(0.0, 2 * np.pi, sh).astype(np.float32),
        "influx_direct": rng.uniform(0.0, 900.0, sh).astype(np.float32),
        "height": rng.uniform(0.0, 2000.0, (ny, nx)).astype(np.float32),
    }
    return Dataset(f, coords=dict(time=time, x=x, y=y, lon=x, lat=y), attrs={"module": "era5"})
