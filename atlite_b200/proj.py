"""The coordinate reference systems the availability path supports, in float64 NumPy.

* EPSG:4326 -- WGS 84 longitude / latitude in degrees.
* EPSG:3035 -- ETRS89-LAEA Europe: Lambert azimuthal equal-area on GRS80, phi0 = 52 N,
  lambda0 = 10 E, false easting 4 321 000 m, false northing 3 210 000 m (EPSG method 9820,
  IOGP Guidance Note 7-2).
* EPSG:3857 -- WGS 84 / Pseudo-Mercator (EPSG method 1024): spherical Mercator with R = 6 378 137 m
  applied to the geodetic latitude.
* ESRI:54009 -- World Mollweide: spherical Mollweide with R = 6 378 137 m applied to the geodetic
  latitude, lambda0 = 0 (what PROJ's ``moll`` does on WGS 84).

Every pair goes through longitude / latitude.  Polygon vertices are projected here on the host;
pixel centres are projected on the device by the same formulas (csrc/proj.cuh), with the constants
``device_projection`` hands it.  ETRS89 and WGS 84
are taken as the same datum, as PROJ does for EPSG:3035 <-> EPSG:4326 without a grid.  A point
that has no image (a pole in Mercator, a point off the Mercator map or outside the Mollweide
ellipse) projects to NaN.

CRS keys: ``epsg`` returns the int EPSG code for the EPSG CRSs and the string ``"ESRI:54009"``
for World Mollweide.
"""

from __future__ import annotations

import numpy as np

from . import _lib
from .hydro import GRS80_A, GRS80_F, authalic_q

MOLLWEIDE = "ESRI:54009"
# CRS key -> its ATL_CRS_* kind on the device (csrc/proj.cuh)
CRS_KIND = {4326: _lib.CRS_LONLAT, 3035: _lib.CRS_LAEA, 3857: _lib.CRS_MERCATOR, MOLLWEIDE: _lib.CRS_MOLLWEIDE}
SUPPORTED = tuple(CRS_KIND)

E2 = GRS80_F * (2.0 - GRS80_F)
E = np.sqrt(E2)
PHI0, LAM0 = np.radians(52.0), np.radians(10.0)
FE, FN = 4321000.0, 3210000.0
QP = float(authalic_q(90.0))
Q0 = float(authalic_q(52.0))
RQ = GRS80_A * np.sqrt(QP / 2.0)
BETA0 = np.arcsin(Q0 / QP)
D = GRS80_A * (np.cos(PHI0) / np.sqrt(1.0 - E2 * np.sin(PHI0) ** 2)) / (RQ * np.cos(BETA0))
# phi from the authalic latitude beta: the three-term series (GN 7-2), then Newton steps on q(phi)
SERIES = (E2 / 3.0 + 31.0 * E2 ** 2 / 180.0 + 517.0 * E2 ** 3 / 5040.0,
          23.0 * E2 ** 2 / 360.0 + 251.0 * E2 ** 3 / 3780.0,
          761.0 * E2 ** 3 / 45360.0)
NEWTON_STEPS = 2

R_SPHERE = 6378137.0  # the sphere of EPSG:3857 and of ESRI:54009 on WGS 84
MOLL_NEWTON_STEPS = 4  # from the start below: converged to the last bit everywhere (tests/test_availability_crs.py)
EDGE = 1e-12  # slack of the map edges, so that a vertex on the antimeridian survives a round trip
HALF_PI_LO = 6.123233995736766e-17  # pi / 2 - float(pi / 2)
# 1 / 3!, 1 / 5!, ..., 1 / 17!: u - sin u = u^3 (C0 - u^2 (C1 - u^2 (...))), to 5e-17 relative for u < 1
SIN_TAIL = (1 / 6, 1 / 120, 1 / 5040, 1 / 362880, 1 / 39916800, 1 / 6227020800, 1 / 1307674368000,
            1 / 355687428096000)


def epsg(crs):
    """Key of ``crs`` (one of ``SUPPORTED``): from an int EPSG code, ``"EPSG:n"``, ``"ESRI:54009"``
    (any case), or an object with ``to_epsg()`` (pyproj / rasterio CRS), or whose ``to_authority()``
    is ``("ESRI", "54009")``.  An int is always an EPSG code.  Anything else raises
    ``NotImplementedError``."""
    code = None
    if hasattr(crs, "to_epsg"):
        code = crs.to_epsg()
        if code is None and hasattr(crs, "to_authority"):
            auth = crs.to_authority()
            if auth is not None and str(auth[0]).upper() == "ESRI" and str(auth[1]) == "54009":
                code = MOLLWEIDE
    elif isinstance(crs, (int, np.integer)) and not isinstance(crs, bool):
        code = int(crs)
    elif isinstance(crs, str):
        s = crs.strip().upper()
        if s.startswith("EPSG:") and s[5:].isdigit():
            code = int(s[5:])
        elif s == MOLLWEIDE:
            code = MOLLWEIDE
    if code not in SUPPORTED:
        raise NotImplementedError(f"CRS {crs!r} is not supported; the availability path supports "
                                  "EPSG:4326 and EPSG:3035, EPSG:3857 and ESRI:54009 (given as an int EPSG code, "
                                  "'EPSG:n', 'ESRI:54009' or an object with to_epsg() / to_authority())")
    return code


def name(crs):
    """``"EPSG:n"`` or ``"ESRI:54009"`` for a supported ``crs``."""
    code = epsg(crs)
    return code if isinstance(code, str) else f"EPSG:{code}"


def laea_forward(lon_deg, lat_deg):
    """EPSG:4326 degrees -> EPSG:3035 metres (easting, northing)."""
    lam = np.radians(np.asarray(lon_deg, dtype=np.float64))
    q = authalic_q(lat_deg)
    beta = np.arcsin(np.clip(q / QP, -1.0, 1.0))
    dl = lam - LAM0
    sb, cb, cdl = np.sin(beta), np.cos(beta), np.cos(dl)
    B = RQ * np.sqrt(2.0 / (1.0 + np.sin(BETA0) * sb + np.cos(BETA0) * cb * cdl))
    return FE + (B * D) * cb * np.sin(dl), FN + (B / D) * (np.cos(BETA0) * sb - np.sin(BETA0) * cb * cdl)


def phi_from_authalic(beta, q):
    """Geodetic latitude (radians) whose authalic q is ``q`` (beta = asin(q / qP))."""
    phi = beta + SERIES[0] * np.sin(2 * beta) + SERIES[1] * np.sin(4 * beta) + SERIES[2] * np.sin(6 * beta)
    for _ in range(NEWTON_STEPS):
        s = np.sin(phi)
        w = 1.0 - E2 * s * s
        c = np.cos(phi)
        c = np.where(c == 0.0, 1e-300, c)
        phi = phi + w * w / (2.0 * c) * (q / (1.0 - E2) - s / w + np.log((1.0 - E * s) / (1.0 + E * s)) / (2.0 * E))
    return phi


def laea_inverse(x, y):
    """EPSG:3035 metres -> EPSG:4326 degrees (lon, lat)."""
    x = np.asarray(x, dtype=np.float64) - FE
    y = np.asarray(y, dtype=np.float64) - FN
    rho = np.sqrt((x / D) ** 2 + (D * y) ** 2)
    C = 2.0 * np.arcsin(np.clip(rho / (2.0 * RQ), -1.0, 1.0))
    sC, cC = np.sin(C), np.cos(C)
    safe = np.where(rho == 0.0, 1.0, rho)
    sbeta = np.where(rho == 0.0, np.sin(BETA0), cC * np.sin(BETA0) + D * y * sC * np.cos(BETA0) / safe)
    beta = np.arcsin(np.clip(sbeta, -1.0, 1.0))
    lam = LAM0 + np.arctan2(x * sC, D * rho * np.cos(BETA0) * cC - D * D * y * np.sin(BETA0) * sC)
    phi = phi_from_authalic(beta, QP * np.sin(beta))
    return np.degrees(lam), np.degrees(phi)


def mercator_forward(lon_deg, lat_deg):
    """EPSG:4326 degrees -> EPSG:3857 metres: x = R lambda, y = R asinh(tan phi); NaN at |phi| >= 90."""
    lon = np.asarray(lon_deg, dtype=np.float64)
    lat = np.asarray(lat_deg, dtype=np.float64)
    with np.errstate(invalid="ignore"):
        ok = np.abs(lat) < 90.0
        y = np.where(ok, R_SPHERE * np.arcsinh(np.tan(np.radians(np.where(ok, lat, 0.0)))), np.nan)
    return np.where(ok, R_SPHERE * np.radians(lon), np.nan), y


def mercator_inverse(x, y):
    """EPSG:3857 metres -> EPSG:4326 degrees: lambda = x / R, phi = atan(sinh(y / R)); NaN off the
    map (|x| > pi R)."""
    x = np.asarray(x, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        ok = np.abs(x) <= np.pi * R_SPHERE * (1.0 + EDGE)
        return (np.where(ok, np.degrees(np.clip(x / R_SPHERE, -np.pi, np.pi)), np.nan),
                np.where(ok, np.degrees(np.arctan(np.sinh(y / R_SPHERE))), np.nan))


def _sin_tail(d):
    """2 d - sin 2 d for d in [0, pi / 2], without the cancellation near 0."""
    u = 2.0 * d
    v = u * u
    p = SIN_TAIL[-1]
    for c in SIN_TAIL[-2::-1]:
        p = c - v * p
    return np.where(u >= 1.0, u - np.sin(u), u * v * p)


def mollweide_delta(phi):
    """pi / 2 - |theta| of the Mollweide auxiliary angle theta (2 theta + sin 2 theta = pi sin phi)
    for the latitude ``phi`` in radians, |phi| <= pi / 2.  Solved for delta, which keeps the
    equation well conditioned at the poles: 2 delta - sin 2 delta = pi (1 - sin |phi|)
    = 2 pi sin^2(eps / 2), eps = pi / 2 - |phi|.  Start: the polar asymptote delta^3 = 3 / 4 of the
    right-hand side; then MOLL_NEWTON_STEPS Newton steps.  0 exactly at the poles."""
    a = np.abs(np.asarray(phi, dtype=np.float64))
    eps = np.where(a >= np.pi / 2, 0.0, (np.pi / 2 - a) + HALF_PI_LO)
    s = np.sin(0.5 * eps)
    rhs = 2.0 * np.pi * s * s
    d = np.cbrt(0.75 * rhs)
    for _ in range(MOLL_NEWTON_STEPS):
        sd = np.sin(d)
        gp = 4.0 * sd * sd
        step = np.where(gp > 0.0, (_sin_tail(d) - rhs) / np.where(gp > 0.0, gp, 1.0), 0.0)
        d = np.clip(d - step, 0.0, np.pi / 2)
    return d


def mollweide_forward(lon_deg, lat_deg):
    """EPSG:4326 degrees -> ESRI:54009 metres: x = 2 sqrt2 / pi R lambda cos theta,
    y = sqrt2 R sin theta; NaN at |phi| > 90."""
    lon = np.asarray(lon_deg, dtype=np.float64)
    lat = np.asarray(lat_deg, dtype=np.float64)
    ok = np.abs(lat) <= 90.0
    phi = np.radians(np.where(ok, lat, 0.0))
    d = mollweide_delta(phi)
    x = (2.0 * np.sqrt(2.0) / np.pi) * R_SPHERE * np.radians(lon) * np.sin(d)
    y = np.copysign(np.sqrt(2.0) * R_SPHERE * np.cos(d), phi)
    return np.where(ok, x, np.nan), np.where(ok, y, np.nan)


def mollweide_inverse(x, y):
    """ESRI:54009 metres -> EPSG:4326 degrees: theta = asin(y / (sqrt2 R)),
    phi = asin((2 theta + sin 2 theta) / pi), lambda = pi x / (2 sqrt2 R cos theta), the latitude
    taken through delta = pi / 2 - |theta| as in ``mollweide_delta`` so that it keeps its precision
    at the poles: pi / 2 - |phi| = 2 asin(sqrt((2 delta - sin 2 delta) / (2 pi))).  NaN outside the
    ellipse x^2 / (8 R^2) + y^2 / (2 R^2) <= 1 (|lambda| > pi or |y| > sqrt2 R), which is tested with
    the slack EDGE: near the poles the longitude of a point is not determined to 1e-12 by its float
    coordinates."""
    x = np.asarray(x, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    s = y / (np.sqrt(2.0) * R_SPHERE)
    t = x / (2.0 * np.sqrt(2.0) * R_SPHERE)
    ok = t * t + s * s <= 1.0 + EDGE
    s = np.clip(s, -1.0, 1.0)
    c = np.sqrt((1.0 - s) * (1.0 + s))
    with np.errstate(invalid="ignore", divide="ignore"):
        lam = np.where(c > 0.0, np.clip(np.pi * t / c, -np.pi, np.pi), 0.0)
    d = np.arctan2(c, np.abs(s))
    eps = 2.0 * np.arcsin(np.sqrt(_sin_tail(d) / (2.0 * np.pi)))
    phi = np.copysign((np.pi / 2 - eps) + HALF_PI_LO, s)
    return np.where(ok, np.degrees(lam), np.nan), np.where(ok, np.degrees(phi), np.nan)


_TO_LONLAT = {3035: laea_inverse, 3857: mercator_inverse, MOLLWEIDE: mollweide_inverse}
_FROM_LONLAT = {3035: laea_forward, 3857: mercator_forward, MOLLWEIDE: mollweide_forward}


def transform(x, y, src, dst):
    """Coordinates (x, y) from CRS ``src`` to ``dst`` (each one of ``SUPPORTED``), through
    longitude / latitude.  Points without an image in ``dst`` become NaN."""
    src, dst = epsg(src), epsg(dst)
    x, y = np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)
    if src == dst:
        return x, y
    if src != 4326:
        x, y = _TO_LONLAT[src](x, y)
    if dst != 4326:
        x, y = _FROM_LONLAT[dst](x, y)
    return x, y


def device_projection(src, dst):
    """The C ABI's AtlProjection (``_lib.Projection``) from CRS ``src`` to CRS ``dst``: their kinds
    and this module's constants, so that the device projects as ``transform`` does."""
    laea = _lib.Laea(*(float(v) for v in (E2, E, QP, RQ, np.sin(BETA0), np.cos(BETA0), D, LAM0, FE, FN, *SERIES)),
                     NEWTON_STEPS)

    def crs(key):
        return _lib.Crs(CRS_KIND[epsg(key)], MOLL_NEWTON_STEPS, R_SPHERE)

    return _lib.Projection(crs(src), crs(dst), laea)


def laea_cell_area(lon_lo, lon_hi, lat_lo, lat_hi):
    """Ellipsoidal area in m^2 of the lon / lat box: a^2 / 2 * dlambda * (q(phi2) - q(phi1)).
    LAEA is equal-area, so this is also the box's area in EPSG:3035."""
    dl = np.radians(np.asarray(lon_hi, dtype=np.float64) - np.asarray(lon_lo, dtype=np.float64))
    return GRS80_A ** 2 / 2.0 * dl * (authalic_q(lat_hi) - authalic_q(lat_lo))


def mollweide_cell_area(lon_lo, lon_hi, lat_lo, lat_hi):
    """Area in m^2 of the lon / lat box on the sphere of ESRI:54009: R^2 dlambda (sin phi2 - sin phi1).
    Mollweide is equal-area on that sphere, so this is also the box's area in ESRI:54009."""
    dl = np.radians(np.asarray(lon_hi, dtype=np.float64) - np.asarray(lon_lo, dtype=np.float64))
    return R_SPHERE ** 2 * dl * (np.sin(np.radians(lat_hi)) - np.sin(np.radians(lat_lo)))


def mercator_cell_area(lon_lo, lon_hi, lat_lo, lat_hi):
    """Area in EPSG:3857 m^2 of the lon / lat box: R^2 dlambda (asinh tan phi2 - asinh tan phi1)."""
    dl = np.radians(np.asarray(lon_hi, dtype=np.float64) - np.asarray(lon_lo, dtype=np.float64))
    return R_SPHERE ** 2 * dl * (np.arcsinh(np.tan(np.radians(lat_hi))) - np.arcsinh(np.tan(np.radians(lat_lo))))


def cell_area(crs, lon_lo, lon_hi, lat_lo, lat_hi):
    """Area in m^2 of the lon / lat box in the projected ``crs``."""
    return {3035: laea_cell_area, 3857: mercator_cell_area, MOLLWEIDE: mollweide_cell_area}[epsg(crs)](
        lon_lo, lon_hi, lat_lo, lat_hi)
