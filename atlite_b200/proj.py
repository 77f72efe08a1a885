"""The two coordinate reference systems the availability path supports, in float64 NumPy.

* EPSG:4326 -- WGS 84 longitude / latitude in degrees.
* EPSG:3035 -- ETRS89-LAEA Europe: Lambert azimuthal equal-area on GRS80, phi0 = 52 N,
  lambda0 = 10 E, false easting 4 321 000 m, false northing 3 210 000 m (EPSG method 9820,
  IOGP Guidance Note 7-2).

Polygon vertices are projected here on the host; pixel centres are projected on the device by
the same formulas (csrc/proj.cuh).  ETRS89 and WGS 84 are taken as the same datum, as PROJ does
for EPSG:3035 <-> EPSG:4326 without a grid.
"""

from __future__ import annotations

import numpy as np

from .hydro import GRS80_A, GRS80_F, authalic_q

SUPPORTED = (4326, 3035)

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


def epsg(crs):
    """EPSG code of ``crs``: an int, ``"EPSG:n"`` (any case), or an object with ``to_epsg()``
    (pyproj / rasterio CRS).  Anything that is not one of ``SUPPORTED`` raises
    ``NotImplementedError``."""
    code = None
    if hasattr(crs, "to_epsg"):
        code = crs.to_epsg()
    elif isinstance(crs, (int, np.integer)) and not isinstance(crs, bool):
        code = int(crs)
    elif isinstance(crs, str):
        s = crs.strip().upper()
        if s.startswith("EPSG:") and s[5:].isdigit():
            code = int(s[5:])
    if code not in SUPPORTED:
        raise NotImplementedError(f"CRS {crs!r} is not supported; the availability path supports "
                                  f"EPSG:4326 and EPSG:3035 (given as an int, 'EPSG:n' or an object with to_epsg())")
    return code


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


def transform(x, y, src, dst):
    """Coordinates (x, y) from CRS ``src`` to ``dst`` (each one of ``SUPPORTED``)."""
    src, dst = epsg(src), epsg(dst)
    x, y = np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)
    if src == dst:
        return x, y
    return laea_forward(x, y) if dst == 3035 else laea_inverse(x, y)


def laea_cell_area(lon_lo, lon_hi, lat_lo, lat_hi):
    """Ellipsoidal area in m^2 of the lon / lat box: a^2 / 2 * dlambda * (q(phi2) - q(phi1)).
    LAEA is equal-area, so this is also the box's area in EPSG:3035."""
    dl = np.radians(np.asarray(lon_hi, dtype=np.float64) - np.asarray(lon_lo, dtype=np.float64))
    return GRS80_A ** 2 / 2.0 * dl * (authalic_q(lat_hi) - authalic_q(lat_lo))
