"""
CPU ORACLE for the dynamic line rating  --  TEST INFRASTRUCTURE ONLY.

A float64 NumPy restatement of the reference's ``convert_line_rating`` and
``line_rating`` (atlite/convert.py:1152-1367), in the conventions of
``atlite_oracle``: fields keep their dtypes and the per-line parameters are
``np.float64`` scalars (``df.iloc[i].values``), so NumPy's promotion rules put the
float32 roundings where the reference has them.  ``tests/golden/make_golden_line_rating.py``
pins it to the reference's own source; ``tests/test_line_rating.py`` holds it to
``tests/golden/reference_line_rating.npz`` at 1e-9 relative.
"""

from __future__ import annotations

import warnings

import numpy as np
import pandas as pd

import atlite_oracle as O

pi = np.pi


def convert_line_rating(ds, psi, R, D=0.028, Ts=373, epsilon=0.6, alpha=0.6, per_unit=False):
    """convert.py:1152-1252 on a mapping of arrays; the solar position is taken from
    ``ds["solar_altitude"]`` / ``ds["solar_azimuth"]`` when present (the dict branch, :1240-1243),
    else computed at a 0 h shift (``SolarPosition(ds)``, :1244; needs time / lon / lat)."""
    Ta = ds["temperature"]
    Tfilm = (Ta + Ts) / 2  # :1197
    T0 = 273.15

    V = ds["wnd100m"]  # :1201
    mu = (1.458e-6 * Tfilm**1.5) / (Tfilm + 383.4 - T0)  # (13a) :1202-1204
    H = ds["height"]
    rho = (1.293 - 1.525e-4 * H + 6.379e-9 * H**2) / (1 + 0.00367 * (Tfilm - T0))  # (14a) :1206-1208

    reynold = D * V * rho / mu  # :1210

    k = 2.424e-2 + 7.477e-5 * (Tfilm - T0) - 4.407e-9 * (Tfilm - T0) ** 2  # :1212-1214
    anglediff = ds["wnd_azimuth"] - np.radians(psi)  # :1215
    Phi = np.absolute(np.mod(anglediff + pi / 2, pi) - pi / 2)  # :1216
    K = 1.194 - np.cos(Phi) + 0.194 * np.cos(2 * Phi) + 0.368 * np.sin(2 * Phi)  # :1217-1220

    Tdiff = Ts - Ta  # :1221
    qcf1 = K * (1.01 + 1.347 * reynold**0.52) * k * Tdiff  # (3a) :1222
    qcf2 = K * 0.754 * reynold**0.6 * k * Tdiff  # (3b) :1223

    qcf = np.maximum(qcf1, qcf2)  # :1225

    qcn = 3.645 * np.sqrt(rho) * D**0.75 * Tdiff**1.25  # :1228

    qc = np.maximum(qcf, qcn)  # :1231

    qr = 17.8 * D * epsilon * ((Ts / 100) ** 4 - (Ta / 100) ** 4)  # :1234

    Q = ds["influx_direct"]  # :1237
    A = D * 1  # :1238

    if "solar_altitude" in ds and "solar_azimuth" in ds:
        alt, az = ds["solar_altitude"], ds["solar_azimuth"]
    else:
        sp = O.solar_position(ds, time_shift="0h")
        alt, az = sp["altitude"], sp["azimuth"]
    Phi_s = np.arccos(np.cos(alt) * np.cos(az - np.radians(psi)))  # :1245-1247

    qs = alpha * Q * A * np.sin(Phi_s)  # :1249

    return np.sqrt((qc + qr - qs) / R)  # :1251


def line_azimuth(xy):
    """get_azimuth (convert.py:1333-1337) of an (N, 2) coordinate array."""
    xy = np.asarray(xy, dtype=np.float64)
    return np.arctan2(xy[0, 0] - xy[-1, 0], xy[0, 1] - xy[-1, 1])


def line_rating(ds, I, azimuth, line_resistance, **params):
    """convert.py:1325-1367 after the intersection matrix: ``I`` (n_lines, ny*nx) CSR, ``azimuth``
    a pandas Series of the raw ``get_azimuth`` values (its index is the shapes' index).  Returns
    (n_lines, nt) float64; line i is ``Imax.min("spatial")`` (skipna) over the cells
    ``cols[rows == i]``, NaN when it has none.  The solar position is resolved once for the whole
    cutout, as ``cutout.data`` carries it (:1331)."""
    rows, cols = I.nonzero()  # :1329
    azimuth = azimuth.where(azimuth >= 0, azimuth + np.pi)  # :1340

    params.setdefault("D", 0.028)  # :1342-1345
    params.setdefault("Ts", 373)
    params.setdefault("epsilon", 0.6)
    params.setdefault("alpha", 0.6)

    df = pd.DataFrame({"psi": azimuth, "R": line_resistance}).assign(**params)  # :1347

    assert df.notnull().all().all(), "Nan values encountered."  # :1349
    assert df.columns.equals(pd.Index(["psi", "R", "D", "Ts", "epsilon", "alpha"]))  # :1350

    nt = len(ds["time"])
    flat = {}  # data.stack(spatial=["y", "x"])  :1331
    for n in ("temperature", "wnd100m", "wnd_azimuth", "influx_direct"):
        a = np.asarray(ds[n])
        flat[n] = a.reshape(nt, -1)
    flat["height"] = np.asarray(ds["height"]).reshape(-1)
    if "solar_altitude" in ds and "solar_azimuth" in ds:
        sp = {"altitude": ds["solar_altitude"], "azimuth": ds["solar_azimuth"]}
    else:
        sp = O.solar_position(ds, time_shift="0h")
    flat["solar_altitude"] = np.broadcast_to(np.asarray(sp["altitude"]), np.shape(ds["temperature"])).reshape(nt, -1)
    flat["solar_azimuth"] = np.broadcast_to(np.asarray(sp["azimuth"]), np.shape(ds["temperature"])).reshape(nt, -1)

    out = np.full((len(df), nt), np.nan)  # dummy  :1352
    for i in range(len(df)):  # :1354-1360
        cells_i = cols[rows == i]
        if cells_i.size:
            sub = {k: (v[cells_i] if v.ndim == 1 else v[:, cells_i]) for k, v in flat.items()}
            imax = convert_line_rating(sub, *df.iloc[i].values)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore", RuntimeWarning)  # all-NaN step -> NaN, as skipna min
                out[i] = np.nanmin(imax, axis=1)
    return out
