#!/usr/bin/env python
"""Generate ``reference_line_rating.npz``: the REFERENCE'S OWN ``convert_line_rating``
(atlite/convert.py:1152-1252) and ``SolarPosition`` (pv/solar_position.py), loaded from the
reference's source files under the stand-ins of ``xr_shim.py`` as ``make_golden.py`` does,
on a small seeded cutout and line network.

``convert_line_rating`` runs unchanged through its ``dict`` branch on the NumPy arrays of one
line's cells.  The ~15 lines of ``line_rating``'s glue (convert.py:1325-1367: azimuth, its wrap,
the parameter DataFrame, the per-line loop over ``cols[rows == i]``, the skipna min and the NaN
row of a line without cells) need geopandas and xarray's concat, so they are restated below; the
intersection matrix comes from the exact CPU checker ``oracle/intersection_exact.py``.

    python tests/golden/make_golden_line_rating.py     # writes tests/golden/reference_line_rating.npz
"""

import os
import sys
import warnings

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, HERE)

import xr_shim  # noqa: E402

import intersection_exact as IX  # noqa: E402
from atlite_b200 import gis, synthetic as syn  # noqa: E402  (inputs and geometry reading only)

warnings.simplefilter("ignore")
conv = xr_shim.install()
from atlite.pv.solar_position import SolarPosition as RefSolarPosition  # noqa: E402


def lines_and_index(x, y):
    """The line network of the cases: a seeded network, a line outside the grid (no cell) and a
    line inside one cell, under string labels."""
    lines = [ln["coordinates"] for ln in syn.make_line_network(x, y, 7)]
    dx = x[1] - x[0]
    lines.append(np.array([[x[-1] + 5 * dx, y[0]], [x[-1] + 9 * dx, y[-1]]]))  # outside the grid
    lines.append(np.array([[x[4] - 0.2 * dx, y[3] + 0.1 * dx], [x[4] + 0.3 * dx, y[3] - 0.2 * dx]]))  # one cell
    return lines, [f"line{i}" for i in range(len(lines))]


def glue(flat, I, azimuth, line_resistance, params):
    """convert.py:1329-1367 after the intersection matrix, per line on NumPy arrays."""
    rows, cols = I.nonzero()
    azimuth = azimuth.where(azimuth >= 0, azimuth + np.pi)
    params = dict(params)
    params.setdefault("D", 0.028)
    params.setdefault("Ts", 373)
    params.setdefault("epsilon", 0.6)
    params.setdefault("alpha", 0.6)
    df = pd.DataFrame({"psi": azimuth, "R": line_resistance}).assign(**params)
    assert df.notnull().all().all()
    assert df.columns.equals(pd.Index(["psi", "R", "D", "Ts", "epsilon", "alpha"]))
    nt = flat["temperature"].shape[0]
    out = np.full((len(df), nt), np.nan)
    for i in range(len(df)):
        cells_i = cols[rows == i]
        if cells_i.size:
            sub = {k: (v[cells_i] if v.ndim == 1 else v[:, cells_i]) for k, v in flat.items()}
            imax = conv.convert_line_rating(sub, *df.iloc[i].values)  # the reference's own function
            out[i] = np.nanmin(imax, axis=1)  # Imax.min("spatial"): skipna
    return out


def main():
    nx, ny, nt = 13, 9, 30
    ds = syn.make_line_rating_dataset(nx, ny, nt, x0=5.0, y0=45.0, start="2013-06-21 02:00")
    x, y, time = ds.coords["x"], ds.coords["y"], ds.coords["time"]
    F = {k: np.array(ds.raw(k)) for k in ds.keys()}
    # planted: a NaN cell at some steps, a cell hotter than Ts (Tdiff < 0 -> NaN) at others
    F["temperature"][3:9, 4, 6] = np.nan
    F["wnd100m"][12, 2, 2] = np.nan
    F["temperature"][5:20, 1, 9] = 380.0
    lines, index = lines_and_index(x, y)
    I = IX.intersectionmatrix(x, y, [gis.geometry_parts({"type": "LineString", "coordinates": c}) for c in lines])
    import scipy.sparse as sp

    I = sp.csr_matrix(I)
    az_raw = pd.Series([np.arctan2(c[0, 0] - c[-1, 0], c[0, 1] - c[-1, 1]) for c in lines], index=index)

    ref = xr_shim.Dataset({k: ((("time", "y", "x") if v.ndim == 3 else ("y", "x")), v) for k, v in F.items()},
                          coords=dict(time=time, x=x, y=y, lon=x, lat=y))
    sp0 = RefSolarPosition(ref)  # the default 0 h shift: what a cutout without stored position gets
    alt0 = np.asarray(sp0["altitude"].transpose("time", "y", "x").values, dtype=np.float64)
    azi0 = np.asarray(sp0["azimuth"].transpose("time", "y", "x").values, dtype=np.float64)
    sp30 = RefSolarPosition(ref, time_shift="-30min")  # what ERA5 cutouts store (era5.py:182-188)
    alt30 = np.asarray(sp30["altitude"].transpose("time", "y", "x").values, dtype=np.float64)
    azi30 = np.asarray(sp30["azimuth"].transpose("time", "y", "x").values, dtype=np.float64)

    out = {"x": x, "y": y, "time_ns": pd.DatetimeIndex(time).as_unit("ns").asi8,
           "I_indptr": I.indptr, "I_indices": I.indices, "I_shape": np.array(I.shape),
           "index": np.array(index), "azimuth_raw": az_raw.values,
           "stored_alt": alt30, "stored_az": azi30}
    for k, v in F.items():
        out["in_" + k] = v
    for i, c in enumerate(lines):
        out[f"line_{i}"] = c

    def flat(alt, azi):
        f = {k: F[k].reshape(nt, -1) for k in ("temperature", "wnd100m", "wnd_azimuth", "influx_direct")}
        f["height"] = F["height"].reshape(-1)
        f["solar_altitude"], f["solar_azimuth"] = alt.reshape(nt, -1), azi.reshape(nt, -1)
        return f

    n = len(index)
    R_series = pd.Series(np.linspace(8e-5, 1.6e-4, n)[::-1], index=index[::-1])  # aligned by index
    D_series = pd.Series(np.linspace(0.02, 0.04, n), index=index)
    alpha_big = pd.Series(np.where(np.arange(n) == 1, 60.0, 0.6), index=index)  # line1: qs > qc + qr by day
    cases = {
        "computed": (flat(alt0, azi0), 9.39e-5, {}),
        "stored_f64": (flat(alt30, azi30), 9.39e-5, {}),
        "stored_f32": (flat(alt30.astype(np.float32), azi30.astype(np.float32)), 9.39e-5, {}),
        "series": (flat(alt30, azi30), R_series, {"D": D_series, "Ts": 363.0, "epsilon": 0.8}),
        "negative": (flat(alt0, azi0), 9.39e-5, {"D": 0.028, "Ts": 373.0, "epsilon": 0.6, "alpha": alpha_big}),
    }
    out["R_series_index"], out["R_series_values"] = np.array(list(R_series.index), dtype=str), R_series.values
    out["D_series_values"], out["alpha_big_values"] = D_series.values, alpha_big.values
    for name, (fl, R, params) in cases.items():
        out[f"out_{name}"] = glue(fl, I, az_raw, R, params)

    # convert_line_rating's dict branch on broadcast arrays (what the flat evaluator serves)
    rng = np.random.default_rng(5)
    m = 64
    d = {"temperature": rng.uniform(250, 310, m), "wnd100m": rng.uniform(0, 25, m),
         "height": rng.uniform(0, 2500, m), "wnd_azimuth": rng.uniform(0, 2 * np.pi, m),
         "influx_direct": rng.uniform(0, 1000, m), "solar_altitude": rng.uniform(-0.5, 1.5, m),
         "solar_azimuth": rng.uniform(0, 2 * np.pi, m)}
    psi = rng.uniform(0, 360, m)
    for k, v in d.items():
        out["flat_" + k] = v
    out["flat_psi"] = psi
    out["out_flat"] = conv.convert_line_rating(d, psi, 1e-4, D=0.03, Ts=368.0, epsilon=0.7, alpha=0.5)
    out["cases"] = np.array(list(cases))
    np.savez_compressed(os.path.join(HERE, "reference_line_rating.npz"), **out)
    print("wrote reference_line_rating.npz:", list(cases) + ["flat"])


if __name__ == "__main__":
    main()
