// proj.cuh -- EPSG:3035 (ETRS89-LAEA, EPSG method 9820) on the device, float64, for pixel centres.
// The constants come from the host (AtlLaea, filled from atlite_b200/proj.py), so host-projected
// polygon vertices and device-projected centres use the same ellipsoid and origin.
#pragma once
#include <cuda_runtime.h>

#include "../../include/atlite_b200.h"

namespace atl {

constexpr double kDeg = 0.017453292519943295;  // pi / 180

// authalic q(phi) from s = sin(phi)
__device__ __forceinline__ double laea_q(const AtlLaea& P, double s) {
  return (1.0 - P.e2) * (s / (1.0 - P.e2 * s * s) - log((1.0 - P.e * s) / (1.0 + P.e * s)) / (2.0 * P.e));
}

// degrees -> metres
__device__ __forceinline__ void laea_forward(const AtlLaea& P, double lon, double lat, double& x, double& y) {
  const double q = laea_q(P, sin(lat * kDeg));
  const double beta = asin(fmin(fmax(q / P.qp, -1.0), 1.0));
  const double dl = lon * kDeg - P.lam0;
  double sb, cb, sdl, cdl;
  sincos(beta, &sb, &cb);
  sincos(dl, &sdl, &cdl);
  const double B = P.rq * sqrt(2.0 / (1.0 + P.sin_b0 * sb + P.cos_b0 * cb * cdl));
  x = P.fe + (B * P.d) * cb * sdl;
  y = P.fn + (B / P.d) * (P.cos_b0 * sb - P.sin_b0 * cb * cdl);
}

// metres -> degrees: authalic latitude from the inverse azimuthal formulas, then the three-term
// series to geodetic latitude and P.newton Newton steps on q(phi) (Snyder 1987, eq. 3-16).
__device__ __forceinline__ void laea_inverse(const AtlLaea& P, double x, double y, double& lon, double& lat) {
  x -= P.fe;
  y -= P.fn;
  const double rho = sqrt((x / P.d) * (x / P.d) + (P.d * y) * (P.d * y));
  const double C = 2.0 * asin(fmin(rho / (2.0 * P.rq), 1.0));
  double sC, cC;
  sincos(C, &sC, &cC);
  const double sbeta = rho == 0.0 ? P.sin_b0 : cC * P.sin_b0 + P.d * y * sC * P.cos_b0 / rho;
  const double beta = asin(fmin(fmax(sbeta, -1.0), 1.0));
  const double lam = P.lam0 + atan2(x * sC, P.d * rho * P.cos_b0 * cC - P.d * P.d * y * P.sin_b0 * sC);
  const double q = P.qp * sin(beta);
  double phi = beta + P.s1 * sin(2.0 * beta) + P.s2 * sin(4.0 * beta) + P.s3 * sin(6.0 * beta);
  for (int k = 0; k < P.newton; ++k) {
    double s, c;
    sincos(phi, &s, &c);
    const double w = 1.0 - P.e2 * s * s;
    if (c == 0.0) c = 1e-300;
    phi += w * w / (2.0 * c) * (q / (1.0 - P.e2) - s / w + log((1.0 - P.e * s) / (1.0 + P.e * s)) / (2.0 * P.e));
  }
  lon = lam / kDeg;
  lat = phi / kDeg;
}

// A pixel centre taken from the lattice's CRS into the other one (ATL_PROJ_*).
__device__ __forceinline__ void project(int mode, const AtlLaea& P, double& x, double& y) {
  double u, v;
  if (mode == ATL_PROJ_LAEA_INVERSE) {
    laea_inverse(P, x, y, u, v);
  } else if (mode == ATL_PROJ_LAEA_FORWARD) {
    laea_forward(P, x, y, u, v);
  } else {
    return;
  }
  x = u;
  y = v;
}

}  // namespace atl
