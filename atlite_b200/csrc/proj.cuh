// proj.cuh -- the availability path's CRSs on the device, float64, for pixel centres: EPSG:3035
// (ETRS89-LAEA, EPSG method 9820), EPSG:3857 (spherical Mercator) and ESRI:54009 (spherical
// Mollweide), each to and from EPSG:4326 degrees.  The constants come from the host (AtlProjection,
// filled by atlite_b200/proj.py device_projection), so host-projected polygon vertices and
// device-projected centres use the same ellipsoid, sphere and origin.  A point without an image
// becomes NaN.
#pragma once
#include <cuda_runtime.h>
#include <math_constants.h>

#include "../../include/atlite_b200.h"

namespace atl {

constexpr double kDeg = 0.017453292519943295;  // pi / 180

// x = c + k * a, each product and sum rounded (as NumPy computes a transform's points); a pixel
// centre is k = i + 0.5, which is exact
__device__ __forceinline__ double lattice_point(double c, double a, double k) { return __dadd_rn(c, __dmul_rn(k, a)); }

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

// degrees -> metres; NaN at the poles
__device__ __forceinline__ void mercator_forward(const AtlCrs& C, double lon, double lat, double& x, double& y) {
  const bool ok = fabs(lat) < 90.0;
  x = ok ? C.r * (lon * kDeg) : CUDART_NAN;
  y = ok ? C.r * asinh(tan(lat * kDeg)) : CUDART_NAN;
}

constexpr double kPi = 3.141592653589793;
constexpr double kHalfPi = 1.5707963267948966;
constexpr double kHalfPiLo = 6.123233995736766e-17;  // pi / 2 - kHalfPi
constexpr double kSqrt2 = 1.4142135623730951;
constexpr double kEdge = 1e-12;  // map edges' slack (proj.EDGE)

// metres -> degrees; NaN off the map
__device__ __forceinline__ void mercator_inverse(const AtlCrs& C, double x, double y, double& lon, double& lat) {
  const bool ok = fabs(x) <= kPi * C.r * (1.0 + kEdge);
  lon = ok ? fmin(fmax(x / C.r, -kPi), kPi) / kDeg : CUDART_NAN;
  lat = ok ? atan(sinh(y / C.r)) / kDeg : CUDART_NAN;
}

// 2 d - sin 2 d for d in [0, pi / 2]: the sine's Taylor tail below 2 d = 1 (no cancellation)
__device__ __forceinline__ double sin_tail(double d) {
  const double u = 2.0 * d;
  if (u >= 1.0) return u - sin(u);
  const double v = u * u;
  double p = 1.0 / 355687428096000.0;
  p = 1.0 / 1307674368000.0 - v * p;
  p = 1.0 / 6227020800.0 - v * p;
  p = 1.0 / 39916800.0 - v * p;
  p = 1.0 / 362880.0 - v * p;
  p = 1.0 / 5040.0 - v * p;
  p = 1.0 / 120.0 - v * p;
  p = 1.0 / 6.0 - v * p;
  return u * v * p;
}

// degrees -> metres.  delta = pi / 2 - |theta| solves 2 delta - sin 2 delta = 2 pi sin^2(eps / 2),
// eps = pi / 2 - |phi| (proj.mollweide_delta): the polar asymptote as the start, then C.newton
// Newton steps.
__device__ __forceinline__ void mollweide_forward(const AtlCrs& C, double lon, double lat, double& x, double& y) {
  if (!(fabs(lat) <= 90.0)) {
    x = y = CUDART_NAN;
    return;
  }
  const double phi = lat * kDeg, a = fabs(phi);
  const double eps = a >= kHalfPi ? 0.0 : (kHalfPi - a) + kHalfPiLo;
  const double s = sin(0.5 * eps);
  const double rhs = 2.0 * kPi * s * s;
  double d = cbrt(0.75 * rhs);
  for (int k = 0; k < C.newton; ++k) {
    const double sd = sin(d);
    const double gp = 4.0 * sd * sd;
    if (gp > 0.0) d -= (sin_tail(d) - rhs) / gp;
    d = fmin(fmax(d, 0.0), kHalfPi);
  }
  double sd, cd;
  sincos(d, &sd, &cd);
  x = (2.0 * kSqrt2 / kPi) * C.r * (lon * kDeg) * sd;
  y = copysign(kSqrt2 * C.r * cd, phi);
}

// metres -> degrees; NaN outside the ellipse x^2 / (8 r^2) + y^2 / (2 r^2) <= 1 (+ kEdge)
__device__ __forceinline__ void mollweide_inverse(const AtlCrs& C, double x, double y, double& lon, double& lat) {
  double s = y / (kSqrt2 * C.r);
  const double t = x / (2.0 * kSqrt2 * C.r);
  if (!(t * t + s * s <= 1.0 + kEdge)) {
    lon = lat = CUDART_NAN;
    return;
  }
  s = fmin(fmax(s, -1.0), 1.0);
  const double c = sqrt((1.0 - s) * (1.0 + s));
  const double lam = c > 0.0 ? fmin(fmax(kPi * t / c, -kPi), kPi) : 0.0;
  // the latitude through delta = pi / 2 - |theta|, precise at the poles (proj.mollweide_inverse)
  const double eps = 2.0 * asin(sqrt(sin_tail(atan2(c, fabs(s))) / (2.0 * kPi)));
  lon = lam / kDeg;
  lat = copysign((kHalfPi - eps) + kHalfPiLo, s) / kDeg;
}

// A lattice point taken from p.from into p.to, FROM and TO being their kinds (ATL_CRS_*): the inverse
// of FROM to lon / lat, then the forward of TO, EPSG:4326 being the identity.  The pair is a template
// argument, so a kernel carries only the arithmetic (and the registers) of its own pair.
template <int FROM, int TO>
__device__ __forceinline__ void project(const AtlProjection& p, double& x, double& y) {
  if constexpr (FROM == TO) return;
  double u = x, v = y;
  if constexpr (FROM == ATL_CRS_LAEA) laea_inverse(p.laea, x, y, u, v);
  if constexpr (FROM == ATL_CRS_MERCATOR) mercator_inverse(p.from, x, y, u, v);
  if constexpr (FROM == ATL_CRS_MOLLWEIDE) mollweide_inverse(p.from, x, y, u, v);
  x = u;
  y = v;
  if constexpr (TO == ATL_CRS_LAEA) laea_forward(p.laea, u, v, x, y);
  if constexpr (TO == ATL_CRS_MERCATOR) mercator_forward(p.to, u, v, x, y);
  if constexpr (TO == ATL_CRS_MOLLWEIDE) mollweide_forward(p.to, u, v, x, y);
}

// Both CRSs of p are known kinds, with the sphere and Newton steps their formulas need
inline bool projection_ok(const AtlProjection& p) {
  const auto ok = [](const AtlCrs& C) {
    return C.kind == ATL_CRS_LONLAT || C.kind == ATL_CRS_LAEA ||
           ((C.kind == ATL_CRS_MERCATOR || C.kind == ATL_CRS_MOLLWEIDE) && C.r > 0.0 && C.newton >= 0 &&
            C.newton <= 64);
  };
  return ok(p.from) && ok(p.to);
}

// K<FROM, TO> for a runtime pair that passed projection_ok
template <template <int, int> class K, int FROM>
auto pair_kernel_to(int to) {
  switch (to) {
    case ATL_CRS_LAEA: return K<FROM, ATL_CRS_LAEA>::get();
    case ATL_CRS_MERCATOR: return K<FROM, ATL_CRS_MERCATOR>::get();
    case ATL_CRS_MOLLWEIDE: return K<FROM, ATL_CRS_MOLLWEIDE>::get();
    default: return K<FROM, ATL_CRS_LONLAT>::get();
  }
}
template <template <int, int> class K>
auto pair_kernel(int from, int to) {
  if (from == to) return K<ATL_CRS_LONLAT, ATL_CRS_LONLAT>::get();  // any CRS to itself: the identity
  switch (from) {
    case ATL_CRS_LAEA: return pair_kernel_to<K, ATL_CRS_LAEA>(to);
    case ATL_CRS_MERCATOR: return pair_kernel_to<K, ATL_CRS_MERCATOR>(to);
    case ATL_CRS_MOLLWEIDE: return pair_kernel_to<K, ATL_CRS_MOLLWEIDE>(to);
    default: return pair_kernel_to<K, ATL_CRS_LONLAT>(to);
  }
}

}  // namespace atl
