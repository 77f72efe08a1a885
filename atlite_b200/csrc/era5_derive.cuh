// era5_derive.cuh -- the per-value arithmetic of the ERA5 derivations (atlite/datasets/era5.py),
// shared by the prepare-time kernels (era5.cu) and the fused conversion kernels that read raw
// ERA5 variables directly (pv.cu, wind.cu, csp.cu, line_rating.cu).  One definition, so a raw cutout converted in one
// pass computes exactly what `era5.prepare` stores and the prepared cutout's conversion reads.
#pragma once

namespace atl {

constexpr float ERA5_TWO_PI_F = 6.283185307179586f;

// get_data_influx (:168 + :175) + sanitize_influx (:199-200) of the direct influx alone: fdir (an
// hourly J m-2 accumulation) in W m-2, clipped at 0 (NaN stays) when sanitizing
__device__ __forceinline__ float era5_direct(float fd, int sanitize) {
  const float inv_h = 1.0f / 3600.0f;
  fd = fd * inv_h;
  if (sanitize) fd = fd < 0.f ? 0.f : fd;
  return fd;
}

// get_data_influx (:163-175) + sanitize_influx (:195-201) of one value.  In: ssrd `sd`, ssr `sn`,
// and tisr / fdir in `ti` / `fd` (hourly J m-2 accumulations); out: influx_toa in `ti`,
// influx_direct in `fd`, influx_diffuse `df` (W m-2) and albedo `al`.
__device__ __forceinline__ void era5_influx(float sd, float sn, float& ti, float& fd, float& df, float& al,
                                            int sanitize) {
  const float inv_h = 1.0f / 3600.0f;
  // :164-167  ((ssrd - ssr) / ssrd.where(ssrd != 0)).fillna(0)
  const float a = (sd - sn) / sd;
  al = (sd != 0.f && a == a) ? a : 0.f;
  df = (sd - fd) * inv_h;                                             // :168 + :175
  fd = era5_direct(fd, sanitize);
  ti = ti * inv_h;
  if (sanitize) {                                                     // :199-200 clip(min = 0), NaN stays
    df = df < 0.f ? 0.f : df;
    ti = ti < 0.f ? 0.f : ti;
  }
}

// get_data_wind (:121): wind speed from its components
__device__ __forceinline__ float era5_wind_speed(float u, float v) { return sqrtf(u * u + v * v); }

// get_data_wind (:129-130): wind azimuth, 0 = north, pi/2 = east, mapped into [0, 2 pi) by
// .where(az >= 0, az + 2 pi) (NaN stays NaN)
__device__ __forceinline__ float era5_wind_azimuth(float u, float v) {
  const float a = atan2f(u, v);
  return (a >= 0.f || a != a) ? a : a + ERA5_TWO_PI_F;
}

// get_data_wind (:124-126): shear exponent ln(w10 / w100) / ln(10 / 100), inv_ln = 1 / ln(10 / 100)
__device__ __forceinline__ float era5_shear(float w10, float w100, float inv_ln) {
  return logf(w10 / w100) * inv_ln;
}

// sanitize_wind (:145): roughness < 0 -> 2e-4 (NaN -> 2e-4 like .where)
__device__ __forceinline__ float era5_roughness(float z) { return (z >= 0.f) ? z : 2e-4f; }

}  // namespace atl
