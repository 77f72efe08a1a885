// era5.cu -- prepare-time derivations of an ERA5 cutout as streaming kernels
// (SURVEY section 8 f4): the arithmetic of atlite/datasets/era5.py
//   get_data_wind   :120-135  wind speed from (u, v), shear exponent, azimuth
//   sanitize_wind   :141-146  negative roughness -> 2e-4
//   get_data_influx :163-175  albedo, diffuse = ssrd - fdir, J m-2 -> W m-2
//   sanitize_influx :195-201  clip(min = 0)
//   get_data_influx :182-188  SolarPosition(ds, time_shift = -30 min) stored in the cutout
//                             (pv/solar_position.py:69-116)
// so that raw downloads (u100, v100, ..., ssrd, fdir, ...) become a device-resident
// cutout without a pass over host memory.  Pure HBM streams: wind 20 B in / 16 B
// out, influx 16 B in / 16 B out per cell-step; the solar position writes two
// float64 values per cell-step from per-step / per-row / per-column tables.
#include <cmath>
#include <vector>

#include "common.cuh"
#include "era5_derive.cuh"
#include "solar_host.cuh"

namespace atl {

struct WindRaw {
  const float *u100, *v100, *u10, *v10, *fsr;
};
struct WindOut {
  float *wnd100m, *shear, *azimuth, *roughness;
};

template <int V>  // V = 4: 128-bit accesses, V = 1: scalar tail / unaligned
__device__ __forceinline__ void wind_elem(const WindRaw& in, const WindOut& out, int64_t i,
                                          float inv_ln, int sanitize) {
  float u1[V], v1[V], u0[V], v0[V], z[V], w[V], sh[V], az[V];
  if (V == 4) {
    *reinterpret_cast<float4*>(u1) = __ldg(reinterpret_cast<const float4*>(in.u100 + i));
    *reinterpret_cast<float4*>(v1) = __ldg(reinterpret_cast<const float4*>(in.v100 + i));
    *reinterpret_cast<float4*>(u0) = __ldg(reinterpret_cast<const float4*>(in.u10 + i));
    *reinterpret_cast<float4*>(v0) = __ldg(reinterpret_cast<const float4*>(in.v10 + i));
    *reinterpret_cast<float4*>(z) = __ldg(reinterpret_cast<const float4*>(in.fsr + i));
  } else {
    u1[0] = in.u100[i];
    v1[0] = in.v100[i];
    u0[0] = in.u10[i];
    v0[0] = in.v10[i];
    z[0] = in.fsr[i];
  }
#pragma unroll
  for (int k = 0; k < V; ++k) {
    w[k] = era5_wind_speed(u1[k], v1[k]);                               // :121
    sh[k] = era5_shear(era5_wind_speed(u0[k], v0[k]), w[k], inv_ln);    // :124-126
    az[k] = era5_wind_azimuth(u1[k], v1[k]);                            // :129-130
    if (sanitize) z[k] = era5_roughness(z[k]);                          // :145
  }
  if (V == 4) {
    *reinterpret_cast<float4*>(out.wnd100m + i) = *reinterpret_cast<float4*>(w);
    *reinterpret_cast<float4*>(out.shear + i) = *reinterpret_cast<float4*>(sh);
    *reinterpret_cast<float4*>(out.azimuth + i) = *reinterpret_cast<float4*>(az);
    *reinterpret_cast<float4*>(out.roughness + i) = *reinterpret_cast<float4*>(z);
  } else {
    out.wnd100m[i] = w[0];
    out.shear[i] = sh[0];
    out.azimuth[i] = az[0];
    out.roughness[i] = z[0];
  }
}

__global__ void k_era5_wind(WindRaw in, WindOut out, int64_t n, float inv_ln, int sanitize, int vec) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n4 = vec ? n / 4 : 0;
  for (int64_t q = i; q < n4; q += stride) wind_elem<4>(in, out, q * 4, inv_ln, sanitize);
  for (int64_t q = n4 * 4 + i; q < n; q += stride) wind_elem<1>(in, out, q, inv_ln, sanitize);
}

struct InfluxRaw {
  const float *ssrd, *ssr, *tisr, *fdir;
};
struct InfluxOut {
  float *toa, *direct, *diffuse, *albedo;
};

template <int V>
__device__ __forceinline__ void influx_elem(const InfluxRaw& in, const InfluxOut& out, int64_t i,
                                            int sanitize) {
  float sd[V], sn[V], ti[V], fd[V], al[V], df[V];
  if (V == 4) {
    *reinterpret_cast<float4*>(sd) = __ldg(reinterpret_cast<const float4*>(in.ssrd + i));
    *reinterpret_cast<float4*>(sn) = __ldg(reinterpret_cast<const float4*>(in.ssr + i));
    *reinterpret_cast<float4*>(ti) = __ldg(reinterpret_cast<const float4*>(in.tisr + i));
    *reinterpret_cast<float4*>(fd) = __ldg(reinterpret_cast<const float4*>(in.fdir + i));
  } else {
    sd[0] = in.ssrd[i];
    sn[0] = in.ssr[i];
    ti[0] = in.tisr[i];
    fd[0] = in.fdir[i];
  }
#pragma unroll
  for (int k = 0; k < V; ++k) era5_influx(sd[k], sn[k], ti[k], fd[k], df[k], al[k], sanitize);
  if (V == 4) {
    *reinterpret_cast<float4*>(out.toa + i) = *reinterpret_cast<float4*>(ti);
    *reinterpret_cast<float4*>(out.direct + i) = *reinterpret_cast<float4*>(fd);
    *reinterpret_cast<float4*>(out.diffuse + i) = *reinterpret_cast<float4*>(df);
    *reinterpret_cast<float4*>(out.albedo + i) = *reinterpret_cast<float4*>(al);
  } else {
    out.toa[i] = ti[0];
    out.direct[i] = fd[0];
    out.diffuse[i] = df[0];
    out.albedo[i] = al[0];
  }
}

__global__ void k_era5_influx(InfluxRaw in, InfluxOut out, int64_t n, int sanitize, int vec) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n4 = vec ? n / 4 : 0;
  for (int64_t q = i; q < n4; q += stride) influx_elem<4>(in, out, q * 4, sanitize);
  for (int64_t q = n4 * 4 + i; q < n; q += stride) influx_elem<1>(in, out, q, sanitize);
}

// pv/solar_position.py:95-114 for every (t, y, x) in float64 from the per-step tables
// {sin dec, cos dec, H0 = radians(lmst at lon 0) - ra}, per-row {sin lat, cos lat}
// and per-column lon (rad).
__global__ void k_solar_position(const double* __restrict__ tt /* 3 * nt */,
                                 const double* __restrict__ lat_sc /* 2 * ny */,
                                 const double* __restrict__ lon /* nx */, int nt, int ny, int nx,
                                 double* __restrict__ alt_out, double* __restrict__ az_out) {
  const double PI = 3.14159265358979323846;
  const int64_t plane = (int64_t)ny * nx;
  const int64_t n = (int64_t)nt * plane;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int t = (int)(i / plane);
    const int r = (int)(i - (int64_t)t * plane);
    const int y = r / nx, x = r - y * nx;
    const double sd = tt[3 * t], cd = tt[3 * t + 1], H0 = tt[3 * t + 2];
    const double sl = lat_sc[2 * y], cl = lat_sc[2 * y + 1];
    double h = fmod(H0 + lon[x] + PI, 2.0 * PI);  // python %: result in [0, 2 pi)
    if (h < 0.0) h += 2.0 * PI;
    h -= PI;                                                                          // :95
    const double ch = cos(h);
    const double alt = asin(fmin(fmax(sd * sl + cd * cl * ch, -1.0), 1.0));          // :103-105
    double az = acos(fmin(fmax((sd * cl - cd * sl * ch) / cos(alt), -1.0), 1.0));    // :109-113
    if (h > 0.0) az = 2.0 * PI - az;                                                  // :114
    alt_out[i] = alt;
    az_out[i] = az;
  }
}

static int grid_for(int64_t work, int threads) {
  int64_t blocks = (work + threads - 1) / threads;
  const int64_t cap = (int64_t)sm_count() * 16;  // grid-stride loops: a few waves of resident CTAs
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

static bool all_aligned16(std::initializer_list<const void*> ps) {
  for (const void* p : ps)
    if (reinterpret_cast<uintptr_t>(p) & 15u) return false;
  return true;
}

}  // namespace atl

using namespace atl;

extern "C" {

int atl_era5_wind(int device, int64_t n, const float* u100, const float* v100, const float* u10,
                  const float* v10, const float* fsr, int32_t sanitize, float* wnd100m,
                  float* wnd_shear_exp, float* wnd_azimuth, float* roughness, void* stream) {
  ATL_REQUIRE(n >= 0, "negative size");
  if (n == 0) return ATL_OK;
  ATL_REQUIRE(u100 && v100 && u10 && v10 && fsr && wnd100m && wnd_shear_exp && wnd_azimuth && roughness,
              "NULL argument");
  ATL_CUDA(cudaSetDevice(device));
  const int vec = all_aligned16({u100, v100, u10, v10, fsr, wnd100m, wnd_shear_exp, wnd_azimuth, roughness});
  const float inv_ln = (float)(1.0 / std::log(10.0 / 100.0));
  k_era5_wind<<<grid_for(vec ? (n + 3) / 4 : n, 256), 256, 0, (cudaStream_t)stream>>>(
      WindRaw{u100, v100, u10, v10, fsr}, WindOut{wnd100m, wnd_shear_exp, wnd_azimuth, roughness}, n,
      inv_ln, sanitize, vec);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

int atl_era5_influx(int device, int64_t n, const float* ssrd, const float* ssr, const float* tisr,
                    const float* fdir, int32_t sanitize, float* influx_toa, float* influx_direct,
                    float* influx_diffuse, float* albedo, void* stream) {
  ATL_REQUIRE(n >= 0, "negative size");
  if (n == 0) return ATL_OK;
  ATL_REQUIRE(ssrd && ssr && tisr && fdir && influx_toa && influx_direct && influx_diffuse && albedo,
              "NULL argument");
  ATL_CUDA(cudaSetDevice(device));
  const int vec = all_aligned16({ssrd, ssr, tisr, fdir, influx_toa, influx_direct, influx_diffuse, albedo});
  k_era5_influx<<<grid_for(vec ? (n + 3) / 4 : n, 256), 256, 0, (cudaStream_t)stream>>>(
      InfluxRaw{ssrd, ssr, tisr, fdir}, InfluxOut{influx_toa, influx_direct, influx_diffuse, albedo}, n,
      sanitize, vec);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

int atl_solar_position(int device, const int64_t* time_ns_host, int64_t nt, int64_t time_shift_ns,
                       const double* lon_deg_host, int32_t nx, const double* lat_deg_host, int32_t ny,
                       double* altitude_dev, double* azimuth_dev, void* stream) {
  ATL_REQUIRE(nt >= 0 && nx > 0 && ny > 0, "bad shape");
  if (nt == 0) return ATL_OK;
  ATL_REQUIRE(time_ns_host && lon_deg_host && lat_deg_host && altitude_dev && azimuth_dev, "NULL argument");
  ATL_REQUIRE(nt < (1LL << 31), "time axis too long");
  ATL_CUDA(cudaSetDevice(device));
  const double D2R = 3.14159265358979323846 / 180.0;
  std::vector<double> tt, lat_sc((size_t)2 * ny), lon((size_t)nx);
  solar_almanac_f64(time_ns_host, nt, time_shift_ns, tt);
  for (int y = 0; y < ny; ++y) {
    lat_sc[2 * (size_t)y] = std::sin(lat_deg_host[y] * D2R);
    lat_sc[2 * (size_t)y + 1] = std::cos(lat_deg_host[y] * D2R);
  }
  for (int x = 0; x < nx; ++x) lon[(size_t)x] = lon_deg_host[x] * D2R;
  cudaStream_t st = (cudaStream_t)stream;
  double *d_tt = nullptr, *d_lat = nullptr, *d_lon = nullptr;
  ATL_CUDA(cudaMallocAsync((void**)&d_tt, tt.size() * 8, st));
  ATL_CUDA(cudaMallocAsync((void**)&d_lat, lat_sc.size() * 8, st));
  ATL_CUDA(cudaMallocAsync((void**)&d_lon, lon.size() * 8, st));
  ATL_CUDA(cudaMemcpyAsync(d_tt, tt.data(), tt.size() * 8, cudaMemcpyHostToDevice, st));
  ATL_CUDA(cudaMemcpyAsync(d_lat, lat_sc.data(), lat_sc.size() * 8, cudaMemcpyHostToDevice, st));
  ATL_CUDA(cudaMemcpyAsync(d_lon, lon.data(), lon.size() * 8, cudaMemcpyHostToDevice, st));
  ATL_CUDA(cudaStreamSynchronize(st));  // the host vectors go out of scope
  k_solar_position<<<grid_for(nt * (int64_t)ny * nx, 256), 256, 0, st>>>(d_tt, d_lat, d_lon, (int)nt, ny, nx,
                                                                       altitude_dev, azimuth_dev);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  cudaFreeAsync(d_tt, st);
  cudaFreeAsync(d_lat, st);
  cudaFreeAsync(d_lon, st);
  return ATL_OK;
}

}  // extern "C"
