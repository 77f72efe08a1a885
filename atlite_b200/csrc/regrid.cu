// regrid.cu -- resample (..., y, x) fields onto another regular grid of the same CRS (gis.py:791-871,
// rasterio's reproject with Resampling.average or .nearest).
//
// Both resamplings are separable: destination cell (i, j) takes source pixel (r, c) with weight
// wy[i, r] * wx[j, c], and
//   out[i, j] = sum_rc wy wx v[r, c] / sum_rc wy wx [v[r, c] is not NaN]       (NaN if the sum is 0).
// The per-axis tables {first source index, count, weights} are built once per grid pair on the host
// in float64 (gis.py here: padding, flipped axes and the nearest pick are folded into them), so the
// kernel only sees contiguous runs of real source indices.  nearest is the same sum with one weight
// of 1 per axis.
//
// One CTA owns one (band of RG_ROWS destination rows, tile of destination columns) and walks the
// batch (time steps) from blockIdx.y.  The band is a list of steps (source row, destination row,
// y weight), destination row by destination row.  For one batch entry the CTA streams the steps'
// source rows through a ring of RG_STAGES shared-memory row buffers with cp.async, so each source
// element leaves HBM once apart from the rows two destination rows share.  Thread j reduces each
// buffered row along x for its destination column (sum and valid weight) and adds the pair, times
// the y weight, into one pair of accumulators, written out when its destination row ends.
// Everything accumulates in float64 in a fixed order, so the result does not depend on the launch
// and is bitwise repeatable.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace atl {

constexpr int RG_THREADS = 128;  // destination columns per CTA at most; every thread also loads
constexpr int RG_ROWS = 8;       // destination rows per band
constexpr int RG_STAGES = 4;     // source rows in flight per CTA
constexpr size_t RG_SMEM_MAX = 160 * 1024;

struct RegridTables {
  const int32_t* xfirst;  // (nx_dst) first source column of destination column j, its count, and
  const int32_t* xcount;  // weights xw[j * kx + k] for columns xfirst[j] + k
  const double* xw;
  const int32_t* band_ptr;  // (n_bands + 1) CSR over the steps
  const int32_t* step_row;  // source row of a step (-1: a destination row no source row reaches)
  const int32_t* step_t;    // destination row of a step within its band; a band's steps ascend in it
  const double* step_w;     // y weight of a step
  const int32_t* tile_lo;   // (n_ctiles) first source column a column tile reads, and its span
  const int32_t* tile_span;
  int ny_dst, nx_dst, kx, tj, n_ctiles;
};

__device__ __forceinline__ void cp_async(void* smem, const float* g) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(s), "l"(g));
}
__device__ __forceinline__ void cp_async(void* smem, const double* g) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(s), "l"(g));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// Shared memory: the tile's x weights (kx * tj, k-major so a warp's reads are conflict-free), then
// RG_STAGES row buffers of max_span elements.  blockDim.x is tj rounded up to a warp.
template <typename T>
__global__ void __launch_bounds__(RG_THREADS) k_regrid(const T* __restrict__ src, int64_t batch, int64_t src_row,
                                                       int64_t src_batch, RegridTables tb, int max_span,
                                                       T* __restrict__ out) {
  extern __shared__ double smem[];
  double* s_xw = smem;
  T* s_buf = reinterpret_cast<T*>(s_xw + (size_t)tb.kx * tb.tj);

  const int tid = threadIdx.x, nthr = blockDim.x;
  const int ctile = blockIdx.x % tb.n_ctiles;
  const int band = blockIdx.x / tb.n_ctiles;
  const int j0 = ctile * tb.tj, i0 = band * RG_ROWS;
  const int c_lo = tb.tile_lo[ctile], span = tb.tile_span[ctile];
  const int e0 = tb.band_ptr[band], ne = tb.band_ptr[band + 1] - e0;
  const int32_t* __restrict__ srow = tb.step_row + e0;
  const int32_t* __restrict__ st = tb.step_t + e0;
  const double* __restrict__ sw = tb.step_w + e0;

  for (int e = tid; e < tb.kx * tb.tj; e += nthr) {
    const int k = e / tb.tj, j = j0 + e % tb.tj;
    s_xw[e] = (j < tb.nx_dst && k < tb.xcount[j]) ? tb.xw[(int64_t)j * tb.kx + k] : 0.0;
  }
  const int j = j0 + tid;
  const bool active = tid < tb.tj && j < tb.nx_dst;
  const int my_first = active ? tb.xfirst[j] - c_lo : 0;
  const int my_count = active ? tb.xcount[j] : 0;
  __syncthreads();

  for (int64_t b = blockIdx.y; b < batch; b += gridDim.y) {
    const T* sb = src + b * src_batch + c_lo;
    T* ob = out + (b * tb.ny_dst + i0) * (int64_t)tb.nx_dst + j;
    auto issue = [&](int q) {  // the source row of step q -> ring slot q % RG_STAGES
      if (q < ne && srow[q] >= 0) {
        const T* g = sb + (int64_t)srow[q] * src_row;
        T* s = s_buf + (size_t)(q % RG_STAGES) * max_span;
        for (int c = tid; c < span; c += nthr) cp_async(s + c, g + c);
      }
      cp_async_commit();  // an empty group keeps the wait count below uniform
    };
#pragma unroll
    for (int q = 0; q < RG_STAGES - 1; ++q) issue(q);
    double acc_s = 0.0, acc_w = 0.0;
    for (int q = 0; q < ne; ++q) {
      cp_async_wait<RG_STAGES - 2>();
      __syncthreads();  // step q's row is in place for every thread; slot (q - 1) % RG_STAGES is free again
      issue(q + RG_STAGES - 1);
      if (srow[q] >= 0) {
        const T* row = s_buf + (size_t)(q % RG_STAGES) * max_span + my_first;
        double s = 0.0, w = 0.0;
        for (int k = 0; k < my_count; ++k) {
          const double v = (double)row[k];
          if (v == v) {
            const double wk = s_xw[k * tb.tj + tid];
            s = fma(wk, v, s);
            w += wk;
          }
        }
        const double wy = sw[q];
        acc_s = fma(wy, s, acc_s);
        acc_w = fma(wy, w, acc_w);
      }
      if (q + 1 == ne || st[q + 1] != st[q]) {  // the destination row is complete
        if (active) ob[(int64_t)st[q] * tb.nx_dst] = acc_w > 0.0 ? (T)(acc_s / acc_w) : (T)NAN;
        acc_s = acc_w = 0.0;
      }
    }
    cp_async_wait<0>();
    __syncthreads();  // every thread is done with the ring before the next batch entry refills it
  }
}

struct RegridPlan {
  int device;
  int ny_src, nx_src;
  RegridTables tb;
  int n_bands, max_span;
  void* dmem;  // one allocation holding every table
};

size_t regrid_smem(const RegridPlan& p, size_t elem) {
  return sizeof(double) * (size_t)p.tb.kx * p.tb.tj + elem * RG_STAGES * (size_t)p.max_span;
}

template <typename T>
int regrid_run(const RegridPlan* p, int64_t batch, const T* src, int64_t src_row, int64_t src_batch, T* out,
               void* stream) {
  ATL_REQUIRE(p, "NULL plan");
  ATL_REQUIRE(batch >= 0, "negative batch");
  if (batch == 0 || p->tb.ny_dst == 0 || p->tb.nx_dst == 0) return ATL_OK;
  ATL_REQUIRE(src && out, "NULL argument");
  ATL_REQUIRE(src_row >= p->nx_src && src_batch >= src_row * p->ny_src, "source strides smaller than its rows");
  ATL_CUDA(cudaSetDevice(p->device));
  const size_t smem = regrid_smem(*p, sizeof(T));
  ATL_CUDA(cudaFuncSetAttribute(k_regrid<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const dim3 grid((unsigned)(p->n_bands * p->tb.n_ctiles), (unsigned)(batch < 65535 ? batch : 65535));
  const int threads = (p->tb.tj + 31) / 32 * 32;
  k_regrid<T><<<grid, threads, smem, (cudaStream_t)stream>>>(src, batch, src_row, src_batch, p->tb, p->max_span, out);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

}  // namespace atl

using namespace atl;

extern "C" {

int atl_regrid_create(int device, int32_t ny_src, int32_t nx_src, int32_t ny_dst, int32_t nx_dst, int32_t ky,
                      const int32_t* yfirst, const int32_t* ycount, const double* yw, int32_t kx,
                      const int32_t* xfirst, const int32_t* xcount, const double* xw, void** out) {
  ATL_REQUIRE(out, "NULL output handle");
  *out = nullptr;
  ATL_REQUIRE(ny_src > 0 && nx_src > 0 && ny_dst >= 0 && nx_dst >= 0 && ky >= 1 && kx >= 1, "bad size");
  ATL_REQUIRE(yfirst && ycount && yw && xfirst && xcount && xw, "NULL table");
  for (int32_t i = 0; i < ny_dst; ++i)
    ATL_REQUIRE(ycount[i] >= 0 && ycount[i] <= ky && (ycount[i] == 0 || (yfirst[i] >= 0 && yfirst[i] + ycount[i] <= ny_src)),
                "y table entry outside the source rows");
  for (int32_t j = 0; j < nx_dst; ++j)
    ATL_REQUIRE(xcount[j] >= 0 && xcount[j] <= kx && (xcount[j] == 0 || (xfirst[j] >= 0 && xfirst[j] + xcount[j] <= nx_src)),
                "x table entry outside the source columns");

  RegridPlan p{};
  p.device = device;
  p.ny_src = ny_src;
  p.nx_src = nx_src;
  p.tb.ny_dst = ny_dst;
  p.tb.nx_dst = nx_dst;
  p.tb.kx = kx;

  // bands: their steps, destination row by destination row
  p.n_bands = (ny_dst + RG_ROWS - 1) / RG_ROWS;
  std::vector<int32_t> band_ptr(1, 0), step_row, step_t;
  std::vector<double> step_w;
  for (int bnd = 0; bnd < p.n_bands; ++bnd) {
    for (int i = bnd * RG_ROWS; i < std::min(ny_dst, (bnd + 1) * RG_ROWS); ++i) {
      for (int k = 0; k < std::max(ycount[i], 1); ++k) {
        step_row.push_back(ycount[i] ? yfirst[i] + k : -1);
        step_t.push_back(i - bnd * RG_ROWS);
        step_w.push_back(ycount[i] ? yw[(size_t)i * ky + k] : 0.0);
      }
    }
    band_ptr.push_back((int32_t)step_row.size());
  }
  // column tiles: as few as RG_THREADS allows, split further until the row ring fits in shared memory
  std::vector<int32_t> tile_lo, tile_span;
  for (int n_ct = nx_dst ? (nx_dst + RG_THREADS - 1) / RG_THREADS : 1;; ++n_ct) {
    p.tb.n_ctiles = n_ct;
    p.tb.tj = nx_dst ? (nx_dst + n_ct - 1) / n_ct : 1;
    tile_lo.assign(n_ct, 0);
    tile_span.assign(n_ct, 0);
    p.max_span = 1;
    for (int t = 0; t < n_ct; ++t) {
      int lo = nx_src, hi = 0;
      for (int j = t * p.tb.tj; j < std::min(nx_dst, (t + 1) * p.tb.tj); ++j)
        if (xcount[j] > 0) {
          lo = std::min(lo, xfirst[j]);
          hi = std::max(hi, xfirst[j] + xcount[j]);
        }
      tile_lo[t] = hi > lo ? lo : 0;
      tile_span[t] = hi > lo ? hi - lo : 0;
      p.max_span = std::max(p.max_span, tile_span[t]);
    }
    if (regrid_smem(p, sizeof(double)) <= RG_SMEM_MAX) break;
    ATL_REQUIRE(p.tb.tj > 1, "a destination cell spans more source columns than shared memory holds");
  }

  // one device block: int32 tables first, then the float64 weights (8-byte aligned)
  const size_t n_int = 2 * (size_t)nx_dst + band_ptr.size() + 2 * step_row.size() + 2 * tile_lo.size();
  const size_t int_bytes = (n_int * sizeof(int32_t) + 7) & ~(size_t)7;
  const size_t bytes = int_bytes + sizeof(double) * ((size_t)nx_dst * kx + step_w.size());
  std::vector<char> h(bytes, 0);
  int32_t* hi = reinterpret_cast<int32_t*>(h.data());
  size_t off = 0;
  auto put_i = [&](const int32_t* a, size_t n) {
    if (n) memcpy(hi + off, a, n * sizeof(int32_t));
    off += n;
    return off - n;
  };
  const size_t o_xf = put_i(xfirst, nx_dst), o_xc = put_i(xcount, nx_dst), o_bp = put_i(band_ptr.data(), band_ptr.size()),
               o_sr = put_i(step_row.data(), step_row.size()), o_st = put_i(step_t.data(), step_t.size()),
               o_tl = put_i(tile_lo.data(), tile_lo.size()), o_ts = put_i(tile_span.data(), tile_span.size());
  double* hd = reinterpret_cast<double*>(h.data() + int_bytes);
  if (nx_dst) memcpy(hd, xw, sizeof(double) * nx_dst * kx);
  if (!step_w.empty()) memcpy(hd + (size_t)nx_dst * kx, step_w.data(), sizeof(double) * step_w.size());

  ATL_CUDA(cudaSetDevice(device));
  void* d = nullptr;
  ATL_CUDA(cudaMalloc(&d, bytes));
  cudaError_t e = cudaMemcpy(d, h.data(), bytes, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    cudaFree(d);
    return cuda_fail(e, "cudaMemcpy(regrid tables)");
  }
  const int32_t* di = reinterpret_cast<const int32_t*>(d);
  const double* dd = reinterpret_cast<const double*>(static_cast<char*>(d) + int_bytes);
  p.tb.xfirst = di + o_xf;
  p.tb.xcount = di + o_xc;
  p.tb.band_ptr = di + o_bp;
  p.tb.step_row = di + o_sr;
  p.tb.step_t = di + o_st;
  p.tb.tile_lo = di + o_tl;
  p.tb.tile_span = di + o_ts;
  p.tb.xw = dd;
  p.tb.step_w = dd + (size_t)nx_dst * kx;
  p.dmem = d;
  *out = new RegridPlan(p);
  return ATL_OK;
}

int atl_regrid_info(const void* plan, int32_t* n_bands, int32_t* n_ctiles, int32_t* tile_cols, int32_t* max_span) {
  ATL_REQUIRE(plan, "NULL plan");
  const RegridPlan* p = static_cast<const RegridPlan*>(plan);
  if (n_bands) *n_bands = p->n_bands;
  if (n_ctiles) *n_ctiles = p->tb.n_ctiles;
  if (tile_cols) *tile_cols = p->tb.tj;
  if (max_span) *max_span = p->max_span;
  return ATL_OK;
}

int atl_regrid_f32(const void* plan, int64_t batch, const float* src_dev, int64_t src_row, int64_t src_batch,
                   float* out_dev, void* stream) {
  return regrid_run(static_cast<const RegridPlan*>(plan), batch, src_dev, src_row, src_batch, out_dev, stream);
}

int atl_regrid_f64(const void* plan, int64_t batch, const double* src_dev, int64_t src_row, int64_t src_batch,
                   double* out_dev, void* stream) {
  return regrid_run(static_cast<const RegridPlan*>(plan), batch, src_dev, src_row, src_batch, out_dev, stream);
}

void atl_regrid_destroy(void* plan) {
  if (!plan) return;
  RegridPlan* p = static_cast<RegridPlan*>(plan);
  cudaSetDevice(p->device);
  cudaFree(p->dmem);
  delete p;
}

}  // extern "C"
