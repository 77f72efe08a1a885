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
// source rows through a ring of RG_STAGES shared-memory row buffers with 16-byte cp.async, so each
// source element leaves HBM once apart from the rows two destination rows share.  Thread j reduces
// each buffered row along x for its destination column (sum and valid weight) and adds the pair,
// times the y weight, into one pair of accumulators, written out when its destination row ends.
// Everything accumulates in float64 in a fixed order, so the result does not depend on the launch
// and is bitwise repeatable.
//
// The same kernel averages a 2-D int16 (or float) window of a terrain grid (GEBCO, gebco.py):
// values equal to the file's fill value are skipped like NaN, a cell with no valid value gets the
// fill value, integer results are rounded half away from zero, and a launch may cover only some
// bands, reading its source rows from a buffer that starts at source row row0 (host windows are
// streamed band by band).  gis.reproject within one CRS skips a nodata value the same way and gives
// an empty cell its own value (atl_regrid_nodata).
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

// A source row goes to its ring slot as the 16-byte-aligned chunks that cover it, so every element
// type (the 2-byte int16 of a terrain window too) moves with 16-byte cp.async: element k of the
// row lands at slot[phase + k], phase = (row address mod 16) / sizeof(T).  The chunks at the two
// ends also carry up to 15 bytes outside the row; an aligned 16-byte chunk never crosses a page,
// and it holds a byte of the row, so those bytes are mapped memory.  They are never used.
__device__ __forceinline__ void cp_async16(void* smem, const void* g) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(g));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

template <typename T>
__device__ __forceinline__ int row_phase(const T* g) {
  return (int)(((uintptr_t)g & 15) / sizeof(T));
}

// Bytes of one ring slot: a row span of max_span elements at any phase.
size_t regrid_slot_bytes(int max_span, size_t elem) { return ((size_t)max_span * elem + 15) / 16 * 16 + 16; }

// Values equal to `value` (when `on`) are skipped like NaN.  A float cell without a valid value gets
// `empty`; an int16 one gets `value` (0 when off).
struct RegridFill {
  int on;
  double value;
  double empty;
};

template <typename T>
__device__ __forceinline__ T regrid_result(double s, double w, const RegridFill& f) {
  if (w > 0.0) return (T)(s / w);
  return (T)f.empty;
}
template <>
__device__ __forceinline__ int16_t regrid_result<int16_t>(double s, double w, const RegridFill& f) {
  if (w > 0.0) return (int16_t)round(s / w);  // half away from zero; a mean of int16 stays in range
  return f.on ? (int16_t)f.value : (int16_t)0;
}

// Shared memory: the tile's x weights (kx * tj, k-major so a warp's reads are conflict-free, padded
// to 16 bytes), then RG_STAGES row slots of regrid_slot_bytes.  blockDim.x is tj rounded up to a
// warp.  The CTA's band is band0 + blockIdx.x / n_ctiles; source row r is read at
// src + (r - row0) * src_row.
template <typename T>
__global__ void __launch_bounds__(RG_THREADS) k_regrid(const T* __restrict__ src, int64_t batch, int64_t src_row,
                                                       int64_t src_batch, int row0, int band0, RegridTables tb,
                                                       int slot_elems, RegridFill fill, T* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* s_xw = reinterpret_cast<double*>(smem_raw);
  T* s_buf = reinterpret_cast<T*>(smem_raw + ((size_t)tb.kx * tb.tj * sizeof(double) + 15) / 16 * 16);

  const int tid = threadIdx.x, nthr = blockDim.x;
  const int ctile = blockIdx.x % tb.n_ctiles;
  const int band = band0 + blockIdx.x / tb.n_ctiles;
  const int j0 = ctile * tb.tj, i0 = band * RG_ROWS;
  const int c_lo = tb.tile_lo[ctile], span = tb.tile_span[ctile];
  const int e0 = tb.band_ptr[band], ne = tb.band_ptr[band + 1] - e0;
  const int32_t* __restrict__ srow = tb.step_row + e0;
  const int32_t* __restrict__ st = tb.step_t + e0;
  const double* __restrict__ sw = tb.step_w + e0;
  const T fill_t = fill.on ? (T)fill.value : (T)0;

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
    auto row_of = [&](int q) { return sb + (int64_t)(srow[q] - row0) * src_row; };
    auto issue = [&](int q) {  // the source row of step q -> ring slot q % RG_STAGES
      if (q < ne && srow[q] >= 0 && span > 0) {
        const T* g = row_of(q);
        const char* c0 = reinterpret_cast<const char*>((uintptr_t)g & ~(uintptr_t)15);
        const int nchunk = (int)(((uintptr_t)(g + span) - (uintptr_t)c0 + 15) / 16);
        char* s = reinterpret_cast<char*>(s_buf + (size_t)(q % RG_STAGES) * slot_elems);
        for (int v = tid; v < nchunk; v += nthr) cp_async16(s + 16 * v, c0 + 16 * v);
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
        const T* row = s_buf + (size_t)(q % RG_STAGES) * slot_elems + row_phase(row_of(q)) + my_first;
        double s = 0.0, w = 0.0;
#pragma unroll 2  // the sum is one dependent chain; the compiler's deeper unroll spills in the int16 case
        for (int k = 0; k < my_count; ++k) {
          const T raw = row[k];
          const double v = (double)raw;
          if (v == v && !(fill.on && raw == fill_t)) {
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
        if (active) ob[(int64_t)st[q] * tb.nx_dst] = regrid_result<T>(acc_s, acc_w, fill);
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
  std::vector<int32_t> band_lo, band_hi;  // source rows [lo, hi) each band reads (lo = hi = 0: none)
  void* dmem;  // one allocation holding every table
};

size_t regrid_smem(const RegridPlan& p, size_t elem) {
  return ((size_t)p.tb.kx * p.tb.tj * sizeof(double) + 15) / 16 * 16 + RG_STAGES * regrid_slot_bytes(p.max_span, elem);
}

template <typename T>
int regrid_run(const RegridPlan* p, int64_t batch, const T* src, int64_t src_row, int64_t src_batch, int row0,
               int band0, int n_bands, RegridFill fill, T* out, void* stream) {
  if (batch == 0 || n_bands == 0 || p->tb.ny_dst == 0 || p->tb.nx_dst == 0) return ATL_OK;
  ATL_REQUIRE(src && out, "NULL argument");
  ATL_CUDA(cudaSetDevice(p->device));
  const size_t smem = regrid_smem(*p, sizeof(T));
  ATL_CUDA(cudaFuncSetAttribute(k_regrid<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const dim3 grid((unsigned)(n_bands * p->tb.n_ctiles), (unsigned)(batch < 65535 ? batch : 65535));
  const int threads = (p->tb.tj + 31) / 32 * 32;
  const int slot_elems = (int)(regrid_slot_bytes(p->max_span, sizeof(T)) / sizeof(T));
  k_regrid<T><<<grid, threads, smem, (cudaStream_t)stream>>>(src, batch, src_row, src_batch, row0, band0, p->tb,
                                                             slot_elems, fill, out);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

template <typename T>
int regrid_batch(const RegridPlan* p, int64_t batch, const T* src, int64_t src_row, int64_t src_batch, T* out,
                 void* stream) {
  ATL_REQUIRE(p, "NULL plan");
  ATL_REQUIRE(batch >= 0, "negative batch");
  if (batch == 0 || p->tb.ny_dst == 0 || p->tb.nx_dst == 0) return ATL_OK;
  ATL_REQUIRE(src_row >= p->nx_src && src_batch >= src_row * p->ny_src, "source strides smaller than its rows");
  return regrid_run(p, batch, src, src_row, src_batch, 0, 0, p->n_bands, RegridFill{0, 0.0, NAN}, out, stream);
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
    int lo = ny_src, hi = 0;
    for (int i = bnd * RG_ROWS; i < std::min(ny_dst, (bnd + 1) * RG_ROWS); ++i) {
      for (int k = 0; k < std::max(ycount[i], 1); ++k) {
        step_row.push_back(ycount[i] ? yfirst[i] + k : -1);
        step_t.push_back(i - bnd * RG_ROWS);
        step_w.push_back(ycount[i] ? yw[(size_t)i * ky + k] : 0.0);
      }
      if (ycount[i]) {
        lo = std::min(lo, yfirst[i]);
        hi = std::max(hi, yfirst[i] + ycount[i]);
      }
    }
    band_ptr.push_back((int32_t)step_row.size());
    p.band_lo.push_back(hi > lo ? lo : 0);
    p.band_hi.push_back(hi > lo ? hi : 0);
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

int atl_regrid_band_rows(const void* plan, int32_t* row_lo, int32_t* row_hi) {
  ATL_REQUIRE(plan && row_lo && row_hi, "NULL argument");
  const RegridPlan* p = static_cast<const RegridPlan*>(plan);
  if (p->n_bands) {
    memcpy(row_lo, p->band_lo.data(), sizeof(int32_t) * p->n_bands);
    memcpy(row_hi, p->band_hi.data(), sizeof(int32_t) * p->n_bands);
  }
  return ATL_OK;
}

int atl_regrid_f32(const void* plan, int64_t batch, const float* src_dev, int64_t src_row, int64_t src_batch,
                   float* out_dev, void* stream) {
  return regrid_batch(static_cast<const RegridPlan*>(plan), batch, src_dev, src_row, src_batch, out_dev, stream);
}

int atl_regrid_f64(const void* plan, int64_t batch, const double* src_dev, int64_t src_row, int64_t src_batch,
                   double* out_dev, void* stream) {
  return regrid_batch(static_cast<const RegridPlan*>(plan), batch, src_dev, src_row, src_batch, out_dev, stream);
}

int atl_regrid_window(const void* plan, int32_t dtype, int32_t band0, int32_t n_bands, const void* src_dev,
                      int32_t row0, int32_t n_rows, int64_t src_row, int32_t has_fill, double fill, void* out_dev,
                      void* stream) {
  ATL_REQUIRE(plan, "NULL plan");
  const RegridPlan* p = static_cast<const RegridPlan*>(plan);
  ATL_REQUIRE(band0 >= 0 && n_bands >= 0 && band0 + n_bands <= p->n_bands, "bands outside the plan");
  ATL_REQUIRE(row0 >= 0 && n_rows >= 0 && src_row >= p->nx_src, "bad source rows");
  for (int b = band0; b < band0 + n_bands; ++b)
    ATL_REQUIRE(p->band_hi[b] == 0 || (p->band_lo[b] >= row0 && p->band_hi[b] <= row0 + n_rows),
                "a band reads source rows outside the buffer");
  const RegridFill f{has_fill ? 1 : 0, fill, has_fill ? fill : NAN};
  switch (dtype) {
    case ATL_REGRID_I16:
      ATL_REQUIRE(!has_fill || (fill >= -32768.0 && fill <= 32767.0 && fill == floor(fill)), "fill value is not an int16");
      return regrid_run(p, 1, static_cast<const int16_t*>(src_dev), src_row, 0, row0, band0, n_bands, f,
                        static_cast<int16_t*>(out_dev), stream);
    case ATL_REGRID_F32:
      return regrid_run(p, 1, static_cast<const float*>(src_dev), src_row, 0, row0, band0, n_bands, f,
                        static_cast<float*>(out_dev), stream);
    case ATL_REGRID_F64:
      return regrid_run(p, 1, static_cast<const double*>(src_dev), src_row, 0, row0, band0, n_bands, f,
                        static_cast<double*>(out_dev), stream);
  }
  ATL_REQUIRE(false, "dtype must be ATL_REGRID_I16, _F32 or _F64");
  return ATL_ERR_INVALID;
}

int atl_regrid_nodata(const void* plan, int32_t dtype, int64_t batch, const void* src_dev, int64_t src_row,
                      int64_t src_batch, int32_t has_nodata, double nodata, double empty, void* out_dev, void* stream) {
  ATL_REQUIRE(plan, "NULL plan");
  const RegridPlan* p = static_cast<const RegridPlan*>(plan);
  ATL_REQUIRE(batch >= 0, "negative batch");
  if (batch == 0 || p->tb.ny_dst == 0 || p->tb.nx_dst == 0) return ATL_OK;
  ATL_REQUIRE(src_row >= p->nx_src && src_batch >= src_row * p->ny_src, "source strides smaller than its rows");
  const RegridFill f{has_nodata ? 1 : 0, nodata, empty};
  switch (dtype) {
    case ATL_REGRID_F32:
      return regrid_run(p, batch, static_cast<const float*>(src_dev), src_row, src_batch, 0, 0, p->n_bands, f,
                        static_cast<float*>(out_dev), stream);
    case ATL_REGRID_F64:
      return regrid_run(p, batch, static_cast<const double*>(src_dev), src_row, src_batch, 0, 0, p->n_bands, f,
                        static_cast<double*>(out_dev), stream);
  }
  ATL_REQUIRE(false, "dtype must be ATL_REGRID_F32 or _F64");
  return ATL_ERR_INVALID;
}

void atl_regrid_destroy(void* plan) {
  if (!plan) return;
  RegridPlan* p = static_cast<RegridPlan*>(plan);
  cudaSetDevice(p->device);
  cudaFree(p->dmem);
  delete p;
}

}  // extern "C"
