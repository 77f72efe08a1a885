// sarah.cu -- SARAH's half-hourly SIS / SID: gap filling within time blocks, then the hourly pair
// mean (datasets/sarah.py:91-159 of the reference: interpolate, fillna(0), hourly_mean).
//
// One thread owns one (variable, cell) series and walks the launch's steps in order, block by block.
// Per block [b0, b1):
//   * interpolate: a NaN step s between the valid steps i0 < s < i1 gets np.interp's value
//       slope = (f1 - f0) / (i1 - i0),  v = slope * (s - i0) + f0      in float64, rounded once to
//     float32; NaNs before the first / after the last valid step take that step's value; a block
//     with no valid step stays NaN.  (np.interp's fallbacks for a NaN result are kept as well.)
//   * zero filling: NaN -> 0;  no filling: NaN stays (hourly_mean alone).
// The filled steps are emitted in increasing order; with pair_mean, steps (2k, 2k + 1) give output
// step k = (a + b) / 2 in float32, and a trailing odd step is dropped.
//
// Traffic: a NaN run is written when its closing valid step arrives, and needs nothing but
// (i0, f0, i1, f1), which sit in registers, so every input element is read from HBM once and every
// output element written once.  The loads are issued SF_UNROLL steps at a time into registers (a warp
// reads 128 contiguous bytes per step), so each thread keeps that many independent loads in flight.
// The float32 and float64 arithmetic is written as round-to-nearest PTX without .ftz and without
// contraction, so the results are NumPy's bit for bit whatever the build's -ftz / -fmad flags.
#include <math.h>

#include "common.cuh"

namespace atl {

constexpr int SF_THREADS = 256;
constexpr int SF_UNROLL = 8;

struct SarahBlocks {
  int32_t start[ATL_SARAH_MAX_BLOCKS + 1];  // block b is [start[b], start[b + 1]); start[n] = nt
  int32_t n;
};

__device__ __forceinline__ float f32_add(float a, float b) {
  float r;
  asm("add.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float f32_mul(float a, float b) {
  float r;
  asm("mul.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float f64_to_f32(double a) {
  float r;
  asm("cvt.rn.f32.f64 %0, %1;" : "=f"(r) : "d"(a));
  return r;
}

// np.interp between (i0, f0) and (i1, f1) at s, i0 < s < i1 (numpy/core/src/multiarray/compiled_base.c)
__device__ __forceinline__ float interp(int i0, float f0, int i1, float f1, int s) {
  const double d0 = f0, d1 = f1;
  const double slope = __ddiv_rn(__dadd_rn(d1, -d0), (double)(i1 - i0));
  double v = __dadd_rn(__dmul_rn(slope, (double)(s - i0)), d0);
  if (isnan(v)) {
    v = __dadd_rn(__dmul_rn(slope, (double)(s - i1)), d1);
    if (isnan(v) && d0 == d1) v = d0;
  }
  return f64_to_f32(v);
}

__global__ void __launch_bounds__(SF_THREADS) k_sarah_fill(const float* __restrict__ sis, const float* __restrict__ sid,
                                                           int64_t n_cells, int32_t nt, const SarahBlocks blocks,
                                                           int fill, int pair_mean, float* __restrict__ sis_out,
                                                           float* __restrict__ sid_out) {
  const int64_t cell = (int64_t)blockIdx.x * SF_THREADS + threadIdx.x;
  if (cell >= n_cells) return;
  const float* __restrict__ in = (blockIdx.y ? sid : sis) + cell;
  float* __restrict__ out = (blockIdx.y ? sid_out : sis_out) + cell;

  float first = 0.f;  // the first value of the current pair
  auto emit = [&](int s, float v) {
    if (!pair_mean) {
      out[(int64_t)s * n_cells] = v;
    } else if (s & 1) {
      out[(int64_t)(s >> 1) * n_cells] = f32_mul(f32_add(first, v), 0.5f);
    } else {
      first = v;
    }
  };

  for (int b = 0; b < blocks.n; ++b) {
    const int b0 = blocks.start[b], b1 = blocks.start[b + 1];
    int prev = -1;      // last valid step of this block so far
    float fprev = 0.f;  // its value
    int pend = b0;      // first step not yet emitted
    for (int t = b0; t < b1; t += SF_UNROLL) {
      float v[SF_UNROLL];
#pragma unroll
      for (int u = 0; u < SF_UNROLL; ++u) v[u] = t + u < b1 ? __ldcs(in + (int64_t)(t + u) * n_cells) : 0.f;
#pragma unroll
      for (int u = 0; u < SF_UNROLL; ++u) {
        const int s = t + u;
        if (s >= b1) break;
        if (v[u] == v[u]) {
          for (int q = pend; q < s; ++q) emit(q, prev < 0 ? v[u] : interp(prev, fprev, s, v[u], q));
          emit(s, v[u]);
          prev = s;
          fprev = v[u];
          pend = s + 1;
        } else if (fill != ATL_SARAH_FILL_INTERP) {
          emit(s, fill == ATL_SARAH_FILL_ZERO ? 0.f : v[u]);
          pend = s + 1;
        }
      }
    }
    for (int q = pend; q < b1; ++q) emit(q, prev < 0 ? __int_as_float(0x7fc00000) : fprev);
  }
}

}  // namespace atl

using namespace atl;

extern "C" {

int atl_sarah_fill(int device, int32_t nt, int64_t n_cells, const float* sis_dev, const float* sid_dev, int32_t n_blocks,
                   const int32_t* block_start, int32_t fill, int32_t pair_mean, float* sis_out_dev,
                   float* sid_out_dev, void* stream) {
  ATL_REQUIRE(nt >= 0 && n_cells >= 0, "negative size");
  if (nt == 0 || n_cells == 0) return ATL_OK;
  ATL_REQUIRE(n_blocks >= 1 && n_blocks <= ATL_SARAH_MAX_BLOCKS, "n_blocks must be in [1, ATL_SARAH_MAX_BLOCKS]");
  ATL_REQUIRE(block_start, "NULL block table");
  ATL_REQUIRE(fill == ATL_SARAH_FILL_NONE || fill == ATL_SARAH_FILL_ZERO || fill == ATL_SARAH_FILL_INTERP, "bad fill");
  ATL_REQUIRE(block_start[0] == 0, "the first block must start at step 0");
  SarahBlocks blocks{};
  blocks.n = n_blocks;
  for (int32_t b = 0; b < n_blocks; ++b) {
    const int32_t end = b + 1 < n_blocks ? block_start[b + 1] : nt;
    ATL_REQUIRE(end > block_start[b], "block starts must ascend strictly and lie below nt");
    blocks.start[b] = block_start[b];
  }
  blocks.start[n_blocks] = nt;
  ATL_REQUIRE(sis_dev && sid_dev && sis_out_dev && sid_out_dev, "NULL argument");
  ATL_REQUIRE((n_cells + SF_THREADS - 1) / SF_THREADS < (int64_t)1 << 31, "too many cells");
  ATL_CUDA(cudaSetDevice(device));
  const dim3 grid((unsigned)((n_cells + SF_THREADS - 1) / SF_THREADS), 2);
  k_sarah_fill<<<grid, SF_THREADS, 0, (cudaStream_t)stream>>>(sis_dev, sid_dev, n_cells, nt, blocks, fill,
                                                               pair_mean ? 1 : 0, sis_out_dev, sid_out_dev);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

}  // extern "C"
