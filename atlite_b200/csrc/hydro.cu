// hydro.cu -- basin-routed inflow per plant (hydro.py:81-104): every plant sums the runoff of its
// upstream basins, each rolled in time by the basin's travel time to the plant,
//   out[p, t] = sum_e  w_e * R[row_e, (t - shift_e) mod nt],   e over the plant's entries in order.
//
// The reference rolls a year-long series once per (plant, upstream basin): sum |upstream(p)| * nt
// values, 1e5-1e6 rolls for a continent's run-of-river fleet.  Here one CTA owns one (plant, time
// tile) pair and its threads run along t, so each entry reads one contiguous segment of its basin's
// row (with at most one wrap point) and adds it into registers.  Plants vary fastest across the grid:
// the CTAs in flight work on the same time tile, and the row segments that nested plants on one river
// share come from L2.
//
// The products and sums are rounded separately, in entry order, exactly as the reference's
// `inflow += runoff.roll(...)` over float64 arrays: the result does not depend on the launch and is
// bitwise repeatable.
#include "kernels.cuh"

namespace atl {

constexpr int HY_THREADS = 256;  // time steps per CTA (one per thread)

// Entries are staged per chunk of HY_THREADS in shared memory: row offset row * nt, the shift
// reduced into [0, nt), and the weight.
__global__ void __launch_bounds__(HY_THREADS) k_hydro_shift_sum(const double* __restrict__ R, int64_t nt,
                                                                const int64_t* __restrict__ entry_ptr,
                                                                const int32_t* __restrict__ rows,
                                                                const int64_t* __restrict__ shifts,
                                                                const double* __restrict__ weights,
                                                                double* __restrict__ out) {
  __shared__ int64_t s_base[HY_THREADS];
  __shared__ int64_t s_shift[HY_THREADS];
  __shared__ double s_w[HY_THREADS];
  const int64_t p = blockIdx.x;
  const int64_t t = (int64_t)blockIdx.y * HY_THREADS + threadIdx.x;
  const bool live = t < nt;
  const int64_t e0 = entry_ptr[p], e1 = entry_ptr[p + 1];
  double acc = 0.0;
  for (int64_t c = e0; c < e1; c += HY_THREADS) {
    const int n = e1 - c < HY_THREADS ? (int)(e1 - c) : HY_THREADS;
    if (threadIdx.x < n) {
      const int64_t e = c + threadIdx.x;
      int64_t s = shifts[e] % nt;  // C remainder: in (-nt, nt)
      if (s < 0) s += nt;
      s_base[threadIdx.x] = (int64_t)rows[e] * nt;
      s_shift[threadIdx.x] = s;
      s_w[threadIdx.x] = weights[e];
    }
    __syncthreads();
    if (live) {
#pragma unroll 8
      for (int j = 0; j < n; ++j) {
        int64_t src = t - s_shift[j];
        if (src < 0) src += nt;
        acc = __dadd_rn(acc, __dmul_rn(__ldg(R + s_base[j] + src), s_w[j]));
      }
    }
    __syncthreads();
  }
  if (live) out[p * nt + t] = acc;
}

}  // namespace atl

using namespace atl;

extern "C" {

int atl_hydro_shift_sum(int device, int32_t n_rows, int64_t nt, const double* runoff_dev, int32_t n_plants,
                        const int64_t* entry_ptr_dev, const int32_t* rows_dev, const int64_t* shifts_dev,
                        const double* weights_dev, double* out_dev, void* stream) {
  ATL_REQUIRE(n_rows >= 0 && n_plants >= 0 && nt >= 0, "negative size");
  if (n_plants == 0 || nt == 0) return ATL_OK;
  ATL_REQUIRE(out_dev && entry_ptr_dev, "NULL argument");
  ATL_REQUIRE(n_rows == 0 || runoff_dev, "NULL runoff");
  ATL_CUDA(cudaSetDevice(device));
  const int64_t tiles = (nt + HY_THREADS - 1) / HY_THREADS;
  ATL_REQUIRE(tiles <= 65535, "time axis too long (more than 65535 tiles of 256 steps)");
  const dim3 grid((unsigned)n_plants, (unsigned)tiles);
  k_hydro_shift_sum<<<grid, HY_THREADS, 0, (cudaStream_t)stream>>>(runoff_dev, nt, entry_ptr_dev, rows_dev,
                                                                   shifts_dev, weights_dev, out_dev);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

}  // extern "C"
