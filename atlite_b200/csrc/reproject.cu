// reproject.cu -- warp (..., y, x) rasters onto an axis-aligned grid of another CRS (gis.reproject,
// rasterio.warp.reproject with Resampling.average or .nearest), for EPSG:4326, 3035, 3857 and
// ESRI:54009 (proj.cuh).
//
// Nothing is tabulated per destination cell: a cell's footprint is computed in the kernel, in float64,
// once per cell for every batch entry the CTA walks.
//
// average (k_reproject_avg): destination cell (i, j) has the corners T_dst (j, i) and T_dst (j + 1,
// i + 1).  Both are projected into the source CRS and taken to source pixel coordinates (u, v) by the
// inverse source affine; the footprint is the axis-aligned box they span, clipped to the source
// (footprint.cuh, shared with the reprojected availability).  A
// pixel's weight is its overlap with the box along u times its overlap along v (pixels overlapping by
// no more than 1e-10 along an axis are left out, as in regrid), NaN and nodata are skipped, and a cell
// without a valid pixel (or with a corner that has no image) gets dst_nodata.
//   A CTA owns a tile of tile_y x tile_x destination cells (at most RP_THREADS).  It projects the
//   tile's (tile_y + 1) x (tile_x + 1) lattice corners once into shared memory, so neighbouring cells
//   share their corners, and every thread turns its cell's two corners into a box.  The box decides
//   who sums it, so the result of a cell does not depend on the tile:
//   * at most RP_SMALL pixels (upsampling and similar resolutions): the cell's own thread, each
//     source row's x-sum and then the rows in ascending order (regrid's order);
//   * more (downsampling): the whole CTA, one such cell after the other.  Thread t takes pixels t,
//     t + RP_THREADS, ... of the box in row-major order with weight wy * wx, and the RP_THREADS
//     partial sums are added in a fixed tree (warp shuffles, then the warps in order).  The loads of a
//     row are consecutive threads' consecutive columns, and neighbouring boxes abut, so each source
//     pixel leaves HBM about once.
//   The host picks the tile from the typical box size (a launch shape only).
// nearest (k_reproject_nearest): one thread per cell projects the cell's centre T_dst (j + 1/2,
// i + 1/2) and takes the pixel floor((u, v)) when it lies inside the source; NaN and nodata there,
// a centre outside the source and one without an image give dst_nodata.
//
// Every sum is float64 in an order fixed by the geometry alone, so results are bitwise repeatable and
// do not depend on the batch slab, the tile or the launch.
#include <math.h>

#include <algorithm>

#include "common.cuh"
#include "footprint.cuh"
#include "proj.cuh"

namespace atl {

template <typename T>
__device__ __forceinline__ bool valid_pixel(T raw, const AtlReproject& r, T nodata) {
  return raw == raw && !(r.has_nodata && raw == nodata);
}

template <typename T, int FROM, int TO>
__global__ void __launch_bounds__(RP_THREADS, 4) k_reproject_avg(AtlReproject r, const T* __restrict__ src, int64_t batch,
                                                              int64_t src_row, int64_t src_batch, int tile_y,
                                                              int tile_x, int64_t n_tx, T* __restrict__ out) {
  __shared__ double2 s_uv[RP_THREADS * 2 + 2];  // (tile_y + 1) * (tile_x + 1) <= 2 RP_THREADS + 1 corners
  __shared__ Box s_box[RP_THREADS];  // thread t's cell
  __shared__ int s_big[RP_THREADS], s_nbig;  // the cells whose box the whole CTA sums
  __shared__ double s_red[2][RP_THREADS / 32];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t i0 = blockIdx.x / n_tx * tile_y, j0 = blockIdx.x % n_tx * tile_x;
  const int lx = tile_x + 1, n_corner = (tile_y + 1) * lx;
  if (tid == 0) s_nbig = 0;
  for (int k = tid; k < n_corner; k += RP_THREADS) {
    double u, v;
    to_source<FROM, TO>(r.dst, r.src, r.proj, (double)(j0 + k % lx), (double)(i0 + k / lx), u, v);
    s_uv[k] = make_double2(u, v);
  }
  __syncthreads();

  // this thread's cell and its box (empty: hi <= lo along an axis)
  const int ti = tid / tile_x, tj = tid % tile_x;
  const int64_t i = i0 + ti, j = j0 + tj;
  bool mine = tid < tile_y * tile_x && i < r.dst.ny && j < r.dst.nx;
  if (mine) {
    const double2 a = s_uv[ti * lx + tj], b = s_uv[(ti + 1) * lx + tj + 1];
    Box bx{};
    bx.cell = i * r.dst.nx + j;
    corner_box(a, b, 0, r.src.nx, 0, r.src.ny, bx);
    s_box[tid] = bx;
    if (bx.c.hi > bx.c.lo && bx.r.hi > bx.r.lo && (int64_t)(bx.c.hi - bx.c.lo) * (bx.r.hi - bx.r.lo) > RP_SMALL) {
      s_big[atomicAdd(&s_nbig, 1)] = tid;
      mine = false;
    }
  }
  __syncthreads();
  const int n_big = s_nbig;
  const T nodata = (T)r.src_nodata, fill = (T)r.dst_nodata;
  const int64_t plane = r.dst.ny * r.dst.nx;

  for (int64_t bt = blockIdx.y; bt < batch; bt += gridDim.y) {
    const T* sb = src + bt * src_batch;
    T* ob = out + bt * plane;
    if (mine) {  // a small box: this thread, row x-sums, then the rows in ascending order
      const Box& B = s_box[tid];
      double acc_s = 0.0, acc_w = 0.0;
      const T* p = sb + (int64_t)B.r.lo * src_row;
      for (int rr = B.r.lo; rr < B.r.hi; ++rr, p += src_row) {
        double s = 0.0, w = 0.0;
        for (int cc = B.c.lo; cc < B.c.hi; ++cc) {
          const T raw = p[cc];
          if (valid_pixel(raw, r, nodata)) {
            const double wx = cc == B.c.lo ? B.c.w_lo : (cc == B.c.hi - 1 ? B.c.w_hi : 1.0);
            s = fma(wx, (double)raw, s);
            w += wx;
          }
        }
        const double wy = rr == B.r.lo ? B.r.w_lo : (rr == B.r.hi - 1 ? B.r.w_hi : 1.0);
        acc_s = fma(wy, s, acc_s);
        acc_w = fma(wy, w, acc_w);
      }
      ob[B.cell] = acc_w > 0.0 ? (T)(acc_s / acc_w) : fill;
    }
    for (int q = 0; q < n_big; ++q) {  // the large boxes: the whole CTA, one after the other
      const Box& B = s_box[s_big[q]];
      const int w = B.c.hi - B.c.lo, h = B.r.hi - B.r.lo;
      const int64_t n = (int64_t)w * h;
      const int dr = RP_THREADS / w, dc = RP_THREADS % w;
      const T* base = sb + (int64_t)B.r.lo * src_row + B.c.lo;
      const double wr_lo = B.r.w_lo, wr_hi = B.r.w_hi, wc_lo = B.c.w_lo, wc_hi = B.c.w_hi;
      int rr = tid / w, cc = tid % w;
      double s = 0.0, ws = 0.0;
#pragma unroll 4
      for (int64_t e = tid; e < n; e += RP_THREADS) {
        const T raw = base[(int64_t)rr * src_row + cc];
        if (valid_pixel(raw, r, nodata)) {
          const double wy = rr == 0 ? wr_lo : (rr == h - 1 ? wr_hi : 1.0);
          const double wx = cc == 0 ? wc_lo : (cc == w - 1 ? wc_hi : 1.0);
          const double wt = wy * wx;
          s = fma(wt, (double)raw, s);
          ws += wt;
        }
        cc += dc;
        rr += dr;
        if (cc >= w) {
          cc -= w;
          ++rr;
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, o);
        ws += __shfl_xor_sync(0xffffffffu, ws, o);
      }
      if (lane == 0) {
        s_red[0][warp] = s;
        s_red[1][warp] = ws;
      }
      __syncthreads();
      if (tid == 0) {
        double ts = 0.0, tw = 0.0;
        for (int k = 0; k < RP_THREADS / 32; ++k) {
          ts += s_red[0][k];
          tw += s_red[1][k];
        }
        ob[s_box[s_big[q]].cell] = tw > 0.0 ? (T)(ts / tw) : fill;
      }
      __syncthreads();  // s_red is free again
    }
  }
}

template <typename T, int FROM, int TO>
__global__ void __launch_bounds__(RP_THREADS) k_reproject_nearest(AtlReproject r, const T* __restrict__ src,
                                                                  int64_t batch, int64_t src_row, int64_t src_batch,
                                                                  T* __restrict__ out) {
  const int64_t plane = r.dst.ny * r.dst.nx;
  const int64_t cell = (int64_t)blockIdx.x * RP_THREADS + threadIdx.x;
  if (cell >= plane) return;
  const int64_t i = cell / r.dst.nx, j = cell % r.dst.nx;
  double u, v;
  to_source<FROM, TO>(r.dst, r.src, r.proj, (double)j + 0.5, (double)i + 0.5, u, v);
  const double fu = floor(u), fv = floor(v);
  const bool in = fu >= 0.0 && fu < (double)r.src.nx && fv >= 0.0 && fv < (double)r.src.ny;  // false for NaN
  const T* p = src + (in ? (int64_t)fv * src_row + (int64_t)fu : 0);
  const T nodata = (T)r.src_nodata, fill = (T)r.dst_nodata;
  for (int64_t bt = blockIdx.y; bt < batch; bt += gridDim.y) {
    T val = fill;
    if (in) {
      const T raw = p[bt * src_batch];
      if (valid_pixel(raw, r, nodata)) val = raw;
    }
    out[bt * plane + cell] = val;
  }
}

template <class T>
struct ReprojectKernel {
  template <int FROM, int TO>
  struct Avg {
    static auto get() { return k_reproject_avg<T, FROM, TO>; }
  };
  template <int FROM, int TO>
  struct Nearest {
    static auto get() { return k_reproject_nearest<T, FROM, TO>; }
  };
};

// batch entries per CTA: enough CTAs to fill the device a few times over, each still walking a run of
// the batch with its boxes in registers
unsigned batch_chunks(int64_t batch, int64_t n_ctas, int device) {
  int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  const int64_t want = (32LL * sms + n_ctas - 1) / std::max<int64_t>(n_ctas, 1);
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>({want, batch, 65535}));
}

template <typename T>
int reproject_run(int device, const AtlReproject& r, int64_t batch, const T* src, int64_t src_row, int64_t src_batch,
                  T* out, cudaStream_t stream) {
  const int64_t plane = r.dst.ny * r.dst.nx;
  if (batch == 0 || plane == 0) return ATL_OK;
  ATL_CUDA(cudaSetDevice(device));
  const int from = r.proj.from.kind, to = r.proj.to.kind;  // destination lattice -> source CRS
  if (r.resampling == ATL_RESAMPLING_NEAREST) {
    const int64_t blocks = (plane + RP_THREADS - 1) / RP_THREADS;
    ATL_REQUIRE(blocks <= 0x7fffffffLL, "destination grid too large");
    const dim3 grid((unsigned)blocks, batch_chunks(batch, blocks, device));
    pair_kernel<ReprojectKernel<T>::template Nearest>(from, to)<<<grid, RP_THREADS, 0, stream>>>(
        r, src, batch, src_row, src_batch, out);
  } else {
    const int64_t n_ty = (r.dst.ny + r.tile_y - 1) / r.tile_y, n_tx = (r.dst.nx + r.tile_x - 1) / r.tile_x;
    ATL_REQUIRE(n_ty * n_tx <= 0x7fffffffLL, "destination grid too large");
    const dim3 grid((unsigned)(n_ty * n_tx), batch_chunks(batch, n_ty * n_tx, device));
    pair_kernel<ReprojectKernel<T>::template Avg>(from, to)<<<grid, RP_THREADS, 0, stream>>>(
        r, src, batch, src_row, src_batch, r.tile_y, r.tile_x, n_tx, out);
  }
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

}  // namespace atl

using namespace atl;

extern "C" {

int atl_reproject(int device, const AtlReproject* r, int32_t dtype, int64_t batch, const void* src_dev,
                  int64_t src_row, int64_t src_batch, void* out_dev, void* stream) {
  ATL_REQUIRE(r, "NULL argument");
  ATL_REQUIRE(batch >= 0, "negative batch");
  const AtlLattice &S = r->src, &D = r->dst;
  ATL_REQUIRE(S.nx > 0 && S.ny > 0 && S.nx <= 0x7fffffffLL && S.ny <= 0x7fffffffLL && D.nx >= 0 && D.ny >= 0,
              "bad size");
  ATL_REQUIRE(S.a != 0.0 && S.e != 0.0 && isfinite(S.a) && isfinite(S.e) && isfinite(S.c) && isfinite(S.f) &&
                  isfinite(D.a) && isfinite(D.e) && isfinite(D.c) && isfinite(D.f),
              "transforms must be finite, with a non-zero source pixel size");
  ATL_REQUIRE(projection_ok(r->proj), "unknown CRS in the projection");
  ATL_REQUIRE(r->resampling == ATL_RESAMPLING_NEAREST || r->resampling == ATL_RESAMPLING_AVERAGE,
              "resampling must be ATL_RESAMPLING_NEAREST or _AVERAGE");
  ATL_REQUIRE(r->resampling == ATL_RESAMPLING_NEAREST ||
                  (r->tile_y >= 1 && r->tile_x >= 1 && r->tile_y * r->tile_x <= RP_THREADS),
              "tile_y * tile_x must lie in [1, 256]");
  if (batch == 0 || D.nx == 0 || D.ny == 0) return ATL_OK;
  ATL_REQUIRE(src_dev && out_dev, "NULL argument");
  ATL_REQUIRE(src_row >= S.nx && (batch == 1 || src_batch >= src_row * S.ny),
              "source strides smaller than its rows");
  const cudaStream_t s = (cudaStream_t)stream;
  switch (dtype) {
    case ATL_REGRID_F32:
      return reproject_run(device, *r, batch, static_cast<const float*>(src_dev), src_row, src_batch,
                           static_cast<float*>(out_dev), s);
    case ATL_REGRID_F64:
      return reproject_run(device, *r, batch, static_cast<const double*>(src_dev), src_row, src_batch,
                           static_cast<double*>(out_dev), s);
  }
  ATL_REQUIRE(false, "dtype must be ATL_REGRID_F32 or _F64");
  return ATL_ERR_INVALID;
}

}  // extern "C"
