// reproject.cu -- warp (..., y, x) rasters onto an axis-aligned grid of another CRS (gis.reproject,
// rasterio.warp.reproject with Resampling.average, .nearest, .sum, .rms, .min, .max, .med, .q1, .q3
// or .mode), for EPSG:4326, 3035, 3857 and ESRI:54009 (proj.cuh).
//
// Nothing is tabulated per destination cell: a cell's footprint is computed in the kernel, in float64,
// once per cell for every batch entry the CTA walks.
//
// average (k_reproject_box with Moments): destination cell (i, j) has the corners T_dst (j, i) and
// T_dst (j + 1, i + 1).  Both are projected into the source CRS and taken to source pixel coordinates
// (u, v) by the inverse source affine; the footprint is the axis-aligned box they span, clipped to the
// source (footprint.cuh, shared with the reprojected availability).  A
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
// sum, rms, min and max are the same walk with another accumulator (Moments, Extreme).
// Within one CRS the boxes may come from regrid's tables instead (atl_reproject_ex's spans): cell
// (i, j) takes row_spans[i] x col_spans[j], and nothing is projected.
// med, q1, q3 and mode (select_run) take the same boxes and the integer weights q = llround(w 2^40):
//   k_select_boxes writes every cell's box once; k_select_small selects the boxes of at most
//   select_small pixels in the cell's thread (an insertion sort of at most RP_SMALL pairs); the larger
//   ones are gathered as (order key, q) pairs into device scratch (k_select_gather), sorted per cell
//   with CUB's segmented radix sort, and finished by one thread per cell walking its sorted pairs
//   (k_select_finish).  The scratch holds one band of cells, or a slab of batch entries of the whole
//   plane, at a time, within a fixed budget.  Integer sums are exact, so both tiers give the same
//   bits as any other correct order.
// nearest (k_reproject_nearest): one thread per cell projects the cell's centre T_dst (j + 1/2,
// i + 1/2) and takes the pixel floor((u, v)) when it lies inside the source; NaN and nodata there,
// a centre outside the source and one without an image give dst_nodata.
//
// Every sum is float64 in an order fixed by the geometry alone, so results are bitwise repeatable and
// do not depend on the batch slab, the tile or the launch.
#include <math.h>

#include <algorithm>
#include <climits>
#include <cub/device/device_segmented_radix_sort.cuh>
#include <vector>

#include "common.cuh"
#include "footprint.cuh"
#include "proj.cuh"

namespace atl {

constexpr int64_t RP_SELECT_SCRATCH = 1LL << 30;  // default scratch budget of the selections, bytes
constexpr double RP_Q_SCALE = 1099511627776.0;   // 2^40: q = llround(w * 2^40)

template <typename T>
__device__ __forceinline__ bool valid_pixel(T raw, const AtlReproject& r, T nodata) {
  return raw == raw && !(r.has_nodata && raw == nodata);
}

// The boxes of atl_reproject_ex's spans on the device (rows == nullptr: the two-corner boxes).
struct SpanBoxes {
  const AtlSpan* rows;
  const AtlSpan* cols;
};
__device__ __forceinline__ Span to_span(const AtlSpan& s) { return Span{s.lo, s.hi, s.w_lo, s.w_hi}; }

// ---------------------------------------------------------------- order keys
// An unsigned key per value whose order is the values' order (-0.0 below +0.0; never for NaN).  Built
// from the bits, so no float32 denormal is flushed on the way.
template <typename T>
struct KeyOf;
template <>
struct KeyOf<float> {
  using K = uint32_t;
  static constexpr K SIGN = 0x80000000u;
  __device__ static K bits(float v) { return __float_as_uint(v); }
  __device__ static float value(K b) { return __uint_as_float(b); }
};
template <>
struct KeyOf<double> {
  using K = unsigned long long;
  static constexpr K SIGN = 0x8000000000000000ull;
  __device__ static K bits(double v) { return (K)__double_as_longlong(v); }
  __device__ static double value(K b) { return __longlong_as_double((long long)b); }
};
template <typename T>
__device__ __forceinline__ typename KeyOf<T>::K key_of_bits(typename KeyOf<T>::K b) {
  return (b & KeyOf<T>::SIGN) ? (typename KeyOf<T>::K)~b : (typename KeyOf<T>::K)(b | KeyOf<T>::SIGN);
}
template <typename T>
__device__ __forceinline__ typename KeyOf<T>::K order_key(T v) {
  return key_of_bits<T>(KeyOf<T>::bits(v));
}
template <typename T>
__device__ __forceinline__ typename KeyOf<T>::K select_key(T v) {  // -0.0 counts as +0.0
  auto b = KeyOf<T>::bits(v);
  if ((b & ~KeyOf<T>::SIGN) == 0) b = 0;
  return key_of_bits<T>(b);
}
template <typename T>
__device__ __forceinline__ T key_value(typename KeyOf<T>::K k) {
  using K = typename KeyOf<T>::K;
  return KeyOf<T>::value((k & KeyOf<T>::SIGN) ? (K)(k ^ KeyOf<T>::SIGN) : (K)~k);
}

// ---------------------------------------------------------------- the box walk's accumulators
// add: a valid pixel with weight wt; row: a row's accumulator times its y weight (the one-thread
// order); merge / shfl_xor: the CTA's tree; result: the cell's value.
template <typename T, int OP>
struct Moments {  // average, sum, rms: sum w v (w v^2 for rms) and sum w
  double s = 0.0, w = 0.0;
  __device__ __forceinline__ void add(double wt, T raw) {
    const double v = (double)raw;
    s = fma(wt, OP == ATL_RESAMPLING_RMS ? v * v : v, s);
    w += wt;
  }
  __device__ __forceinline__ void row(double wy, const Moments& o) {
    s = fma(wy, o.s, s);
    w = fma(wy, o.w, w);
  }
  __device__ __forceinline__ void merge(const Moments& o) {
    s += o.s;
    w += o.w;
  }
  __device__ __forceinline__ void shfl_xor(int o) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    w += __shfl_xor_sync(0xffffffffu, w, o);
  }
  __device__ __forceinline__ T result(T fill) const {
    if (!(w > 0.0)) return fill;
    if (OP == ATL_RESAMPLING_SUM) return (T)s;
    if (OP == ATL_RESAMPLING_RMS) return (T)sqrt(s / w);
    return (T)(s / w);
  }
};

template <typename T, int OP>
struct Extreme {  // min / max of the order keys
  using K = typename KeyOf<T>::K;
  static constexpr K NONE = OP == ATL_RESAMPLING_MIN ? (K)~(K)0 : (K)0;  // the keys of NaNs
  K k = NONE;
  __device__ __forceinline__ void take(K o) { k = OP == ATL_RESAMPLING_MIN ? (o < k ? o : k) : (o > k ? o : k); }
  __device__ __forceinline__ void add(double, T raw) { take(order_key(raw)); }
  __device__ __forceinline__ void row(double, const Extreme& o) { take(o.k); }
  __device__ __forceinline__ void merge(const Extreme& o) { take(o.k); }
  __device__ __forceinline__ void shfl_xor(int o) { take(__shfl_xor_sync(0xffffffffu, k, o)); }
  __device__ __forceinline__ T result(T fill) const { return k == NONE ? fill : key_value<T>(k); }
};

template <typename T, int FROM, int TO, class Acc>
__global__ void __launch_bounds__(RP_THREADS, 4) k_reproject_box(AtlReproject r, SpanBoxes sp, const T* __restrict__ src,
                                                              int64_t batch, int64_t src_row, int64_t src_batch,
                                                              int tile_y, int tile_x, int64_t n_tx, T* __restrict__ out) {
  __shared__ double2 s_uv[RP_THREADS * 2 + 2];  // (tile_y + 1) * (tile_x + 1) <= 2 RP_THREADS + 1 corners
  __shared__ Box s_box[RP_THREADS];  // thread t's cell
  __shared__ int s_big[RP_THREADS], s_nbig;  // the cells whose box the whole CTA sums
  __shared__ __align__(16) unsigned char s_red_raw[sizeof(Acc) * (RP_THREADS / 32)];  // Acc has initialisers
  Acc* s_red = reinterpret_cast<Acc*>(s_red_raw);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t i0 = blockIdx.x / n_tx * tile_y, j0 = blockIdx.x % n_tx * tile_x;
  const int lx = tile_x + 1, n_corner = (tile_y + 1) * lx;
  if (tid == 0) s_nbig = 0;
  if (!sp.rows) {
    for (int k = tid; k < n_corner; k += RP_THREADS) {
      double u, v;
      to_source<FROM, TO>(r.dst, r.src, r.proj, (double)(j0 + k % lx), (double)(i0 + k / lx), u, v);
      s_uv[k] = make_double2(u, v);
    }
  }
  __syncthreads();

  // this thread's cell and its box (empty: hi <= lo along an axis)
  const int ti = tid / tile_x, tj = tid % tile_x;
  const int64_t i = i0 + ti, j = j0 + tj;
  bool mine = tid < tile_y * tile_x && i < r.dst.ny && j < r.dst.nx;
  if (mine) {
    Box bx{};
    bx.cell = i * r.dst.nx + j;
    if (sp.rows) {
      bx.r = to_span(sp.rows[i]);
      bx.c = to_span(sp.cols[j]);
    } else {
      const double2 a = s_uv[ti * lx + tj], b = s_uv[(ti + 1) * lx + tj + 1];
      corner_box(a, b, 0, r.src.nx, 0, r.src.ny, bx);
    }
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
      Acc acc;
      const T* p = sb + (int64_t)B.r.lo * src_row;
      for (int rr = B.r.lo; rr < B.r.hi; ++rr, p += src_row) {
        Acc row;
        for (int cc = B.c.lo; cc < B.c.hi; ++cc) {
          const T raw = p[cc];
          if (valid_pixel(raw, r, nodata)) {
            const double wx = cc == B.c.lo ? B.c.w_lo : (cc == B.c.hi - 1 ? B.c.w_hi : 1.0);
            row.add(wx, raw);
          }
        }
        const double wy = rr == B.r.lo ? B.r.w_lo : (rr == B.r.hi - 1 ? B.r.w_hi : 1.0);
        acc.row(wy, row);
      }
      ob[B.cell] = acc.result(fill);
    }
    for (int q = 0; q < n_big; ++q) {  // the large boxes: the whole CTA, one after the other
      const Box& B = s_box[s_big[q]];
      const int w = B.c.hi - B.c.lo, h = B.r.hi - B.r.lo;
      const int64_t n = (int64_t)w * h;
      const int dr = RP_THREADS / w, dc = RP_THREADS % w;
      const T* base = sb + (int64_t)B.r.lo * src_row + B.c.lo;
      const double wr_lo = B.r.w_lo, wr_hi = B.r.w_hi, wc_lo = B.c.w_lo, wc_hi = B.c.w_hi;
      int rr = tid / w, cc = tid % w;
      Acc acc;
#pragma unroll 4
      for (int64_t e = tid; e < n; e += RP_THREADS) {
        const T raw = base[(int64_t)rr * src_row + cc];
        if (valid_pixel(raw, r, nodata)) {
          const double wy = rr == 0 ? wr_lo : (rr == h - 1 ? wr_hi : 1.0);
          const double wx = cc == 0 ? wc_lo : (cc == w - 1 ? wc_hi : 1.0);
          acc.add(wy * wx, raw);
        }
        cc += dc;
        rr += dr;
        if (cc >= w) {
          cc -= w;
          ++rr;
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc.shfl_xor(o);
      if (lane == 0) s_red[warp] = acc;
      __syncthreads();
      if (tid == 0) {
        Acc tot;
        for (int k = 0; k < RP_THREADS / 32; ++k) tot.merge(s_red[k]);
        ob[s_box[s_big[q]].cell] = tot.result(fill);
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

// ---------------------------------------------------------------- selections (med, q1, q3, mode)

__device__ __forceinline__ int64_t weight_q(double w) { return llround(w * RP_Q_SCALE); }

// The answer over n (key, q) pairs sorted by key; pairs with q = 0 take no part.  The sums are exact
// (128-bit), so the answer does not depend on the order of equal keys.
template <typename T, typename K>
__device__ T select_sorted(const K* key, const int64_t* q, int64_t n, int op, T fill) {
  using U = unsigned __int128;
  U W = 0;
  for (int64_t e = 0; e < n; ++e) W += (uint64_t)q[e];
  if (W == 0) return fill;
  if (op == ATL_RESAMPLING_MODE) {
    U best = 0, run = 0;
    K best_k = 0;
    for (int64_t e = 0; e < n; ++e) {
      run += (uint64_t)q[e];
      if (e + 1 == n || key[e + 1] != key[e]) {
        if (run > best) {  // strictly: a tie keeps the smaller value
          best = run;
          best_k = key[e];
        }
        run = 0;
      }
    }
    return key_value<T>(best_k);
  }
  const U need = W * (U)(op == ATL_RESAMPLING_Q1 ? 1 : op == ATL_RESAMPLING_MED ? 2 : 3);
  U c = 0;
  for (int64_t e = 0; e < n; ++e) {
    c += (uint64_t)q[e];
    if (4 * c >= need) return key_value<T>(key[e]);
  }
  return fill;  // not reached: 4 C reaches 4 W
}

__device__ __forceinline__ int64_t box_pixels(const Box& B) {
  return B.c.hi > B.c.lo && B.r.hi > B.r.lo ? (int64_t)(B.c.hi - B.c.lo) * (B.r.hi - B.r.lo) : 0;
}

// every cell's box, and its pixels when more than `small` (else 0)
template <int FROM, int TO>
__global__ void __launch_bounds__(RP_THREADS) k_select_boxes(AtlReproject r, SpanBoxes sp, int small, Box* boxes,
                                                             int64_t* big) {
  const int64_t plane = r.dst.ny * r.dst.nx;
  const int64_t cell = (int64_t)blockIdx.x * RP_THREADS + threadIdx.x;
  if (cell >= plane) return;
  const int64_t i = cell / r.dst.nx, j = cell % r.dst.nx;
  Box bx{};
  bx.cell = cell;
  if (sp.rows) {
    bx.r = to_span(sp.rows[i]);
    bx.c = to_span(sp.cols[j]);
  } else {  // the corners exactly as k_reproject_box projects them
    double2 a, b;
    to_source<FROM, TO>(r.dst, r.src, r.proj, (double)j, (double)i, a.x, a.y);
    to_source<FROM, TO>(r.dst, r.src, r.proj, (double)(j + 1), (double)(i + 1), b.x, b.y);
    corner_box(a, b, 0, r.src.nx, 0, r.src.ny, bx);
  }
  boxes[cell] = bx;
  const int64_t n = box_pixels(bx);
  big[cell] = n > small ? n : 0;
}

// the cells of at most `small` pixels (and the empty ones): the cell's own thread
template <typename T>
__global__ void __launch_bounds__(RP_THREADS) k_select_small(AtlReproject r, const Box* __restrict__ boxes,
                                                             const T* __restrict__ src, int64_t batch, int64_t src_row,
                                                             int64_t src_batch, int small, T* __restrict__ out) {
  using K = typename KeyOf<T>::K;
  const int64_t plane = r.dst.ny * r.dst.nx;
  const int64_t cell = (int64_t)blockIdx.x * RP_THREADS + threadIdx.x;
  if (cell >= plane) return;
  const Box B = boxes[cell];
  if (box_pixels(B) > small) return;
  const T nodata = (T)r.src_nodata, fill = (T)r.dst_nodata;
  K key[RP_SMALL];
  int64_t qq[RP_SMALL];
  for (int64_t bt = blockIdx.y; bt < batch; bt += gridDim.y) {
    const T* sb = src + bt * src_batch;
    int n = 0;
    for (int rr = B.r.lo; rr < B.r.hi; ++rr) {
      const double wy = rr == B.r.lo ? B.r.w_lo : (rr == B.r.hi - 1 ? B.r.w_hi : 1.0);
      for (int cc = B.c.lo; cc < B.c.hi; ++cc) {
        const T raw = sb[(int64_t)rr * src_row + cc];
        const double wx = cc == B.c.lo ? B.c.w_lo : (cc == B.c.hi - 1 ? B.c.w_hi : 1.0);
        const int64_t q = weight_q(wy * wx);
        if (valid_pixel(raw, r, nodata) && q > 0) {  // insertion by key
          const K k = select_key(raw);
          int p = n++;
          for (; p > 0 && key[p - 1] > k; --p) {
            key[p] = key[p - 1];
            qq[p] = qq[p - 1];
          }
          key[p] = k;
          qq[p] = q;
        }
      }
    }
    out[bt * plane + cell] = n ? select_sorted<T>(key, qq, n, r.resampling, fill) : fill;
  }
}

// off[s] (s <= n_seg = slab entries * n_cells): segment s = (entry s / n_cells, cell c0 + s % n_cells)
// starts at entry * slab_px + big_off[cell] - big_off[c0] of the scratch
__global__ void k_select_offsets(const int64_t* __restrict__ big_off, int64_t c0, int64_t n_cells, int64_t n_seg,
                                 int64_t slab_px, int* __restrict__ off) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s > n_seg) return;
  const int64_t b = s / n_cells, c = c0 + s % n_cells;
  off[s] = (int)(b * slab_px + big_off[c] - big_off[c0]);
}

// one CTA per (cell, slab entry): the box's (key, q) pairs in row-major order, invalid pixels as
// (the largest key, 0)
template <typename T>
__global__ void __launch_bounds__(RP_THREADS) k_select_gather(AtlReproject r, const Box* __restrict__ boxes,
                                                              const int64_t* __restrict__ big_off, int64_t c0,
                                                              int64_t slab_px, const T* __restrict__ src,
                                                              int64_t src_row, int64_t src_batch,
                                                              typename KeyOf<T>::K* __restrict__ keys,
                                                              int64_t* __restrict__ qs) {
  using K = typename KeyOf<T>::K;
  const int64_t cell = c0 + blockIdx.x;
  const int n = (int)(big_off[cell + 1] - big_off[cell]);
  if (n == 0) return;
  const Box B = boxes[cell];
  const int w = B.c.hi - B.c.lo, h = B.r.hi - B.r.lo;
  const int64_t o = (int64_t)blockIdx.y * slab_px + big_off[cell] - big_off[c0];
  const T* base = src + blockIdx.y * src_batch + (int64_t)B.r.lo * src_row + B.c.lo;
  const T nodata = (T)r.src_nodata;
  for (int e = threadIdx.x; e < n; e += RP_THREADS) {
    const int rr = e / w, cc = e - rr * w;
    const T raw = base[(int64_t)rr * src_row + cc];
    K k = ~(K)0;
    int64_t q = 0;
    if (valid_pixel(raw, r, nodata)) {
      const double wy = rr == 0 ? B.r.w_lo : (rr == h - 1 ? B.r.w_hi : 1.0);
      const double wx = cc == 0 ? B.c.w_lo : (cc == w - 1 ? B.c.w_hi : 1.0);
      k = select_key(raw);
      q = weight_q(wy * wx);
    }
    keys[o + e] = k;
    qs[o + e] = q;
  }
}

// one thread per segment with pixels: its cell's answer from the sorted pairs
template <typename T>
__global__ void k_select_finish(const typename KeyOf<T>::K* __restrict__ keys, const int64_t* __restrict__ qs,
                                const int* __restrict__ off, int64_t n_seg, int64_t n_cells, int64_t c0, int64_t b0,
                                int64_t plane, int op, T fill, T* __restrict__ out) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_seg || off[s + 1] == off[s]) return;
  const int64_t b = b0 + s / n_cells, cell = c0 + s % n_cells;
  out[b * plane + cell] = select_sorted<T>(keys + off[s], qs + off[s], off[s + 1] - off[s], op, fill);
}

template <class T, class Acc>
struct BoxKernel {
  template <int FROM, int TO>
  struct K {
    static auto get() { return k_reproject_box<T, FROM, TO, Acc>; }
  };
};
template <class T>
struct NearestKernel {
  template <int FROM, int TO>
  struct K {
    static auto get() { return k_reproject_nearest<T, FROM, TO>; }
  };
};
template <int FROM, int TO>
struct SelectBoxesKernel {
  static auto get() { return k_select_boxes<FROM, TO>; }
};

// batch entries per CTA: enough CTAs to fill the device a few times over, each still walking a run of
// the batch with its boxes in registers
unsigned batch_chunks(int64_t batch, int64_t n_ctas, int device) {
  int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  const int64_t want = (32LL * sms + n_ctas - 1) / std::max<int64_t>(n_ctas, 1);
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>({want, batch, 65535}));
}

// device memory from the stream's pool, given back on every return path
struct StreamBuf {
  void* p = nullptr;
  cudaStream_t s;
  explicit StreamBuf(cudaStream_t st) : s(st) {}
  StreamBuf(const StreamBuf&) = delete;
  ~StreamBuf() {
    if (p) cudaFreeAsync(p, s);
  }
  cudaError_t alloc(size_t n) {
    if (p) cudaFreeAsync(p, s);
    p = nullptr;
    return cudaMallocAsync(&p, std::max<size_t>(n, 16), s);
  }
  template <class X>
  X* as() const {
    return static_cast<X*>(p);
  }
};

template <typename T, class Acc>
int box_run(int device, const AtlReproject& r, const SpanBoxes& sp, int64_t batch, const T* src, int64_t src_row,
            int64_t src_batch, T* out, cudaStream_t stream) {
  const int64_t n_ty = (r.dst.ny + r.tile_y - 1) / r.tile_y, n_tx = (r.dst.nx + r.tile_x - 1) / r.tile_x;
  ATL_REQUIRE(n_ty * n_tx <= 0x7fffffffLL, "destination grid too large");
  const dim3 grid((unsigned)(n_ty * n_tx), batch_chunks(batch, n_ty * n_tx, device));
  pair_kernel<BoxKernel<T, Acc>::template K>(r.proj.from.kind, r.proj.to.kind)<<<grid, RP_THREADS, 0, stream>>>(
      r, sp, src, batch, src_row, src_batch, r.tile_y, r.tile_x, n_tx, out);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

template <typename T>
int select_run(int device, const AtlReproject& r, const SpanBoxes& sp, int small, int64_t budget, int64_t batch,
               const T* src, int64_t src_row, int64_t src_batch, T* out, cudaStream_t stream) {
  using K = typename KeyOf<T>::K;
  const int64_t plane = r.dst.ny * r.dst.nx;
  const int64_t blocks = (plane + RP_THREADS - 1) / RP_THREADS;
  ATL_REQUIRE(blocks <= 0x7fffffffLL, "destination grid too large");
  StreamBuf boxes(stream), big(stream);
  ATL_CUDA(boxes.alloc(sizeof(Box) * plane));
  ATL_CUDA(big.alloc(sizeof(int64_t) * (plane + 1)));
  pair_kernel<SelectBoxesKernel>(r.proj.from.kind, r.proj.to.kind)<<<(unsigned)blocks, RP_THREADS, 0, stream>>>(
      r, sp, small, boxes.as<Box>(), big.as<int64_t>());
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  k_select_small<T><<<dim3((unsigned)blocks, batch_chunks(batch, blocks, device)), RP_THREADS, 0, stream>>>(
      r, boxes.as<Box>(), src, batch, src_row, src_batch, small, out);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());

  // the large boxes' pixels, their prefix over the plane, and the bands and slabs that fit the budget
  std::vector<int64_t> off(plane + 1, 0);
  ATL_CUDA(cudaMemcpyAsync(off.data() + 1, big.as<int64_t>(), sizeof(int64_t) * plane, cudaMemcpyDeviceToHost, stream));
  ATL_CUDA(cudaStreamSynchronize(stream));
  for (int64_t c = 0; c < plane; ++c) off[c + 1] += off[c];
  const int64_t total = off[plane];
  if (total == 0) return ATL_OK;
  ATL_CUDA(cudaMemcpyAsync(big.p, off.data(), sizeof(int64_t) * (plane + 1), cudaMemcpyHostToDevice, stream));
  const int64_t px_bytes = 2 * (int64_t)sizeof(K) + 2 * (int64_t)sizeof(int64_t), seg_bytes = sizeof(int);
  const auto cost = [&](int64_t c0, int64_t c1) { return (off[c1] - off[c0]) * px_bytes + (c1 - c0) * seg_bytes; };
  struct Chunk {
    int64_t b0, nb, c0, c1;
  };
  std::vector<Chunk> chunks;
  int64_t slab = std::min<int64_t>({budget / std::max<int64_t>(cost(0, plane), 1), batch, 65535,
                                    (int64_t)INT_MAX / (std::max(total, plane) + 1)});
  if (slab >= 1) {
    for (int64_t b = 0; b < batch; b += slab) chunks.push_back({b, std::min(slab, batch - b), 0, plane});
  } else {  // bands of cells, each at least one cell
    std::vector<Chunk> bands;
    for (int64_t c0 = 0; c0 < plane;) {
      int64_t lo = c0 + 1, hi = plane;  // the last c1 with cost(c0, c1) <= budget, at least c0 + 1
      while (lo < hi) {
        const int64_t mid = (lo + hi + 1) / 2;
        if (cost(c0, mid) <= budget && off[mid] - off[c0] < INT_MAX) lo = mid; else hi = mid - 1;
      }
      ATL_REQUIRE(off[lo] - off[c0] < INT_MAX, "a cell's footprint exceeds 2^31 pixels");
      if (off[lo] > off[c0]) bands.push_back({0, 1, c0, lo});
      c0 = lo;
    }
    for (int64_t b = 0; b < batch; ++b)
      for (const Chunk& k : bands) chunks.push_back({b, 1, k.c0, k.c1});
  }
  int64_t max_px = 0, max_seg = 0;
  for (const Chunk& k : chunks) {
    max_px = std::max(max_px, k.nb * (off[k.c1] - off[k.c0]));
    max_seg = std::max(max_seg, k.nb * (k.c1 - k.c0));
  }
  StreamBuf keys(stream), qs(stream), offs(stream), temp(stream);
  ATL_CUDA(keys.alloc(2 * sizeof(K) * max_px));
  ATL_CUDA(qs.alloc(2 * sizeof(int64_t) * max_px));
  ATL_CUDA(offs.alloc(sizeof(int) * (max_seg + 1)));
  size_t temp_bytes = 0;
  K *k_in = keys.as<K>(), *k_out = k_in + max_px;
  int64_t *q_in = qs.as<int64_t>(), *q_out = q_in + max_px;
  const T fill = (T)r.dst_nodata;
  for (const Chunk& k : chunks) {
    const int64_t n_cells = k.c1 - k.c0, n_seg = k.nb * n_cells, slab_px = off[k.c1] - off[k.c0];
    if (slab_px == 0) continue;
    const int* off_d = offs.as<int>();
    k_select_offsets<<<(unsigned)((n_seg + 1 + RP_THREADS - 1) / RP_THREADS), RP_THREADS, 0, stream>>>(
        big.as<int64_t>(), k.c0, n_cells, n_seg, slab_px, offs.as<int>());
    k_select_gather<T><<<dim3((unsigned)n_cells, (unsigned)k.nb), RP_THREADS, 0, stream>>>(
        r, boxes.as<Box>(), big.as<int64_t>(), k.c0, slab_px, src + k.b0 * src_batch, src_row, src_batch, k_in, q_in);
    g_launches += 2;
    ATL_CUDA(cudaGetLastError());
    const int n_items = (int)(k.nb * slab_px);
    size_t need = 0;
    ATL_CUDA(cub::DeviceSegmentedRadixSort::SortPairs(nullptr, need, k_in, k_out, q_in, q_out, n_items, (int)n_seg,
                                                      off_d, off_d + 1, 0, (int)sizeof(K) * 8, stream));
    if (need > temp_bytes) {
      ATL_CUDA(temp.alloc(need));
      temp_bytes = need;
    }
    ATL_CUDA(cub::DeviceSegmentedRadixSort::SortPairs(temp.p, need, k_in, k_out, q_in, q_out, n_items, (int)n_seg,
                                                      off_d, off_d + 1, 0, (int)sizeof(K) * 8, stream));
    k_select_finish<T><<<(unsigned)((n_seg + RP_THREADS - 1) / RP_THREADS), RP_THREADS, 0, stream>>>(
        k_out, q_out, off_d, n_seg, n_cells, k.c0, k.b0, plane, r.resampling, fill, out);
    g_launches += 2;
    ATL_CUDA(cudaGetLastError());
  }
  return ATL_OK;
}

template <typename T>
int reproject_run(int device, const AtlReproject& r, const AtlReprojectOptions& o, int64_t batch, const T* src,
                  int64_t src_row, int64_t src_batch, T* out, cudaStream_t stream) {
  const int64_t plane = r.dst.ny * r.dst.nx;
  if (batch == 0 || plane == 0) return ATL_OK;
  ATL_CUDA(cudaSetDevice(device));
  const int from = r.proj.from.kind, to = r.proj.to.kind;  // destination lattice -> source CRS
  if (r.resampling == ATL_RESAMPLING_NEAREST) {
    const int64_t blocks = (plane + RP_THREADS - 1) / RP_THREADS;
    ATL_REQUIRE(blocks <= 0x7fffffffLL, "destination grid too large");
    const dim3 grid((unsigned)blocks, batch_chunks(batch, blocks, device));
    pair_kernel<NearestKernel<T>::template K>(from, to)<<<grid, RP_THREADS, 0, stream>>>(r, src, batch, src_row,
                                                                                        src_batch, out);
    ++g_launches;
    ATL_CUDA(cudaGetLastError());
    return ATL_OK;
  }
  StreamBuf spans(stream);
  SpanBoxes sp{nullptr, nullptr};
  if (o.row_spans) {
    ATL_CUDA(spans.alloc(sizeof(AtlSpan) * (r.dst.ny + r.dst.nx)));
    ATL_CUDA(cudaMemcpyAsync(spans.p, o.row_spans, sizeof(AtlSpan) * r.dst.ny, cudaMemcpyHostToDevice, stream));
    ATL_CUDA(cudaMemcpyAsync(spans.as<AtlSpan>() + r.dst.ny, o.col_spans, sizeof(AtlSpan) * r.dst.nx,
                             cudaMemcpyHostToDevice, stream));
    sp = SpanBoxes{spans.as<AtlSpan>(), spans.as<AtlSpan>() + r.dst.ny};
  }
  switch (r.resampling) {
    case ATL_RESAMPLING_AVERAGE:
      return box_run<T, Moments<T, ATL_RESAMPLING_AVERAGE>>(device, r, sp, batch, src, src_row, src_batch, out, stream);
    case ATL_RESAMPLING_SUM:
      return box_run<T, Moments<T, ATL_RESAMPLING_SUM>>(device, r, sp, batch, src, src_row, src_batch, out, stream);
    case ATL_RESAMPLING_RMS:
      return box_run<T, Moments<T, ATL_RESAMPLING_RMS>>(device, r, sp, batch, src, src_row, src_batch, out, stream);
    case ATL_RESAMPLING_MIN:
      return box_run<T, Extreme<T, ATL_RESAMPLING_MIN>>(device, r, sp, batch, src, src_row, src_batch, out, stream);
    case ATL_RESAMPLING_MAX:
      return box_run<T, Extreme<T, ATL_RESAMPLING_MAX>>(device, r, sp, batch, src, src_row, src_batch, out, stream);
  }
  return select_run(device, r, sp, o.select_small < 0 ? RP_SMALL : o.select_small,
                    o.scratch_bytes > 0 ? o.scratch_bytes : RP_SELECT_SCRATCH, batch, src, src_row, src_batch, out,
                    stream);
}

bool resampling_ok(int32_t m) {
  switch (m) {
    case ATL_RESAMPLING_NEAREST:
    case ATL_RESAMPLING_AVERAGE:
    case ATL_RESAMPLING_MODE:
    case ATL_RESAMPLING_MAX:
    case ATL_RESAMPLING_MIN:
    case ATL_RESAMPLING_MED:
    case ATL_RESAMPLING_Q1:
    case ATL_RESAMPLING_Q3:
    case ATL_RESAMPLING_SUM:
    case ATL_RESAMPLING_RMS:
      return true;
  }
  return false;
}

bool spans_ok(const AtlSpan* s, int64_t n, int64_t n_src) {
  for (int64_t k = 0; k < n; ++k)
    if (s[k].hi > s[k].lo && !(s[k].lo >= 0 && s[k].hi <= n_src && isfinite(s[k].w_lo) && isfinite(s[k].w_hi) &&
                               s[k].w_lo > 0.0 && s[k].w_hi > 0.0))
      return false;
  return true;
}

}  // namespace atl

using namespace atl;

extern "C" {

int atl_reproject_ex(int device, const AtlReproject* r, const AtlReprojectOptions* o, int32_t dtype, int64_t batch,
                     const void* src_dev, int64_t src_row, int64_t src_batch, void* out_dev, void* stream) {
  ATL_REQUIRE(r, "NULL argument");
  ATL_REQUIRE(batch >= 0, "negative batch");
  const AtlLattice &S = r->src, &D = r->dst;
  ATL_REQUIRE(S.nx > 0 && S.ny > 0 && S.nx <= 0x7fffffffLL && S.ny <= 0x7fffffffLL && D.nx >= 0 && D.ny >= 0,
              "bad size");
  ATL_REQUIRE(S.a != 0.0 && S.e != 0.0 && isfinite(S.a) && isfinite(S.e) && isfinite(S.c) && isfinite(S.f) &&
                  isfinite(D.a) && isfinite(D.e) && isfinite(D.c) && isfinite(D.f),
              "transforms must be finite, with a non-zero source pixel size");
  ATL_REQUIRE(projection_ok(r->proj), "unknown CRS in the projection");
  ATL_REQUIRE(resampling_ok(r->resampling),
              "resampling must be ATL_RESAMPLING_NEAREST, _AVERAGE, _MODE, _MAX, _MIN, _MED, _Q1, _Q3, _SUM or _RMS");
  ATL_REQUIRE(r->resampling == ATL_RESAMPLING_NEAREST ||
                  (r->tile_y >= 1 && r->tile_x >= 1 && r->tile_y * r->tile_x <= RP_THREADS),
              "tile_y * tile_x must lie in [1, 256]");
  const AtlReprojectOptions opt = o ? *o : AtlReprojectOptions{nullptr, nullptr, 0, -1, 0};
  ATL_REQUIRE(!opt.row_spans == !opt.col_spans, "row_spans and col_spans go together");
  ATL_REQUIRE(!opt.row_spans || r->resampling != ATL_RESAMPLING_NEAREST, "nearest takes no spans");
  ATL_REQUIRE(opt.select_small <= RP_SMALL, "select_small must be at most 32");
  ATL_REQUIRE(!opt.row_spans || (spans_ok(opt.row_spans, D.ny, S.ny) && spans_ok(opt.col_spans, D.nx, S.nx)),
              "spans must lie inside the source, with finite positive weights");
  if (batch == 0 || D.nx == 0 || D.ny == 0) return ATL_OK;
  ATL_REQUIRE(src_dev && out_dev, "NULL argument");
  ATL_REQUIRE(src_row >= S.nx && (batch == 1 || src_batch >= src_row * S.ny),
              "source strides smaller than its rows");
  const cudaStream_t s = (cudaStream_t)stream;
  switch (dtype) {
    case ATL_REGRID_F32:
      return reproject_run(device, *r, opt, batch, static_cast<const float*>(src_dev), src_row, src_batch,
                           static_cast<float*>(out_dev), s);
    case ATL_REGRID_F64:
      return reproject_run(device, *r, opt, batch, static_cast<const double*>(src_dev), src_row, src_batch,
                           static_cast<double*>(out_dev), s);
  }
  ATL_REQUIRE(false, "dtype must be ATL_REGRID_F32 or _F64");
  return ATL_ERR_INVALID;
}

int atl_reproject(int device, const AtlReproject* r, int32_t dtype, int64_t batch, const void* src_dev,
                  int64_t src_row, int64_t src_batch, void* out_dev, void* stream) {
  return atl_reproject_ex(device, r, nullptr, dtype, batch, src_dev, src_row, src_batch, out_dev, stream);
}

}  // extern "C"
