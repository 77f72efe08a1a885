// availability.cu -- land eligibility on a fine pixel lattice (gis.py:263-325 shape_availability) and
// its aggregation to the cutout grid (availabilitymatrix).
//
// The reference rasterises every shape with GDAL, masks and warps every raster with rasterio, dilates
// with scipy.ndimage and averages with a GDAL warp, one shape at a time in a process pool.  The work
// per 100 m pixel is small and uniform and a continent has 1e8-1e9 of them, so here every stage is a
// kernel over the window of one shape:
//
//   k_mask_cross / k_mask_scan   polygon mask: one thread per (edge, row) finds the first centre of
//                                the row that is not strictly left of the edge (exact orient2d sign)
//                                and adds the edge's weight there; a warp per row then sums from the
//                                right, so a pixel holds the sum over the edges right of its centre
//                                (even-odd: its parity; nonzero winding: != 0).
//   k_raster_sample<T>           nearest raster pixel under each centre, nodata rules, lookup table.
//   k_dist_rows / k_dist_cols    buffer: L1 distance transform capped at k, a warp-scan along rows and
//                                per-column sweeps over row chunks with a k-row halo.
//   k_bin_* / k_geometry         buffered geometries: segments binned to 16 x 16 pixel tiles, each
//                                pixel tests only its tile's segments.
//   k_count                      eligible pixels counted per cutout cell: per-CTA shared histogram
//                                over the cells near the tile, global 64-bit atomics for the rest.
//   k_avail_rect / _average /    the reprojected average (compute_shape_availability with dst_*):
//   _finalize                    the rectangle of destination cells with a footprint, each band's
//                                nine class counts per cell of it, then the cells' values.
#include <algorithm>
#include <climits>
#include <cmath>

#include "common.cuh"
#include "footprint.cuh"
#include "orient.cuh"
#include "proj.cuh"

namespace atl {

// ---------------------------------------------------------------- polygon mask
__global__ void k_mask_cross(AtlLattice L, int64_t lat_row0, int64_t n_edges, const double4* __restrict__ edges,
                             const int32_t* __restrict__ edge_w, const int64_t* __restrict__ pair_ptr,
                             const int32_t* __restrict__ row0, int64_t n_pairs, int32_t* __restrict__ cnt) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_pairs) return;
  int64_t lo = 0, hi = n_edges;  // edge e with pair_ptr[e] <= p < pair_ptr[e + 1]
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (pair_ptr[mid] <= p) lo = mid; else hi = mid;
  }
  const int64_t e = lo;
  const int64_t j = (int64_t)row0[e] + (p - pair_ptr[e]);
  if (j < 0 || j >= L.ny) return;
  const double cy = lattice_point(L.f, L.e, (double)(lat_row0 + j) + 0.5);
  const double4 ed = edges[e];
  if ((ed.y > cy) == (ed.w > cy)) return;
  const bool up = ed.w > ed.y;
  const double ax = up ? ed.x : ed.z, ay = up ? ed.y : ed.w;
  const double bx = up ? ed.z : ed.x, by = up ? ed.w : ed.y;
  // first column whose centre is not strictly left of the upward edge a -> b
  const double xi = ax + (cy - ay) * ((bx - ax) / (by - ay));
  double t = ceil((xi - L.c) / L.a - 0.5);
  t = fmin(fmax(t, 0.0), (double)L.nx);
  int64_t i = (int64_t)t;
  while (i > 0 && orient2d_sign(ax, ay, bx, by, lattice_point(L.c, L.a, (double)(i - 1) + 0.5), cy) <= 0) --i;
  while (i < L.nx && orient2d_sign(ax, ay, bx, by, lattice_point(L.c, L.a, (double)i + 0.5), cy) > 0) ++i;
  if (i == 0) return;
  atomicAdd(cnt + j * L.nx + (i - 1), up ? edge_w[e] : -edge_w[e]);
}

// one warp per row: inclusive suffix sum -> mask
__global__ void k_mask_scan(int64_t ny, int64_t nx, const int32_t* __restrict__ cnt, uint8_t* __restrict__ out,
                            int mode, int flip) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= ny) return;
  const int32_t* row = cnt + r * nx;
  uint8_t* o = out + r * nx;
  int32_t carry = 0;
  for (int64_t base = nx - 1; base >= 0; base -= 32) {
    const int64_t i = base - lane;
    int32_t x = i >= 0 ? row[i] : 0;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      const int32_t y = __shfl_up_sync(0xffffffffu, x, s);
      if (lane >= s) x += y;
    }
    x += carry;
    carry = __shfl_sync(0xffffffffu, x, 31);
    if (i >= 0) {
      const int in = mode == ATL_MASK_EVEN_ODD ? (x & 1) : (x != 0);
      o[i] = (uint8_t)(in ^ flip);
    }
  }
}

// ---------------------------------------------------------------- raster sample
template <class T, int FROM, int TO>
__global__ void k_raster_sample(AtlRasterSample s, int64_t j0) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t j = j0 + blockIdx.y;
  if (i >= s.win.nx) return;
  double x = lattice_point(s.win.c, s.win.a, (double)i + 0.5);
  double y = lattice_point(s.win.f, s.win.e, (double)(s.win_row0 + j) + 0.5);
  project<FROM, TO>(s.proj, x, y);
  const double u = floor(__ddiv_rn(__dsub_rn(x, s.ras.c), s.ras.a));
  const double v = floor(__ddiv_rn(__dsub_rn(y, s.ras.f), s.ras.e));
  int ex = s.ex_nodata;
  if (u >= 0.0 && u < (double)s.ras.nx && v >= 0.0 && v < (double)s.ras.ny) {
    const int64_t col = (int64_t)u, row = (int64_t)v;
    const int64_t mi = col - s.mask_i0, mj = row - s.mask_j0;
    if (s.mask && mi >= 0 && mi < s.mask_nx && mj >= 0 && mj < s.mask_ny && s.mask[mj * s.mask_nx + mi])
      ex = s.lut[(int64_t)static_cast<const T*>(s.idx)[row * s.ras.nx + col]];
  }
  uint8_t* o = s.out + j * s.win.nx + i;
  if (s.or_into) {
    if (ex) *o = 1;
  } else {
    *o = (uint8_t)ex;
  }
}

// ---------------------------------------------------------------- buffer (L1 dilation)
constexpr int32_t kFar = 1 << 30;

// One warp per row: distance along the row to the nearest set pixel, min(prefix, suffix) of
// f(i') -/+ i' with f = 0 on set pixels and kFar elsewhere.
__global__ void k_dist_rows(int64_t ny, int64_t nx, const uint8_t* __restrict__ src, int32_t* __restrict__ rd) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= ny) return;
  const uint8_t* row = src + r * nx;
  int32_t* d = rd + r * nx;
  int32_t carry = kFar;  // forward: d(i) = i + min_{i' <= i} (f(i') - i')
  for (int64_t base = 0; base < nx; base += 32) {
    const int64_t i = base + lane;
    int32_t v = (i < nx && row[i]) ? -(int32_t)i : kFar;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      const int32_t y = __shfl_up_sync(0xffffffffu, v, s);
      if (lane >= s) v = min(v, y);
    }
    v = min(v, carry);
    carry = __shfl_sync(0xffffffffu, v, 31);
    if (i < nx) d[i] = v >= kFar ? kFar : v + (int32_t)i;
  }
  carry = kFar;  // backward: d(i) = min_{i' >= i} (f(i') + i') - i
  for (int64_t base = nx - 1; base >= 0; base -= 32) {
    const int64_t i = base - lane;
    int32_t v = (i >= 0 && row[i]) ? (int32_t)i : kFar;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      const int32_t y = __shfl_up_sync(0xffffffffu, v, s);
      if (lane >= s) v = min(v, y);
    }
    v = min(v, carry);
    carry = __shfl_sync(0xffffffffu, v, 31);
    if (i >= 0 && v < kFar) d[i] = min(d[i], v - (int32_t)i);
  }
}

// Thread (column i, chunk of kChunk rows): D(j) = min_j' rd(j') + |j - j'| <= k needs only rows within
// k of the chunk, so a forward sweep from k rows above and a backward sweep from k rows below set
// every pixel of the chunk that lies within k.  Only the chunk's own pixels are written.
constexpr int64_t kChunk = 64;
__global__ void k_dist_cols(int64_t ny, int64_t nx, int32_t k, const int32_t* __restrict__ rd,
                            uint8_t* __restrict__ excl) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nx) return;
  const int64_t j0 = (int64_t)blockIdx.y * kChunk, j1 = min(j0 + kChunk, ny);
  int64_t run = kFar;
  for (int64_t j = max(j0 - (int64_t)k, (int64_t)0); j < j1; ++j) {
    run = min(run + 1, (int64_t)__ldg(rd + j * nx + i));
    if (j >= j0 && run <= k) excl[j * nx + i] = 1;
  }
  run = kFar;
  for (int64_t j = min(j1 + (int64_t)k, ny) - 1; j >= j0; --j) {
    run = min(run + 1, (int64_t)__ldg(rd + j * nx + i));
    if (j < j1 && run <= k) excl[j * nx + i] = 1;
  }
}

// ---------------------------------------------------------------- buffered geometries
__device__ __forceinline__ double seg_dist2(double px, double py, const double4 s) {
  const double dx = s.z - s.x, dy = s.w - s.y;
  const double l2 = dx * dx + dy * dy;
  double t = l2 > 0.0 ? ((px - s.x) * dx + (py - s.y) * dy) / l2 : 0.0;
  t = fmin(fmax(t, 0.0), 1.0);
  const double ex = px - (s.x + t * dx), ey = py - (s.y + t * dy);
  return ex * ex + ey * ey;
}

struct TileGrid {
  int64_t ntx, nty;
};
__device__ __forceinline__ TileGrid tile_grid(const AtlLattice& L) {
  return {(L.nx + ATL_AVAIL_TILE - 1) / ATL_AVAIL_TILE, (L.ny + ATL_AVAIL_TILE - 1) / ATL_AVAIL_TILE};
}

// The tiles a segment may matter to: its box widened by |buffer| in pixel units, then each tile of
// that range kept when its centre lies within |buffer| + half its diagonal (+ one pixel of slack).
template <bool FILL>
__global__ void k_bin(AtlGeomExclusion g, int64_t row0) {
  const int64_t sidx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (sidx >= g.n_segs) return;
  const AtlLattice L = g.win;
  const TileGrid tg = tile_grid(L);
  const double4 s = reinterpret_cast<const double4*>(g.segs)[sidx];
  const double b = fabs(g.buffer);
  const double u0 = (fmin(s.x, s.z) - b - L.c) / L.a, u1 = (fmax(s.x, s.z) + b - L.c) / L.a;
  const double v0 = (fmax(s.y, s.w) + b - L.f) / L.e - (double)row0, v1 = (fmin(s.y, s.w) - b - L.f) / L.e - (double)row0;
  const int64_t ti0 = (int64_t)fmax(floor(u0 / ATL_AVAIL_TILE), 0.0);
  const int64_t ti1 = (int64_t)fmin(floor(u1 / ATL_AVAIL_TILE), (double)(tg.ntx - 1));
  const int64_t tj0 = (int64_t)fmax(floor(v0 / ATL_AVAIL_TILE), 0.0);
  const int64_t tj1 = (int64_t)fmin(floor(v1 / ATL_AVAIL_TILE), (double)(tg.nty - 1));
  const double half = 0.5 * ATL_AVAIL_TILE * L.a;
  const double reach = b + half * 1.4142135623730951 + L.a;
  for (int64_t tj = tj0; tj <= tj1; ++tj)
    for (int64_t ti = ti0; ti <= ti1; ++ti) {
      const double cx = L.c + (double)(ti * ATL_AVAIL_TILE) * L.a + half;
      const double cy = L.f + (double)(row0 + tj * ATL_AVAIL_TILE) * L.e - half;
      if (seg_dist2(cx, cy, s) > reach * reach) continue;
      const int64_t t = tj * tg.ntx + ti;
      if (FILL)
        g.tile_list[atomicAdd(reinterpret_cast<unsigned long long*>(g.tile_cursor + t), 1ull)] = (int32_t)sidx;
      else
        atomicAdd(g.tile_cnt + t, 1);
    }
}

// one CTA per tile, one thread per pixel
__global__ void __launch_bounds__(ATL_AVAIL_TILE* ATL_AVAIL_TILE) k_geometry(AtlGeomExclusion g, int64_t row0) {
  const AtlLattice L = g.win;
  const TileGrid tg = tile_grid(L);
  const int64_t t = blockIdx.x;
  const int64_t i = (t % tg.ntx) * ATL_AVAIL_TILE + threadIdx.x % ATL_AVAIL_TILE;
  const int64_t j = (t / tg.ntx) * ATL_AVAIL_TILE + threadIdx.x / ATL_AVAIL_TILE;
  if (i >= L.nx || j >= L.ny) return;
  const double px = lattice_point(L.c, L.a, (double)i + 0.5), py = lattice_point(L.f, L.e, (double)(row0 + j) + 0.5);
  const double b2 = g.buffer * g.buffer;
  bool near = false;
  if (g.n_segs) {
    const double4* segs = reinterpret_cast<const double4*>(g.segs);
    for (int64_t k = g.tile_ptr[t], k1 = g.tile_ptr[t + 1]; k < k1 && !near; ++k)
      near = seg_dist2(px, py, segs[g.tile_list[k]]) <= b2;
  }
  const int64_t o = j * L.nx + i;
  const bool in = g.inside && g.inside[o];
  bool ex = g.buffer >= 0.0 ? (in || near) : (in && !near);
  if (g.invert) ex = !ex;
  if (ex) g.excl[o] = 1;
}

// ---------------------------------------------------------------- counting
constexpr int kCountTile = 64;   // pixels per CTA side
constexpr int kHist = 8;         // shared histogram: kHist x kHist cells around the tile
template <int FROM, int TO>
__global__ void __launch_bounds__(256) k_count(AtlAvailCount c) {
  __shared__ unsigned int hist[kHist * kHist];
  __shared__ int64_t base_x, base_y;
  __shared__ bool use_hist;
  const AtlLattice L = c.win;
  const int64_t i0 = (int64_t)blockIdx.x * kCountTile, j0 = (int64_t)blockIdx.y * kCountTile;
  for (int k = threadIdx.x; k < kHist * kHist; k += blockDim.x) hist[k] = 0;
  if (threadIdx.x == 0) {
    double x = lattice_point(L.c, L.a, (double)min(i0 + kCountTile / 2, L.nx - 1) + 0.5);
    double y = lattice_point(L.f, L.e, (double)(c.win_row0 + min(j0 + kCountTile / 2, L.ny - 1)) + 0.5);
    project<FROM, TO>(c.proj, x, y);
    const double bx = floor((x - c.gx0) / c.gdx), by = floor((y - c.gy0) / c.gdy);
    // a tile centre without an image (NaN) or far off the grid: every pixel takes the global path
    use_hist = fabs(bx) < 1e18 && fabs(by) < 1e18;
    base_x = use_hist ? (int64_t)bx - kHist / 2 : 0;
    base_y = use_hist ? (int64_t)by - kHist / 2 : 0;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < kCountTile * kCountTile; k += blockDim.x) {
    const int64_t i = i0 + k % kCountTile, j = j0 + k / kCountTile;
    if (i >= L.nx || j >= L.ny || c.excl[j * L.nx + i]) continue;
    double x = lattice_point(L.c, L.a, (double)i + 0.5), y = lattice_point(L.f, L.e, (double)(c.win_row0 + j) + 0.5);
    project<FROM, TO>(c.proj, x, y);
    const double u = floor(__ddiv_rn(__dsub_rn(x, c.gx0), c.gdx));
    const double v = floor(__ddiv_rn(__dsub_rn(y, c.gy0), c.gdy));
    if (!(u >= 0.0 && u < (double)c.gnx && v >= 0.0 && v < (double)c.gny)) continue;
    const int64_t ix = (int64_t)u, iy = (int64_t)v;
    const int64_t hx = ix - base_x, hy = iy - base_y;
    if (use_hist && hx >= 0 && hx < kHist && hy >= 0 && hy < kHist)
      atomicAdd(hist + hy * kHist + hx, 1u);
    else
      atomicAdd(c.counts + iy * c.gnx + ix, 1ull);
  }
  __syncthreads();
  for (int k = threadIdx.x; k < kHist * kHist; k += blockDim.x)
    if (hist[k]) atomicAdd(c.counts + (base_y + k / kHist) * c.gnx + (base_x + k % kHist), (unsigned long long)hist[k]);
}

// ---------------------------------------------------------------- reprojected average
// Window pixel coordinates of dst's lattice point (jj, ii).  Not inlined: the kernels of a pair all
// call this one compiled function, so the box pass, the band kernels, the finalize and
// atl_avail_average_corners see the same bits (inlined, the compiler may contract the projection's
// products and sums differently in each kernel).
template <int FROM, int TO>
__device__ __noinline__ double2 window_uv(const AtlAvailAverage& A, double jj, double ii) {
  double u, v;
  to_source<FROM, TO>(A.dst, A.win, A.proj, jj, ii, u, v);
  return make_double2(u, v);
}

// One destination cell's box on the padded window (footprint.cuh), the same in every pass.
template <int FROM, int TO>
__device__ __noinline__ Box average_box(const AtlAvailAverage& A, int64_t i, int64_t j) {
  Box bx{};
  corner_box(window_uv<FROM, TO>(A, (double)j, (double)i), window_uv<FROM, TO>(A, (double)(j + 1), (double)(i + 1)),
             -A.pad, A.win.nx + A.pad, -A.pad, A.win.ny + A.pad, bx);
  return bx;
}

// The pixels of a span's three classes (first, interior, last) within [lo, hi): [k[c], k[c + 1]) for
// class c = 0, 1, 2 after clipping, empty when k[c + 1] <= k[c].  A one-pixel span is only "first".
struct Classes {
  int lo[3], hi[3];
};
__device__ __forceinline__ Classes span_classes(const Span& s, int lo, int hi) {
  Classes k;
  const bool two = s.hi - s.lo >= 2;
  k.lo[0] = max(s.lo, lo), k.hi[0] = min(s.lo + 1, hi);
  k.lo[1] = max(s.lo + 1, lo), k.hi[1] = min(s.hi - 1, hi);
  k.lo[2] = two ? max(s.hi - 1, lo) : 0, k.hi[2] = two ? min(s.hi, hi) : 0;
  return k;
}
__device__ __forceinline__ int class_size(const Classes& k, int c) {  // selects: c may be a runtime value
  const int lo = c == 0 ? k.lo[0] : (c == 1 ? k.lo[1] : k.lo[2]), hi = c == 0 ? k.hi[0] : (c == 1 ? k.hi[1] : k.hi[2]);
  return max(hi - lo, 0);
}

// sum of the bytes of w at offsets [lo, hi) (clipped to [0, 4))
__device__ __forceinline__ unsigned bytes_in(unsigned w, int64_t lo, int64_t hi) {
  const int l = (int)min(max(lo, (int64_t)0), (int64_t)4), h = (int)min(max(hi, (int64_t)0), (int64_t)4);
  if (h <= l) return 0u;
  const unsigned mask = (unsigned)((1ull << (8 * h)) - 1) & ~(unsigned)((1ull << (8 * l)) - 1);
  return __dp4a(w & mask, 0x01010101u, 0u);
}
// sum of the bytes of the 16-byte chunk w at offsets [lo, hi)
__device__ __forceinline__ unsigned chunk_sum(const uint4& w, int64_t lo, int64_t hi) {
  if (hi <= 0 || lo >= 16 || hi <= lo) return 0u;
  if (lo <= 0 && hi >= 16) return __dp4a(w.x, 0x01010101u, __dp4a(w.y, 0x01010101u, __dp4a(w.z, 0x01010101u,
                                         __dp4a(w.w, 0x01010101u, 0u))));
  return bytes_in(w.x, lo, hi) + bytes_in(w.y, lo - 4, hi - 4) + bytes_in(w.z, lo - 8, hi - 8) +
         bytes_in(w.w, lo - 12, hi - 12);
}

// Box pass: the bounding rectangle of the cells with a non-empty box (rect: row0, col0, row1, col1).
// CTA (x, y) takes columns x * RP_THREADS ... of the rows y, y + gridDim.y, ...
template <int FROM, int TO>
__global__ void __launch_bounds__(RP_THREADS) k_avail_rect(const __grid_constant__ AtlAvailAverage A,
                                                           int* __restrict__ rect) {
  __shared__ int s_rect[4];
  if (threadIdx.x == 0) s_rect[0] = s_rect[1] = INT_MAX, s_rect[2] = s_rect[3] = 0;
  __syncthreads();
  const int j = blockIdx.x * RP_THREADS + threadIdx.x;
  if (j < A.dst.nx) {
    for (int i = blockIdx.y; i < A.dst.ny; i += gridDim.y) {
      const Box bx = average_box<FROM, TO>(A, i, j);
      if (bx.c.hi > bx.c.lo && bx.r.hi > bx.r.lo) {
        atomicMin(s_rect + 0, i);
        atomicMin(s_rect + 1, j);
        atomicMax(s_rect + 2, i + 1);
        atomicMax(s_rect + 3, j + 1);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_rect[2] > 0) {
    atomicMin(rect + 0, s_rect[0]);
    atomicMin(rect + 1, s_rect[1]);
    atomicMax(rect + 2, s_rect[2]);
    atomicMax(rect + 3, s_rect[3]);
  }
}

// Band pass: a CTA owns a tile of tile_y x tile_x cells of the rectangle and adds the band's nine
// counts of each cell whose box meets the band.  Boxes of at most RP_SMALL band pixels are counted by
// the cell's thread, larger ones by the whole CTA (as in k_reproject_avg): thread t takes the 16-byte
// aligned chunks t, t + RP_THREADS, ... of the big boxes' rows (one list for all of them) and sums
// their excluded bytes with __dp4a per column class; the counts are exact, so neither the split nor
// the order matters, and each cell has one owner per launch.  An aligned chunk never leaves the 16-byte segment of a byte of the row,
// so it stays inside the allocation.
template <int FROM, int TO>
__global__ void __launch_bounds__(RP_THREADS) k_avail_average(const __grid_constant__ AtlAvailAverage A, const uint8_t* __restrict__ excl,
                                                              int64_t band_row0, int64_t band_ny, int64_t n_tx,
                                                              long long* __restrict__ counts) {
  __shared__ Box s_box[RP_THREADS];
  __shared__ int s_big[RP_THREADS], s_nbig;
  __shared__ int64_t s_item[RP_THREADS + 1];  // the big cells' first items
  __shared__ unsigned s_ex[RP_THREADS][9];     // their excluded pixels per class pair

  const int tid = threadIdx.x;
  const int64_t rw = A.col1 - A.col0, nx = A.win.nx;
  const int64_t i = A.row0 + blockIdx.x / n_tx * A.tile_y + tid / A.tile_x;
  const int64_t j = A.col0 + blockIdx.x % n_tx * A.tile_x + tid % A.tile_x;
  const int r_lo = (int)band_row0, r_hi = (int)(band_row0 + band_ny);  // the band's window rows
  if (tid == 0) s_nbig = 0;
  __syncthreads();
  bool mine = tid < A.tile_y * A.tile_x && i < A.row1 && j < A.col1;
  if (mine) {
    Box bx = average_box<FROM, TO>(A, i, j);
    bx.cell = (i - A.row0) * rw + (j - A.col0);
    s_box[tid] = bx;
    // the box's pixels in the band: rows [r_lo, r_hi), real columns [0, nx)
    const int64_t h = min(bx.r.hi, r_hi) - max(bx.r.lo, r_lo), w = min((int64_t)bx.c.hi, nx) - max(bx.c.lo, 0);
    if (h <= 0 || w <= 0 || bx.c.hi <= bx.c.lo || bx.r.hi <= bx.r.lo) {
      mine = false;
    } else if (h * w > RP_SMALL) {
      s_big[atomicAdd(&s_nbig, 1)] = tid;
      mine = false;
    }
  }
  __syncthreads();

  if (mine) {  // a small box: this thread, every class pair
    const Box& B = s_box[tid];
    const Classes R = span_classes(B.r, r_lo, r_hi), K = span_classes(B.c, 0, (int)nx);
    long long* n = counts + B.cell * 9;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      int got[3] = {0, 0, 0};
      for (int rr = R.lo[a]; rr < R.hi[a]; ++rr) {
        const uint8_t* p = excl + (int64_t)(rr - r_lo) * nx;
#pragma unroll
        for (int b = 0; b < 3; ++b)
          for (int cc = K.lo[b]; cc < K.hi[b]; ++cc) got[b] += p[cc] == 0;
      }
#pragma unroll
      for (int b = 0; b < 3; ++b) n[3 * a + b] += got[b];
    }
  }

  // the large boxes: the whole CTA walks one list of their (row, 16-byte chunk) items, each cell's
  // items in a run, and adds the excluded bytes of each class pair up in shared memory
  const int n_big = s_nbig;
  if (n_big == 0) return;
  for (int q = tid; q < n_big; q += RP_THREADS) {
    const Box& B = s_box[s_big[q]];
    const int rows = min(B.r.hi, r_hi) - max(B.r.lo, r_lo);
    const int cols = (int)(min((int64_t)B.c.hi, nx) - max(B.c.lo, 0));
    s_item[q + 1] = (int64_t)rows * ((cols + 15) / 16 + 1);  // chunks per row, at most
#pragma unroll
    for (int t = 0; t < 9; ++t) s_ex[q][t] = 0u;
  }
  __syncthreads();
  if (tid == 0) {
    s_item[0] = 0;
    for (int q = 0; q < n_big; ++q) s_item[q + 1] += s_item[q];
  }
  __syncthreads();
  const int64_t n_items = s_item[n_big];
  int q = -1, rlo = 0, clo = 0, chi = 0, kw = 1, blo = 0, bhi = 0;
  Classes K{};
  int64_t first = 0, next = 0;
  for (int64_t e = tid; e < n_items; e += RP_THREADS) {
    if (e >= next) {  // the item belongs to a later cell: take its box
      do ++q;
      while (s_item[q + 1] <= e);
      const Box& B = s_box[s_big[q]];
      K = span_classes(B.c, 0, (int)nx);
      rlo = max(B.r.lo, r_lo), clo = max(B.c.lo, 0), chi = (int)min((int64_t)B.c.hi, nx);
      kw = (chi - clo + 15) / 16 + 1, blo = B.r.lo, bhi = B.r.hi;
      first = s_item[q], next = s_item[q + 1];
    }
    const int64_t l = e - first;
    int64_t dr, k;
    if (l <= 0xffffffffLL) {
      dr = (unsigned)l / (unsigned)kw, k = (unsigned)l % (unsigned)kw;
    } else {
      dr = l / kw, k = l % kw;
    }
    const int64_t rr = rlo + dr;
    const uint8_t* p = excl + (rr - r_lo) * nx;
    const uintptr_t at = (reinterpret_cast<uintptr_t>(p + clo) & ~(uintptr_t)15) + 16 * (uintptr_t)k;
    if (at > reinterpret_cast<uintptr_t>(p + chi - 1)) continue;  // this row needs one chunk less
    const uint4 w = __ldg(reinterpret_cast<const uint4*>(at));
    const int64_t o = (int64_t)(reinterpret_cast<uintptr_t>(p) - at);  // column c is byte o + c
    const int ra = rr == blo ? 0 : (rr == bhi - 1 ? 2 : 1);
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      const unsigned x = K.hi[b] > K.lo[b] ? chunk_sum(w, o + K.lo[b], o + K.hi[b]) : 0u;
      if (x) atomicAdd(&s_ex[q][3 * ra + b], x);
    }
  }
  __syncthreads();
  for (int t = tid; t < n_big * 9; t += RP_THREADS) {
    const Box& B = s_box[s_big[t / 9]];
    const Classes R = span_classes(B.r, r_lo, r_hi), K = span_classes(B.c, 0, (int)nx);
    const int ab = t % 9;
    counts[B.cell * 9 + ab] += (long long)class_size(R, ab / 3) * class_size(K, ab % 3) - s_ex[t / 9][ab];
  }
}

// Finalize: the value of each cell of the rectangle from its counts and its box's weights.
template <int FROM, int TO>
__global__ void __launch_bounds__(RP_THREADS) k_avail_finalize(const __grid_constant__ AtlAvailAverage A, const long long* __restrict__ counts,
                                                               double* __restrict__ out) {
  const int64_t rw = A.col1 - A.col0;
  const int64_t cell = (int64_t)blockIdx.x * RP_THREADS + threadIdx.x;
  if (cell >= (A.row1 - A.row0) * rw) return;
  const Box B = average_box<FROM, TO>(A, A.row0 + cell / rw, A.col0 + cell % rw);
  if (B.c.hi <= B.c.lo || B.r.hi <= B.r.lo) {
    out[cell] = 0.0;
    return;
  }
  const long long* n = counts + cell * 9;
  double S[3];
#pragma unroll
  for (int a = 0; a < 3; ++a)
    S[a] = __dadd_rn(__dadd_rn(__dmul_rn(B.c.w_lo, (double)n[3 * a]), (double)n[3 * a + 1]),
                     __dmul_rn(B.c.w_hi, (double)n[3 * a + 2]));
  const double num = __dadd_rn(__dadd_rn(__dmul_rn(B.r.w_lo, S[0]), S[1]), __dmul_rn(B.r.w_hi, S[2]));
  const int mx = B.c.hi - B.c.lo, my = B.r.hi - B.r.lo;
  const double Wx = mx == 1 ? B.c.w_lo : __dadd_rn(__dadd_rn(B.c.w_lo, B.c.w_hi), (double)(mx - 2));
  const double Wy = my == 1 ? B.r.w_lo : __dadd_rn(__dadd_rn(B.r.w_lo, B.r.w_hi), (double)(my - 2));
  out[cell] = __ddiv_rn(num, __dmul_rn(Wy, Wx));
}

// The window pixel coordinates of dst's lattice points (col, row) = (k % (nx + 1), k / (nx + 1)).
template <int FROM, int TO>
__global__ void __launch_bounds__(RP_THREADS) k_avail_corners(const __grid_constant__ AtlAvailAverage A, double* __restrict__ uv) {
  const int64_t k = (int64_t)blockIdx.x * RP_THREADS + threadIdx.x, lx = A.dst.nx + 1;
  if (k >= (A.dst.ny + 1) * lx) return;
  const double2 p = window_uv<FROM, TO>(A, (double)(k % lx), (double)(k / lx));
  uv[2 * k] = p.x;
  uv[2 * k + 1] = p.y;
}

template <int FROM, int TO>
struct AvgRectKernel {
  static auto get() { return k_avail_rect<FROM, TO>; }
};
template <int FROM, int TO>
struct AvgCountKernel {
  static auto get() { return k_avail_average<FROM, TO>; }
};
template <int FROM, int TO>
struct AvgFinalizeKernel {
  static auto get() { return k_avail_finalize<FROM, TO>; }
};
template <int FROM, int TO>
struct AvgCornersKernel {
  static auto get() { return k_avail_corners<FROM, TO>; }
};

template <class T>
struct RasterSampleKernel {
  template <int FROM, int TO>
  struct K {
    static auto get() { return k_raster_sample<T, FROM, TO>; }
  };
};
template <int FROM, int TO>
struct CountKernel {
  static auto get() { return k_count<FROM, TO>; }
};

int lattice_ok(const AtlLattice* L) {
  return L && L->nx > 0 && L->ny > 0 && L->a > 0.0 && L->e < 0.0 && std::isfinite(L->c) && std::isfinite(L->f);
}

// The descriptor of the reprojected average, checked on the host; with_rect: its rectangle and tile too
int average_check(const AtlAvailAverage* A, bool with_rect) {
  ATL_REQUIRE(A && lattice_ok(&A->win) && std::isfinite(A->win.a) && std::isfinite(A->win.e),
              "bad window lattice (need nx, ny > 0, a > 0, e < 0)");
  const AtlLattice& D = A->dst;
  ATL_REQUIRE(D.nx > 0 && D.ny > 0 && D.nx < 0x7fffffffLL && D.ny < 0x7fffffffLL && D.a != 0.0 && D.e != 0.0 &&
                  std::isfinite(D.a) && std::isfinite(D.e) && std::isfinite(D.c) && std::isfinite(D.f),
              "bad destination lattice (need nx, ny > 0 and finite, non-zero a and e)");
  ATL_REQUIRE(A->pad >= 0 && A->win.nx + A->pad < 0x7fffffffLL && A->win.ny + A->pad < 0x7fffffffLL, "bad pad");
  ATL_REQUIRE(projection_ok(A->proj), "unknown CRS in the projection");
  if (with_rect) {
    ATL_REQUIRE(A->row0 >= 0 && A->row0 <= A->row1 && A->row1 <= D.ny && A->col0 >= 0 && A->col0 <= A->col1 &&
                    A->col1 <= D.nx,
                "the rectangle must lie within the destination grid");
    ATL_REQUIRE(A->tile_y >= 1 && A->tile_x >= 1 && A->tile_y * A->tile_x <= RP_THREADS,
                "tile_y * tile_x must lie in [1, 256]");
  }
  return ATL_OK;
}

}  // namespace atl

using namespace atl;

extern "C" {

int atl_avail_mask(int device, const AtlLattice* lat, int64_t lat_row0, int64_t n_edges, const double* edges,
                   const int32_t* edge_w, const int64_t* pair_ptr, const int32_t* row0, int32_t* cnt, uint8_t* out,
                   int32_t mode, int32_t flip, void* stream) {
  ATL_REQUIRE(lattice_ok(lat) && lat_row0 >= 0, "bad lattice (need nx, ny > 0, a > 0, e < 0, row0 >= 0)");
  ATL_REQUIRE(cnt && out && n_edges >= 0 && (n_edges == 0 || (edges && edge_w && pair_ptr && row0)), "NULL argument");
  ATL_REQUIRE(mode == ATL_MASK_EVEN_ODD || mode == ATL_MASK_NONZERO, "unknown mask mode");
  ATL_CUDA(cudaSetDevice(device));
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t n = lat->nx * lat->ny;
  ATL_CUDA(cudaMemsetAsync(cnt, 0, n * sizeof(int32_t), st));
  if (n_edges > 0) {
    int64_t n_pairs = 0;
    ATL_CUDA(cudaMemcpyAsync(&n_pairs, pair_ptr + n_edges, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    ATL_CUDA(cudaStreamSynchronize(st));
    if (n_pairs > 0) {
      k_mask_cross<<<(unsigned)((n_pairs + 255) / 256), 256, 0, st>>>(
          *lat, lat_row0, n_edges, reinterpret_cast<const double4*>(edges), edge_w, pair_ptr, row0, n_pairs, cnt);
      ++g_launches;
    }
  }
  k_mask_scan<<<(unsigned)((lat->ny * 32 + 255) / 256), 256, 0, st>>>(lat->ny, lat->nx, cnt, out, mode, flip ? 1 : 0);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

int atl_avail_raster_sample(int device, const AtlRasterSample* s, void* stream) {
  ATL_REQUIRE(s && lattice_ok(&s->win) && lattice_ok(&s->ras), "bad lattice (need nx, ny > 0, a > 0, e < 0)");
  ATL_REQUIRE(s->idx && s->lut && s->out, "NULL argument");
  ATL_REQUIRE(s->idx_bytes == 1 || s->idx_bytes == 4, "idx_bytes must be 1 or 4");
  ATL_REQUIRE(projection_ok(s->proj), "unknown CRS in the projection");
  ATL_REQUIRE(s->win_row0 >= 0, "negative band row");
  ATL_CUDA(cudaSetDevice(device));
  const int from = s->proj.from.kind, to = s->proj.to.kind;
  const auto kern = s->idx_bytes == 1 ? pair_kernel<RasterSampleKernel<uint8_t>::K>(from, to)
                                      : pair_kernel<RasterSampleKernel<int32_t>::K>(from, to);
  for (int64_t j0 = 0; j0 < s->win.ny; j0 += 65535) {  // the grid's y limit: slabs of rows
    const dim3 grid((unsigned)((s->win.nx + 255) / 256), (unsigned)std::min<int64_t>(65535, s->win.ny - j0));
    kern<<<grid, 256, 0, (cudaStream_t)stream>>>(*s, j0);
    ++g_launches;
  }
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

int atl_avail_dilate(int device, int64_t ny, int64_t nx, int32_t k, const uint8_t* src, int32_t* rowdist,
                     uint8_t* excl, void* stream) {
  ATL_REQUIRE(ny > 0 && nx > 0 && k >= 0 && nx < kFar / 2, "bad window");
  ATL_REQUIRE(src && rowdist && excl, "NULL argument");
  ATL_CUDA(cudaSetDevice(device));
  cudaStream_t st = (cudaStream_t)stream;
  k_dist_rows<<<(unsigned)((ny * 32 + 255) / 256), 256, 0, st>>>(ny, nx, src, rowdist);
  const int64_t chunks = (ny + kChunk - 1) / kChunk;
  ATL_REQUIRE(chunks <= 65535, "window too tall");
  k_dist_cols<<<dim3((unsigned)((nx + 127) / 128), (unsigned)chunks), 128, 0, st>>>(ny, nx, k, rowdist, excl);
  g_launches += 2;
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

int atl_avail_geom_bin(int device, const AtlGeomExclusion* g, int64_t win_row0, int32_t phase, void* stream) {
  ATL_REQUIRE(g && lattice_ok(&g->win) && win_row0 >= 0, "bad lattice (need nx, ny > 0, a > 0, e < 0, row0 >= 0)");
  ATL_REQUIRE(g->n_segs >= 0 && (g->n_segs == 0 || g->segs), "NULL segments");
  ATL_REQUIRE(phase == 0 ? g->tile_cnt != nullptr : (g->tile_cursor && g->tile_list), "NULL tile arrays");
  if (g->n_segs == 0) return ATL_OK;
  ATL_CUDA(cudaSetDevice(device));
  const unsigned blocks = (unsigned)((g->n_segs + 127) / 128);
  if (phase == 0)
    k_bin<false><<<blocks, 128, 0, (cudaStream_t)stream>>>(*g, win_row0);
  else
    k_bin<true><<<blocks, 128, 0, (cudaStream_t)stream>>>(*g, win_row0);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

int atl_avail_geometry(int device, const AtlGeomExclusion* g, int64_t win_row0, void* stream) {
  ATL_REQUIRE(g && lattice_ok(&g->win) && win_row0 >= 0, "bad lattice (need nx, ny > 0, a > 0, e < 0, row0 >= 0)");
  ATL_REQUIRE(g->excl && (g->n_segs == 0 || (g->segs && g->tile_ptr && g->tile_list)), "NULL argument");
  ATL_CUDA(cudaSetDevice(device));
  const int64_t tiles = ((g->win.nx + ATL_AVAIL_TILE - 1) / ATL_AVAIL_TILE) *
                        ((g->win.ny + ATL_AVAIL_TILE - 1) / ATL_AVAIL_TILE);
  ATL_REQUIRE(tiles < (1LL << 31), "window too large");
  k_geometry<<<(unsigned)tiles, ATL_AVAIL_TILE * ATL_AVAIL_TILE, 0, (cudaStream_t)stream>>>(*g, win_row0);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

int atl_avail_count(int device, const AtlAvailCount* c, void* stream) {
  ATL_REQUIRE(c && lattice_ok(&c->win), "bad lattice (need nx, ny > 0, a > 0, e < 0)");
  ATL_REQUIRE(c->excl && c->counts, "NULL argument");
  ATL_REQUIRE(c->gnx > 0 && c->gny > 0 && c->gdx > 0.0 && c->gdy > 0.0, "bad cutout grid");
  ATL_REQUIRE(projection_ok(c->proj), "unknown CRS in the projection");
  ATL_REQUIRE(c->win_row0 >= 0, "negative band row");
  ATL_CUDA(cudaSetDevice(device));
  const int64_t bx = (c->win.nx + kCountTile - 1) / kCountTile, by = (c->win.ny + kCountTile - 1) / kCountTile;
  ATL_REQUIRE(by <= 65535, "window too tall");
  const auto kern = pair_kernel<CountKernel>(c->proj.from.kind, c->proj.to.kind);
  kern<<<dim3((unsigned)bx, (unsigned)by), 256, 0, (cudaStream_t)stream>>>(*c);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

int atl_avail_average_rect(int device, const AtlAvailAverage* a, int32_t* rect_dev, int32_t* rect_host,
                           void* stream) {
  if (int rc = average_check(a, false)) return rc;
  ATL_REQUIRE(rect_dev && rect_host, "NULL argument");
  const dim3 grid((unsigned)((a->dst.nx + RP_THREADS - 1) / RP_THREADS), (unsigned)std::min<int64_t>(a->dst.ny, 65535));
  ATL_CUDA(cudaSetDevice(device));
  const cudaStream_t st = (cudaStream_t)stream;
  int32_t r[4] = {INT_MAX, INT_MAX, 0, 0};
  ATL_CUDA(cudaMemcpyAsync(rect_dev, r, sizeof(r), cudaMemcpyHostToDevice, st));
  pair_kernel<AvgRectKernel>(a->proj.from.kind, a->proj.to.kind)<<<grid, RP_THREADS, 0, st>>>(*a, rect_dev);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  ATL_CUDA(cudaMemcpyAsync(r, rect_dev, sizeof(r), cudaMemcpyDeviceToHost, st));
  ATL_CUDA(cudaStreamSynchronize(st));
  if (r[2] == 0) r[0] = r[1] = r[3] = 0;  // no cell has a box
  for (int k = 0; k < 4; ++k) rect_host[k] = r[k];
  return ATL_OK;
}

int atl_avail_average_counts(int device, const AtlAvailAverage* a, const uint8_t* excl, int64_t band_row0,
                             int64_t band_ny, int64_t* counts, void* stream) {
  if (int rc = average_check(a, true)) return rc;
  ATL_REQUIRE(band_row0 >= 0 && band_ny > 0 && band_row0 + band_ny <= a->win.ny, "the band must lie within the window");
  ATL_REQUIRE(excl && counts, "NULL argument");
  const int64_t n_ty = (a->row1 - a->row0 + a->tile_y - 1) / a->tile_y;
  const int64_t n_tx = (a->col1 - a->col0 + a->tile_x - 1) / a->tile_x;
  if (n_ty * n_tx == 0) return ATL_OK;
  ATL_REQUIRE(n_ty * n_tx <= 0x7fffffffLL, "rectangle too large");
  ATL_CUDA(cudaSetDevice(device));
  pair_kernel<AvgCountKernel>(a->proj.from.kind, a->proj.to.kind)<<<(unsigned)(n_ty * n_tx), RP_THREADS, 0,
                                                                    (cudaStream_t)stream>>>(
      *a, excl, band_row0, band_ny, n_tx, reinterpret_cast<long long*>(counts));
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

int atl_avail_average_finalize(int device, const AtlAvailAverage* a, const int64_t* counts, double* out,
                               void* stream) {
  if (int rc = average_check(a, true)) return rc;
  ATL_REQUIRE(counts && out, "NULL argument");
  const int64_t cells = (int64_t)(a->row1 - a->row0) * (a->col1 - a->col0);
  if (cells == 0) return ATL_OK;
  ATL_CUDA(cudaSetDevice(device));
  pair_kernel<AvgFinalizeKernel>(a->proj.from.kind, a->proj.to.kind)<<<(unsigned)((cells + RP_THREADS - 1) /
                                                                                  RP_THREADS),
                                                                       RP_THREADS, 0, (cudaStream_t)stream>>>(
      *a, reinterpret_cast<const long long*>(counts), out);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

int atl_avail_average_corners(int device, const AtlAvailAverage* a, double* uv, void* stream) {
  if (int rc = average_check(a, false)) return rc;
  ATL_REQUIRE(uv, "NULL argument");
  const int64_t pts = (a->dst.ny + 1) * (a->dst.nx + 1), blocks = (pts + RP_THREADS - 1) / RP_THREADS;
  ATL_REQUIRE(blocks <= 0x7fffffffLL, "destination grid too large");
  ATL_CUDA(cudaSetDevice(device));
  pair_kernel<AvgCornersKernel>(a->proj.from.kind, a->proj.to.kind)<<<(unsigned)blocks, RP_THREADS, 0,
                                                                      (cudaStream_t)stream>>>(*a, uv);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

}  // extern "C"
