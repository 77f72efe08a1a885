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
#include <algorithm>
#include <cmath>

#include "common.cuh"
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

}  // extern "C"
