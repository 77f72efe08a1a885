// overlay.cu -- area overlap of two polygon collections: I[i, j] = area(dest_i ∩ orig_j) / area(orig_j).
//
// The general form of the reference's compute_indicatormatrix (gis.py:104-145), where `orig` is any
// collection of polygons rather than the cells of a grid (that case is indicator.cu).  The reference
// finds candidates with an STRtree and intersects each pair with shapely in a Python loop; here
// every stage runs on the device:
//
//   k_box_area     one warp per shape: closed bounding box, and the area of an orig shape (shoelace
//                  about its box corner).
//   band index     per shape, its y range cut into nb bands; every edge is listed in the bands its
//                  y range meets, in edge order (k_band_count / _fill, then a stable radix sort).
//   candidates     the orig boxes binned on a uniform grid over their extent (same scheme); one
//                  thread per dest box walks the bins it covers and keeps the orig boxes whose
//                  interior it overlaps, each pair in one bin only (the bin of the lower-left corner
//                  of the two boxes' intersection).  A radix sort puts the pairs in (dest, orig) order.
//   k_pair_area    one warp per pair: Green's theorem on the boundary of D ∩ O,
//                      area(D ∩ O) = sum over edges e of D of ∫_e w_O x dy + sum over edges g of O of ∫_g w_D x dy
//                  with w_S the winding number of S (1 inside, 0 outside; rings are oriented on the
//                  host with the interior on the left, holes clockwise).  Along an edge w changes only
//                  where it crosses an edge of the other shape, so an edge's integral is
//                      w(start) T(ta, tb) + sum over crossings k of s_k T(t_k, tb)
//                  (T = ∫ x dy over a parameter interval, s_k = +1 entering, -1 leaving, [ta, tb]
//                  the part of the edge inside the pair box R): no sorting of crossings.  Only the
//                  edges whose box meets R do any work, found through the band index; the winding
//                  number at a start point is a ray cast over one band of the other shape.
//   compaction     fractions above kKeep, in pair order, into CSR.
//
// Degeneracies (shared edges, vertices on edges, collinear overlaps) are decided exactly by
// simulation of simplicity: every predicate is evaluated for O translated by the infinitesimal
// (eps, eps^2), in which no vertex of one shape lies on the other's boundary.  The area is
// continuous under the translation, so the limit is the area of the unperturbed pair: a boundary
// piece both shapes share counts once when their interiors lie on the same side and not at all
// when they lie on opposite sides, and shapes that only touch get area 0.  The signs come from
// orient2d_sign (orient.cuh) with the symbolic tie-breaks below; the crossing points and the
// integrals are evaluated in float64 on the unperturbed coordinates, relative to the lower-left
// corner of R.
//
// Repeatability: every pair is summed by one warp in an order fixed by the input (lane k takes
// entries k, k+32, ... of band lists sorted by edge index, then a fixed butterfly), so the result
// and its sparsity pattern are bitwise identical from run to run.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "indicator.cuh"
#include "orient.cuh"

namespace atl {
namespace {

constexpr int kBandEdges = 4;         // edges per band of a shape's y-band index (on average)
constexpr int kMaxBands = 1 << 15;    // bands per shape at most
constexpr int kMaxBinsAxis = 2048;    // candidate bins per axis at most
constexpr int kBinsPerShape = 4;      // candidate bins per non-empty orig shape at most
constexpr int kThreads = 256;

// edge = (ax, ay, bx, by) as double4 {x, y, z, w}; box = (xlo, ylo, xhi, yhi) likewise
struct SideDev {
  const double4* edge;       // oriented: the shape's interior on the left
  const int64_t* edge_ptr;   // [n + 1] edges of each shape
  const double4* box;        // [n]; empty shapes (inf, inf, -inf, -inf)
  const int64_t* band0;      // [n] first global band of each shape
  const int32_t* nband;      // [n]
  const int64_t* band_ptr;   // [n_bands + 1] entries of each band
  const uint32_t* band_key;  // [entries] global band of each entry (sorted)
  const int32_t* band_edge;  // [entries] global edge index of each entry
};

struct BinGrid {
  double x0, y0, ibx, iby;  // bin = floor((v - v0) * ib), clamped
  int32_t nbx, nby;
};

// Band of y in a shape's index.  Monotone in y, and computed with explicit round-to-nearest
// operations so that building and querying the index agree in every kernel.
__device__ __forceinline__ int band_of(const double4& box, int nb, double y) {
  const double h = __dsub_rn(box.w, box.y);
  if (nb <= 1 || !(h > 0.0)) return 0;
  const double f = floor(__dmul_rn(__dsub_rn(y, box.y), __ddiv_rn((double)nb, h)));
  return (int)fmin(fmax(f, 0.0), (double)(nb - 1));
}

__device__ __forceinline__ int bin_of(double v, double v0, double ib, int n) {
  const double f = floor(__dmul_rn(__dsub_rn(v, v0), ib));
  return (int)fmin(fmax(f, 0.0), (double)(n - 1));
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One warp per shape: bounding box of its edges; with `area`, the shoelace area about the box's
// lower-left corner (exteriors counter-clockwise and holes clockwise, so holes subtract).
__global__ void k_box_area(const double4* __restrict__ edge, const int64_t* __restrict__ edge_ptr, int32_t n,
                           double4* __restrict__ box, double* __restrict__ area) {
  const int64_t s = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (s >= n) return;
  const int64_t e0 = edge_ptr[s], e1 = edge_ptr[s + 1];
  double xlo = INFINITY, ylo = INFINITY, xhi = -INFINITY, yhi = -INFINITY;
  for (int64_t k = e0 + lane; k < e1; k += 32) {
    const double4 e = edge[k];
    xlo = fmin(xlo, fmin(e.x, e.z));
    xhi = fmax(xhi, fmax(e.x, e.z));
    ylo = fmin(ylo, fmin(e.y, e.w));
    yhi = fmax(yhi, fmax(e.y, e.w));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    xlo = fmin(xlo, __shfl_xor_sync(0xffffffffu, xlo, o));
    ylo = fmin(ylo, __shfl_xor_sync(0xffffffffu, ylo, o));
    xhi = fmax(xhi, __shfl_xor_sync(0xffffffffu, xhi, o));
    yhi = fmax(yhi, __shfl_xor_sync(0xffffffffu, yhi, o));
  }
  if (area) {
    double a = 0.0;
    for (int64_t k = e0 + lane; k < e1; k += 32) {
      const double4 e = edge[k];
      a += (e.x - xlo) * (e.w - ylo) - (e.z - xlo) * (e.y - ylo);
    }
    a = warp_sum(a);
    if (lane == 0) area[s] = 0.5 * a;
  }
  if (lane == 0) box[s] = make_double4(xlo, ylo, xhi, yhi);
}

// Band index, pass 1: bands per edge (span[e]) and entries per band (band_count, integer atomics).
__global__ void k_band_count(const double4* __restrict__ edge, const int32_t* __restrict__ edge_shape, int64_t n_edges,
                             const double4* __restrict__ box, const int64_t* __restrict__ band0,
                             const int32_t* __restrict__ nband, int64_t* __restrict__ span,
                             int32_t* __restrict__ band_count) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const int s = edge_shape[e];
  const double4 g = edge[e], b = box[s];
  const int nb = nband[s];
  const int b0 = band_of(b, nb, fmin(g.y, g.w)), b1 = band_of(b, nb, fmax(g.y, g.w));
  span[e] = b1 - b0 + 1;
  for (int k = b0; k <= b1; ++k) atomicAdd(band_count + band0[s] + k, 1);
}

// pass 2: the (band, edge) entries of every edge at its scanned offset, in edge order.
__global__ void k_band_fill(const double4* __restrict__ edge, const int32_t* __restrict__ edge_shape, int64_t n_edges,
                            const double4* __restrict__ box, const int64_t* __restrict__ band0,
                            const int32_t* __restrict__ nband, const int64_t* __restrict__ off,
                            uint32_t* __restrict__ key, int32_t* __restrict__ val) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const int s = edge_shape[e];
  const double4 g = edge[e], b = box[s];
  const int nb = nband[s];
  const int b0 = band_of(b, nb, fmin(g.y, g.w)), b1 = band_of(b, nb, fmax(g.y, g.w));
  int64_t o = off[e];
  for (int k = b0; k <= b1; ++k, ++o) {
    key[o] = (uint32_t)(band0[s] + k);
    val[o] = (int32_t)e;
  }
}

// Extent and count of the non-empty orig boxes, by one CTA in a fixed order:
// out = {xlo, ylo, xhi, yhi, count}.
__global__ void k_extent(const double4* __restrict__ box, int32_t n, double* __restrict__ out) {
  __shared__ double sh[5][kThreads];
  double v[5] = {INFINITY, INFINITY, -INFINITY, -INFINITY, 0.0};
  for (int s = threadIdx.x; s < n; s += blockDim.x) {
    const double4 b = box[s];
    if (!(b.x <= b.z)) continue;
    v[0] = fmin(v[0], b.x);
    v[1] = fmin(v[1], b.y);
    v[2] = fmax(v[2], b.z);
    v[3] = fmax(v[3], b.w);
    v[4] += 1.0;
  }
  for (int k = 0; k < 5; ++k) sh[k][threadIdx.x] = v[k];
  __syncthreads();
  for (int w = kThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) {
      const int t = threadIdx.x, u = threadIdx.x + w;
      sh[0][t] = fmin(sh[0][t], sh[0][u]);
      sh[1][t] = fmin(sh[1][t], sh[1][u]);
      sh[2][t] = fmax(sh[2][t], sh[2][u]);
      sh[3][t] = fmax(sh[3][t], sh[3][u]);
      sh[4][t] += sh[4][u];
    }
    __syncthreads();
  }
  if (threadIdx.x < 5) out[threadIdx.x] = sh[threadIdx.x][0];
}

// Width and height of every orig box, +inf for an empty one (sorted last).
__global__ void k_box_sizes(const double4* __restrict__ box, int32_t n, double* __restrict__ w,
                            double* __restrict__ h) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const double4 b = box[s];
  const bool empty = !(b.x <= b.z);
  w[s] = empty ? INFINITY : b.z - b.x;
  h[s] = empty ? INFINITY : b.w - b.y;
}

// Candidate bins, pass 1 and 2: the bins each orig box covers (span) and the orig ids per bin.
__global__ void k_bin_count(const double4* __restrict__ box, int32_t n, BinGrid g, int64_t* __restrict__ span,
                            int32_t* __restrict__ bin_count) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const double4 b = box[s];
  if (!(b.x <= b.z)) {
    span[s] = 0;
    return;
  }
  const int i0 = bin_of(b.x, g.x0, g.ibx, g.nbx), i1 = bin_of(b.z, g.x0, g.ibx, g.nbx);
  const int j0 = bin_of(b.y, g.y0, g.iby, g.nby), j1 = bin_of(b.w, g.y0, g.iby, g.nby);
  span[s] = (int64_t)(i1 - i0 + 1) * (j1 - j0 + 1);
  for (int j = j0; j <= j1; ++j)
    for (int i = i0; i <= i1; ++i) atomicAdd(bin_count + (int64_t)j * g.nbx + i, 1);
}

__global__ void k_bin_fill(const double4* __restrict__ box, int32_t n, BinGrid g, const int64_t* __restrict__ off,
                           uint32_t* __restrict__ key, int32_t* __restrict__ val) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const double4 b = box[s];
  if (!(b.x <= b.z)) return;
  const int i0 = bin_of(b.x, g.x0, g.ibx, g.nbx), i1 = bin_of(b.z, g.x0, g.ibx, g.nbx);
  const int j0 = bin_of(b.y, g.y0, g.iby, g.nby), j1 = bin_of(b.w, g.y0, g.iby, g.nby);
  int64_t o = off[s];
  for (int j = j0; j <= j1; ++j)
    for (int i = i0; i <= i1; ++i, ++o) {
      key[o] = (uint32_t)((int64_t)j * g.nbx + i);
      val[o] = s;
    }
}

// One thread per dest box: the orig boxes whose interiors its interior overlaps (a pair of boxes
// that only touch cannot give area).  Each pair is reported in the bin of the lower-left corner of
// the boxes' intersection only.  FILL = false counts, FILL = true writes the (dest << 32 | orig) keys.
template <bool FILL>
__global__ void k_pairs(const double4* __restrict__ dbox, int32_t n_dest, const double4* __restrict__ obox, BinGrid g,
                        const int64_t* __restrict__ bin_ptr, const int32_t* __restrict__ bin_orig,
                        int64_t* __restrict__ count, const int64_t* __restrict__ off, uint64_t* __restrict__ keys) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= n_dest) return;
  const double4 b = dbox[d];
  int64_t c = 0, o = FILL ? off[d] : 0;
  if (b.x < b.z && b.y < b.w) {
    const int i0 = bin_of(b.x, g.x0, g.ibx, g.nbx), i1 = bin_of(b.z, g.x0, g.ibx, g.nbx);
    const int j0 = bin_of(b.y, g.y0, g.iby, g.nby), j1 = bin_of(b.w, g.y0, g.iby, g.nby);
    for (int j = j0; j <= j1; ++j)
      for (int i = i0; i <= i1; ++i) {
        const int64_t bin = (int64_t)j * g.nbx + i;
        for (int64_t k = bin_ptr[bin]; k < bin_ptr[bin + 1]; ++k) {
          const int s = bin_orig[k];
          const double4 q = obox[s];
          if (!(q.x < b.z && b.x < q.z && q.y < b.w && b.y < q.w)) continue;
          if (bin_of(fmax(b.x, q.x), g.x0, g.ibx, g.nbx) != i || bin_of(fmax(b.y, q.y), g.y0, g.iby, g.nby) != j)
            continue;
          if (FILL) keys[o++] = ((uint64_t)d << 32) | (uint32_t)s;
          ++c;
        }
      }
  }
  if (!FILL) count[d] = c;
}

// ---------------------------------------------------------------- exact predicates, O perturbed
// O is translated by delta = (eps, eps^2), eps -> 0+.  Both functions return a non-zero sign.

// sign of orient(P + delta, Q + delta, A): an orig edge (P, Q) against a dest point A.
// = orient(P, Q, A) + (Qy - Py) eps - (Qx - Px) eps^2
__device__ __forceinline__ int side_o(const double4& g, double ax, double ay) {
  const int s = orient2d_sign(g.x, g.y, g.z, g.w, ax, ay);
  if (s) return s;
  if (g.w != g.y) return g.w > g.y ? 1 : -1;
  return g.z > g.x ? -1 : 1;
}

// sign of orient(A, B, P + delta): a dest edge (A, B) against an orig point P.
// = orient(A, B, P) - (By - Ay) eps + (Bx - Ax) eps^2
__device__ __forceinline__ int side_d(const double4& e, double px, double py) {
  const int s = orient2d_sign(e.x, e.y, e.z, e.w, px, py);
  if (s) return s;
  if (e.w != e.y) return e.w > e.y ? -1 : 1;
  return e.z > e.x ? 1 : -1;
}

// Change of the other shape's winding number along edge e where it crosses edge g of the other
// shape (+1 when e passes from the right of g to its left), 0 when they do not cross.
// SELF_O: e is an orig edge (perturbed) and g a dest edge; else the reverse.
template <bool SELF_O>
__device__ __forceinline__ int crossing(const double4& e, const double4& g) {
  if (!SELF_O) {
    const int sa = side_o(g, e.x, e.y), sb = side_o(g, e.z, e.w);
    if (sa == sb) return 0;
    if (side_d(e, g.x, g.y) == side_d(e, g.z, g.w)) return 0;
    return sb;
  }
  const int sp = side_d(g, e.x, e.y), sq = side_d(g, e.z, e.w);
  if (sp == sq) return 0;
  if (side_o(e, g.x, g.y) == side_o(e, g.z, g.w)) return 0;
  return sq;
}

// Winding number of the shape `t` of side T at the start (px, py) of an edge of the other side: a
// ray to +x over the one band of t that holds py (every edge that spans py is listed there).
template <bool SELF_O>
__device__ int winding(double px, double py, const SideDev& T, int t, const double4& bt) {
  const int nb = T.nband[t];
  const int64_t band = T.band0[t] + band_of(bt, nb, py);
  int w = 0;
  for (int64_t k = T.band_ptr[band]; k < T.band_ptr[band + 1]; ++k) {
    const double4 g = T.edge[T.band_edge[k]];
    if (!SELF_O) {  // dest point against orig edges (P + delta, Q + delta)
      if (g.y < py && py <= g.w) {
        if (side_o(g, px, py) > 0) ++w;
      } else if (g.w < py && py <= g.y) {
        if (side_o(g, px, py) < 0) --w;
      }
    } else {  // orig point + delta against dest edges
      if (g.y <= py && py < g.w) {
        if (side_d(g, px, py) > 0) ++w;
      } else if (g.w <= py && py < g.y) {
        if (side_d(g, px, py) < 0) --w;
      }
    }
  }
  return w;
}

// ∫ (x - x0) dy along e over the parameter interval [t1, t2]
__device__ __forceinline__ double seg(const double4& e, double t1, double t2, double x0) {
  return (t2 - t1) * (e.w - e.y) * ((e.x - x0) + 0.5 * (t1 + t2) * (e.z - e.x));
}

// Liang-Barsky: narrow [ta, tb] to the parameters where a0 + t (a1 - a0) lies in [lo, hi].
__device__ __forceinline__ void clip_axis(double a0, double a1, double lo, double hi, double& ta, double& tb) {
  if (a0 == a1) {
    if (a0 < lo || a0 > hi) tb = -1.0;
    return;
  }
  const double inv = 1.0 / (a1 - a0);
  double u = (lo - a0) * inv, v = (hi - a0) * inv;
  if (u > v) {
    const double w = u;
    u = v;
    v = w;
  }
  ta = fmax(ta, u);
  tb = fmin(tb, v);
}

// y of the crossing of dest edge d and orig edge o, computed once for the pair: both edges switch
// weight at this y, so the two boundary pieces that meet there are joined by a horizontal step, on
// which ∫ x dy is 0, and the boundary of D ∩ O stays closed however ill-conditioned the crossing is
// (nearly collinear edges of a border digitised twice).  Along d, then clamped into the y range the
// two edges share.  Not inlined and with explicit roundings, so both kernels' callers get the same bits.
__device__ __noinline__ double crossing_y(double4 d, double4 o) {
  const double dx = __dsub_rn(d.z, d.x), dy = __dsub_rn(d.w, d.y);
  const double ox = __dsub_rn(o.z, o.x), oy = __dsub_rn(o.w, o.y);
  const double num = __dsub_rn(__dmul_rn(__dsub_rn(o.x, d.x), oy), __dmul_rn(__dsub_rn(o.y, d.y), ox));
  const double den = __dsub_rn(__dmul_rn(dx, oy), __dmul_rn(dy, ox));
  double t = __ddiv_rn(num, den);
  t = t > 0.0 ? (t < 1.0 ? t : 1.0) : 0.0;  // NaN (parallel round-off) -> 0
  const double y = __dadd_rn(d.y, __dmul_rn(t, dy));
  const double lo = fmax(fmin(d.y, d.w), fmin(o.y, o.w)), hi = fmin(fmax(d.y, d.w), fmax(o.y, o.w));
  return fmin(fmax(y, lo), hi);
}

// ∫ w_T (x - x0) dy along the part of edge e (of side S) inside the pair box r; e is not horizontal.
template <bool SELF_O>
__device__ double edge_integral(const double4& e, const SideDev& T, int t, const double4& r) {
  double ta = 0.0, tb = 1.0;
  clip_axis(e.x, e.z, r.x, r.z, ta, tb);
  clip_axis(e.y, e.w, r.y, r.w, ta, tb);
  if (!(ta < tb)) return 0.0;
  const double4 bt = T.box[t];
  double acc = 0.0;
  if (!(e.x < bt.x || e.x > bt.z || e.y < bt.y || e.y > bt.w)) {
    const int w = winding<SELF_O>(e.x, e.y, T, t, bt);
    if (w) acc = (double)w * seg(e, ta, tb, r.x);
  }
  const double ylo = fmax(fmin(e.y, e.w), r.y), yhi = fmin(fmax(e.y, e.w), r.w);
  if (!(ylo <= yhi)) return acc;
  const double exlo = fmin(e.x, e.z), exhi = fmax(e.x, e.z);
  const int nb = T.nband[t];
  const int64_t base = T.band0[t];
  const int c0 = band_of(bt, nb, ylo), c1 = band_of(bt, nb, yhi);
  const double ey = __dsub_rn(e.w, e.y);
  for (int64_t k = T.band_ptr[base + c0]; k < T.band_ptr[base + c1 + 1]; ++k) {
    const double4 g = T.edge[T.band_edge[k]];
    if ((int)(T.band_key[k] - base) != max(band_of(bt, nb, fmin(g.y, g.w)), c0)) continue;  // seen in a lower band
    if (fmax(g.x, g.z) < exlo || fmin(g.x, g.z) > exhi || fmax(g.y, g.w) < ylo || fmin(g.y, g.w) > yhi) continue;
    const int s = crossing<SELF_O>(e, g);
    if (!s) continue;
    const double yc = SELF_O ? crossing_y(g, e) : crossing_y(e, g);
    const double tc = __ddiv_rn(__dsub_rn(yc, e.y), ey);  // where e reaches the pair's crossing y
    acc += (double)s * seg(e, fmin(fmax(tc, ta), tb), tb, r.x);
  }
  return acc;
}

// Lane's share of the edges of shape s (side S) that meet r, each integrated against shape t.
template <bool SELF_O>
__device__ double side_sum(const SideDev& S, int s, const SideDev& T, int t, const double4& r, int lane) {
  const double4 bs = S.box[s];
  const int nb = S.nband[s];
  const int64_t base = S.band0[s];
  const int b0 = band_of(bs, nb, r.y), b1 = band_of(bs, nb, r.w);
  double acc = 0.0;
  for (int64_t k = S.band_ptr[base + b0] + lane; k < S.band_ptr[base + b1 + 1]; k += 32) {
    const double4 e = S.edge[S.band_edge[k]];
    if (e.y == e.w) continue;  // horizontal: no x dy
    if ((int)(S.band_key[k] - base) != max(band_of(bs, nb, fmin(e.y, e.w)), b0)) continue;
    if (fmax(e.x, e.z) < r.x || fmin(e.x, e.z) > r.z || fmax(e.y, e.w) < r.y || fmin(e.y, e.w) > r.w) continue;
    acc += edge_integral<SELF_O>(e, T, t, r);
  }
  return acc;
}

// One warp per candidate pair: frac = area(dest ∩ orig) / area(orig), keep = frac > kKeep.
__global__ void k_pair_area(const uint64_t* __restrict__ keys, int64_t n_pairs, SideDev D, SideDev O,
                            const double* __restrict__ area_o, double* __restrict__ frac, int32_t* __restrict__ keep) {
  const int64_t p = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (p >= n_pairs) return;
  const int d = (int)(keys[p] >> 32), o = (int)(keys[p] & 0xffffffffu);
  const double4 bd = D.box[d], bo = O.box[o];
  const double4 r = make_double4(fmax(bd.x, bo.x), fmax(bd.y, bo.y), fmin(bd.z, bo.z), fmin(bd.w, bo.w));
  double acc = side_sum<false>(D, d, O, o, r, lane) + side_sum<true>(O, o, D, d, r, lane);
  acc = warp_sum(acc);
  if (lane == 0) {
    const double f = acc / area_o[o];
    const bool k = f > kKeep;
    frac[p] = k ? f : 0.0;
    keep[p] = k;
  }
}

__global__ void k_compact(const uint64_t* __restrict__ keys, const double* __restrict__ frac,
                          const int32_t* __restrict__ keep, const int32_t* __restrict__ pos, int64_t n_pairs,
                          int32_t* __restrict__ row, int32_t* __restrict__ col, double* __restrict__ val) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_pairs || !keep[p]) return;
  const int32_t q = pos[p];
  row[q] = (int32_t)(keys[p] >> 32);
  col[q] = (int32_t)(keys[p] & 0xffffffffu);
  val[q] = frac[p];
}

// indptr[d] = first kept entry of a row >= d (rows sorted)
__global__ void k_indptr(const int32_t* __restrict__ row, int64_t nnz, int32_t n_dest, int64_t* __restrict__ indptr) {
  const int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (d > n_dest) return;
  int64_t lo = 0, hi = nnz;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (row[mid] < d) lo = mid + 1;
    else hi = mid;
  }
  indptr[d] = lo;
}

template <class T>
struct DevBuf {
  T* p = nullptr;
  ~DevBuf() { cudaFree(p); }
  cudaError_t alloc(size_t n) { return cudaMalloc((void**)&p, std::max<size_t>(n, 1) * sizeof(T)); }
};

// CUB scratch that grows as needed
struct Temp {
  DevBuf<char> buf;
  size_t bytes = 0;
  cudaError_t need(size_t b) {
    if (b <= bytes) return cudaSuccess;
    cudaFree(buf.p);
    buf.p = nullptr;
    bytes = 0;
    cudaError_t e = buf.alloc(b);
    if (e == cudaSuccess) bytes = b;
    return e;
  }
};

int bits_for(uint64_t v) {  // bits needed to represent every value < v
  int b = 1;
  while (b < 64 && (1ull << b) < v) ++b;
  return b;
}

unsigned blocks(int64_t n, int per = kThreads) { return (unsigned)std::max<int64_t>((n + per - 1) / per, 1); }

// Host copy of one side: edges oriented with the interior on the left, grouped by shape.
struct HostSide {
  int32_t n = 0;
  std::vector<double4> edge;
  std::vector<int32_t> edge_shape;
  std::vector<int64_t> edge_ptr, band0;
  std::vector<int32_t> nband;
  int64_t n_bands = 0;
};

// `need_area`: every shape with a ring must enclose a positive area (orig shapes are divided by it).
int orient_side(HostSide& H, int32_t n, const int64_t* srp, const int64_t* rp, const int8_t* hole, const double* xy,
                bool need_area) {
  H.n = n;
  H.edge_ptr.assign((size_t)n + 1, 0);
  H.band0.assign(n, 0);
  H.nband.assign(n, 1);
  for (int32_t s = 0; s < n; ++s) {
    ATL_REQUIRE(srp[s + 1] >= srp[s], "shape_ring_ptr must be non-decreasing");
    double shape_area2 = 0.0;  // exteriors minus holes
    for (int64_t r = srp[s]; r < srp[s + 1]; ++r) {
      const int64_t a = rp[r], b = rp[r + 1];
      ATL_REQUIRE(b >= a, "ring_ptr must be non-decreasing");
      if (b - a < 3) continue;  // no area
      double area2 = 0.0;  // shoelace about the first vertex
      const double x0 = xy[2 * a], y0 = xy[2 * a + 1];
      for (int64_t k = a; k < b; ++k) {
        const int64_t k1 = k + 1 < b ? k + 1 : a;
        ATL_REQUIRE(std::isfinite(xy[2 * k]) && std::isfinite(xy[2 * k + 1]), "non-finite vertex");
        area2 += (xy[2 * k] - x0) * (xy[2 * k1 + 1] - y0) - (xy[2 * k1] - x0) * (xy[2 * k + 1] - y0);
      }
      if (area2 == 0.0) continue;
      shape_area2 += hole[r] ? -std::fabs(area2) : std::fabs(area2);
      const bool flip = (area2 > 0.0) == (hole[r] != 0);  // exteriors counter-clockwise, holes clockwise
      for (int64_t k = a; k < b; ++k) {
        const int64_t k1 = k + 1 < b ? k + 1 : a;
        double4 e = make_double4(xy[2 * k], xy[2 * k + 1], xy[2 * k1], xy[2 * k1 + 1]);
        if (e.x == e.z && e.y == e.w) continue;
        if (flip) e = make_double4(e.z, e.w, e.x, e.y);
        H.edge.push_back(e);
        H.edge_shape.push_back(s);
      }
    }
    if (need_area && srp[s + 1] > srp[s] && !(shape_area2 > 0.0)) {
      set_error("orig shape " + std::to_string(s) + " has zero area");
      return ATL_ERR_INVALID;
    }
    H.edge_ptr[s + 1] = (int64_t)H.edge.size();
    const int64_t ne = H.edge_ptr[s + 1] - H.edge_ptr[s];
    H.band0[s] = H.n_bands;
    H.nband[s] = (int32_t)std::min<int64_t>(std::max<int64_t>(ne / kBandEdges, 1), kMaxBands);
    H.n_bands += H.nband[s];
  }
  ATL_REQUIRE(H.edge.size() < (1ull << 31) && H.n_bands < (1ll << 32), "too many edges");
  return ATL_OK;
}

// Device copy of one side with its boxes, (orig) areas and band index.
struct DevSide {
  DevBuf<double4> edge, box;
  DevBuf<int32_t> edge_shape, nband, band_count, band_edge, val_in;
  DevBuf<int64_t> edge_ptr, band0, band_ptr, span, off;
  DevBuf<uint32_t> band_key, key_in;
  DevBuf<double> area;
  SideDev view() const {
    return SideDev{edge.p, edge_ptr.p, box.p, band0.p, nband.p, band_ptr.p, band_key.p, band_edge.p};
  }
};

int build_side(DevSide& D, const HostSide& H, bool with_area, Temp& temp) {
  const int64_t ne = (int64_t)H.edge.size();
  ATL_CUDA(D.edge.alloc(ne));
  ATL_CUDA(D.edge_shape.alloc(ne));
  ATL_CUDA(D.edge_ptr.alloc(H.n + 1));
  ATL_CUDA(D.band0.alloc(H.n));
  ATL_CUDA(D.nband.alloc(H.n));
  ATL_CUDA(D.box.alloc(H.n));
  ATL_CUDA(D.band_count.alloc(H.n_bands + 1));
  ATL_CUDA(D.band_ptr.alloc(H.n_bands + 1));
  ATL_CUDA(D.span.alloc(ne + 1));
  ATL_CUDA(D.off.alloc(ne + 1));
  if (ne) {
    ATL_CUDA(cudaMemcpy(D.edge.p, H.edge.data(), ne * sizeof(double4), cudaMemcpyHostToDevice));
    ATL_CUDA(cudaMemcpy(D.edge_shape.p, H.edge_shape.data(), ne * 4, cudaMemcpyHostToDevice));
  }
  ATL_CUDA(cudaMemcpy(D.edge_ptr.p, H.edge_ptr.data(), (H.n + 1) * 8, cudaMemcpyHostToDevice));
  ATL_CUDA(cudaMemcpy(D.band0.p, H.band0.data(), H.n * 8, cudaMemcpyHostToDevice));
  ATL_CUDA(cudaMemcpy(D.nband.p, H.nband.data(), H.n * 4, cudaMemcpyHostToDevice));
  if (with_area) ATL_CUDA(D.area.alloc(H.n));
  k_box_area<<<blocks((int64_t)H.n * 32), kThreads>>>(D.edge.p, D.edge_ptr.p, H.n, D.box.p, D.area.p);
  ++g_launches;
  ATL_CUDA(cudaMemset(D.band_count.p, 0, (H.n_bands + 1) * 4));
  ATL_CUDA(cudaMemset(D.span.p, 0, (ne + 1) * 8));
  if (ne) {
    k_band_count<<<blocks(ne), kThreads>>>(D.edge.p, D.edge_shape.p, ne, D.box.p, D.band0.p, D.nband.p, D.span.p,
                                           D.band_count.p);
    ++g_launches;
  }
  size_t b = 0;
  ATL_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, b, D.span.p, D.off.p, ne + 1));
  ATL_CUDA(temp.need(b));
  ATL_CUDA(cub::DeviceScan::ExclusiveSum(temp.buf.p, b, D.span.p, D.off.p, ne + 1));
  b = 0;
  ATL_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, b, D.band_count.p, D.band_ptr.p, H.n_bands + 1));
  ATL_CUDA(temp.need(b));
  ATL_CUDA(cub::DeviceScan::ExclusiveSum(temp.buf.p, b, D.band_count.p, D.band_ptr.p, H.n_bands + 1));
  int64_t n_ent = 0;
  ATL_CUDA(cudaMemcpy(&n_ent, D.off.p + ne, 8, cudaMemcpyDeviceToHost));
  ATL_CUDA(D.key_in.alloc(n_ent));
  ATL_CUDA(D.val_in.alloc(n_ent));
  ATL_CUDA(D.band_key.alloc(n_ent));
  ATL_CUDA(D.band_edge.alloc(n_ent));
  if (n_ent) {
    k_band_fill<<<blocks(ne), kThreads>>>(D.edge.p, D.edge_shape.p, ne, D.box.p, D.band0.p, D.nband.p, D.off.p,
                                          D.key_in.p, D.val_in.p);
    ++g_launches;
    const int end_bit = bits_for((uint64_t)H.n_bands);
    b = 0;
    ATL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, b, D.key_in.p, D.band_key.p, D.val_in.p, D.band_edge.p, n_ent,
                                             0, end_bit));
    ATL_CUDA(temp.need(b));
    ATL_CUDA(cub::DeviceRadixSort::SortPairs(temp.buf.p, b, D.key_in.p, D.band_key.p, D.val_in.p, D.band_edge.p,
                                             n_ent, 0, end_bit));
  }
  ATL_CUDA(cudaGetLastError());
  return ATL_OK;
}

// The matrix of one call into R (rows = dest shapes, columns = orig shapes).
int overlay(AtlIndicator* R, const HostSide& HO, const HostSide& HD) {
  Temp temp;
  DevSide O, D;
  int rc = build_side(O, HO, true, temp);
  if (rc != ATL_OK) return rc;
  rc = build_side(D, HD, false, temp);
  if (rc != ATL_OK) return rc;

  // candidate bins over the orig boxes
  // Bins are sized to the MEDIAN orig box, so that a few huge shapes among many small ones (cells
  // plus a continent) do not make every bin hold every small shape; the huge ones are listed in
  // many bins instead.  At most kBinsPerShape bins per non-empty orig shape.
  const int32_t n_o = HO.n, n_d = HD.n;
  DevBuf<double> d_ext, w_in, h_in, w_sorted, h_sorted;
  ATL_CUDA(d_ext.alloc(5));
  k_extent<<<1, kThreads>>>(O.box.p, n_o, d_ext.p);
  ++g_launches;
  double ext[5];
  ATL_CUDA(cudaMemcpy(ext, d_ext.p, sizeof(ext), cudaMemcpyDeviceToHost));
  if (!(ext[4] > 0.0)) return ATL_OK;  // no orig shape has an edge
  ATL_CUDA(w_in.alloc(n_o));
  ATL_CUDA(h_in.alloc(n_o));
  ATL_CUDA(w_sorted.alloc(n_o));
  ATL_CUDA(h_sorted.alloc(n_o));
  k_box_sizes<<<blocks(n_o), kThreads>>>(O.box.p, n_o, w_in.p, h_in.p);
  ++g_launches;
  size_t b = 0;
  ATL_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, b, w_in.p, w_sorted.p, n_o));
  ATL_CUDA(temp.need(b));
  ATL_CUDA(cub::DeviceRadixSort::SortKeys(temp.buf.p, b, w_in.p, w_sorted.p, n_o));
  ATL_CUDA(cub::DeviceRadixSort::SortKeys(temp.buf.p, b, h_in.p, h_sorted.p, n_o));
  const int64_t mid = (int64_t)ext[4] / 2;  // the non-empty boxes come first
  double med_w = 0.0, med_h = 0.0;
  ATL_CUDA(cudaMemcpy(&med_w, w_sorted.p + mid, 8, cudaMemcpyDeviceToHost));
  ATL_CUDA(cudaMemcpy(&med_h, h_sorted.p + mid, 8, cudaMemcpyDeviceToHost));
  BinGrid g{};
  const double W = ext[2] - ext[0], H = ext[3] - ext[1];
  auto axis = [&](double extent, double size) -> int32_t {
    if (!(extent > 0.0)) return 1;
    size = std::max(size, extent / kMaxBinsAxis);
    return (int32_t)std::min<double>(std::max(std::ceil(extent / size), 1.0), kMaxBinsAxis);
  };
  g.x0 = ext[0];
  g.y0 = ext[1];
  g.nbx = axis(W, med_w);
  g.nby = axis(H, med_h);
  const double cap = kBinsPerShape * ext[4] + 64.0;
  if ((double)g.nbx * g.nby > cap) {  // coarsen both axes alike
    const double f = std::sqrt((double)g.nbx * g.nby / cap);
    g.nbx = std::max<int32_t>((int32_t)(g.nbx / f), 1);
    g.nby = std::max<int32_t>((int32_t)(g.nby / f), 1);
  }
  g.ibx = W > 0.0 ? g.nbx / W : 0.0;
  g.iby = H > 0.0 ? g.nby / H : 0.0;
  const int64_t n_bins = (int64_t)g.nbx * g.nby;

  DevBuf<int64_t> o_span, o_off, bin_ptr, p_count, p_off;
  DevBuf<int32_t> bin_count, bin_val_in, bin_orig;
  DevBuf<uint32_t> bin_key_in, bin_key;
  ATL_CUDA(o_span.alloc(n_o + 1));
  ATL_CUDA(o_off.alloc(n_o + 1));
  ATL_CUDA(bin_count.alloc(n_bins + 1));
  ATL_CUDA(bin_ptr.alloc(n_bins + 1));
  ATL_CUDA(cudaMemset(o_span.p, 0, (n_o + 1) * 8));
  ATL_CUDA(cudaMemset(bin_count.p, 0, (n_bins + 1) * 4));
  k_bin_count<<<blocks(n_o), kThreads>>>(O.box.p, n_o, g, o_span.p, bin_count.p);
  ++g_launches;
  b = 0;
  ATL_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, b, o_span.p, o_off.p, n_o + 1));
  ATL_CUDA(temp.need(b));
  ATL_CUDA(cub::DeviceScan::ExclusiveSum(temp.buf.p, b, o_span.p, o_off.p, n_o + 1));
  b = 0;
  ATL_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, b, bin_count.p, bin_ptr.p, n_bins + 1));
  ATL_CUDA(temp.need(b));
  ATL_CUDA(cub::DeviceScan::ExclusiveSum(temp.buf.p, b, bin_count.p, bin_ptr.p, n_bins + 1));
  int64_t n_ent = 0;
  ATL_CUDA(cudaMemcpy(&n_ent, o_off.p + n_o, 8, cudaMemcpyDeviceToHost));
  ATL_CUDA(bin_key_in.alloc(n_ent));
  ATL_CUDA(bin_val_in.alloc(n_ent));
  ATL_CUDA(bin_key.alloc(n_ent));
  ATL_CUDA(bin_orig.alloc(n_ent));
  k_bin_fill<<<blocks(n_o), kThreads>>>(O.box.p, n_o, g, o_off.p, bin_key_in.p, bin_val_in.p);
  ++g_launches;
  const int bin_bits = bits_for((uint64_t)n_bins);
  b = 0;
  ATL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, b, bin_key_in.p, bin_key.p, bin_val_in.p, bin_orig.p, n_ent, 0,
                                           bin_bits));
  ATL_CUDA(temp.need(b));
  ATL_CUDA(cub::DeviceRadixSort::SortPairs(temp.buf.p, b, bin_key_in.p, bin_key.p, bin_val_in.p, bin_orig.p, n_ent, 0,
                                           bin_bits));

  // candidate pairs in (dest, orig) order
  ATL_CUDA(p_count.alloc(n_d + 1));
  ATL_CUDA(p_off.alloc(n_d + 1));
  ATL_CUDA(cudaMemset(p_count.p, 0, (n_d + 1) * 8));
  k_pairs<false><<<blocks(n_d), kThreads>>>(D.box.p, n_d, O.box.p, g, bin_ptr.p, bin_orig.p, p_count.p, nullptr,
                                            nullptr);
  ++g_launches;
  b = 0;
  ATL_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, b, p_count.p, p_off.p, n_d + 1));
  ATL_CUDA(temp.need(b));
  ATL_CUDA(cub::DeviceScan::ExclusiveSum(temp.buf.p, b, p_count.p, p_off.p, n_d + 1));
  int64_t n_pairs = 0;
  ATL_CUDA(cudaMemcpy(&n_pairs, p_off.p + n_d, 8, cudaMemcpyDeviceToHost));
  if (n_pairs == 0) return ATL_OK;
  ATL_REQUIRE(n_pairs < (1ll << 31), "too many candidate pairs");
  DevBuf<uint64_t> keys_in, keys;
  ATL_CUDA(keys_in.alloc(n_pairs));
  ATL_CUDA(keys.alloc(n_pairs));
  k_pairs<true><<<blocks(n_d), kThreads>>>(D.box.p, n_d, O.box.p, g, bin_ptr.p, bin_orig.p, nullptr, p_off.p,
                                           keys_in.p);
  ++g_launches;
  const int key_bits = 32 + bits_for((uint64_t)n_d);
  b = 0;
  ATL_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, b, keys_in.p, keys.p, n_pairs, 0, key_bits));
  ATL_CUDA(temp.need(b));
  ATL_CUDA(cub::DeviceRadixSort::SortKeys(temp.buf.p, b, keys_in.p, keys.p, n_pairs, 0, key_bits));

  // pair areas, then the kept entries in pair order
  DevBuf<double> frac, val;
  DevBuf<int32_t> keep, pos, row, col;
  DevBuf<int64_t> indptr;
  ATL_CUDA(frac.alloc(n_pairs));
  ATL_CUDA(keep.alloc(n_pairs + 1));
  ATL_CUDA(pos.alloc(n_pairs + 1));
  ATL_CUDA(cudaMemset(keep.p + n_pairs, 0, 4));
  k_pair_area<<<blocks(n_pairs * 32), kThreads>>>(keys.p, n_pairs, D.view(), O.view(), O.area.p, frac.p, keep.p);
  ++g_launches;
  ATL_CUDA(cudaGetLastError());
  b = 0;
  ATL_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, b, keep.p, pos.p, n_pairs + 1));
  ATL_CUDA(temp.need(b));
  ATL_CUDA(cub::DeviceScan::ExclusiveSum(temp.buf.p, b, keep.p, pos.p, n_pairs + 1));
  int32_t nnz = 0;
  ATL_CUDA(cudaMemcpy(&nnz, pos.p + n_pairs, 4, cudaMemcpyDeviceToHost));
  ATL_CUDA(row.alloc(nnz));
  ATL_CUDA(col.alloc(nnz));
  ATL_CUDA(val.alloc(nnz));
  ATL_CUDA(indptr.alloc(n_d + 1));
  k_compact<<<blocks(n_pairs), kThreads>>>(keys.p, frac.p, keep.p, pos.p, n_pairs, row.p, col.p, val.p);
  k_indptr<<<blocks(n_d + 1), kThreads>>>(row.p, nnz, n_d, indptr.p);
  g_launches += 2;
  ATL_CUDA(cudaGetLastError());
  R->indices.resize(nnz);
  R->data.resize(nnz);
  ATL_CUDA(cudaMemcpy(R->indptr.data(), indptr.p, (n_d + 1) * 8, cudaMemcpyDeviceToHost));
  if (nnz) {
    ATL_CUDA(cudaMemcpy(R->indices.data(), col.p, (size_t)nnz * 4, cudaMemcpyDeviceToHost));
    ATL_CUDA(cudaMemcpy(R->data.data(), val.p, (size_t)nnz * 8, cudaMemcpyDeviceToHost));
  }
  return ATL_OK;
}

}  // namespace
}  // namespace atl

using namespace atl;

extern "C" {

int atl_overlay_compute(int device, int32_t n_orig, const int64_t* orig_shape_ring_ptr, const int64_t* orig_ring_ptr,
                        const int8_t* orig_ring_is_hole, const double* orig_xy, int32_t n_dest,
                        const int64_t* dest_shape_ring_ptr, const int64_t* dest_ring_ptr,
                        const int8_t* dest_ring_is_hole, const double* dest_xy, AtlIndicator** out) {
  ATL_REQUIRE(out, "NULL argument");
  *out = nullptr;
  ATL_REQUIRE(n_orig >= 0 && n_dest >= 0, "negative shape count");
  ATL_REQUIRE(orig_shape_ring_ptr && (n_orig == 0 || (orig_ring_ptr && orig_ring_is_hole && orig_xy)),
              "NULL argument");
  ATL_REQUIRE(dest_shape_ring_ptr && (n_dest == 0 || (dest_ring_ptr && dest_ring_is_hole && dest_xy)),
              "NULL argument");
  HostSide HO, HD;
  int rc = orient_side(HO, n_orig, orig_shape_ring_ptr, orig_ring_ptr, orig_ring_is_hole, orig_xy, true);
  if (rc != ATL_OK) return rc;
  rc = orient_side(HD, n_dest, dest_shape_ring_ptr, dest_ring_ptr, dest_ring_is_hole, dest_xy, false);
  if (rc != ATL_OK) return rc;
  AtlIndicator* R = new AtlIndicator();
  R->n_shapes = n_dest;
  R->nx = n_orig;
  R->ny = 1;
  R->indptr.assign((size_t)n_dest + 1, 0);
  if (n_orig > 0 && n_dest > 0 && !HO.edge.empty() && !HD.edge.empty()) {
    cudaError_t ce = cudaSetDevice(device);
    rc = ce == cudaSuccess ? overlay(R, HO, HD) : cuda_fail(ce, "atl_overlay_compute");
    if (rc == ATL_OK) {
      ce = cudaDeviceSynchronize();
      if (ce != cudaSuccess) rc = cuda_fail(ce, "atl_overlay_compute");
    }
  }
  if (rc != ATL_OK) {
    delete R;
    return rc;
  }
  *out = R;
  return ATL_OK;
}

}  // extern "C"
