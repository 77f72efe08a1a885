// indicator.cu -- shapes -> (n_shapes, ny*nx) overlap matrix on a regular grid.
//
// Replaces the step in front of the hot path, Cutout.indicatormatrix ->
// gis.py:104-145 compute_indicatormatrix: I[i, j] = area(shape_i ∩ cell_j) /
// area(cell_j), where the cells are the boxes of Cutout.grid (cutout.py:355-376:
// centre (x, y), half-width (dx/2, dy/2)).  The reference loops over shapely
// intersections in Python; on a regular grid the same areas follow exactly from
// the polygon edges alone.
//
// Method (signed-area accumulation, the exact-coverage technique of vector
// rasterisers): in grid units (cells = unit squares) and for one row band
// j <= v < j+1, the part of cell i covered by a polygon is
//     cov(j, i) = - sum over edges  dir * ∫ clamp(i + 1 - u_e(v), 0, 1) dv
// (dir = +1 for an edge running towards +v; counter-clockwise rings).  For one
// edge piece the integral is 0 left of it, its full height h right of it, and a
// closed-form quadratic inside the cells it crosses, so an edge only touches the
// cells it passes through if the DIFFERENCES D(i) = F(i) - F(i-1) are
// accumulated and a prefix sum along x follows.
//
//   k_edges   one thread per edge: walks the rows / cells it crosses, adds the
//             differences into the shape's bounding-box buffer.  Sums are kept
//             as 2^-52 fixed point in 64-bit integer atomics: associative, so the
//             result (and with it the sparsity pattern) is identical run to run.
//   k_scan    one warp per buffer row: prefix sum -> coverage in [0, 1], counts
//             the entries above the keep threshold.
//   k_emit    one warp per buffer row: ordered compaction into CSR
//             (column = iy * nx + ix, the order of cutout.grid).
//
// Holes carry the opposite sign; ring orientation is normalised on the host.
// Not bandwidth-critical (O(edges + bounding-box cells)); float64 arithmetic.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "indicator.cuh"
#include "orient.cuh"

namespace atl {

constexpr double kFix = 4503599627370496.0;  // 2^52: one ulp of a coverage fraction; sums wrap
                                              // harmlessly (mod 2^64) as long as the final coverage is < 2048
// kKeep (indicator.cuh): coverage fractions at or below it are dropped

struct EdgeDev {
  double u0, v0, u1, v1;  // grid units relative to the cutout's lower-left cell corner
  int32_t shape;          // index into the batch's box arrays
  int32_t sign;           // +1 / -1: ring weight x orientation normalisation
};

struct BoxDev {
  int32_t i0, j0, w, h;  // bounding box in cells (clipped to the grid)
  int64_t off;           // offset of the box buffer (w*h entries)
  int64_t row0;          // index of its first row in the batch's row list
};

// Mean of c(t) = clamp(1 - t, 0, 1) over [t0, t1] (t = u - i, the cell-local
// coordinate).  Built from the lengths of the pieces t <= 0 (c = 1) and
// 0 < t < 1 (c linear) rather than from an antiderivative difference, so nearly
// vertical edges (t1 - t0 -> 0) lose no precision.
__device__ __forceinline__ double cell_mean(double t0, double t1) {
  const double span = t1 - t0;
  if (!(span > 0.0)) return fmin(fmax(1.0 - t0, 0.0), 1.0);
  const double la = fmax(fmin(t1, 0.0) - t0, 0.0);
  const double a = fmax(t0, 0.0), b = fmin(t1, 1.0);
  const double lb = fmax(b - a, 0.0);
  return (la + lb * (1.0 - 0.5 * (a + b))) / span;
}

__global__ void k_edges(const EdgeDev* __restrict__ edges, int64_t n_edges,
                        const BoxDev* __restrict__ boxes, unsigned long long* __restrict__ buf) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  const EdgeDev ed = edges[e];
  if (ed.v0 == ed.v1) return;  // horizontal: no contribution
  const BoxDev bx = boxes[ed.shape];
  const bool up = ed.v1 > ed.v0;
  const double sgn = (up ? -1.0 : 1.0) * (double)ed.sign;
  const double va = up ? ed.v0 : ed.v1, vb = up ? ed.v1 : ed.v0;
  const double ua = up ? ed.u0 : ed.u1, ub = up ? ed.u1 : ed.u0;
  const double m = (ub - ua) / (vb - va);  // du/dv
  int jlo = (int)floor(va), jhi = (int)ceil(vb) - 1;
  jlo = max(jlo, bx.j0);
  jhi = min(jhi, bx.j0 + bx.h - 1);
  for (int j = jlo; j <= jhi; ++j) {
    const double vlo = fmax(va, (double)j), vhi = fmin(vb, (double)j + 1.0);
    const double h = vhi - vlo;
    if (!(h > 0.0)) continue;
    // end points of the piece inside this row band (exact at the edge's own ends)
    const double p = (vlo == va) ? ua : ua + m * (vlo - va);
    const double q = (vhi == vb) ? ub : ua + m * (vhi - va);
    const double umin = fmin(p, q) - bx.i0, umax = fmax(p, q) - bx.i0;
    unsigned long long* row = buf + bx.off + (int64_t)(j - bx.j0) * bx.w;
    if (umax <= 0.0) {  // entirely left of the box: full height for every cell
      atomicAdd(row, (unsigned long long)llrint(sgn * h * kFix));
      continue;
    }
    if (umin >= (double)bx.w) continue;  // entirely right of it
    const int ia = max((int)floor(umin), 0);
    const int ib = min((int)floor(umax), bx.w - 1);
    double prev = 0.0;
    for (int i = ia; i <= ib + 1 && i < bx.w; ++i) {
      const double F = (i > ib) ? h : h * cell_mean(umin - i, umax - i);
      const double d = F - prev;
      prev = F;
      if (d != 0.0) atomicAdd(row + i, (unsigned long long)llrint(sgn * d * kFix));
    }
  }
}

// rows[r] = {box index}; one warp per row.  In place: fixed-point differences ->
// coverage as double bits.  row_count[r] = entries kept.
__global__ void k_scan(const int32_t* __restrict__ row_box, int64_t n_rows,
                       const BoxDev* __restrict__ boxes, unsigned long long* __restrict__ buf,
                       int32_t* __restrict__ row_count) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= n_rows) return;
  const BoxDev bx = boxes[row_box[r]];
  unsigned long long* row = buf + bx.off + (r - bx.row0) * bx.w;
  long long carry = 0;
  int cnt = 0;
  for (int base = 0; base < bx.w; base += 32) {
    const int i = base + lane;
    long long x = i < bx.w ? (long long)row[i] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    x += carry;
    carry = __shfl_sync(0xffffffffu, x, 31);
    if (i < bx.w) {
      double c = (double)x * (1.0 / kFix);
      c = fmin(fmax(c, 0.0), 1.0);
      if (!(c > kKeep)) c = 0.0;
      row[i] = (unsigned long long)__double_as_longlong(c);
      cnt += c > 0.0;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if (lane == 0) row_count[r] = cnt;
}

__global__ void k_emit(const int32_t* __restrict__ row_box, int64_t n_rows,
                       const BoxDev* __restrict__ boxes, const unsigned long long* __restrict__ buf,
                       const int64_t* __restrict__ row_out, int nx, int32_t* __restrict__ indices,
                       double* __restrict__ data) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= n_rows) return;
  const BoxDev bx = boxes[row_box[r]];
  const int j = (int)(r - bx.row0);
  const unsigned long long* row = buf + bx.off + (int64_t)j * bx.w;
  int64_t out = row_out[r];
  for (int base = 0; base < bx.w; base += 32) {
    const int i = base + lane;
    const double c = i < bx.w ? __longlong_as_double((long long)row[i]) : 0.0;
    const unsigned keep = __ballot_sync(0xffffffffu, c > 0.0);
    if (c > 0.0) {
      const int64_t o = out + __popc(keep & ((1u << lane) - 1u));
      indices[o] = (bx.j0 + j) * nx + bx.i0 + i;
      data[o] = c;
    }
    out += __popc(keep);
  }
}

// ------------------------------------------------------------------ intersection matrix
// Cutout.intersectionmatrix -> gis.py:148-183: entry [i, j] = 1 when shape i and the
// CLOSED box of cell j intersect (shapely `intersects`).  The boxes are the
// reference's own float64 boxes (cutout.py:369-372), given as per-column and per-row
// edge tables; on non-dyadic grids they leave gaps and overlaps of an ulp, and the
// decision is taken against them exactly:
//   k_touch        one thread per ring edge, line segment or point: exact closed
//                  segment-vs-box test on the candidate cells around it, hits marked
//                  in a byte mask over the shape's bounding box (idempotent stores).
//   k_edges        (above, unchanged) coverage of the polygon parts on the uniform grid.
//   k_touch_scan   one warp per row: keep = touched || coverage > 1/2 (a cell no ring
//                  edge touches is wholly inside or wholly outside, and the uniform
//                  cell differs from the reference box by < 1/8 cell per side, so the
//                  coverage is > 0.56 or < 0.44), counts the kept cells.
//   k_touch_emit   ordered compaction into CSR, data = 1.

struct SegDev {
  double ax, ay, bx, by;  // end points in the caller's coordinates; a == b is a point
  int32_t shape;          // index into the batch's box arrays
  int32_t pad;
};

struct CellEdges {
  const double *xlo, *xhi;  // [nx] reference box edges per column
  const double *ylo, *yhi;  // [ny] per row
};

// two_sum / orient2d_exact / orient2d_sign: orient.cuh

// Closed segment [a, b] vs closed box: separating-axis test.  The box axes are the
// bounding-box comparisons (exact); the segment's normal separates iff all four
// corners lie strictly on one side of its line.  A point (a == b) and an axis-parallel
// segment are decided by the bounding boxes alone.
__device__ __forceinline__ bool seg_box(double ax, double ay, double bx, double by, double xlo, double xhi,
                                        double ylo, double yhi) {
  if (fmax(ax, bx) < xlo || fmin(ax, bx) > xhi || fmax(ay, by) < ylo || fmin(ay, by) > yhi) return false;
  if (ax == bx || ay == by) return true;
  const int s0 = orient2d_sign(ax, ay, bx, by, xlo, ylo);
  const int s1 = orient2d_sign(ax, ay, bx, by, xhi, ylo);
  const int s2 = orient2d_sign(ax, ay, bx, by, xhi, yhi);
  const int s3 = orient2d_sign(ax, ay, bx, by, xlo, yhi);
  return !((s0 > 0 && s1 > 0 && s2 > 0 && s3 > 0) || (s0 < 0 && s1 < 0 && s2 < 0 && s3 < 0));
}

__device__ __forceinline__ int floor_clamped(double v) {  // floor, kept inside int range
  return (int)floor(fmin(fmax(v, -1e9), 1e9));
}

// One thread per primitive.  Candidates: the uniform-grid rows the segment spans,
// widened by one on each side, and in row j the columns under the part of the segment
// with j - 1 <= v <= j + 2, widened by one.  The reference box of cell (j, i) lies
// within 1/8 cell of [i, i+1] x [j, j+1], so this holds every cell it can touch; the
// candidate arithmetic only has to be a superset, the exact test decides.
__global__ void k_touch(const SegDev* __restrict__ segs, int64_t n_segs, const BoxDev* __restrict__ boxes,
                        CellEdges ce, double uo, double dx, double vo, double dy, uint8_t* __restrict__ mask) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_segs) return;
  const SegDev s = segs[e];
  const BoxDev bx = boxes[s.shape];
  if (bx.w == 0) return;
  const double ua = (s.ax - uo) / dx, va = (s.ay - vo) / dy;
  const double ub = (s.bx - uo) / dx, vb = (s.by - vo) / dy;
  const int jlo = max(floor_clamped(fmin(va, vb)) - 1, bx.j0);
  const int jhi = min(floor_clamped(fmax(va, vb)) + 1, bx.j0 + bx.h - 1);
  const double dv = vb - va;
  for (int j = jlo; j <= jhi; ++j) {
    double umin = fmin(ua, ub), umax = fmax(ua, ub);
    if (dv != 0.0) {  // the part of the segment inside the widened row band
      const double t0 = fmin(fmax(((double)j - 1.0 - va) / dv, 0.0), 1.0);
      const double t1 = fmin(fmax(((double)j + 2.0 - va) / dv, 0.0), 1.0);
      const double p = ua + t0 * (ub - ua), q = ua + t1 * (ub - ua);
      umin = fmin(p, q);
      umax = fmax(p, q);
    }
    const int ilo = max(floor_clamped(umin) - 1, bx.i0);
    const int ihi = min(floor_clamped(umax) + 1, bx.i0 + bx.w - 1);
    const double ylo = ce.ylo[j], yhi = ce.yhi[j];
    uint8_t* row = mask + bx.off + (int64_t)(j - bx.j0) * bx.w;
    for (int i = ilo; i <= ihi; ++i)
      if (seg_box(s.ax, s.ay, s.bx, s.by, ce.xlo[i], ce.xhi[i], ylo, yhi)) row[i - bx.i0] = 1;
  }
}

// One warp per box row: prefix sum of the coverage differences (as k_scan), then
// mask[i] = touched || coverage > 1/2 in place; row_count[r] = cells kept.
__global__ void k_touch_scan(const int32_t* __restrict__ row_box, int64_t n_rows, const BoxDev* __restrict__ boxes,
                             const unsigned long long* __restrict__ buf, uint8_t* __restrict__ mask,
                             int32_t* __restrict__ row_count) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= n_rows) return;
  const BoxDev bx = boxes[row_box[r]];
  const unsigned long long* row = buf + bx.off + (r - bx.row0) * bx.w;
  uint8_t* mrow = mask + bx.off + (r - bx.row0) * bx.w;
  long long carry = 0;
  int cnt = 0;
  for (int base = 0; base < bx.w; base += 32) {
    const int i = base + lane;
    long long x = i < bx.w ? (long long)row[i] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    x += carry;
    carry = __shfl_sync(0xffffffffu, x, 31);
    if (i < bx.w) {
      const bool keep = mrow[i] != 0 || (double)x * (1.0 / kFix) > 0.5;
      mrow[i] = keep;
      cnt += keep;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if (lane == 0) row_count[r] = cnt;
}

__global__ void k_touch_emit(const int32_t* __restrict__ row_box, int64_t n_rows, const BoxDev* __restrict__ boxes,
                             const uint8_t* __restrict__ mask, const int64_t* __restrict__ row_out, int nx,
                             int32_t* __restrict__ indices, double* __restrict__ data) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= n_rows) return;
  const BoxDev bx = boxes[row_box[r]];
  const int j = (int)(r - bx.row0);
  const uint8_t* mrow = mask + bx.off + (int64_t)j * bx.w;
  int64_t out = row_out[r];
  for (int base = 0; base < bx.w; base += 32) {
    const int i = base + lane;
    const bool hit = i < bx.w && mrow[i] != 0;
    const unsigned keep = __ballot_sync(0xffffffffu, hit);
    if (hit) {
      const int64_t o = out + __popc(keep & ((1u << lane) - 1u));
      indices[o] = (bx.j0 + j) * nx + bx.i0 + i;
      data[o] = 1.0;
    }
    out += __popc(keep);
  }
}

}  // namespace atl

using namespace atl;

namespace {

struct HostBox {
  int32_t i0 = 0, j0 = 0, w = 0, h = 0;
};

template <class T>
struct DevBuf {
  T* p = nullptr;
  ~DevBuf() { cudaFree(p); }
  cudaError_t alloc(size_t n) { return cudaMalloc((void**)&p, std::max<size_t>(n, 1) * sizeof(T)); }
};

// One batch of shapes [s_beg, s_end): all of their box buffers fit the scratch budget.
int run_batch(AtlIndicator* R, int s_beg, int s_end, const std::vector<HostBox>& hb,
              const std::vector<EdgeDev>& all_edges, const std::vector<int64_t>& shape_edge_ptr) {
  const int nb = s_end - s_beg;
  std::vector<BoxDev> boxes(nb);
  std::vector<int32_t> row_box;
  int64_t off = 0;
  for (int k = 0; k < nb; ++k) {
    const HostBox& b = hb[s_beg + k];
    boxes[k] = BoxDev{b.i0, b.j0, b.w, b.h, off, (int64_t)row_box.size()};
    off += (int64_t)b.w * b.h;
    row_box.insert(row_box.end(), b.h, k);
  }
  const int64_t n_rows = (int64_t)row_box.size();
  const int64_t e_beg = shape_edge_ptr[s_beg], e_end = shape_edge_ptr[s_end];
  std::vector<int64_t> counts_cum(n_rows + 1, 0);
  if (n_rows > 0 && off > 0) {
    std::vector<EdgeDev> edges(all_edges.begin() + e_beg, all_edges.begin() + e_end);
    for (auto& e : edges) e.shape -= s_beg;
    DevBuf<EdgeDev> d_edges;
    DevBuf<BoxDev> d_boxes;
    DevBuf<int32_t> d_row_box, d_row_count, d_indices;
    DevBuf<unsigned long long> d_buf;
    DevBuf<int64_t> d_row_out;
    DevBuf<double> d_data;
    ATL_CUDA(d_edges.alloc(edges.size()));
    ATL_CUDA(d_boxes.alloc(nb));
    ATL_CUDA(d_row_box.alloc(n_rows));
    ATL_CUDA(d_row_count.alloc(n_rows));
    ATL_CUDA(d_row_out.alloc(n_rows));
    ATL_CUDA(d_buf.alloc(off));
    ATL_CUDA(cudaMemcpy(d_edges.p, edges.data(), edges.size() * sizeof(EdgeDev), cudaMemcpyHostToDevice));
    ATL_CUDA(cudaMemcpy(d_boxes.p, boxes.data(), nb * sizeof(BoxDev), cudaMemcpyHostToDevice));
    ATL_CUDA(cudaMemcpy(d_row_box.p, row_box.data(), n_rows * 4, cudaMemcpyHostToDevice));
    ATL_CUDA(cudaMemset(d_buf.p, 0, off * 8));
    const int T = 128;
    if (!edges.empty()) {
      k_edges<<<(unsigned)((edges.size() + T - 1) / T), T>>>(d_edges.p, (int64_t)edges.size(), d_boxes.p, d_buf.p);
      ++g_launches;
    }
    const unsigned row_blocks = (unsigned)((n_rows * 32 + T - 1) / T);
    k_scan<<<row_blocks, T>>>(d_row_box.p, n_rows, d_boxes.p, d_buf.p, d_row_count.p);
    ++g_launches;
    ATL_CUDA(cudaGetLastError());
    std::vector<int32_t> counts(n_rows);
    ATL_CUDA(cudaMemcpy(counts.data(), d_row_count.p, n_rows * 4, cudaMemcpyDeviceToHost));
    for (int64_t r = 0; r < n_rows; ++r) counts_cum[r + 1] = counts_cum[r] + counts[r];
    const int64_t nnz = counts_cum[n_rows];
    if (nnz > 0) {
      ATL_CUDA(d_indices.alloc(nnz));
      ATL_CUDA(d_data.alloc(nnz));
      ATL_CUDA(cudaMemcpy(d_row_out.p, counts_cum.data(), n_rows * 8, cudaMemcpyHostToDevice));
      k_emit<<<row_blocks, T>>>(d_row_box.p, n_rows, d_boxes.p, d_buf.p, d_row_out.p, R->nx, d_indices.p,
                                d_data.p);
      ++g_launches;
      ATL_CUDA(cudaGetLastError());
      const size_t base = R->indices.size();
      R->indices.resize(base + nnz);
      R->data.resize(base + nnz);
      ATL_CUDA(cudaMemcpy(R->indices.data() + base, d_indices.p, nnz * 4, cudaMemcpyDeviceToHost));
      ATL_CUDA(cudaMemcpy(R->data.data() + base, d_data.p, nnz * 8, cudaMemcpyDeviceToHost));
    }
  }
  // CSR row pointers of the batch's shapes
  for (int k = 0; k < nb; ++k) {
    const int64_t r0 = boxes[k].row0, r1 = r0 + boxes[k].h;
    R->indptr[s_beg + k + 1] = R->indptr[s_beg + k] + (counts_cum[r1] - counts_cum[r0]);
  }
  return ATL_OK;
}

// Box cells per scratch batch, the budget atl_indicator_compute uses (9 bytes per cell
// here; ATL_INDICATOR_BUDGET forces small batches in the tests).
int64_t batch_budget() {
  int64_t budget = 64LL << 20;
  if (const char* b = getenv("ATL_INDICATOR_BUDGET")) budget = std::max<int64_t>(atoll(b), 1);
  return budget;
}

struct TouchGrid {
  CellEdges ce;  // device pointers
  double uo, dx, vo, dy;
};

// Intersection matrix, one batch of shapes [s_beg, s_end): touch mask and coverage of
// every box, then keep = touched || coverage > 1/2, compacted into R.
int run_touch_batch(AtlIndicator* R, int s_beg, int s_end, const std::vector<HostBox>& hb,
                    const std::vector<EdgeDev>& all_edges, const std::vector<int64_t>& shape_edge_ptr,
                    const std::vector<SegDev>& all_segs, const std::vector<int64_t>& shape_seg_ptr,
                    const TouchGrid& g) {
  const int nb = s_end - s_beg;
  std::vector<BoxDev> boxes(nb);
  std::vector<int32_t> row_box;
  int64_t off = 0;
  for (int k = 0; k < nb; ++k) {
    const HostBox& b = hb[s_beg + k];
    boxes[k] = BoxDev{b.i0, b.j0, b.w, b.h, off, (int64_t)row_box.size()};
    off += (int64_t)b.w * b.h;
    row_box.insert(row_box.end(), b.h, k);
  }
  const int64_t n_rows = (int64_t)row_box.size();
  std::vector<int64_t> counts_cum(n_rows + 1, 0);
  if (n_rows > 0 && off > 0) {
    std::vector<EdgeDev> edges(all_edges.begin() + shape_edge_ptr[s_beg], all_edges.begin() + shape_edge_ptr[s_end]);
    for (auto& e : edges) e.shape -= s_beg;
    std::vector<SegDev> segs(all_segs.begin() + shape_seg_ptr[s_beg], all_segs.begin() + shape_seg_ptr[s_end]);
    for (auto& s : segs) s.shape -= s_beg;
    DevBuf<EdgeDev> d_edges;
    DevBuf<SegDev> d_segs;
    DevBuf<BoxDev> d_boxes;
    DevBuf<int32_t> d_row_box, d_row_count, d_indices;
    DevBuf<unsigned long long> d_buf;
    DevBuf<uint8_t> d_mask;
    DevBuf<int64_t> d_row_out;
    DevBuf<double> d_data;
    ATL_CUDA(d_edges.alloc(edges.size()));
    ATL_CUDA(d_segs.alloc(segs.size()));
    ATL_CUDA(d_boxes.alloc(nb));
    ATL_CUDA(d_row_box.alloc(n_rows));
    ATL_CUDA(d_row_count.alloc(n_rows));
    ATL_CUDA(d_row_out.alloc(n_rows));
    ATL_CUDA(d_buf.alloc(off));
    ATL_CUDA(d_mask.alloc(off));
    ATL_CUDA(cudaMemcpy(d_edges.p, edges.data(), edges.size() * sizeof(EdgeDev), cudaMemcpyHostToDevice));
    ATL_CUDA(cudaMemcpy(d_segs.p, segs.data(), segs.size() * sizeof(SegDev), cudaMemcpyHostToDevice));
    ATL_CUDA(cudaMemcpy(d_boxes.p, boxes.data(), nb * sizeof(BoxDev), cudaMemcpyHostToDevice));
    ATL_CUDA(cudaMemcpy(d_row_box.p, row_box.data(), n_rows * 4, cudaMemcpyHostToDevice));
    ATL_CUDA(cudaMemset(d_buf.p, 0, off * 8));
    ATL_CUDA(cudaMemset(d_mask.p, 0, off));
    const int T = 128;
    if (!segs.empty()) {
      k_touch<<<(unsigned)((segs.size() + T - 1) / T), T>>>(d_segs.p, (int64_t)segs.size(), d_boxes.p, g.ce, g.uo,
                                                            g.dx, g.vo, g.dy, d_mask.p);
      ++g_launches;
    }
    if (!edges.empty()) {
      k_edges<<<(unsigned)((edges.size() + T - 1) / T), T>>>(d_edges.p, (int64_t)edges.size(), d_boxes.p, d_buf.p);
      ++g_launches;
    }
    const unsigned row_blocks = (unsigned)((n_rows * 32 + T - 1) / T);
    k_touch_scan<<<row_blocks, T>>>(d_row_box.p, n_rows, d_boxes.p, d_buf.p, d_mask.p, d_row_count.p);
    ++g_launches;
    ATL_CUDA(cudaGetLastError());
    std::vector<int32_t> counts(n_rows);
    ATL_CUDA(cudaMemcpy(counts.data(), d_row_count.p, n_rows * 4, cudaMemcpyDeviceToHost));
    for (int64_t r = 0; r < n_rows; ++r) counts_cum[r + 1] = counts_cum[r] + counts[r];
    const int64_t nnz = counts_cum[n_rows];
    if (nnz > 0) {
      ATL_CUDA(d_indices.alloc(nnz));
      ATL_CUDA(d_data.alloc(nnz));
      ATL_CUDA(cudaMemcpy(d_row_out.p, counts_cum.data(), n_rows * 8, cudaMemcpyHostToDevice));
      k_touch_emit<<<row_blocks, T>>>(d_row_box.p, n_rows, d_boxes.p, d_mask.p, d_row_out.p, R->nx, d_indices.p,
                                      d_data.p);
      ++g_launches;
      ATL_CUDA(cudaGetLastError());
      const size_t base = R->indices.size();
      R->indices.resize(base + nnz);
      R->data.resize(base + nnz);
      ATL_CUDA(cudaMemcpy(R->indices.data() + base, d_indices.p, nnz * 4, cudaMemcpyDeviceToHost));
      ATL_CUDA(cudaMemcpy(R->data.data() + base, d_data.p, nnz * 8, cudaMemcpyDeviceToHost));
    }
  }
  for (int k = 0; k < nb; ++k) {
    const int64_t r0 = boxes[k].row0, r1 = r0 + boxes[k].h;
    R->indptr[s_beg + k + 1] = R->indptr[s_beg + k] + (counts_cum[r1] - counts_cum[r0]);
  }
  return ATL_OK;
}

// The reference box edges must be ordered and lie within 1/8 cell of the uniform
// grid's cell borders (lo[k] ~ c0 + (k - 1/2) d): then a cell's reference box and
// its uniform cell overlap by more than (3/4)^2 > 1/2 of a cell, which is what makes
// the coverage > 1/2 rule exact for untouched cells.
bool edges_near_uniform(const double* lo, const double* hi, int32_t n, double c0, double d) {
  for (int32_t k = 0; k < n; ++k) {
    if (!(std::isfinite(lo[k]) && std::isfinite(hi[k]) && lo[k] <= hi[k])) return false;
    if (k > 0 && !(lo[k] >= lo[k - 1] && hi[k] >= hi[k - 1])) return false;
    const double ulo = c0 + ((double)k - 0.5) * d, uhi = c0 + ((double)k + 0.5) * d;
    if (!(std::fabs(lo[k] - ulo) < 0.125 * d && std::fabs(hi[k] - uhi) < 0.125 * d)) return false;
  }
  return true;
}

}  // namespace

extern "C" {

int atl_indicator_compute(int device, int32_t ny, int32_t nx, double x0, double dx, double y0,
                          double dy, int32_t n_shapes, const int64_t* shape_ring_ptr,
                          const int64_t* ring_ptr, const int8_t* ring_is_hole, const double* xy,
                          AtlIndicator** out) {
  ATL_REQUIRE(out, "NULL argument");
  *out = nullptr;
  ATL_REQUIRE(ny > 0 && nx > 0 && (int64_t)ny * nx < (1LL << 31), "bad grid");
  ATL_REQUIRE(dx > 0 && dy > 0, "cell sizes must be positive (coordinates ascending)");
  ATL_REQUIRE(n_shapes >= 0 && shape_ring_ptr && (n_shapes == 0 || (ring_ptr && ring_is_hole && xy)),
              "NULL argument");
  ATL_CUDA(cudaSetDevice(device));
  const double uo = x0 - 0.5 * dx, vo = y0 - 0.5 * dy;  // lower-left corner of cell (0, 0)

  std::vector<EdgeDev> edges;
  std::vector<int64_t> shape_edge_ptr(n_shapes + 1, 0);
  std::vector<HostBox> hb(n_shapes);
  for (int s = 0; s < n_shapes; ++s) {
    double ulo = INFINITY, uhi = -INFINITY, vlo = INFINITY, vhi = -INFINITY;
    ATL_REQUIRE(shape_ring_ptr[s + 1] >= shape_ring_ptr[s], "shape_ring_ptr must be non-decreasing");
    for (int64_t r = shape_ring_ptr[s]; r < shape_ring_ptr[s + 1]; ++r) {
      const int64_t a = ring_ptr[r], b = ring_ptr[r + 1];
      ATL_REQUIRE(b >= a, "ring_ptr must be non-decreasing");
      if (b - a < 3) continue;  // degenerate ring: no area
      // orientation from the shoelace sum in grid units (about the first vertex)
      double area2 = 0.0;
      const double ux0 = (xy[2 * a] - uo) / dx, vy0 = (xy[2 * a + 1] - vo) / dy;
      for (int64_t k = a; k < b; ++k) {
        const int64_t k1 = (k + 1 < b) ? k + 1 : a;
        const double u0 = (xy[2 * k] - uo) / dx - ux0, v0 = (xy[2 * k + 1] - vo) / dy - vy0;
        const double u1 = (xy[2 * k1] - uo) / dx - ux0, v1 = (xy[2 * k1 + 1] - vo) / dy - vy0;
        ATL_REQUIRE(std::isfinite(u0) && std::isfinite(v0), "non-finite vertex");
        area2 += u0 * v1 - u1 * v0;
      }
      if (area2 == 0.0) continue;
      const int32_t sign = (ring_is_hole[r] ? -1 : 1) * (area2 > 0.0 ? 1 : -1);
      for (int64_t k = a; k < b; ++k) {
        const int64_t k1 = (k + 1 < b) ? k + 1 : a;
        EdgeDev e;
        e.u0 = (xy[2 * k] - uo) / dx;
        e.v0 = (xy[2 * k + 1] - vo) / dy;
        e.u1 = (xy[2 * k1] - uo) / dx;
        e.v1 = (xy[2 * k1 + 1] - vo) / dy;
        e.shape = s;
        e.sign = sign;
        if (!ring_is_hole[r]) {
          ulo = std::min(ulo, e.u0);
          uhi = std::max(uhi, e.u0);
          vlo = std::min(vlo, e.v0);
          vhi = std::max(vhi, e.v0);
        }
        if (e.v0 != e.v1 || e.u0 != e.u1) edges.push_back(e);
      }
    }
    shape_edge_ptr[s + 1] = (int64_t)edges.size();
    HostBox& b = hb[s];
    if (uhi > ulo && vhi > vlo) {
      const double i0 = std::max(std::floor(ulo), 0.0), i1 = std::min(std::ceil(uhi), (double)nx);
      const double j0 = std::max(std::floor(vlo), 0.0), j1 = std::min(std::ceil(vhi), (double)ny);
      if (i1 > i0 && j1 > j0) {
        b.i0 = (int32_t)i0;
        b.j0 = (int32_t)j0;
        b.w = (int32_t)(i1 - i0);
        b.h = (int32_t)(j1 - j0);
      }
    }
  }

  AtlIndicator* R = new AtlIndicator();
  R->n_shapes = n_shapes;
  R->ny = ny;
  R->nx = nx;
  R->indptr.assign((size_t)n_shapes + 1, 0);
  int64_t budget = 64LL << 20;  // box cells per batch (512 MiB of scratch)
  if (const char* b = getenv("ATL_INDICATOR_BUDGET")) budget = std::max<int64_t>(atoll(b), 1);  // tests
  int rc = ATL_OK;
  for (int s = 0; s < n_shapes && rc == ATL_OK;) {
    int e = s;
    int64_t cells = 0;
    while (e < n_shapes && (e == s || cells + (int64_t)hb[e].w * hb[e].h <= budget)) {
      cells += (int64_t)hb[e].w * hb[e].h;
      ++e;
    }
    rc = run_batch(R, s, e, hb, edges, shape_edge_ptr);
    s = e;
  }
  if (rc == ATL_OK) {
    cudaError_t ce = cudaDeviceSynchronize();
    if (ce != cudaSuccess) rc = cuda_fail(ce, "atl_indicator_compute");
  }
  if (rc != ATL_OK) {
    delete R;
    return rc;
  }
  *out = R;
  return ATL_OK;
}

int atl_intersection_compute(int device, int32_t ny, int32_t nx, double x0, double dx, double y0, double dy,
                             const double* cell_x_lo, const double* cell_x_hi, const double* cell_y_lo,
                             const double* cell_y_hi, int32_t n_shapes, const int64_t* shape_part_ptr,
                             const int64_t* part_ptr, const int8_t* part_kind, const double* xy,
                             AtlIndicator** out) {
  ATL_REQUIRE(out, "NULL argument");
  *out = nullptr;
  ATL_REQUIRE(ny > 0 && nx > 0 && (int64_t)ny * nx < (1LL << 31), "bad grid");
  ATL_REQUIRE(dx > 0 && dy > 0, "cell sizes must be positive (coordinates ascending)");
  ATL_REQUIRE(cell_x_lo && cell_x_hi && cell_y_lo && cell_y_hi, "NULL argument");
  ATL_REQUIRE(n_shapes >= 0 && shape_part_ptr && (n_shapes == 0 || (part_ptr && part_kind && xy)),
              "NULL argument");
  ATL_REQUIRE(edges_near_uniform(cell_x_lo, cell_x_hi, nx, x0, dx) &&
                  edges_near_uniform(cell_y_lo, cell_y_hi, ny, y0, dy),
              "cell edge tables must be finite, ordered and within 1/8 cell of the regular grid");
  ATL_CUDA(cudaSetDevice(device));
  const double uo = x0 - 0.5 * dx, vo = y0 - 0.5 * dy;  // lower-left corner of uniform cell (0, 0)

  std::vector<EdgeDev> edges;
  std::vector<SegDev> segs;
  std::vector<int64_t> shape_edge_ptr(n_shapes + 1, 0), shape_seg_ptr(n_shapes + 1, 0);
  std::vector<HostBox> hb(n_shapes);
  for (int s = 0; s < n_shapes; ++s) {
    double ulo = INFINITY, uhi = -INFINITY, vlo = INFINITY, vhi = -INFINITY;
    ATL_REQUIRE(shape_part_ptr[s + 1] >= shape_part_ptr[s], "shape_part_ptr must be non-decreasing");
    for (int64_t p = shape_part_ptr[s]; p < shape_part_ptr[s + 1]; ++p) {
      const int64_t a = part_ptr[p], b = part_ptr[p + 1];
      const int kind = part_kind[p];
      ATL_REQUIRE(b >= a, "part_ptr must be non-decreasing");
      ATL_REQUIRE(kind >= ATL_PART_EXTERIOR && kind <= ATL_PART_POINTS, "unknown part kind");
      for (int64_t k = a; k < b; ++k) {
        ATL_REQUIRE(std::isfinite(xy[2 * k]) && std::isfinite(xy[2 * k + 1]), "non-finite vertex");
        const double u = (xy[2 * k] - uo) / dx, v = (xy[2 * k + 1] - vo) / dy;
        ulo = std::min(ulo, u);
        uhi = std::max(uhi, u);
        vlo = std::min(vlo, v);
        vhi = std::max(vhi, v);
      }
      auto seg = [&](int64_t k0, int64_t k1) {
        segs.push_back(SegDev{xy[2 * k0], xy[2 * k0 + 1], xy[2 * k1], xy[2 * k1 + 1], s, 0});
      };
      if (kind == ATL_PART_POINTS) {
        for (int64_t k = a; k < b; ++k) seg(k, k);
      } else if (kind == ATL_PART_LINE) {
        if (b - a == 1) seg(a, a);  // a one-point line is a point
        for (int64_t k = a; k + 1 < b; ++k) seg(k, k + 1);
      } else {
        // ring: every edge (the closing one included) touches; the area edges go to
        // k_edges exactly as atl_indicator_compute builds them
        for (int64_t k = a; k < b; ++k) seg(k, k + 1 < b ? k + 1 : a);
        if (b - a < 3) continue;
        double area2 = 0.0;
        const double ux0 = (xy[2 * a] - uo) / dx, vy0 = (xy[2 * a + 1] - vo) / dy;
        for (int64_t k = a; k < b; ++k) {
          const int64_t k1 = (k + 1 < b) ? k + 1 : a;
          const double u0 = (xy[2 * k] - uo) / dx - ux0, v0 = (xy[2 * k + 1] - vo) / dy - vy0;
          const double u1 = (xy[2 * k1] - uo) / dx - ux0, v1 = (xy[2 * k1 + 1] - vo) / dy - vy0;
          area2 += u0 * v1 - u1 * v0;
        }
        if (area2 == 0.0) continue;
        const bool hole = kind == ATL_PART_HOLE;
        const int32_t sign = (hole ? -1 : 1) * (area2 > 0.0 ? 1 : -1);
        for (int64_t k = a; k < b; ++k) {
          const int64_t k1 = (k + 1 < b) ? k + 1 : a;
          EdgeDev e;
          e.u0 = (xy[2 * k] - uo) / dx;
          e.v0 = (xy[2 * k + 1] - vo) / dy;
          e.u1 = (xy[2 * k1] - uo) / dx;
          e.v1 = (xy[2 * k1 + 1] - vo) / dy;
          e.shape = s;
          e.sign = sign;
          if (e.v0 != e.v1 || e.u0 != e.u1) edges.push_back(e);
        }
      }
    }
    shape_edge_ptr[s + 1] = (int64_t)edges.size();
    shape_seg_ptr[s + 1] = (int64_t)segs.size();
    // bounding box of every part, widened by one cell (an edge on a border touches the
    // next cell; the reference boxes are within 1/8 cell of the uniform ones), clipped
    HostBox& bx = hb[s];
    if (ulo <= uhi && vlo <= vhi) {
      const double i0 = std::max(std::floor(ulo) - 1.0, 0.0), i1 = std::min(std::floor(uhi) + 2.0, (double)nx);
      const double j0 = std::max(std::floor(vlo) - 1.0, 0.0), j1 = std::min(std::floor(vhi) + 2.0, (double)ny);
      if (i1 > i0 && j1 > j0) {
        bx.i0 = (int32_t)i0;
        bx.j0 = (int32_t)j0;
        bx.w = (int32_t)(i1 - i0);
        bx.h = (int32_t)(j1 - j0);
      }
    }
  }

  AtlIndicator* R = new AtlIndicator();
  R->n_shapes = n_shapes;
  R->ny = ny;
  R->nx = nx;
  R->indptr.assign((size_t)n_shapes + 1, 0);
  int rc = ATL_OK;
  {
    DevBuf<double> d_xlo, d_xhi, d_ylo, d_yhi;
    auto upload = [](DevBuf<double>& d, const double* h, int32_t n) -> cudaError_t {
      cudaError_t ce = d.alloc(n);
      return ce != cudaSuccess ? ce : cudaMemcpy(d.p, h, (size_t)n * 8, cudaMemcpyHostToDevice);
    };
    cudaError_t ce = upload(d_xlo, cell_x_lo, nx);
    if (ce == cudaSuccess) ce = upload(d_xhi, cell_x_hi, nx);
    if (ce == cudaSuccess) ce = upload(d_ylo, cell_y_lo, ny);
    if (ce == cudaSuccess) ce = upload(d_yhi, cell_y_hi, ny);
    if (ce != cudaSuccess) rc = cuda_fail(ce, "atl_intersection_compute");
    const TouchGrid g{CellEdges{d_xlo.p, d_xhi.p, d_ylo.p, d_yhi.p}, uo, dx, vo, dy};
    const int64_t budget = batch_budget();
    for (int s = 0; s < n_shapes && rc == ATL_OK;) {
      int e = s;
      int64_t cells = 0;
      while (e < n_shapes && (e == s || cells + (int64_t)hb[e].w * hb[e].h <= budget)) {
        cells += (int64_t)hb[e].w * hb[e].h;
        ++e;
      }
      rc = run_touch_batch(R, s, e, hb, edges, shape_edge_ptr, segs, shape_seg_ptr, g);
      s = e;
    }
    if (rc == ATL_OK) {
      ce = cudaDeviceSynchronize();
      if (ce != cudaSuccess) rc = cuda_fail(ce, "atl_intersection_compute");
    }
  }
  if (rc != ATL_OK) {
    delete R;
    return rc;
  }
  *out = R;
  return ATL_OK;
}

int atl_indicator_nnz(const AtlIndicator* ind, int64_t* nnz_out) {
  ATL_REQUIRE(ind && nnz_out, "NULL argument");
  *nnz_out = (int64_t)ind->indices.size();
  return ATL_OK;
}

int atl_indicator_export(const AtlIndicator* ind, int64_t* indptr_out, int32_t* indices_out,
                         double* data_out) {
  ATL_REQUIRE(ind && indptr_out, "NULL argument");
  ATL_REQUIRE(ind->indices.empty() || (indices_out && data_out), "NULL argument");
  std::memcpy(indptr_out, ind->indptr.data(), ind->indptr.size() * 8);
  if (!ind->indices.empty()) {
    std::memcpy(indices_out, ind->indices.data(), ind->indices.size() * 4);
    std::memcpy(data_out, ind->data.data(), ind->data.size() * 8);
  }
  return ATL_OK;
}

void atl_indicator_destroy(AtlIndicator* ind) { delete ind; }

}  // extern "C"
