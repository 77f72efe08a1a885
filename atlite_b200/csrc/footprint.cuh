// footprint.cuh -- the average warp's footprint of a destination cell on a source pixel lattice,
// shared by gis.reproject (reproject.cu) and the reprojected availability (availability.cu).
//
// Destination cell (i, j) has the corners T_dst (j, i) and T_dst (j + 1, i + 1).  Both are projected
// into the source CRS and taken to source pixel coordinates (u, v) by the inverse source affine; the
// footprint is the axis-aligned box they span.  Along each axis the box covers the pixels that
// overlap it by more than RP_EPS, clipped to a range of pixels ([0, n) for reproject, [-pad, n + pad)
// for the padded availability window); the first and the last of them carry their overlaps as
// weights, every pixel between them 1.
#pragma once
#include <math.h>

#include "proj.cuh"

namespace atl {

constexpr int RP_THREADS = 256;
constexpr int RP_SMALL = 32;  // pixels of a box its own thread sums
constexpr double RP_EPS = 1e-10;  // gis.REGRID_EPS

// destination lattice point (col jj, row ii) -> source pixel coordinates (u, v); NaN without an image.
// p takes points from dst's CRS into src's.
template <int FROM, int TO>
__device__ __forceinline__ void to_source(const AtlLattice& dst, const AtlLattice& src, const AtlProjection& p,
                                          double jj, double ii, double& u, double& v) {
  double x = lattice_point(dst.c, dst.a, jj), y = lattice_point(dst.f, dst.e, ii);
  project<FROM, TO>(p, x, y);
  u = __ddiv_rn(__dsub_rn(x, src.c), src.a);
  v = __ddiv_rn(__dsub_rn(y, src.f), src.e);
}

// The pixels [lo, hi) of one axis that overlap [t0, t1] by more than RP_EPS, clipped to [lo_clip,
// hi_clip), and the overlaps of the first and the last (1 for every pixel between them).  Empty:
// hi <= lo.
struct Span {
  int lo, hi;
  double w_lo, w_hi;
};
__device__ __forceinline__ Span axis_span(double t0, double t1, int64_t lo_clip, int64_t hi_clip) {
  Span s;
  s.lo = (int)fmin(fmax(floor(t0 + RP_EPS), (double)lo_clip), (double)hi_clip);
  s.hi = (int)fmin(fmax(ceil(t1 - RP_EPS), (double)lo_clip), (double)hi_clip);
  s.w_lo = fmin(s.lo + 1.0, t1) - fmax((double)s.lo, t0);
  s.w_hi = fmin((double)s.hi, t1) - fmax(s.hi - 1.0, t0);
  return s;
}

struct Box {
  Span r, c;
  int64_t cell;  // destination index i * dst.nx + j
};

// The box of the cell whose corners are a = (u, v) of (j, i) and b of (j + 1, i + 1), columns
// clipped to [c_lo, c_hi) and rows to [r_lo, r_hi).  Left untouched (the caller's empty box) when a
// corner has no image.
__device__ __forceinline__ void corner_box(double2 a, double2 b, int64_t c_lo, int64_t c_hi, int64_t r_lo,
                                           int64_t r_hi, Box& bx) {
  if (a.x == a.x && a.y == a.y && b.x == b.x && b.y == b.y) {  // both corners have an image
    bx.c = axis_span(fmin(a.x, b.x), fmax(a.x, b.x), c_lo, c_hi);
    bx.r = axis_span(fmin(a.y, b.y), fmax(a.y, b.y), r_lo, r_hi);
  }
}

}  // namespace atl
