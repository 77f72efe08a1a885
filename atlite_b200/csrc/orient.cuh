// orient.cuh -- exact sign of the 2-D orientation determinant, shared by the kernels that decide
// point / segment / box relations exactly (indicator.cu, availability.cu).
#pragma once
#include <cuda_runtime.h>

namespace atl {

// Knuth's TwoSum: s + e == a + b exactly.  Explicit round-to-nearest intrinsics keep
// the compiler from contracting or reordering the steps.
static __device__ __forceinline__ void two_sum(double a, double b, double& s, double& e) {
  s = __dadd_rn(a, b);
  const double bv = __dsub_rn(s, a);
  const double av = __dsub_rn(s, bv);
  e = __dadd_rn(__dsub_rn(a, av), __dsub_rn(b, bv));
}

// Exact sign of orient2d(a, b, c) = (a - c) x (b - c), expanded into six products
//   ax*by - ax*cy - cx*by - ay*bx + ay*cx + cy*bx
// each split exactly into p + e by an fma (TwoProduct), and summed exactly by
// Grow-Expansion (Shewchuk 1997).  The result is a non-overlapping expansion in
// increasing magnitude, so its sign is that of its last non-zero component.  Exact
// unless a product underflows (|coordinates| < 1e-150), which map coordinates never do.
static __device__ __noinline__ int orient2d_exact(double ax, double ay, double bx, double by, double cx, double cy) {
  const double pa[6] = {ax, -ax, -cx, -ay, ay, cy};
  const double pb[6] = {by, cy, by, bx, cx, bx};
  double h[12];
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    const double p = __dmul_rn(pa[k], pb[k]);
    const double t[2] = {fma(pa[k], pb[k], -p), p};
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      double q = t[m];
      const int n = 2 * k + m;
#pragma unroll
      for (int i = 0; i < n; ++i) {
        double s, e;
        two_sum(q, h[i], s, e);
        h[i] = e;
        q = s;
      }
      h[n] = q;
    }
  }
  int sgn = 0;
#pragma unroll
  for (int i = 0; i < 12; ++i)
    if (h[i] != 0.0) sgn = h[i] > 0.0 ? 1 : -1;
  return sgn;
}

// Sign of orient2d(a, b, c): Shewchuk's filter with the proven bound
// |err| <= (3 + 16 eps) eps (|detleft| + |detright|), eps = 2^-53, and the exact
// expansion when the filter cannot decide.
static __device__ __forceinline__ int orient2d_sign(double ax, double ay, double bx, double by, double cx, double cy) {
  const double detleft = __dmul_rn(__dsub_rn(ax, cx), __dsub_rn(by, cy));
  const double detright = __dmul_rn(__dsub_rn(ay, cy), __dsub_rn(bx, cx));
  const double det = __dsub_rn(detleft, detright);
  double detsum;
  if (detleft > 0.0) {
    if (detright <= 0.0) return det > 0.0 ? 1 : (det < 0.0 ? -1 : 0);
    detsum = __dadd_rn(detleft, detright);
  } else if (detleft < 0.0) {
    if (detright >= 0.0) return det > 0.0 ? 1 : (det < 0.0 ? -1 : 0);
    detsum = __dsub_rn(-detleft, detright);
  } else {
    return det > 0.0 ? 1 : (det < 0.0 ? -1 : 0);
  }
  constexpr double kEps = 0x1p-53;
  const double errbound = __dmul_rn((3.0 + 16.0 * kEps) * kEps, detsum);
  if (det > errbound) return 1;
  if (-det > errbound) return -1;
  return orient2d_exact(ax, ay, bx, by, cx, cy);
}

}  // namespace atl
