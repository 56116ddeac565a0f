// bvh_b200/csrc/exact.cuh -- exact expansion arithmetic and the exact sign of orient2d, shared by the triangle-pair predicate
// (tritri.cuh, DESIGN.md §4.22) and the point-in-polygon walk (segments.cu, §4.23).
//
// A sign is first read from a double-precision evaluation with Shewchuk's static error bound (every operation rounded explicitly: the
// library is built -fmad=false, and the bound assumes no contraction); only when the bound cannot decide it does the exact evaluation
// run: every monomial as a sum of doubles (two_prod through fma, differences through two_sum), accumulated into a nonoverlapping
// expansion whose largest component carries the sign.  The exact evaluation is __noinline__ so the walks' common path keeps its
// registers.  Exactness needs every product and error term to stay clear of underflow and overflow: see the ranges of the callers.
#pragma once
#include "internal.h"

namespace bvhb200 {
#ifdef __CUDACC__

// ---- exact arithmetic (Shewchuk, "Adaptive precision floating-point arithmetic and fast robust geometric predicates", 1997) ----
__device__ __forceinline__ void two_sum(double a, double b, double& s, double& e) {
    s = __dadd_rn(a, b);
    const double bv = __dsub_rn(s, a), av = __dsub_rn(s, bv);
    e = __dadd_rn(__dsub_rn(a, av), __dsub_rn(b, bv));
}
__device__ __forceinline__ void two_prod(double a, double b, double& p, double& e) {
    p = __dmul_rn(a, b);
    e = __fma_rn(a, b, -p);
}
// h[0 .. m) (nonoverlapping, increasing magnitude, no zeros) += b exactly (Grow-Expansion with zero elimination); returns the length.
__device__ __forceinline__ int grow(double* h, int m, double b) {
    double q = b;
    int k = 0;
    for (int i = 0; i < m; ++i) {
        double s, e;
        two_sum(q, h[i], s, e);
        if (e != 0.0) h[k++] = e;
        q = s;
    }
    if (q != 0.0) h[k++] = q;
    return k;
}
__device__ __forceinline__ int grow_prod2(double* h, int m, double x, double y, bool neg) {
    if (x == 0.0 || y == 0.0) return m;
    double p, e;
    two_prod(x, y, p, e);
    if (neg) { p = -p; e = -e; }
    return grow(h, grow(h, m, e), p);
}
__device__ __forceinline__ int expansion_sign(const double* h, int m) { return m == 0 ? 0 : (h[m - 1] > 0.0 ? 1 : -1); }

// Exact sign of orient2d(a, b, c) = (a - c) x (b - c).  inline: defined once across the translation units that include it.
inline __device__ __noinline__ int orient2d_exact(double ax, double ay, double bx, double by, double cx, double cy) {
    double A[2][2], B[2][2];
    two_sum(ax, -cx, A[0][0], A[0][1]); two_sum(ay, -cy, A[1][0], A[1][1]);
    two_sum(bx, -cx, B[0][0], B[0][1]); two_sum(by, -cy, B[1][0], B[1][1]);
    double h[16];
    int m = 0;
    for (int u = 0; u < 4; ++u) {
        m = grow_prod2(h, m, A[0][u & 1], B[1][u >> 1], false);
        m = grow_prod2(h, m, A[1][u & 1], B[0][u >> 1], true);
    }
    return expansion_sign(h, m);
}
// Filtered sign of orient2d(a, b, c) (Shewchuk's orient2d stage A: the same evaluation order and bound): +1 when c lies left of a -> b.
__device__ __forceinline__ int orient2d_sign(double ax, double ay, double bx, double by, double cx, double cy) {
    constexpr double BOUND = (3.0 + 16.0 * 0x1p-53) * 0x1p-53;
    const double l = __dmul_rn(__dsub_rn(ax, cx), __dsub_rn(by, cy));
    const double r = __dmul_rn(__dsub_rn(ay, cy), __dsub_rn(bx, cx));
    const double det = __dsub_rn(l, r), err = __dmul_rn(BOUND, __dadd_rn(fabs(l), fabs(r)));
    if (det > err) return 1;
    if (-det > err) return -1;
    return orient2d_exact(ax, ay, bx, by, cx, cy);
}

#endif  // __CUDACC__
}  // namespace bvhb200
