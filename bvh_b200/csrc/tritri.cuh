// bvh_b200/csrc/tritri.cuh -- the exact triangle-triangle predicate of bvhgpu_triangle_pairs_* (include/bvh_b200.h, DESIGN.md §4.22):
// do two closed triangles, their coordinates taken as exact real numbers, have a point in common?
//
// Every decision is the sign of an orientation determinant: orient3d (degree 3) or, for points in a common plane, orient2d of a
// projection (degree 2).  A sign is first read from a double-precision evaluation with Shewchuk's static error bound (every operation
// rounded explicitly: the library is built -fmad=false, and the bound assumes no contraction); only when the bound cannot decide it does
// the exact evaluation run: every monomial of the determinant as a sum of doubles (two_prod through fma, differences through two_sum),
// accumulated into a nonoverlapping expansion whose largest component carries the sign (exact.cuh holds the arithmetic and orient2d).
// The exact evaluations are __noinline__ so the walk's common path keeps its registers.
//
// Exactness: f32 inputs promoted to double are multiples of 2^-149 below 2^128 in magnitude, f64 inputs that are zero or of magnitude
// in [2^-300, 2^300] are multiples of 2^-352 below 2^301.  A degree-3 monomial of coordinate differences is then a multiple of 2^-447
// (f32) or 2^-1056 (f64), both multiples of 2^-1074, and below 2^390 (f32) or 2^906 (f64): no product, error term or sum underflows
// or overflows, so two_prod and two_sum are exact and the filter's rounding errors are relative.  Outside that range (f64 only) a
// triangle is "unchecked": the predicate does not run on it (TriPairsLeaf keeps its pairs).
#pragma once
#include "exact.cuh"

namespace bvhb200 {
#ifdef __CUDACC__

constexpr double TRI_F64_LO = 0x1p-300, TRI_F64_HI = 0x1p+300;     // the f64 range the predicate is exact on (zero as well)

// ---- exact arithmetic: two_sum, two_prod, grow, grow_prod2, orient2d_exact and orient2d_sign are in exact.cuh ----
// h += sign * x * y * z exactly (four doubles); zero factors add nothing.
__device__ __forceinline__ int grow_prod3(double* h, int m, double x, double y, double z, bool neg) {
    if (x == 0.0 || y == 0.0 || z == 0.0) return m;
    double p, e, p1, e1, p2, e2;
    two_prod(x, y, p, e);
    two_prod(p, z, p1, e1);
    two_prod(e, z, p2, e2);
    if (neg) { p1 = -p1; e1 = -e1; p2 = -p2; e2 = -e2; }
    m = grow(h, m, e2); m = grow(h, m, e1); m = grow(h, m, p2);
    return grow(h, m, p1);
}
// Exact sign of orient3d(a, b, c, d) = det[a - d; b - d; c - d]: each difference is hi + lo (two_sum), the determinant the sum of its
// 6 x 8 monomials of three such parts.  By value, so that the caller's points stay in registers.
__device__ __noinline__ int orient3d_exact(double ax, double ay, double az, double bx, double by, double bz, double cx, double cy, double cz,
                                           double dx, double dy, double dz) {
    double A[3][2], B[3][2], C[3][2];
    two_sum(ax, -dx, A[0][0], A[0][1]); two_sum(ay, -dy, A[1][0], A[1][1]); two_sum(az, -dz, A[2][0], A[2][1]);
    two_sum(bx, -dx, B[0][0], B[0][1]); two_sum(by, -dy, B[1][0], B[1][1]); two_sum(bz, -dz, B[2][0], B[2][1]);
    two_sum(cx, -dx, C[0][0], C[0][1]); two_sum(cy, -dy, C[1][0], C[1][1]); two_sum(cz, -dz, C[2][0], C[2][1]);
    double h[192];
    int m = 0;
    // det = A0 (B1 C2 - B2 C1) + A1 (B2 C0 - B0 C2) + A2 (B0 C1 - B1 C0)
    const int P[6][3] = {{0, 1, 2}, {0, 2, 1}, {1, 2, 0}, {1, 0, 2}, {2, 0, 1}, {2, 1, 0}};
    for (int t = 0; t < 6; ++t) {
        const bool neg = (t & 1) != 0;
        for (int u = 0; u < 8; ++u)
            m = grow_prod3(h, m, A[P[t][0]][u & 1], B[P[t][1]][(u >> 1) & 1], C[P[t][2]][u >> 2], neg);
    }
    return expansion_sign(h, m);
}
// ---- filtered signs (Shewchuk's orient3d / orient2d stage A: the same evaluation order and bounds) ----
// A call, not inlined: tri_tri makes up to 24 of them, and inlined they would spill the walk's registers.
__device__ __noinline__ int orient3_sign(double ax, double ay, double az, double bx, double by, double bz, double cx, double cy, double cz,
                                         double dx, double dy, double dz) {
    constexpr double BOUND = (7.0 + 56.0 * 0x1p-53) * 0x1p-53;
    const double adx = __dsub_rn(ax, dx), ady = __dsub_rn(ay, dy), adz = __dsub_rn(az, dz);
    const double bdx = __dsub_rn(bx, dx), bdy = __dsub_rn(by, dy), bdz = __dsub_rn(bz, dz);
    const double cdx = __dsub_rn(cx, dx), cdy = __dsub_rn(cy, dy), cdz = __dsub_rn(cz, dz);
    const double bdxcdy = __dmul_rn(bdx, cdy), cdxbdy = __dmul_rn(cdx, bdy);
    const double cdxady = __dmul_rn(cdx, ady), adxcdy = __dmul_rn(adx, cdy);
    const double adxbdy = __dmul_rn(adx, bdy), bdxady = __dmul_rn(bdx, ady);
    const double det = __dadd_rn(__dadd_rn(__dmul_rn(adz, __dsub_rn(bdxcdy, cdxbdy)), __dmul_rn(bdz, __dsub_rn(cdxady, adxcdy))),
                                 __dmul_rn(cdz, __dsub_rn(adxbdy, bdxady)));
    const double perm = __dadd_rn(__dadd_rn(__dmul_rn(__dadd_rn(fabs(bdxcdy), fabs(cdxbdy)), fabs(adz)),
                                            __dmul_rn(__dadd_rn(fabs(cdxady), fabs(adxcdy)), fabs(bdz))),
                                  __dmul_rn(__dadd_rn(fabs(adxbdy), fabs(bdxady)), fabs(cdz)));
    const double err = __dmul_rn(BOUND, perm);
    if (det > err) return 1;
    if (-det > err) return -1;
    return orient3d_exact(ax, ay, az, bx, by, bz, cx, cy, cz, dx, dy, dz);
}
__device__ __forceinline__ int orient3(const double a[3], const double b[3], const double c[3], const double d[3]) {
    return orient3_sign(a[0], a[1], a[2], b[0], b[1], b[2], c[0], c[1], c[2], d[0], d[1], d[2]);
}
// Component i of a point by selects, so that a run-time axis does not move the point to local memory.
__device__ __forceinline__ double comp(const double a[3], int i) { return i == 0 ? a[0] : i == 1 ? a[1] : a[2]; }
// orient2d of the projection of a, b, c onto axes (i, j).
__device__ __forceinline__ int orient2(const double a[3], const double b[3], const double c[3], int i, int j) {
    return orient2d_sign(comp(a, i), comp(a, j), comp(b, i), comp(b, j), comp(c, i), comp(c, j));
}

// ---- the predicate on triangles of doubles ----
// A triangle's projection: the first of the planes (x, y), (y, z), (z, x) on which its projection has a nonzero signed area `o` (the
// normal's z, x or y component); o = 0 on all three: (b - a) x (c - a) = 0, the triangle is degenerate.
struct TriProj { int i, j, o; };
__device__ __forceinline__ TriProj projection(const double t[3][3]) {
    int o = orient2(t[0], t[1], t[2], 0, 1);
    if (o) return {0, 1, o};
    o = orient2(t[0], t[1], t[2], 1, 2);
    if (o) return {1, 2, o};
    return {2, 0, orient2(t[0], t[1], t[2], 2, 0)};
}
// p in the closed triangle t (projected, orientation pr.o != 0)
__device__ __forceinline__ bool point_in_tri2(const double p[3], const double t[3][3], TriProj pr) {
    return orient2(t[0], t[1], p, pr.i, pr.j) != -pr.o && orient2(t[1], t[2], p, pr.i, pr.j) != -pr.o &&
           orient2(t[2], t[0], p, pr.i, pr.j) != -pr.o;
}
// q collinear with [p1, p2] (projected): q lies on the closed segment
__device__ __forceinline__ bool on_segment2(const double p1[3], const double p2[3], const double q[3], int i, int j) {
    const double ui = comp(p1, i), vi = comp(p2, i), qi = comp(q, i), uj = comp(p1, j), vj = comp(p2, j), qj = comp(q, j);
    return fmin(ui, vi) <= qi && qi <= fmax(ui, vi) && fmin(uj, vj) <= qj && qj <= fmax(uj, vj);
}
// closed segments [p1, p2] and [q1, q2] of one plane (projected, both non-degenerate) meet
__device__ __forceinline__ bool seg_seg2(const double p1[3], const double p2[3], const double q1[3], const double q2[3], int i, int j) {
    const int d1 = orient2(q1, q2, p1, i, j), d2 = orient2(q1, q2, p2, i, j);
    if (d1 != 0 && d1 == d2) return false;
    const int d3 = orient2(p1, p2, q1, i, j), d4 = orient2(p1, p2, q2, i, j);
    if (d3 != 0 && d3 == d4) return false;
    if (d1 && d2 && d3 && d4) return true;                      // proper crossing
    return (d1 == 0 && on_segment2(q1, q2, p1, i, j)) || (d2 == 0 && on_segment2(q1, q2, p2, i, j)) ||
           (d3 == 0 && on_segment2(p1, p2, q1, i, j)) || (d4 == 0 && on_segment2(p1, p2, q2, i, j));
}
// The closed segment [u, v] meets the closed triangle t.  su, sv: orient3(t, u), orient3(t, v), not both of one nonzero sign.
// Both zero: the segment lies in t's plane, decided in t's projection.  Otherwise it meets the plane in one point, which lies in t
// exactly when the line uv passes every directed edge of t on one side (orient3(u, v, t_k, t_k+1) all >= 0 or all <= 0).
__device__ __forceinline__ bool seg_tri(const double u[3], const double v[3], int su, int sv, const double t[3][3], TriProj pr) {
    if (su == 0 && sv == 0)
        return point_in_tri2(u, t, pr) || point_in_tri2(v, t, pr) || seg_seg2(u, v, t[0], t[1], pr.i, pr.j) ||
               seg_seg2(u, v, t[1], t[2], pr.i, pr.j) || seg_seg2(u, v, t[2], t[0], pr.i, pr.j);
    const int s1 = orient3(u, v, t[0], t[1]);
    const int s2 = orient3(u, v, t[1], t[2]);
    if (s1 * s2 < 0) return false;
    const int s3 = orient3(u, v, t[2], t[0]);
    return !(s1 > 0 || s2 > 0 || s3 > 0) || !(s1 < 0 || s2 < 0 || s3 < 0);
}
// Two non-degenerate closed triangles meet exactly when an edge of one meets the other: the boundary of the (compact, convex)
// intersection lies on the triangles' edges.  First the plane tests: one triangle strictly on one side of the other's plane.
__device__ __forceinline__ bool tri_tri(const double (&p)[3][3], TriProj pp, const double (&q)[3][3], TriProj qp) {
    int sq[3], sp[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) sq[k] = orient3(p[0], p[1], p[2], q[k]);
    if ((sq[0] > 0 && sq[1] > 0 && sq[2] > 0) || (sq[0] < 0 && sq[1] < 0 && sq[2] < 0)) return false;
#pragma unroll
    for (int k = 0; k < 3; ++k) sp[k] = orient3(q[0], q[1], q[2], p[k]);
    if ((sp[0] > 0 && sp[1] > 0 && sp[2] > 0) || (sp[0] < 0 && sp[1] < 0 && sp[2] < 0)) return false;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int l = k == 2 ? 0 : k + 1;
        if (!(sp[k] != 0 && sp[k] == sp[l]) && seg_tri(p[k], p[l], sp[k], sp[l], q, qp)) return true;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int l = k == 2 ? 0 : k + 1;
        if (!(sq[k] != 0 && sq[k] == sq[l]) && seg_tri(q[k], q[l], sq[k], sq[l], p, pp)) return true;
    }
    return false;
}

// ---- the leaf policy of the triangle-pair walk (overlap_walk, csr.cuh) ----
// A triangle is EXCLUDED when a coordinate is not finite or (b - a) x (c - a) = 0; it meets nothing.  An f64 triangle with a nonzero
// coordinate of magnitude outside [TRI_F64_LO, TRI_F64_HI] is UNCHECKED: never excluded as degenerate, and every pair with it that the
// boxes report (the other triangle not excluded) is kept.  Otherwise meets(P, Q): a shared vertex (all three coordinates ==) reports
// the pair, or drops it with skip_shared; else tri_tri.
enum : int { TRI_EXCLUDED = 0, TRI_UNCHECKED = 1, TRI_OK = 2 };
template <class T> __device__ __forceinline__ bool tri_in_range(T x) {
    if (sizeof(T) == 4) return true;
    const double a = fabs((double)x);
    return a == 0.0 || (a >= TRI_F64_LO && a <= TRI_F64_HI);
}
// Loads triangle s as doubles; returns TRI_EXCLUDED for a non-finite coordinate, TRI_UNCHECKED out of range, else TRI_OK (its
// degeneracy still to be decided).
template <class T> __device__ __forceinline__ int load_tri(const DTri<T>* __restrict__ tris, uint32_t s, double (&v)[3][3]) {
    const DTri<T>* t = tris + s;
    bool finite = true, in_range = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const T x = __ldg(t->a + k), y = __ldg(t->b + k), z = __ldg(t->c + k);
        v[0][k] = (double)x; v[1][k] = (double)y; v[2][k] = (double)z;
        finite = finite && isfinite(v[0][k]) && isfinite(v[1][k]) && isfinite(v[2][k]);
        in_range = in_range && tri_in_range<T>(x) && tri_in_range<T>(y) && tri_in_range<T>(z);
    }
    return !finite ? TRI_EXCLUDED : !in_range ? TRI_UNCHECKED : TRI_OK;
}
template <class T> struct TriPairsLeaf {
    const DTri<T>* own;           // the triangles of the row's tree
    const DTri<T>* other;         // the triangles of the walked tree (== own in the self form)
    int skip_shared;
    double p[3][3];
    TriProj pp;
    int pclass;
    // the row's triangle; false: it is excluded and the row is empty
    __device__ __forceinline__ bool row(uint32_t s) {
        pclass = load_tri<T>(own, s, p);
        if (pclass == TRI_OK) {
            pp = projection(p);
            if (!pp.o) pclass = TRI_EXCLUDED;                     // degenerate
        }
        return pclass != TRI_EXCLUDED;
    }
    __device__ __forceinline__ bool keep(uint32_t t) {
        double q[3][3];
        const int qclass = load_tri<T>(other, t, q);
        if (qclass == TRI_EXCLUDED) return false;
        if (qclass == TRI_UNCHECKED || pclass == TRI_UNCHECKED) return true;
        bool shared = false;
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int b = 0; b < 3; ++b) shared = shared || (p[a][0] == q[b][0] && p[a][1] == q[b][1] && p[a][2] == q[b][2]);
        if (shared && skip_shared) return false;                  // decided before Q's degeneracy: either way it is not reported
        const TriProj qp = projection(q);
        if (!qp.o) return false;                                  // degenerate
        return shared || tri_tri(p, pp, q, qp);
    }
};

#endif  // __CUDACC__
}  // namespace bvhb200
