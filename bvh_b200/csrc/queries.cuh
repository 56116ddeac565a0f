// bvh_b200/csrc/queries.cuh -- the IntersectsAabb predicates other than Ray and the nearest_to walks, generic in the dimension D.
// Shared by traverse.cu (D = 3, and D = 2 through the z = 0 embedding of dim2.cu) and dim4.cu (D = 4).  Every sum runs over the axes
// left to right in T without FMA, so the instantiation for D = 3 performs exactly the operations the 3-D kernels always did.
#pragma once
#include "common.cuh"
#include <type_traits>

namespace bvhb200 {

#ifdef __CUDACC__
// ---- query records: Aabb {min, max} (2D T), Point (D T), Ball {center, radius} (D + 1 T) (src/aabb/intersection.rs:35-45,
// src/ball.rs:85-106).  Each is a probe of csr_walk_kernel (csr.cuh): load(src, r) reads record r of the batch at src,
// hit(mn, mx) is the predicate. ----
template <class T, int KIND, int D> struct Query;
template <class T, int D> struct Query<T, BVHGPU_QUERY_AABB, D> {
    T mn[D], mx[D];
    static constexpr int STRIDE = 2 * D;
    __device__ __forceinline__ void load(const void* src, uint32_t r) { const T* p = static_cast<const T*>(src) + (size_t)r * STRIDE; for (int k = 0; k < D; ++k) { mn[k] = __ldg(p + k); mx[k] = __ldg(p + D + k); } }
    __device__ __forceinline__ bool hit(const T bmn[D], const T bmx[D]) const {            // aabb_impl.rs:240-248
        bool h = true;
#pragma unroll
        for (int i = 0; i < D; ++i) if (mx[i] < bmn[i] || bmx[i] < mn[i]) h = false;
        return h;
    }
};
template <class T, int D> struct Query<T, BVHGPU_QUERY_POINT, D> {
    T p[D];
    static constexpr int STRIDE = D;
    __device__ __forceinline__ void load(const void* src, uint32_t r) { const T* q = static_cast<const T*>(src) + (size_t)r * STRIDE; for (int k = 0; k < D; ++k) p[k] = __ldg(q + k); }
    __device__ __forceinline__ bool hit(const T bmn[D], const T bmx[D]) const {            // Aabb::contains, aabb_impl.rs:175-177
        bool h = true;
#pragma unroll
        for (int i = 0; i < D; ++i) if (!(p[i] >= bmn[i]) || !(p[i] <= bmx[i])) h = false;
        return h;
    }
};
template <class T, int D> struct Query<T, BVHGPU_QUERY_BALL, D> {
    T c[D], r2;
    static constexpr int STRIDE = D + 1;
    __device__ __forceinline__ void load(const void* src, uint32_t r) { const T* q = static_cast<const T*>(src) + (size_t)r * STRIDE; for (int k = 0; k < D; ++k) c[k] = __ldg(q + k); const T rad = __ldg(q + D); r2 = mul_rn(rad, rad); }
    __device__ __forceinline__ bool hit(const T bmn[D], const T bmx[D]) const {            // Ball::intersects_aabb, ball.rs:85-99
        T d2 = T(0);
#pragma unroll
        for (int i = 0; i < D; ++i) {
            T x = c[i];
            if (x < bmn[i]) x = bmn[i];
            if (x > bmx[i]) x = bmx[i];
            const T d = sub_rn(x, c[i]);
            d2 = add_rn(d2, mul_rn(d, d));
        }
        return d2 <= r2;
    }
};

// Internal kind: every shape whose AABB lies within squared distance U of a point, record {p, U} (D + 1 T).
//
// The per-axis gap of a box is judged against two distances: the exact one, and the reference's rounded
// Aabb::min_distance_squared (aabb_impl.rs:618-629: |p - centre| - half_size), which cancels badly far from the origin.  The
// reference's gap differs from the exact gap by less than 9 u m (u = eps / 2, m = max(|p|, -min, max, max - min) on that axis,
// plus a few subnormal steps), and min - p, p - max are off by at most 2 u m.  axis_slack is 16 eps m + 16 subnormal steps, so
// the lower bound sum_k max(max(min_k - p_k, p_k - max_k) - slack_k, 0)^2 stays below both distances.  It is monotone under box
// containment in floating point (a larger box has smaller differences and a larger m; subtraction, squaring and addition of
// non-negative terms are monotone), so pruning an inner box can never lose a shape it contains.  An empty child box (min > max
// on some axis: the Aabb::empty() a "no split wins" node stores where surface areas overflow) contains nothing it bounds, so it
// is always entered.
constexpr int QUERY_WITHIN = 4;
template <class T> __device__ __forceinline__ T slack_floor();
template <> __device__ __forceinline__ float slack_floor<float>() { return 0x1p-145f; }        // 16 f32 subnormal steps
template <> __device__ __forceinline__ double slack_floor<double>() { return 0x1p-1070; }      // 16 f64 subnormal steps
// m of one axis of one box; an empty axis (min = +inf, max = -inf) gives |p|, a NaN term is ignored
template <class T> __device__ __forceinline__ T axis_magnitude(T p, T mn, T mx) {
    T m = fabs(p);
    const T nmn = -mn, ext = sub_rn(mx, mn);
    m = nmn > m ? nmn : m;
    m = mx > m ? mx : m;
    return ext > m ? ext : m;
}
template <class T> __device__ __forceinline__ T axis_slack(T m) { return add_rn(mul_rn(m, mul_rn(T(16), Traits<T>::eps())), slack_floor<T>()); }
template <int D, class T> __device__ __forceinline__ T box_lower_d2(const T p[D], const T bmn[D], const T bmx[D]) {
    T d2 = T(0);
#pragma unroll
    for (int i = 0; i < D; ++i) {
        const T a = sub_rn(bmn[i], p[i]), b = sub_rn(p[i], bmx[i]);
        T d = a > b ? a : b;
        d = sub_rn(d, axis_slack(axis_magnitude(p[i], bmn[i], bmx[i])));
        d = d > T(0) ? d : T(0);
        d2 = add_rn(d2, mul_rn(d, d));
    }
    return d2;
}
// The U of nearest_candidates at a shape: the squared distance to the farthest corner, each non-zero axis term widened by the
// slack of m = max(that axis's m of the shape, g[axis]).  g is the magnitude of the root's child boxes: every node below them
// has a smaller m, so U also bounds the reference's rounded distance of any node Bvh::nearest_to prunes (see nearest_bound_kernel).
// A zero farthest distance means min = max = p on that axis, where the reference's term is exactly 0 as well.
template <int D, class T> __device__ __forceinline__ T box_upper_d2(const T p[D], const T bmn[D], const T bmx[D], const T g[D]) {
    T d2 = T(0);
#pragma unroll
    for (int i = 0; i < D; ++i) {
        const T a = fabs(sub_rn(p[i], bmn[i])), b = fabs(sub_rn(p[i], bmx[i]));
        T d = a > b ? a : b;
        if (d > T(0)) {
            const T m = axis_magnitude(p[i], bmn[i], bmx[i]);
            d = add_rn(d, axis_slack(g[i] > m ? g[i] : m));
        }
        d2 = add_rn(d2, mul_rn(d, d));
    }
    return d2;
}
// g of box_upper_d2 for one point: the axis magnitudes of the root's two child boxes.  Empty boxes (those of a root leaf, or of
// a "no split wins" root) give |p|.
template <int D, class T, class Node> __device__ __forceinline__ void root_magnitude(const Node* __restrict__ nodes, const T p[D], T g[D]) {
#pragma unroll
    for (int k = 0; k < D; ++k) {
        const T l = axis_magnitude(p[k], __ldg(&nodes[0].l_aabb.min[k]), __ldg(&nodes[0].l_aabb.max[k]));
        const T r = axis_magnitude(p[k], __ldg(&nodes[0].r_aabb.min[k]), __ldg(&nodes[0].r_aabb.max[k]));
        g[k] = l > r ? l : r;
    }
}
template <class T, int D> struct Query<T, QUERY_WITHIN, D> {
    T p[D], u;
    static constexpr int STRIDE = D + 1;
    __device__ __forceinline__ void load(const void* src, uint32_t r) { const T* q = static_cast<const T*>(src) + (size_t)r * STRIDE; for (int k = 0; k < D; ++k) p[k] = __ldg(q + k); u = __ldg(q + D); }
    __device__ __forceinline__ bool hit(const T bmn[D], const T bmx[D]) const {
        bool empty = false;
#pragma unroll
        for (int i = 0; i < D; ++i) empty |= bmn[i] > bmx[i];
        return empty || box_lower_d2<D>(p, bmn, bmx) <= u;
    }
};

// Aabb::min_distance_squared (aabb_impl.rs:618-629): per axis max(|p - centre| - half_size, 0), then the dot product
// ((o0*o0 + o1*o1) + o2*o2) [+ o3*o3].  An empty box (min = +inf, max = -inf) gives a NaN centre and o = 0 on that axis, as
// NaN.max(0) = 0 in Rust.
template <int D, class T> __device__ __forceinline__ T aabb_min_d2(const T p[D], const T mn[D], const T mx[D]) {
    T o[D];
#pragma unroll
    for (int k = 0; k < D; ++k) {
        const T hs = mul_rn(sub_rn(mx[k], mn[k]), T(0.5));             // half_size(), :479-481
        const T c = add_rn(mn[k], hs);
        const T q = sub_rn(fabs(sub_rn(p[k], c)), hs);
        o[k] = q > T(0) ? q : T(0);
    }
    T acc = add_rn(mul_rn(o[0], o[0]), mul_rn(o[1], o[1]));
#pragma unroll
    for (int k = 2; k < D; ++k) acc = add_rn(acc, mul_rn(o[k], o[k]));
    return acc;
}
template <class T> __device__ __forceinline__ T quiet_nan();                                      // the padding of out_closest
template <> __device__ __forceinline__ float quiet_nan<float>() { return __int_as_float(0x7fc00000); }
template <> __device__ __forceinline__ double quiet_nan<double>() { return __longlong_as_double(0x7ff8000000000000ll); }
__device__ __forceinline__ float sqrt_rn(float x) { return __fsqrt_rn(x); }
__device__ __forceinline__ double sqrt_rn(double x) { return __dsqrt_rn(x); }

// ---- nearest_to: Bvh::nearest_to (bvh_impl.rs:221-238, bvh_node.rs:327-372) over the reference node array ----
// EXACT: reference semantics (children ordered by min_distance_squared, prune with `<`, first minimum kept).
// !EXACT: children ordered and pruned by the monotone lower bound box_lower_d2, ties kept (`<=`).
// leaf(shape) returns the leaf's value.  The recursion is a stackless walk over parent links: on the way back up the two child
// distances are recomputed (same bits), so any tree depth works without a stack.  Node: a bvh_node{D}{f,d} POD.
template <int D, class T, bool EXACT, class Node, class Leaf>
__device__ __forceinline__ void nearest_walk(const Node* __restrict__ nodes, const T p[D], uint32_t& best, T& best_d, Leaf leaf) {
    best = BVH_INVALID;
    best_d = Traits<T>::inf();
    uint32_t node = 0, from = BVH_INVALID;                 // from: the child we are returning from (BVH_INVALID = arriving from the parent)
    for (;;) {
        const uint4 meta = __ldg(reinterpret_cast<const uint4*>(nodes + node));      // parent, child_l, child_r, shape
        if (meta.y == BVH_INVALID) {                       // leaf
            const T d = leaf(meta.w);
            if (best == BVH_INVALID || d < best_d) { best = meta.w; best_d = d; }
            if (node == 0) return;
            from = node; node = meta.x;
            continue;
        }
        const Node& nd = nodes[node];
        T lmn[D], lmx[D], rmn[D], rmx[D];
#pragma unroll
        for (int k = 0; k < D; ++k) { lmn[k] = __ldg(&nd.l_aabb.min[k]); lmx[k] = __ldg(&nd.l_aabb.max[k]); rmn[k] = __ldg(&nd.r_aabb.min[k]); rmx[k] = __ldg(&nd.r_aabb.max[k]); }
        const T dl = EXACT ? aabb_min_d2<D>(p, lmn, lmx) : box_lower_d2<D>(p, lmn, lmx);
        const T dr = EXACT ? aabb_min_d2<D>(p, rmn, rmx) : box_lower_d2<D>(p, rmn, rmx);
        const bool swap = dl > dr;                          // bvh_node.rs:349-351
        const uint32_t near_i = swap ? meta.z : meta.y, far_i = swap ? meta.y : meta.z;
        const T near_d = swap ? dr : dl, far_d = swap ? dl : dr;
        uint32_t next = BVH_INVALID;
        if (from == BVH_INVALID) {                          // first visit: the nearer child, if it can still win
            if (best == BVH_INVALID || (EXACT ? near_d < best_d : near_d <= best_d)) next = near_i;
            else from = near_i;                             // skipped: as if we had just returned from it
        }
        if (next == BVH_INVALID && from == near_i) {        // back from (or past) the nearer child: now the farther one
            if (best == BVH_INVALID || (EXACT ? far_d < best_d : far_d <= best_d)) next = far_i;
            else from = far_i;
        }
        if (next != BVH_INVALID) { node = next; from = BVH_INVALID; continue; }
        if (node == 0) return;                              // back from the farther child of the root
        from = node; node = meta.x;
    }
}

// ---- k nearest shapes (bvhgpu_knn_*): the parent-link walk of nearest_walk<D, T, false> keeping the K best keys ----
// The key of shape s is (d2, s) in lexicographic order, d2 = leaf(s) (aabb_min_d2 of the shape's own current box, never NaN).  The
// list d[0 .. K) / s[0 .. K) is sorted DESCENDING.  Slots 0 .. k-1 start as (+inf, BVH_INVALID), worse than every real key; slots
// k .. K-1 hold (-inf, BVH_INVALID) sentinels that no key passes.  So d[0], s[0] is the current k-th key for any k <= K, the insertion
// shifts towards slot 0, and every array index is a compile-time constant: the list stays in registers when it fits.
// A child is entered when its box is empty or box_lower_d2 <= min(d[0], r2): every shape below it has a key >= that bound (the bound
// is monotone under containment and stays below the rounded distance of the shape's own box, see Query<T, QUERY_WITHIN, D>), so a
// pruned subtree holds no shape that could still enter the list or qualify.  Ties are entered, so an equal key with a lower index is
// never lost, and the result is the brute-force order whatever the visiting order.
template <class T> __device__ __forceinline__ bool key_less(T a, uint32_t ia, T b, uint32_t ib) { return a < b || (a == b && ia < ib); }
template <class T, int K> __device__ __forceinline__ void knn_insert(T (&d)[K], uint32_t (&s)[K], T key, uint32_t id) {
    bool moving = true;                                     // slot 0 (the k-th key) is dropped; (key, id) goes where it belongs
#pragma unroll
    for (int j = 0; j + 1 < K; ++j) {
        const bool shift = moving && key_less(key, id, d[j + 1], s[j + 1]);
        if (moving) { d[j] = shift ? d[j + 1] : key; s[j] = shift ? s[j + 1] : id; }
        moving = shift;
    }
    if (moving) { d[K - 1] = key; s[K - 1] = id; }
}
template <int D, class T, int K, class Node, class Leaf>
__device__ __forceinline__ void knn_walk(const Node* __restrict__ nodes, const T p[D], T r2, T (&d)[K], uint32_t (&s)[K], Leaf leaf) {
    uint32_t node = 0, from = BVH_INVALID;
    for (;;) {
        const uint4 meta = __ldg(reinterpret_cast<const uint4*>(nodes + node));      // parent, child_l, child_r, shape
        if (meta.y == BVH_INVALID) {
            const T key = leaf(meta.w);
            if (key <= r2 && key_less(key, meta.w, d[0], s[0])) knn_insert(d, s, key, meta.w);
            if (node == 0) return;
            from = node; node = meta.x;
            continue;
        }
        const Node& nd = nodes[node];
        T lmn[D], lmx[D], rmn[D], rmx[D];
        bool el = false, er = false;
#pragma unroll
        for (int k = 0; k < D; ++k) {
            lmn[k] = __ldg(&nd.l_aabb.min[k]); lmx[k] = __ldg(&nd.l_aabb.max[k]); rmn[k] = __ldg(&nd.r_aabb.min[k]); rmx[k] = __ldg(&nd.r_aabb.max[k]);
            el |= lmn[k] > lmx[k]; er |= rmn[k] > rmx[k];
        }
        const T dl = box_lower_d2<D>(p, lmn, lmx), dr = box_lower_d2<D>(p, rmn, rmx);
        const bool swap = dl > dr;
        const uint32_t near_i = swap ? meta.z : meta.y, far_i = swap ? meta.y : meta.z;
        const T near_d = swap ? dr : dl, far_d = swap ? dl : dr;
        const bool near_e = swap ? er : el, far_e = swap ? el : er;
        uint32_t next = BVH_INVALID;
        if (from == BVH_INVALID) {                          // first visit: the nearer child
            if (near_e || (near_d <= d[0] && near_d <= r2)) next = near_i;
            else from = near_i;                             // skipped: as if we had just returned from it
        }
        if (next == BVH_INVALID && from == near_i) {        // back from (or past) the nearer child: the farther one, against the new k-th key
            if (far_e || (far_d <= d[0] && far_d <= r2)) next = far_i;
            else from = far_i;
        }
        if (next != BVH_INVALID) { node = next; from = BVH_INVALID; continue; }
        if (node == 0) return;
        from = node; node = meta.x;
    }
}
// One point of a knn batch: limit r (has_limit) qualifies the shapes with d2 <= fl(r * r) (Ball::intersects_aabb's comparison); r < 0
// or NaN qualifies none (-0 >= 0 holds); an empty tree (n_shapes == 0) none.  Row i*k .. i*k+k-1 of the outputs gets the list in
// ascending order, sqrt of each key as the distance, (BVH_INVALID, +inf) past the qualifying shapes.
template <int D, class T, int K, class Node, class Leaf>
__device__ __forceinline__ void knn_point(const Node* __restrict__ nodes, uint32_t n_shapes, const T p[D], bool has_limit, T r, uint32_t k,
                                          uint32_t* __restrict__ out_shape, T* __restrict__ out_dist, Leaf leaf) {
    T d[K];
    uint32_t s[K];
#pragma unroll
    for (int j = 0; j < K; ++j) { d[j] = j < (int)k ? Traits<T>::inf() : -Traits<T>::inf(); s[j] = BVH_INVALID; }
    const T r2 = has_limit ? mul_rn(r, r) : Traits<T>::inf();
    if (n_shapes != 0 && (!has_limit || r >= T(0))) knn_walk<D, T, K>(nodes, p, r2, d, s, leaf);
#pragma unroll
    for (int j = 0; j < K; ++j)
        if (j < (int)k) { out_shape[k - 1 - j] = s[j]; out_dist[k - 1 - j] = d[j]; }
    // the square roots in a loop of its own: one call site of sqrt's slow path instead of K, none with the list live (no spills)
#pragma unroll 1
    for (uint32_t j = 0; j < k; ++j) out_dist[j] = sqrt_rn(out_dist[j]);
}
// The K bucket of knn_walk for 1 <= k <= BVHGPU_KNN_MAX_K: launch(std::integral_constant<int, K>{}).
template <class Launch> inline void knn_bucket(uint32_t k, Launch launch) {
    if (k <= 4) launch(std::integral_constant<int, 4>{});
    else if (k <= 8) launch(std::integral_constant<int, 8>{});
    else if (k <= 16) launch(std::integral_constant<int, 16>{});
    else if (k <= 32) launch(std::integral_constant<int, 32>{});
    else launch(std::integral_constant<int, 64>{});
}

// FlatBvh::nearest_to (flat_bvh.rs:513-562) over the reference FlatNode array.  Flat: a bvh_flat{D}{f,d} POD.
template <int D, class T, class Flat, class Leaf>
__device__ __forceinline__ void nearest_flat(const Flat* __restrict__ flat, uint32_t n_flat, const T p[D], uint32_t& best, T& best_d, Leaf leaf) {
    uint32_t index = 0;
    while (index < n_flat) {                                // flat_bvh.rs:524-558
        const Flat& f = flat[index];
        const uint32_t entry = f.entry_index, exit_i = f.exit_index;
        if (entry == BVH_INVALID) {
            const uint32_t shape = f.shape_index;
            const T d = leaf(shape);
            if (best == BVH_INVALID || d < best_d) { best = shape; best_d = d; }
            index = exit_i;
        } else {
            T mn[D], mx[D];
            for (int k = 0; k < D; ++k) { mn[k] = f.aabb.min[k]; mx[k] = f.aabb.max[k]; }
            const T md = aabb_min_d2<D>(p, mn, mx);
            index = (best == BVH_INVALID || md < best_d) ? entry : exit_i;
        }
    }
}
#endif  // __CUDACC__

}  // namespace bvhb200
