// bvh_b200/csrc/segments.cu -- polygons of 2-D trees (bvhgpu_tree_set_segments_*, include/bvh_b200.h; DESIGN.md §4.23): exact
// point-in-polygon with winding numbers, the k nearest segments and the signed distance to the segments.
//
// A 2-D tree lives embedded in the plane z = 0 (dim2.cu): its records have z = [-1, +1] (empty child boxes z = [+inf, -inf]), its shape
// boxes d_aabb and node boxes z = [0, 0].
//   contains   one thread per point p walks the records with overlap_records (csr.cuh) and the query box [px, +inf] x [py, py] x [0, 0]:
//              a record is entered when its box meets the query box or is empty, a reached shape is tested against its own box, then
//              winding_leaf runs on its segment.  A segment relevant to p (its y range contains py, max(ax, bx) >= px) lies in its
//              shape's box (the caller's condition), so that box meets the query box, and so does every stored box above it that is not
//              empty: no relevant segment is missed, whatever the tree.  The signs are exact (orient2d_sign, exact.cuh).
//   knn        knn_point<3, T, K> (queries.cuh) on the point lifted to z = 0, with segment_key at the leaves: the walk of knn_tri_kernel.
//   signed     the knn row (k = 1, no limit), the contains class, and polygon_sign_kernel: negated where the class is 1 (inside).
#include "exact.cuh"
#include "csr.cuh"

namespace bvhb200 {

// The f64 range on which orient2d_sign is exact (as for the triangle pairs, tritri.cuh): zero or a magnitude in [2^-300, 2^300].  The
// differences are multiples of 2^-352 below 2^301, their products multiples of 2^-704 below 2^602: no two_prod or two_sum underflows or
// overflows.  f32 coordinates promoted to double are exact everywhere (multiples of 2^-149 below 2^128).
constexpr double SEG_F64_LO = 0x1p-300, SEG_F64_HI = 0x1p+300;
template <class T> __device__ __forceinline__ bool seg_in_range(T x) {
    if (sizeof(T) == 4) return true;
    const double a = fabs((double)x);
    return a == 0.0 || (a >= SEG_F64_LO && a <= SEG_F64_HI);
}

__device__ __forceinline__ void load_seg(const DSeg<float>* p, float& ax, float& ay, float& bx, float& by) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(p));
    ax = v.x; ay = v.y; bx = v.z; by = v.w;
}
__device__ __forceinline__ void load_seg(const DSeg<double>* p, double& ax, double& ay, double& bx, double& by) {
    const double2 a = __ldg(reinterpret_cast<const double2*>(p)), b = __ldg(reinterpret_cast<const double2*>(p) + 1);
    ax = a.x; ay = a.y; bx = b.x; by = b.y;
}

// One segment's part of the winding number of p (px, py finite and, in f64, in range).  Excluded (non-finite coordinate, a == b): nothing.
// Not relevant: nothing.  Relevant with an f64 coordinate out of range: undecided.  Otherwise o = sign(orient2d(a, b, p)): boundary when
// o == 0 and p lies in the closed box of a and b; +1 when ay <= py < by and o > 0; -1 when by <= py < ay and o < 0.
template <class T>
__device__ __forceinline__ void winding_leaf(const DSeg<T>* __restrict__ seg, T px, T py, int32_t& w, bool& boundary, bool& undecided) {
    T ax, ay, bx, by;
    load_seg(seg, ax, ay, bx, by);
    if (!(isfinite(ax) && isfinite(ay) && isfinite(bx) && isfinite(by)) || (ax == bx && ay == by)) return;
    const T ylo = ay < by ? ay : by, yhi = ay < by ? by : ay, xlo = ax < bx ? ax : bx, xhi = ax < bx ? bx : ax;
    if (!(ylo <= py && py <= yhi && xhi >= px)) return;
    if (!(seg_in_range(ax) && seg_in_range(ay) && seg_in_range(bx) && seg_in_range(by))) { undecided = true; return; }
    const int o = orient2d_sign((double)ax, (double)ay, (double)bx, (double)by, (double)px, (double)py);
    if (o == 0) {
        if (xlo <= px) boundary = true;                                       // y range and px <= xhi hold already
    } else if (o > 0) {
        if (ay <= py && py < by) ++w;
    } else if (by <= py && py < ay) {
        --w;
    }
}

template <class T>
__global__ void __launch_bounds__(128) polygon_contains_kernel(const typename Traits<T>::TNode* __restrict__ trec, uint32_t n_rec,
                                                               const typename Traits<T>::DAabb* __restrict__ aabb, const DSeg<T>* __restrict__ segs,
                                                               const T* __restrict__ points, uint32_t n, int rule, uint8_t* __restrict__ out_class,
                                                               int32_t* __restrict__ out_winding) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const T px = __ldg(points + 2 * (size_t)i), py = __ldg(points + 2 * (size_t)i + 1);
    int32_t w = 0;
    uint8_t cls = BVHGPU_POINT_OUTSIDE;
    if (!(isfinite(px) && isfinite(py))) {
        // a non-finite point: outside, winding 0
    } else if (!(seg_in_range(px) && seg_in_range(py))) {
        cls = BVHGPU_POINT_UNDECIDED;                                         // not walked
    } else {
        const T smn[3] = {px, py, T(0)}, smx[3] = {Traits<T>::inf(), py, T(0)};
        bool boundary = false, undecided = false;
        overlap_records<3, T>(trec, 0u, n_rec, smn, smx, [&](uint32_t shape) {
            T tmn[3], tmx[3];
            load_box(aabb + shape, tmn, tmx);
            if (overlap_boxes<3, T>(smn, smx, tmn, tmx)) winding_leaf<T>(segs + shape, px, py, w, boundary, undecided);
        });
        const bool inside = rule == BVHGPU_FILL_EVEN_ODD ? (w & 1) != 0 : w != 0;
        cls = boundary ? BVHGPU_POINT_BOUNDARY : undecided ? BVHGPU_POINT_UNDECIDED : inside ? BVHGPU_POINT_INSIDE : BVHGPU_POINT_OUTSIDE;
    }
    out_class[i] = cls;
    if (out_winding) out_winding[i] = w;
}

// The key of bvhgpu_knn_segments_*, operation for operation in T without FMA; q = the closest point it is measured against.  A NaN num
// takes the interior branch, and the key is NaN.
template <class T>
__device__ __forceinline__ T segment_key(T px, T py, T ax, T ay, T bx, T by, T& qx, T& qy) {
    const T ex = sub_rn(bx, ax), ey = sub_rn(by, ay), wx = sub_rn(px, ax), wy = sub_rn(py, ay);
    const T num = add_rn(mul_rn(wx, ex), mul_rn(wy, ey)), den = add_rn(mul_rn(ex, ex), mul_rn(ey, ey));
    if (num <= T(0)) { qx = ax; qy = ay; }
    else if (num >= den) { qx = bx; qy = by; }
    else {
        const T t = div_rn(num, den);
        qx = add_rn(ax, mul_rn(t, ex)); qy = add_rn(ay, mul_rn(t, ey));
    }
    const T dx = sub_rn(px, qx), dy = sub_rn(py, qy);
    return add_rn(mul_rn(dx, dx), mul_rn(dy, dy));
}

// k nearest segments: knn_point on the point lifted to z = 0 over the embedded node array (z = [0, 0]: every z term of box_lower_d2 is
// +0, dim2.cu), segment_key at the leaves.  The closest points are recomputed for the k final slots after the walk, as knn_tri_kernel
// does: the same operations on the same inputs.
template <class T, int K>
__global__ void __launch_bounds__(128) knn_seg_kernel(const typename Traits<T>::Node* __restrict__ nodes, uint32_t n_shapes,
                                                      const DSeg<T>* __restrict__ segs, const T* __restrict__ points, const T* __restrict__ max_dist,
                                                      uint32_t nq, uint32_t k, uint32_t* __restrict__ out_shape, T* __restrict__ out_dist,
                                                      T* __restrict__ out_closest) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    const T p[3] = {__ldg(points + 2 * (size_t)i), __ldg(points + 2 * (size_t)i + 1), T(0)};
    auto leaf = [&](uint32_t shape) {
        T ax, ay, bx, by, qx, qy;
        load_seg(segs + shape, ax, ay, bx, by);
        return segment_key(p[0], p[1], ax, ay, bx, by, qx, qy);
    };
    knn_point<3, T, K>(nodes, n_shapes, p, max_dist != nullptr, max_dist ? max_dist[i] : T(0), k, out_shape + (size_t)i * k,
                       out_dist + (size_t)i * k, leaf);
    if (!out_closest) return;
#pragma unroll 1
    for (uint32_t j = 0; j < k; ++j) {
        const uint32_t s = out_shape[(size_t)i * k + j];
        T qx = quiet_nan<T>(), qy = quiet_nan<T>();
        if (s != BVH_INVALID) {
            T ax, ay, bx, by;
            load_seg(segs + s, ax, ay, bx, by);
            segment_key(p[0], p[1], ax, ay, bx, by, qx, qy);
        }
        T* o = out_closest + 2 * ((size_t)i * k + j);
        o[0] = qx; o[1] = qy;
    }
}

// Signed distance: the k = 1 row negated where the class is 1 (inside); boundary (2) and undecided (3) points keep their distance, and a
// point without a segment keeps +inf.
template <class T>
__global__ void __launch_bounds__(256) polygon_sign_kernel(uint32_t n, const uint8_t* __restrict__ cls, const uint32_t* __restrict__ shape,
                                                           T* __restrict__ dist) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (cls[i] == BVHGPU_POINT_INSIDE && shape[i] != BVH_INVALID) dist[i] = -dist[i];     // inside at distance 0 gives -0
}

template <class T> int set_segments(Tree<T>* tree, const T* segs4, size_t n) {
    bvhgpu_ctx* ctx = tree->ctx;
    if (n != tree->n) { set_error("set_segments: %zu segments for a tree over %u shapes", n, tree->n); return BVHGPU_ERR_INVALID; }
    if (n == 0) return BVHGPU_OK;
    if (!tree->d_segs) BVH_TRY(dalloc(ctx, &tree->d_segs, sizeof(DSeg<T>) * n));
    BVH_CUDA_TRY(cudaMemcpyAsync(tree->d_segs, segs4, sizeof(DSeg<T>) * n, cudaMemcpyHostToDevice, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));                          // the caller's buffer may go away
    return BVHGPU_OK;
}

// The checks the three calls share after their own (pointers, n, rule / k): the tree's status, then the segments.
template <class T> static int segments_check(Tree<T>* tree, const char* what) {
    BVH_TRY(resolve_status(tree));
    if (tree->n && !tree->d_segs) { set_error("%s: needs bvhgpu_tree_set_segments_* first", what); return BVHGPU_ERR_INVALID; }
    return BVHGPU_OK;
}
static int polygon_rule(const char* what, int rule) {
    if (rule != BVHGPU_FILL_EVEN_ODD && rule != BVHGPU_FILL_NONZERO) { set_error("%s: unknown fill rule %d", what, rule); return BVHGPU_ERR_INVALID; }
    return BVHGPU_OK;
}
template <class T> static int contains_launch(Tree<T>* tree, const T* d_points, size_t n, int rule, uint8_t* d_class, int32_t* d_winding) {
    bvhgpu_ctx* ctx = tree->ctx;
    if (tree->n == 0) {                                                        // empty tree: class 0, winding 0
        BVH_CUDA_TRY(cudaMemsetAsync(d_class, 0, n, ctx->stream));
        if (d_winding) BVH_CUDA_TRY(cudaMemsetAsync(d_winding, 0, sizeof(int32_t) * n, ctx->stream));
        return BVHGPU_OK;
    }
    BVH_TRY(ensure_records(tree));
    polygon_contains_kernel<T><<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(
        tree->d_tnodes, tree->n_trec, tree->d_aabb, reinterpret_cast<const DSeg<T>*>(tree->d_segs), d_points, (uint32_t)n, rule, d_class, d_winding);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}
template <class T> int polygon_contains_device(Tree<T>* tree, const T* d_points, size_t n, int rule, uint8_t* d_class, int32_t* d_winding) {
    BVH_TRY(check_n("contains_points", n));
    BVH_TRY(polygon_rule("contains_points", rule));
    BVH_TRY(segments_check(tree, "contains_points"));
    if (n == 0) return BVHGPU_OK;
    return contains_launch(tree, d_points, n, rule, d_class, d_winding);
}
template <class T> static int knn_seg_launch(Tree<T>* tree, const T* d_points, size_t n, uint32_t k, const T* d_max_dist, uint32_t* d_shape, T* d_dist,
                                             T* d_closest) {
    bvhgpu_ctx* ctx = tree->ctx;
    const unsigned grid = (unsigned)((n + 127) / 128);
    knn_bucket(k, [&](auto kb) {
        knn_seg_kernel<T, decltype(kb)::value><<<grid, 128, 0, ctx->stream>>>(tree->d_nodes, tree->n, reinterpret_cast<const DSeg<T>*>(tree->d_segs),
                                                                            d_points, d_max_dist, (uint32_t)n, k, d_shape, d_dist, d_closest);
    });
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}
template <class T> int knn_seg_device(Tree<T>* tree, const T* d_points, size_t n, uint32_t k, const T* d_max_dist, uint32_t* d_shape, T* d_dist,
                                      T* d_closest) {
    BVH_TRY(check_n("knn_segments", n));
    if (k < 1 || k > BVHGPU_KNN_MAX_K) { set_error("knn_segments: k = %u outside 1 .. %d", k, BVHGPU_KNN_MAX_K); return BVHGPU_ERR_INVALID; }
    BVH_TRY(segments_check(tree, "knn_segments"));
    if (n == 0) return BVHGPU_OK;
    return knn_seg_launch(tree, d_points, n, k, d_max_dist, d_shape, d_dist, d_closest);
}
// knn (k = 1, no limit), the contains walk into scratch, the sign: three launches on the context's stream.
template <class T> int polygon_distance_device(Tree<T>* tree, const T* d_points, size_t n, int rule, uint32_t* d_shape, T* d_dist, T* d_closest) {
    BVH_TRY(check_n("signed_distance", n));
    BVH_TRY(polygon_rule("signed_distance", rule));
    BVH_TRY(segments_check(tree, "signed_distance"));
    if (n == 0) return BVHGPU_OK;
    bvhgpu_ctx* ctx = tree->ctx;
    Scratch scratch(ctx);
    uint8_t* cls = nullptr;
    BVH_TRY(scratch.get(&cls, n));
    BVH_TRY(knn_seg_launch<T>(tree, d_points, n, 1, nullptr, d_shape, d_dist, d_closest));
    BVH_TRY(contains_launch(tree, d_points, n, rule, cls, (int32_t*)nullptr));
    polygon_sign_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>((uint32_t)n, cls, d_shape, d_dist);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}

template int set_segments<float>(Tree<float>*, const float*, size_t);
template int set_segments<double>(Tree<double>*, const double*, size_t);
template int polygon_contains_device<float>(Tree<float>*, const float*, size_t, int, uint8_t*, int32_t*);
template int polygon_contains_device<double>(Tree<double>*, const double*, size_t, int, uint8_t*, int32_t*);
template int knn_seg_device<float>(Tree<float>*, const float*, size_t, uint32_t, const float*, uint32_t*, float*, float*);
template int knn_seg_device<double>(Tree<double>*, const double*, size_t, uint32_t, const double*, uint32_t*, double*, double*);
template int polygon_distance_device<float>(Tree<float>*, const float*, size_t, int, uint32_t*, float*, float*);
template int polygon_distance_device<double>(Tree<double>*, const double*, size_t, int, uint32_t*, double*, double*);

}  // namespace bvhb200
