// bvh_b200/csrc/dim2.cu -- D = 2 instantiation of build / flatten / traverse (SURVEY.md 8f N4; the reference is generic in D and
// ships 2-D slab tests: src/ray/intersect_simd.rs:99-133 (f32), :181-191 (f64); default path src/ray/intersect_default.rs:16-37).
//
// A 2-D scene is run through the 3-D kernels embedded in the plane z = 0, which reproduces the 2-D arithmetic bit for bit:
//   build     every AABB gets z = [0, 0]: centres have z = 0, extents have z = 0, so largest_axis (first strict maximum,
//             aabb_impl.rs:594-596) never picks z; surface_area 2*((sx*sx + sy*sy) + 0) == 2*(sx*sx + sy*sy) exactly
//             (aabb_impl.rs:551-554 with a 2-term dot); buckets, costs and child boxes never see z.  Same topology, same boxes.
//   traverse  the traversal records (and the shape AABBs the FLAT leaf re-test reads) get z = [-1, +1]; rays get origin.z = 0 and
//             inv_direction.z = +inf: the z slab is (-1 - 0) * inf = -inf, (1 - 0) * inf = +inf -- never NaN, and max(tmin, -inf),
//             min(tmax, +inf) are identities, so the 3-D slab test returns exactly what the 2-D one does.
//   ordered   the distance-ordered traversal walks the same records with the same lifted rays (ordered_kernel<3, T>, csr.cuh).  The z
//             slab is (-inf, +inf) on every record (an empty child box has z = [+inf, -inf]: (+inf - 0) * inf = +inf and
//             (-inf - 0) * inf = -inf, again no NaN), z is the last axis of the fold, and max(tmin, -inf) / min(tmax, +inf) are
//             identities: the 3-D instance returns the 2-D set and the 2-D entry / exit distances bit for bit.
//   closest   does NOT lift: it slices the node boxes and the shape boxes, which have z = [0, 0], and (0 - 0) * inf = NaN would
//             reject every box.  closest_kernel<2, T> (closest.cu) walks the embedded 3-D nodes and d_aabb, tests x and y only, and
//             reads the 2-D rays (6 T) as they are.
//   queries   Aabb / Point / Ball records and nearest_to points are lifted to z = 0 (lift2_kernel) and run through the 3-D query and
//             nearest kernels.  Every z term is exactly neutral, so the results are the 2-D ones bit for bit:
//               - Aabb and Point tests pass on z: the records and the FLAT re-test boxes span z = [-1, +1] and contain 0.
//               - Ball: the centre's z = 0 clamps to itself, so the z difference is +0 and adds +0 to the sum of squares.
//               - Aabb::min_distance_squared on d_nodes / d_flat / d_aabb (z = [0, 0]): half size 0, centre 0, o_z = max(|0 - 0| - 0, 0)
//                 = 0; on an empty child box (z = [+inf, -inf]) the centre is NaN and o_z = 0 as well (NaN.max(0) = 0, as in Rust).
//               - the QUERY_WITHIN lower bound on a record: max(-1 - 0, 0 - 1) = -1 -> 0; the farthest-corner bound on a shape: |0 - 0| = 0.
//               - adding +0 to a non-negative sum is exact, and the squares are summed left to right, so z comes last.
//   knn       the k nearest shapes: points lifted to z = 0 (lift2_kernel, nvec = 1), knn_kernel<T, K> (traverse.cu) on the embedded
//             tree.  The keys are aabb_min_d2 of d_aabb (z = [0, 0]: o_z = 0, as above); the pruning bound box_lower_d2 of a node box
//             with z = [0, 0] has a z gap of max(0 - 0, 0 - 0) = 0 minus a positive slack, clamped to 0; empty child boxes fall under
//             the always-entered rule.  Every z term is +0 added last, so keys, bounds and rows are the 2-D ones bit for bit.
// The 2-D PODs are converted on the device (expand on the way in, drop z on the way out).
#include "internal.h"

namespace bvhb200 {

template <class T> __global__ void __launch_bounds__(256) expand_aabb2_kernel(const T* __restrict__ in /*4 per box*/, uint32_t n, T* __restrict__ out /*6 per box*/) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const T* p = in + 4 * (size_t)i;
    T* q = out + 6 * (size_t)i;
    q[0] = p[0]; q[1] = p[1]; q[2] = T(0); q[3] = p[2]; q[4] = p[3]; q[5] = T(0);
}
template <class T> __global__ void __launch_bounds__(256) expand_ray2_kernel(const T* __restrict__ in /*6 per ray*/, uint32_t n, T* __restrict__ out /*9 per ray*/) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const T* p = in + 6 * (size_t)i;
    T* q = out + 9 * (size_t)i;
    q[0] = p[0]; q[1] = p[1]; q[2] = T(0);
    q[3] = p[2]; q[4] = p[3]; q[5] = T(0);
    q[6] = p[4]; q[7] = p[5]; q[8] = Traits<T>::inf();
}
// shape AABBs for the FLAT leaf re-test of a 2-D tree: z = [-1, +1]
template <class T> __global__ void __launch_bounds__(256) trav_aabb2_kernel(const typename Traits<T>::DAabb* __restrict__ in, uint32_t n, typename Traits<T>::DAabb* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    typename Traits<T>::DAabb d = in[i];
    d.min[2] = T(-1); d.max[2] = T(1);
    out[i] = d;
}
template <class T, class N2> __global__ void __launch_bounds__(256) shrink_nodes_kernel(const typename Traits<T>::Node* __restrict__ in, uint32_t n, N2* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const typename Traits<T>::Node nd = in[i];
    N2 o;
    o.parent = nd.parent; o.child_l = nd.child_l; o.child_r = nd.child_r; o.shape = nd.shape;
    for (int k = 0; k < 2; ++k) { o.l_aabb.min[k] = nd.l_aabb.min[k]; o.l_aabb.max[k] = nd.l_aabb.max[k]; o.r_aabb.min[k] = nd.r_aabb.min[k]; o.r_aabb.max[k] = nd.r_aabb.max[k]; }
    out[i] = o;
}
template <class T, class F2> __global__ void __launch_bounds__(256) shrink_flat_kernel(const typename Traits<T>::Flat* __restrict__ in, size_t n, F2* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const typename Traits<T>::Flat f = in[i];
    F2 o;
    for (int k = 0; k < 2; ++k) { o.aabb.min[k] = f.aabb.min[k]; o.aabb.max[k] = f.aabb.max[k]; }
    o.entry_index = f.entry_index; o.exit_index = f.exit_index; o.shape_index = f.shape_index;
    out[i] = o;
}

// Query records and points lifted into the plane z = 0: every 2-vector of a record gets z = 0, trailing scalars are copied.
//   Aabb {min, max}: nvec = 2 (z = [0, 0]);  Point and nearest_to points: nvec = 1 (z = 0);  Ball {center, radius}: nvec = 1, nscal = 1.
template <class T> __global__ void __launch_bounds__(256) lift2_kernel(const T* __restrict__ in, uint32_t n, int nvec, int nscal, T* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const T* p = in + (size_t)(2 * nvec + nscal) * i;
    T* q = out + (size_t)(3 * nvec + nscal) * i;
    for (int v = 0; v < nvec; ++v) { q[3 * v] = p[2 * v]; q[3 * v + 1] = p[2 * v + 1]; q[3 * v + 2] = T(0); }
    for (int s = 0; s < nscal; ++s) q[3 * nvec + s] = p[2 * nvec + s];
}

template <class T> int dim2_expand_aabbs(bvhgpu_ctx* ctx, const T* d_in4, uint32_t n, T* d_out6) {
    expand_aabb2_kernel<T><<<(n + 255) / 256, 256, 0, ctx->stream>>>(d_in4, n, d_out6);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}
template <class T> int dim2_expand_rays(bvhgpu_ctx* ctx, const T* d_in6, uint32_t n, T* d_out9) {
    expand_ray2_kernel<T><<<(n + 255) / 256, 256, 0, ctx->stream>>>(d_in6, n, d_out9);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}
template <class T> int dim2_lift(bvhgpu_ctx* ctx, const T* d_in, uint32_t n, int nvec, int nscal, T* d_out) {
    lift2_kernel<T><<<(n + 255) / 256, 256, 0, ctx->stream>>>(d_in, n, nvec, nscal, d_out);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}
template <class T> int dim2_finish_build(Tree<T>* tree) {
    bvhgpu_ctx* ctx = tree->ctx;
    tree->dims = 2;
    if (tree->n == 0) return BVHGPU_OK;
    if (!tree->d_aabb_trav) BVH_TRY(dalloc_t(ctx, &tree->d_aabb_trav, tree->n));
    trav_aabb2_kernel<T><<<(tree->n + 255) / 256, 256, 0, ctx->stream>>>(tree->d_aabb, tree->n, tree->d_aabb_trav);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}
template <class T, class N2> int dim2_nodes_out(Tree<T>* tree, N2* d_out) {
    bvhgpu_ctx* ctx = tree->ctx;
    shrink_nodes_kernel<T, N2><<<(tree->n_nodes + 255) / 256, 256, 0, ctx->stream>>>(tree->d_nodes, tree->n_nodes, d_out);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}
template <class T, class F2> int dim2_flat_out(Tree<T>* tree, F2* d_out) {
    bvhgpu_ctx* ctx = tree->ctx;
    shrink_flat_kernel<T, F2><<<(unsigned)((tree->n_flat + 255) / 256), 256, 0, ctx->stream>>>(tree->d_flat, tree->n_flat, d_out);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}

template int dim2_expand_aabbs<float>(bvhgpu_ctx*, const float*, uint32_t, float*);
template int dim2_expand_aabbs<double>(bvhgpu_ctx*, const double*, uint32_t, double*);
template int dim2_expand_rays<float>(bvhgpu_ctx*, const float*, uint32_t, float*);
template int dim2_expand_rays<double>(bvhgpu_ctx*, const double*, uint32_t, double*);
template int dim2_lift<float>(bvhgpu_ctx*, const float*, uint32_t, int, int, float*);
template int dim2_lift<double>(bvhgpu_ctx*, const double*, uint32_t, int, int, double*);
template int dim2_finish_build<float>(Tree<float>*);
template int dim2_finish_build<double>(Tree<double>*);
template int dim2_nodes_out<float, bvh_node2f>(Tree<float>*, bvh_node2f*);
template int dim2_nodes_out<double, bvh_node2d>(Tree<double>*, bvh_node2d*);
template int dim2_flat_out<float, bvh_flat2f>(Tree<float>*, bvh_flat2f*);
template int dim2_flat_out<double, bvh_flat2d>(Tree<double>*, bvh_flat2d*);

}  // namespace bvhb200
