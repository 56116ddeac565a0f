// bvh_b200/csrc/closest.cu -- closest hit per ray with distance pruning (SURVEY.md 8f N3): the form a ray tracer needs.
//
// The reference gives its callers two things: the candidate set (Bvh::traverse, or the best-effort distance-ordered iterators of
// src/bvh/distance_traverse.rs / child_distance_traverse.rs) and the primitive test Ray::intersects_triangle
// (src/ray/ray_impl.rs:154-213); the closest hit is the caller's loop over both (src/bvh/iter.rs:330-365 does exactly that in its
// benchmark).  Here the loop runs on the device, front to back, and subtrees whose AABB is entered behind the best hit so far are
// never opened:
//   AABB mode      result = the shape whose AABB the ray enters first, key (entry distance, DFS order) -- i.e. the first element of a
//                  perfectly sorted nearest_traverse_iterator.  Entry distances are Ray::intersection_slice_for_aabb
//                  (src/ray/ray_impl.rs:118-145) bit for bit; pruning keeps ties (entry == best), so the result is EXACTLY the
//                  minimum over Bvh::traverse's candidates.
//   triangle mode  result = the triangle with the smallest Ray::intersects_triangle distance (Moeller-Trumbore with backface culling,
//                  same operation order, no FMA), ties to the lower shape index.  A subtree is skipped when its entry distance exceeds
//                  best * (1 + 2^-16): the slab distance and the Moeller-Trumbore distance are different roundings of the same
//                  quantity, so pruning at exactly `entry > best` could drop a hit that wins by an ulp.  The margin does not bound
//                  how far a grazing hit's rounded distance can fall in front of its own box (17 % was seen in f32), so the result
//                  G differs from the unpruned minimum W only where W's Moeller-Trumbore distance lies more than 2^-16 in front of
//                  the slab entry of W's own AABB; then d_W <= d_G, that entry exceeds fl(d_G * (1 + 2^-16)), and W's exact
//                  intersection lies behind d_G.  G's distance, u and v are always the reference's Moeller-Trumbore result for G.
// Any hit (ANY = true): the other loop callers write over the same two calls, traverse(..).iter().any(|s| distance < tmax) -- a
// shadow ray, a line of sight.  The same walk with a per-ray constant bound instead of best * margin: a child is entered while its entry
// is < tmax (AABB mode; exact, since slab entries are monotone under box containment and every stored box contains the boxes below
// it) or <= fl(tmax * (1 + 2^-16)) (triangle mode, the margin above), a leaf is accepted when its own box is entered before tmax /
// its Moeller-Trumbore distance is < tmax, and the first accepted leaf ends the walk.  Only out_shape is written.
// Dimensions: the AABB mode runs in D = 2, 3 and 4 (the same slab_slice over D axes, common.cuh); triangles are 3-D only.
// The walk needs no stack: nodes carry parent links, a lane remembers which child it comes back from and re-derives the near / far
// order from the node (same loads, same bits), so any tree depth works (the reference's iterators use a 32-slot stack / a heap).
// Multi hit (multi_hit_kernel): the first k hits along the ray, the same walk and ray loading with the sorted register list of the k
// nearest shapes (key_less / knn_insert of queries.cuh) in place of the one best hit; see the comment above the kernel.
#include "internal.h"
#include "csr.cuh"
#include "queries.cuh"

namespace bvhb200 {

template <class T> __device__ __forceinline__ void cross_rn(const T a[3], const T b[3], T o[3]) {       // nalgebra 3-D cross
    o[0] = sub_rn(mul_rn(a[1], b[2]), mul_rn(a[2], b[1]));
    o[1] = sub_rn(mul_rn(a[2], b[0]), mul_rn(a[0], b[2]));
    o[2] = sub_rn(mul_rn(a[0], b[1]), mul_rn(a[1], b[0]));
}
template <class T> __device__ __forceinline__ T dot_rn(const T a[3], const T b[3]) { return add_rn(add_rn(mul_rn(a[0], b[0]), mul_rn(a[1], b[1])), mul_rn(a[2], b[2])); }

// Ray::intersects_triangle (src/ray/ray_impl.rs:154-213).  Returns the distance (+inf: miss / back face / behind the origin).
template <class T>
__device__ __forceinline__ T moeller_trumbore(const T o[3], const T dir[3], const T a[3], const T b[3], const T c[3], T& u_out, T& v_out) {
    const T INF = Traits<T>::inf(), EPS = Traits<T>::eps();
    T ab[3], ac[3], uvec[3], ao[3], vvec[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { ab[k] = sub_rn(b[k], a[k]); ac[k] = sub_rn(c[k], a[k]); }
    cross_rn(dir, ac, uvec);
    const T det = dot_rn(ab, uvec);
    u_out = T(0); v_out = T(0);
    if (det < EPS) return INF;
    const T inv_det = div_rn(T(1), det);
#pragma unroll
    for (int k = 0; k < 3; ++k) ao[k] = sub_rn(o[k], a[k]);
    const T u = mul_rn(dot_rn(ao, uvec), inv_det);
    u_out = u;
    if (!(u >= T(0) && u <= T(1))) return INF;
    cross_rn(ao, ab, vvec);
    const T v = mul_rn(dot_rn(dir, vvec), inv_det);
    v_out = v;
    if (v < T(0) || add_rn(u, v) > T(1)) return INF;
    const T dist = mul_rn(dot_rn(ac, vvec), inv_det);
    return dist > EPS ? dist : INF;
}

// Both windings of one triangle for the crossing counts: moeller_trumbore as it is, then the same function with b and c exchanged
// (the back-face test).  Each counts when its distance is < tmax (+inf without a limit: finite).
template <class T>
__device__ __forceinline__ void count_windings(const T o[3], const T dir[3], const T a[3], const T b[3], const T c[3], T tmax,
                                               uint32_t& front, uint32_t& back) {
    T u, v;
    front += moeller_trumbore(o, dir, a, b, c, u, v) < tmax ? 1u : 0u;
    back += moeller_trumbore(o, dir, a, c, b, u, v) < tmax ? 1u : 0u;
}

template <class T>
__global__ void __launch_bounds__(256) pack_tris_kernel(const T* __restrict__ tris9, uint32_t n, DTri<T>* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    DTri<T> t;
    const T* p = tris9 + 9 * (size_t)i;
#pragma unroll
    for (int k = 0; k < 3; ++k) { t.a[k] = p[k]; t.b[k] = p[3 + k]; t.c[k] = p[6 + k]; }
    t.pa = t.pb = t.pc = T(0);
    out[i] = t;
}

template <class T>
__global__ void __launch_bounds__(256) fill_nohit_kernel(uint32_t n, uint32_t* __restrict__ shape, T* __restrict__ dist, T* __restrict__ uv) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    shape[i] = BVH_INVALID; dist[i] = Traits<T>::inf();
    if (uv) { uv[2 * (size_t)i] = T(0); uv[2 * (size_t)i + 1] = T(0); }
}

// The walk tests D axes of the boxes.  D = 3: the 3-D tree, rays of 9 T (origin, direction, inv_direction) or 6 T (origin,
// direction).  D = 4: a Tree4's bvh_node4* and ABI boxes, rays of 12 T.  D = 2: the 3-D nodes and boxes a 2-D tree is embedded in
// (z = [0, 0]), of which only x and y are tested, and the 2-D rays of 6 T as they are.  The lift that serves the other 2-D walks does
// not work here: on z = [0, 0] the z slab would be (0 - 0) * inf = NaN and reject every box.  Triangles: D = 3 only.
// (node and box types: ClosestLayout, internal.h)

template <int D, class T, bool TRI, bool ANY = false>
__global__ void __launch_bounds__(128) closest_kernel(const typename ClosestLayout<D, T>::Node* __restrict__ nodes, uint32_t n_shapes,
                                                      const typename ClosestLayout<D, T>::Box* __restrict__ aabb, const DTri<T>* __restrict__ tris,
                                                      const T* __restrict__ rays, uint32_t ray_stride, uint32_t nrays,
                                                      uint32_t* __restrict__ out_shape, T* __restrict__ out_dist, T* __restrict__ out_uv,
                                                      const T* __restrict__ ray_tmax) {
    static_assert(!TRI || D == 3, "Ray::intersects_triangle is 3-D only");
    constexpr int BD = D == 4 ? 4 : 3;                         // components of the stored boxes
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nrays) return;
    T o[D], dir[D], inv[D];
    {
        const T* p = rays + (size_t)ray_stride * r;
        const bool full = D != 3 || ray_stride == 9;           // only D = 3 has the compact {origin, direction} layout
#pragma unroll
        for (int k = 0; k < D; ++k) { o[k] = __ldg(p + k); dir[k] = __ldg(p + D + k); inv[k] = full ? __ldg(p + 2 * D + k) : div_rn(T(1), dir[k]); }
    }
    const T INF = Traits<T>::inf();
    const T margin = TRI ? add_rn(T(1), T(1.0 / 65536.0)) : T(1);
    uint32_t best = BVH_INVALID, best_key = BVH_INVALID;
    T best_d = INF, bu = T(0), bv = T(0);
    // any hit: a leaf is accepted when its distance is < tmax; children are entered while entry < tmax (AABB mode) or
    // entry <= fl(tmax * (1 + 2^-16)) (triangle mode), a per-ray constant instead of best * margin
    T tmax = INF, any_bound = INF;
    if constexpr (ANY) {
        if (ray_tmax) tmax = __ldg(ray_tmax + r);
        any_bound = mul_rn(tmax, margin);
    }

    auto leaf = [&](uint32_t shape, uint32_t node_idx) {
        if constexpr (ANY) {
            if constexpr (TRI) {
                const DTri<T>& t = tris[shape];
                T a[3], b[3], c[3];
#pragma unroll
                for (int k = 0; k < 3; ++k) { a[k] = __ldg(&t.a[k]); b[k] = __ldg(&t.b[k]); c[k] = __ldg(&t.c[k]); }
                T u, v;
                if (moeller_trumbore(o, dir, a, b, c, u, v) < tmax) best = shape;
            } else {
                T mn[BD], mx[BD], e, x;
                load_box(aabb + shape, mn, mx);
                if (slab_slice<D, T>(o, inv, mn, mx, e, x) && e < tmax) best = shape;
            }
        } else if constexpr (TRI) {
            const DTri<T>& t = tris[shape];
            T a[3], b[3], c[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) { a[k] = __ldg(&t.a[k]); b[k] = __ldg(&t.b[k]); c[k] = __ldg(&t.c[k]); }
            T u, v;
            const T d = moeller_trumbore(o, dir, a, b, c, u, v);
            if (d < best_d || (d == best_d && d < INF && shape < best)) { best = shape; best_d = d; bu = u; bv = v; }
        } else {
            T mn[BD], mx[BD], e, x;
            load_box(aabb + shape, mn, mx);
            if (slab_slice<D, T>(o, inv, mn, mx, e, x)) {
                if (best == BVH_INVALID || e < best_d || (e == best_d && node_idx < best_key)) { best = shape; best_d = e; best_key = node_idx; }
            }
        }
    };

    if (n_shapes == 1) {                                       // root leaf (bvh_node.rs:314 tests the shape's own AABB)
        T mn[BD], mx[BD], e, x;
        load_box(aabb + nodes[0].shape, mn, mx);
        if (slab_slice<D, T>(o, inv, mn, mx, e, x)) leaf(nodes[0].shape, 0u);
    } else {
        uint32_t node = 0, from = BVH_INVALID;                  // from: the child we are coming back from (BVH_INVALID: arriving from the parent)
        for (;;) {
            const uint4 meta = __ldg(reinterpret_cast<const uint4*>(nodes + node));      // parent, child_l, child_r, shape / count
            if (meta.y == BVH_INVALID) {
                leaf(meta.w, node);
                if constexpr (ANY) {
                    if (best != BVH_INVALID) break;             // any hit: the first accepted leaf ends the walk
                }
                from = node; node = meta.x;
                continue;
            }
            const typename ClosestLayout<D, T>::Node& nd = nodes[node];
            T lmn[D], lmx[D], rmn[D], rmx[D], el, er, x;
#pragma unroll
            for (int k = 0; k < D; ++k) { lmn[k] = __ldg(&nd.l_aabb.min[k]); lmx[k] = __ldg(&nd.l_aabb.max[k]); rmn[k] = __ldg(&nd.r_aabb.min[k]); rmx[k] = __ldg(&nd.r_aabb.max[k]); }
            const bool hl = slab_slice<D, T>(o, inv, lmn, lmx, el, x), hr = slab_slice<D, T>(o, inv, rmn, rmx, er, x);
            if (!hl) el = INF;
            if (!hr) er = INF;
            const bool left_first = el <= er;                   // front to back; ties: left (DFS order)
            const uint32_t near_i = left_first ? meta.y : meta.z, far_i = left_first ? meta.z : meta.y;
            const T near_e = left_first ? el : er, far_e = left_first ? er : el;
            const bool near_ok = left_first ? hl : hr, far_ok = left_first ? hr : hl;
            uint32_t next = BVH_INVALID;
            if constexpr (ANY) {
                // AABB mode: entry < tmax, exact (a box entered at or beyond tmax holds no accepted leaf); triangles: the margin
                const bool near_in = near_ok && (TRI ? near_e <= any_bound : near_e < tmax);
                const bool far_in = far_ok && (TRI ? far_e <= any_bound : far_e < tmax);
                if (from == BVH_INVALID) {
                    if (near_in) next = near_i;
                    else from = near_i;
                }
                if (next == BVH_INVALID && from == near_i) {
                    if (far_in) next = far_i;
                    else from = far_i;
                }
            } else {
                const T bound = mul_rn(best_d, margin);             // inf stays inf
                if (from == BVH_INVALID) {
                    if (near_ok && near_e <= bound) next = near_i;
                    else from = near_i;                             // skipped: as if we had just come back from it
                }
                if (next == BVH_INVALID && from == near_i) {
                    if (far_ok && far_e <= bound) next = far_i;
                    else from = far_i;
                }
            }
            if (next != BVH_INVALID) { node = next; from = BVH_INVALID; continue; }
            if (node == 0) break;                               // back from the far child of the root
            from = node; node = meta.x;
        }
    }
    out_shape[r] = best;
    if constexpr (!ANY) {
        out_dist[r] = best_d;
        if (out_uv) { out_uv[2 * (size_t)r] = bu; out_uv[2 * (size_t)r + 1] = bv; }
    }
}

template <class T>
int set_triangles(Tree<T>* tree, const T* tris9, size_t n, bool dev_input) {
    bvhgpu_ctx* ctx = tree->ctx;
    if (n != tree->n) { set_error("set_triangles: %zu triangles for a tree over %u shapes", n, tree->n); return BVHGPU_ERR_INVALID; }
    if (n == 0) return BVHGPU_OK;
    Scratch scratch(ctx);
    const T* d_in = tris9;
    if (!dev_input) {
        T* staged = nullptr;
        BVH_TRY(scratch.get(&staged, 9 * n));
        BVH_CUDA_TRY(cudaMemcpyAsync(staged, tris9, sizeof(T) * 9 * n, cudaMemcpyHostToDevice, ctx->stream));
        d_in = staged;
    }
    if (!tree->d_tris) BVH_TRY(dalloc(ctx, &tree->d_tris, sizeof(DTri<T>) * n));
    pack_tris_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(d_in, (uint32_t)n, reinterpret_cast<DTri<T>*>(tree->d_tris));
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    if (!dev_input) BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));       // the caller's buffer may go away
    return BVHGPU_OK;
}

template <class T>
int closest_hit_device(Tree<T>* tree, const void* d_rays, uint32_t fmt, size_t nrays, int use_triangles, uint32_t* d_shape, T* d_dist, T* d_uv) {
    bvhgpu_ctx* ctx = tree->ctx;
    cudaStream_t st = ctx->stream;
    if (nrays > 0x7FFFFFFFull) { set_error("closest_hit: too many rays"); return BVHGPU_ERR_INVALID; }
    if (fmt != BVHGPU_RAYS_FULL && fmt != BVHGPU_RAYS_OD) { set_error("closest_hit: bad ray layout %u", fmt); return BVHGPU_ERR_INVALID; }
    if (nrays == 0) return BVHGPU_OK;
    BVH_TRY(resolve_status(tree));
    if (tree->n == 0) {                                         // empty tree: no hit
        fill_nohit_kernel<T><<<(unsigned)((nrays + 255) / 256), 256, 0, st>>>((uint32_t)nrays, d_shape, d_dist, d_uv);
        ctx->launches++;
        BVH_CUDA_TRY(cudaGetLastError());
        return BVHGPU_OK;
    }
    if (use_triangles && !tree->d_tris) { set_error("closest_hit: triangle mode needs bvhgpu_tree_set_triangles_* first"); return BVHGPU_ERR_INVALID; }
    const unsigned grid = (unsigned)((nrays + 127) / 128);
    const uint32_t stride = fmt == BVHGPU_RAYS_FULL ? 9u : 6u;
    if (use_triangles)
        closest_kernel<3, T, true><<<grid, 128, 0, st>>>(tree->d_nodes, tree->n, tree->d_aabb, reinterpret_cast<const DTri<T>*>(tree->d_tris), reinterpret_cast<const T*>(d_rays), stride, (uint32_t)nrays, d_shape, d_dist, d_uv, nullptr);
    else
        closest_kernel<3, T, false><<<grid, 128, 0, st>>>(tree->d_nodes, tree->n, tree->d_aabb, nullptr, reinterpret_cast<const T*>(d_rays), stride, (uint32_t)nrays, d_shape, d_dist, d_uv, nullptr);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}

template <int D, class T>
int closest_aabb_device(bvhgpu_ctx* ctx, const typename ClosestLayout<D, T>::Node* nodes, uint32_t n_shapes, const typename ClosestLayout<D, T>::Box* aabb,
                        const T* d_rays, size_t nrays, uint32_t* d_shape, T* d_dist) {
    cudaStream_t st = ctx->stream;
    if (nrays == 0) return BVHGPU_OK;
    if (n_shapes == 0) fill_nohit_kernel<T><<<(unsigned)((nrays + 255) / 256), 256, 0, st>>>((uint32_t)nrays, d_shape, d_dist, nullptr);
    else closest_kernel<D, T, false><<<(unsigned)((nrays + 127) / 128), 128, 0, st>>>(nodes, n_shapes, aabb, nullptr, d_rays, 3 * D, (uint32_t)nrays, d_shape, d_dist, nullptr, nullptr);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}

// Any hit (bvhgpu_any_hit_*): closest_kernel<D, T, TRI, true>, one ray per thread, out_shape only.  d_tmax: nrays limits or
// nullptr (+inf for every ray).  An empty tree reports no hit for every ray (BVH_INVALID bytes, no kernel).
template <class T>
int any_hit_device(Tree<T>* tree, const void* d_rays, uint32_t fmt, size_t nrays, const T* d_tmax, int use_triangles, uint32_t* d_shape) {
    bvhgpu_ctx* ctx = tree->ctx;
    cudaStream_t st = ctx->stream;
    if (nrays > 0x7FFFFFFFull) { set_error("any_hit: too many rays"); return BVHGPU_ERR_INVALID; }
    if (fmt != BVHGPU_RAYS_FULL && fmt != BVHGPU_RAYS_OD) { set_error("any_hit: bad ray layout %u", fmt); return BVHGPU_ERR_INVALID; }
    if (nrays == 0) return BVHGPU_OK;
    BVH_TRY(resolve_status(tree));
    if (tree->n == 0) {
        BVH_CUDA_TRY(cudaMemsetAsync(d_shape, 0xFF, sizeof(uint32_t) * nrays, st));
        return BVHGPU_OK;
    }
    if (use_triangles && !tree->d_tris) { set_error("any_hit: triangle mode needs bvhgpu_tree_set_triangles_* first"); return BVHGPU_ERR_INVALID; }
    const unsigned grid = (unsigned)((nrays + 127) / 128);
    const uint32_t stride = fmt == BVHGPU_RAYS_FULL ? 9u : 6u;
    if (use_triangles)
        closest_kernel<3, T, true, true><<<grid, 128, 0, st>>>(tree->d_nodes, tree->n, tree->d_aabb, reinterpret_cast<const DTri<T>*>(tree->d_tris), reinterpret_cast<const T*>(d_rays), stride, (uint32_t)nrays, d_shape, nullptr, nullptr, d_tmax);
    else
        closest_kernel<3, T, false, true><<<grid, 128, 0, st>>>(tree->d_nodes, tree->n, tree->d_aabb, nullptr, reinterpret_cast<const T*>(d_rays), stride, (uint32_t)nrays, d_shape, nullptr, nullptr, d_tmax);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}

template <int D, class T>
int any_hit_aabb_device(bvhgpu_ctx* ctx, const typename ClosestLayout<D, T>::Node* nodes, uint32_t n_shapes, const typename ClosestLayout<D, T>::Box* aabb,
                        const T* d_rays, size_t nrays, const T* d_tmax, uint32_t* d_shape) {
    cudaStream_t st = ctx->stream;
    if (nrays == 0) return BVHGPU_OK;
    if (n_shapes == 0) {
        BVH_CUDA_TRY(cudaMemsetAsync(d_shape, 0xFF, sizeof(uint32_t) * nrays, st));
        return BVHGPU_OK;
    }
    closest_kernel<D, T, false, true><<<(unsigned)((nrays + 127) / 128), 128, 0, st>>>(nodes, n_shapes, aabb, nullptr, d_rays, 3 * D, (uint32_t)nrays, d_shape, nullptr, nullptr, d_tmax);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}

// ---- multi hit (bvhgpu_multi_hit_*): the first k hits along each ray, one ray per thread ----
// The walk, the near / far order and the ray loading are closest_kernel's.  The one best hit becomes the K-slot list of knn_walk
// (queries.cuh): sorted DESCENDING, slots 0 .. k-1 start as (+inf, BVH_INVALID), slots k .. K-1 hold (-inf, BVH_INVALID) sentinels, so
// (d[0], s[0]) is the current k-th key and every index is a compile-time constant.  Keys, in key_less order:
//   AABB mode      (entry of the shape's own box, the leaf's node index): the DFS tie rule of closest_kernel.  The list holds node
//                  indices; they are mapped to shapes when the row is written.  A leaf qualifies when its own box passes the slab test
//                  (and, with a limit, entry < tmax).  A child is entered when its slab test passes, its entry <= d[0] (ties entered)
//                  and, with a limit, its entry < tmax: exact, since slab entries are monotone under box containment.
//   triangle mode  (Moeller-Trumbore distance, shape): a triangle qualifies when its distance is < tmax (+inf without a limit, so a
//                  miss never qualifies).  A child is entered when its slab test passes and entry <= fl(d[0] * (1 + 2^-16)) and
//                  entry <= fl(tmax * (1 + 2^-16)): closest_kernel's and the any-hit walk's margins.  u and v are recomputed for the
//                  k final triangles after the walk (the same function on the same inputs), so the list carries only (key, id).
// With k = 1 and no limit the bounds are closest_kernel's, so the row is closest_hit's; while the list is empty they are the any-hit
// walk's, so a row is empty exactly where any_hit reports no hit.  Rows start at (size_t)r * k: n * k passes 2^32 from n = 2^26.
template <int D, class T, bool TRI, int K>
__global__ void __launch_bounds__(128) multi_hit_kernel(const typename ClosestLayout<D, T>::Node* __restrict__ nodes, uint32_t n_shapes,
                                                        const typename ClosestLayout<D, T>::Box* __restrict__ aabb, const DTri<T>* __restrict__ tris,
                                                        const T* __restrict__ rays, uint32_t ray_stride, uint32_t nrays, uint32_t k,
                                                        const T* __restrict__ ray_tmax, uint32_t* __restrict__ out_shape, T* __restrict__ out_dist,
                                                        T* __restrict__ out_uv) {
    static_assert(!TRI || D == 3, "Ray::intersects_triangle is 3-D only");
    constexpr int BD = D == 4 ? 4 : 3;
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nrays) return;
    T o[D], dir[D], inv[D];
    {
        const T* p = rays + (size_t)ray_stride * r;
        const bool full = D != 3 || ray_stride == 9;
#pragma unroll
        for (int c = 0; c < D; ++c) { o[c] = __ldg(p + c); dir[c] = __ldg(p + D + c); inv[c] = full ? __ldg(p + 2 * D + c) : div_rn(T(1), dir[c]); }
    }
    const T INF = Traits<T>::inf();
    const T margin = TRI ? add_rn(T(1), T(1.0 / 65536.0)) : T(1);
    const bool has_limit = ray_tmax != nullptr;
    const T tmax = has_limit ? __ldg(ray_tmax + r) : INF;
    const T tmax_bound = mul_rn(tmax, margin);                  // triangle mode; inf stays inf, NaN stays NaN
    T d[K];
    uint32_t s[K];
#pragma unroll
    for (int j = 0; j < K; ++j) { d[j] = j < (int)k ? INF : -INF; s[j] = BVH_INVALID; }

    auto leaf = [&](uint32_t shape, uint32_t node_idx) {
        T key;
        uint32_t id;
        bool ok;
        if constexpr (TRI) {
            const DTri<T>& t = tris[shape];
            T a[3], b[3], c[3];
#pragma unroll
            for (int q = 0; q < 3; ++q) { a[q] = __ldg(&t.a[q]); b[q] = __ldg(&t.b[q]); c[q] = __ldg(&t.c[q]); }
            T u, v;
            key = moeller_trumbore(o, dir, a, b, c, u, v);
            id = shape;
            ok = key < tmax;
        } else {
            T mn[BD], mx[BD], x;
            load_box(aabb + shape, mn, mx);
            ok = slab_slice<D, T>(o, inv, mn, mx, key, x) && (!has_limit || key < tmax);
            id = node_idx;
        }
        if (ok && key_less(key, id, d[0], s[0])) knn_insert(d, s, key, id);
    };
    auto enter = [&](bool hit, T e) {
        if constexpr (TRI) return hit && e <= mul_rn(d[0], margin) && e <= tmax_bound;
        else return hit && e <= d[0] && (!has_limit || e < tmax);
    };

    if (n_shapes == 1) {                                       // root leaf (bvh_node.rs:314 tests the shape's own AABB)
        T mn[BD], mx[BD], e, x;
        load_box(aabb + nodes[0].shape, mn, mx);
        if (slab_slice<D, T>(o, inv, mn, mx, e, x)) leaf(nodes[0].shape, 0u);
    } else {
        uint32_t node = 0, from = BVH_INVALID;
        for (;;) {
            const uint4 meta = __ldg(reinterpret_cast<const uint4*>(nodes + node));      // parent, child_l, child_r, shape / count
            if (meta.y == BVH_INVALID) {
                leaf(meta.w, node);
                from = node; node = meta.x;
                continue;
            }
            const typename ClosestLayout<D, T>::Node& nd = nodes[node];
            T lmn[D], lmx[D], rmn[D], rmx[D], el, er, x;
#pragma unroll
            for (int c = 0; c < D; ++c) { lmn[c] = __ldg(&nd.l_aabb.min[c]); lmx[c] = __ldg(&nd.l_aabb.max[c]); rmn[c] = __ldg(&nd.r_aabb.min[c]); rmx[c] = __ldg(&nd.r_aabb.max[c]); }
            const bool hl = slab_slice<D, T>(o, inv, lmn, lmx, el, x), hr = slab_slice<D, T>(o, inv, rmn, rmx, er, x);
            if (!hl) el = INF;
            if (!hr) er = INF;
            const bool left_first = el <= er;
            const uint32_t near_i = left_first ? meta.y : meta.z, far_i = left_first ? meta.z : meta.y;
            const T near_e = left_first ? el : er, far_e = left_first ? er : el;
            const bool near_ok = left_first ? hl : hr, far_ok = left_first ? hr : hl;
            uint32_t next = BVH_INVALID;
            if (from == BVH_INVALID) {
                if (enter(near_ok, near_e)) next = near_i;
                else from = near_i;                             // skipped: as if we had just come back from it
            }
            if (next == BVH_INVALID && from == near_i) {        // the far child, against the k-th key as it is now
                if (enter(far_ok, far_e)) next = far_i;
                else from = far_i;
            }
            if (next != BVH_INVALID) { node = next; from = BVH_INVALID; continue; }
            if (node == 0) break;
            from = node; node = meta.x;
        }
    }
    const size_t base = (size_t)r * k;
#pragma unroll
    for (int j = 0; j < K; ++j)
        if (j < (int)k) { out_shape[base + k - 1 - j] = s[j]; out_dist[base + k - 1 - j] = d[j]; }
    // node indices -> shapes, and u, v, in loops of their own after the list is dead (no spills, one call site of moeller_trumbore)
#pragma unroll 1
    for (uint32_t j = 0; j < k; ++j) {
        const uint32_t id = out_shape[base + j];
        T u = T(0), v = T(0);
        if constexpr (TRI) {
            if (id != BVH_INVALID && out_uv) {
                const DTri<T>& t = tris[id];
                T a[3], b[3], c[3];
#pragma unroll
                for (int q = 0; q < 3; ++q) { a[q] = __ldg(&t.a[q]); b[q] = __ldg(&t.b[q]); c[q] = __ldg(&t.c[q]); }
                moeller_trumbore(o, dir, a, b, c, u, v);
            }
        } else if (id != BVH_INVALID) {
            out_shape[base + j] = __ldg(&reinterpret_cast<const uint4*>(nodes + id)->w);
        }
        if (out_uv) { out_uv[2 * (base + j)] = u; out_uv[2 * (base + j) + 1] = v; }
    }
}

template <class T>
__global__ void __launch_bounds__(256) fill_multi_pad_kernel(size_t n, uint32_t* __restrict__ shape, T* __restrict__ dist, T* __restrict__ uv) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        shape[i] = BVH_INVALID; dist[i] = Traits<T>::inf();
        if (uv) { uv[2 * i] = T(0); uv[2 * i + 1] = T(0); }
    }
}

// One launch of multi_hit_kernel in the K bucket of k (knn_bucket), or rows of padding for an empty tree.
template <int D, class T, bool TRI>
static int multi_hit_launch(bvhgpu_ctx* ctx, const typename ClosestLayout<D, T>::Node* nodes, uint32_t n_shapes, const typename ClosestLayout<D, T>::Box* aabb,
                            const DTri<T>* tris, const T* d_rays, uint32_t stride, size_t nrays, uint32_t k, const T* d_tmax, uint32_t* d_shape,
                            T* d_dist, T* d_uv) {
    cudaStream_t st = ctx->stream;
    if (n_shapes == 0) {
        const size_t slots = nrays * k;
        fill_multi_pad_kernel<T><<<(unsigned)std::min<size_t>((slots + 255) / 256, 65535), 256, 0, st>>>(slots, d_shape, d_dist, d_uv);
    } else {
        const unsigned grid = (unsigned)((nrays + 127) / 128);
        knn_bucket(k, [&](auto kb) {
            multi_hit_kernel<D, T, TRI, decltype(kb)::value><<<grid, 128, 0, st>>>(nodes, n_shapes, aabb, tris, d_rays, stride, (uint32_t)nrays, k, d_tmax,
                                                                              d_shape, d_dist, d_uv);
        });
    }
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}

template <class T>
int multi_hit_device(Tree<T>* tree, const void* d_rays, uint32_t fmt, size_t nrays, uint32_t k, const T* d_tmax, int use_triangles,
                     uint32_t* d_shape, T* d_dist, T* d_uv) {
    if (nrays > 0x7FFFFFFFull) { set_error("multi_hit: too many rays"); return BVHGPU_ERR_INVALID; }
    if (fmt != BVHGPU_RAYS_FULL && fmt != BVHGPU_RAYS_OD) { set_error("multi_hit: bad ray layout %u", fmt); return BVHGPU_ERR_INVALID; }
    if (nrays == 0) return BVHGPU_OK;
    BVH_TRY(resolve_status(tree));
    if (use_triangles && tree->n && !tree->d_tris) { set_error("multi_hit: triangle mode needs bvhgpu_tree_set_triangles_* first"); return BVHGPU_ERR_INVALID; }
    const uint32_t stride = fmt == BVHGPU_RAYS_FULL ? 9u : 6u;
    const T* rays = reinterpret_cast<const T*>(d_rays);
    if (use_triangles)
        return multi_hit_launch<3, T, true>(tree->ctx, tree->d_nodes, tree->n, tree->d_aabb, reinterpret_cast<const DTri<T>*>(tree->d_tris), rays, stride,
                                            nrays, k, d_tmax, d_shape, d_dist, d_uv);
    return multi_hit_launch<3, T, false>(tree->ctx, tree->d_nodes, tree->n, tree->d_aabb, nullptr, rays, stride, nrays, k, d_tmax, d_shape, d_dist, d_uv);
}

template <int D, class T>
int multi_hit_aabb_device(bvhgpu_ctx* ctx, const typename ClosestLayout<D, T>::Node* nodes, uint32_t n_shapes, const typename ClosestLayout<D, T>::Box* aabb,
                          const T* d_rays, size_t nrays, uint32_t k, const T* d_tmax, uint32_t* d_shape, T* d_dist) {
    if (nrays == 0) return BVHGPU_OK;
    return multi_hit_launch<D, T, false>(ctx, nodes, n_shapes, aabb, nullptr, d_rays, 3 * D, nrays, k, d_tmax, d_shape, d_dist, nullptr);
}

// ---- crossing counts (bvhgpu_count_hits_*), point-in-mesh (bvhgpu_contains_points_*) and the sign of bvhgpu_signed_distance_* ----
// Per ray: front = #shapes of Bvh::traverse's set whose moeller_trumbore(o, d, a, b, c) is < tmax, back = the same with b and c
// exchanged (count_windings).  The walk is closest_kernel's stackless parent-link walk, ray loading and slab test, without a near / far
// order: the left child is judged first, the right one when the walk comes back from the left, and a child is entered when its slab
// test passes and its entry <= fl(tmax * (1 + 2^-16)), the any-hit walk's triangle margin (+inf without a limit: every child whose slab
// test passes, i.e. exactly Bvh::traverse's set).  Only the judged child's box is loaded.  A root leaf (n = 1) tests the shape's own box.
template <class T> __device__ __forceinline__ T crossings_sqrt(T x);
template <> __device__ __forceinline__ float crossings_sqrt(float x) { return __fsqrt_rn(x); }
template <> __device__ __forceinline__ double crossings_sqrt(double x) { return __dsqrt_rn(x); }

template <class T>
__device__ __forceinline__ void crossings_walk(const typename Traits<T>::Node* __restrict__ nodes, uint32_t n_shapes,
                                               const typename Traits<T>::DAabb* __restrict__ aabb, const DTri<T>* __restrict__ tris,
                                               const T o[3], const T dir[3], const T inv[3], T tmax, uint32_t& front, uint32_t& back) {
    const T bound = mul_rn(tmax, add_rn(T(1), T(1.0 / 65536.0)));      // inf stays inf, NaN stays NaN (nothing is entered)
    auto leaf = [&](uint32_t shape) {
        const DTri<T>& t = tris[shape];
        T a[3], b[3], c[3];
#pragma unroll
        for (int q = 0; q < 3; ++q) { a[q] = __ldg(&t.a[q]); b[q] = __ldg(&t.b[q]); c[q] = __ldg(&t.c[q]); }
        count_windings(o, dir, a, b, c, tmax, front, back);
    };
    auto enter = [&](const typename Traits<T>::Aabb& box) {
        T mn[3], mx[3], e, x;
#pragma unroll
        for (int q = 0; q < 3; ++q) { mn[q] = __ldg(&box.min[q]); mx[q] = __ldg(&box.max[q]); }
        return slab_slice<3, T>(o, inv, mn, mx, e, x) && e <= bound;
    };
    if (n_shapes == 1) {                                       // root leaf (bvh_node.rs:314 tests the shape's own AABB)
        T mn[3], mx[3], e, x;
        load_box(aabb + nodes[0].shape, mn, mx);
        if (slab_slice<3, T>(o, inv, mn, mx, e, x)) leaf(nodes[0].shape);
        return;
    }
    uint32_t node = 0, from = BVH_INVALID;                      // from: the child we are coming back from (BVH_INVALID: from the parent)
    for (;;) {
        const uint4 meta = __ldg(reinterpret_cast<const uint4*>(nodes + node));      // parent, child_l, child_r, shape / count
        if (meta.y == BVH_INVALID) {
            leaf(meta.w);
            from = node; node = meta.x;
            continue;
        }
        const typename Traits<T>::Node& nd = nodes[node];
        uint32_t next = BVH_INVALID;
        if (from == BVH_INVALID) {
            if (enter(nd.l_aabb)) next = meta.y;
            else from = meta.y;                                 // skipped: as if we had just come back from it
        }
        if (next == BVH_INVALID && from == meta.y) {
            if (enter(nd.r_aabb)) next = meta.z;
            else from = meta.z;
        }
        if (next != BVH_INVALID) { node = next; from = BVH_INVALID; continue; }
        if (node == 0) break;                                   // back from the right child of the root
        from = node; node = meta.x;
    }
}

// FROM_POINTS = false: one ray per thread, FULL (9 T) or OD (6 T) rays, ray_tmax nrays limits or nullptr; writes out_front / out_back.
// FROM_POINTS = true: one POINT per thread (3 T each); the three rays Ray::new(p, BVHGPU_CONTAINS_DIRECTIONS[j]) are built in registers
// with rays_new_kernel's arithmetic and walked one after the other without a limit, so neighbouring threads walk neighbouring points in
// the same direction at the same time and the vote needs no scratch.  out_inside[i] = 1 when at least two of the three rays vote inside
// (rule EVEN_ODD: front + back odd; NONZERO: back != front).
template <class T, bool FROM_POINTS>
__global__ void __launch_bounds__(128) crossings_kernel(const typename Traits<T>::Node* __restrict__ nodes, uint32_t n_shapes,
                                                        const typename Traits<T>::DAabb* __restrict__ aabb, const DTri<T>* __restrict__ tris,
                                                        const T* __restrict__ in, uint32_t ray_stride, uint32_t n, const T* __restrict__ ray_tmax,
                                                        uint32_t* __restrict__ out_front, uint32_t* __restrict__ out_back, int rule,
                                                        uint8_t* __restrict__ out_inside) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if constexpr (!FROM_POINTS) {
        T o[3], dir[3], inv[3];
        const T* p = in + (size_t)ray_stride * i;
        const bool full = ray_stride == 9;
#pragma unroll
        for (int k = 0; k < 3; ++k) { o[k] = __ldg(p + k); dir[k] = __ldg(p + 3 + k); inv[k] = full ? __ldg(p + 6 + k) : div_rn(T(1), dir[k]); }
        uint32_t front = 0, back = 0;
        crossings_walk<T>(nodes, n_shapes, aabb, tris, o, dir, inv, ray_tmax ? __ldg(ray_tmax + i) : Traits<T>::inf(), front, back);
        out_front[i] = front;
        out_back[i] = back;
    } else {
        constexpr double DIRS[3][3] = BVHGPU_CONTAINS_DIRECTIONS;
        T o[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) o[k] = __ldg(in + 3 * (size_t)i + k);
        uint32_t votes = 0;
#pragma unroll 1
        for (int j = 0; j < 3; ++j) {
            const T dx = T(j == 0 ? DIRS[0][0] : j == 1 ? DIRS[1][0] : DIRS[2][0]);
            const T dy = T(j == 0 ? DIRS[0][1] : j == 1 ? DIRS[1][1] : DIRS[2][1]);
            const T dz = T(j == 0 ? DIRS[0][2] : j == 1 ? DIRS[1][2] : DIRS[2][2]);
            const T nrm = crossings_sqrt(add_rn(add_rn(mul_rn(dx, dx), mul_rn(dy, dy)), mul_rn(dz, dz)));     // rays_new_kernel
            const T dir[3] = {div_rn(dx, nrm), div_rn(dy, nrm), div_rn(dz, nrm)};
            const T inv[3] = {div_rn(T(1), dir[0]), div_rn(T(1), dir[1]), div_rn(T(1), dir[2])};
            uint32_t front = 0, back = 0;
            crossings_walk<T>(nodes, n_shapes, aabb, tris, o, dir, inv, Traits<T>::inf(), front, back);
            votes += (rule == BVHGPU_FILL_EVEN_ODD ? ((front + back) & 1u) != 0u : back != front) ? 1u : 0u;
        }
        out_inside[i] = votes >= 2 ? 1 : 0;
    }
}

// Signed distance: the knn_triangles row (k = 1) negated where the point is inside; a point without a triangle keeps +inf.
template <class T>
__global__ void __launch_bounds__(256) apply_sign_kernel(uint32_t n, const uint8_t* __restrict__ inside, const uint32_t* __restrict__ shape,
                                                         T* __restrict__ dist) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (inside[i] && shape[i] != BVH_INVALID) dist[i] = -dist[i];       // inside at distance 0 gives -0
}

// The checks shared by the three calls, in multi hit's order after the caller's null and layout / rule checks: n, the tree's status,
// then the triangles.  *nothing: n = 0, nothing to launch.
template <class T>
static int crossings_checks(Tree<T>* tree, size_t n, const char* who, bool* nothing) {
    *nothing = false;
    if (n > 0x7FFFFFFFull) { set_error("%s: n = %zu exceeds 2^31-1", who, n); return BVHGPU_ERR_INVALID; }
    if (n == 0) { *nothing = true; return BVHGPU_OK; }
    BVH_TRY(resolve_status(tree));
    if (tree->n && !tree->d_tris) { set_error("%s: needs bvhgpu_tree_set_triangles_* first", who); return BVHGPU_ERR_INVALID; }
    return BVHGPU_OK;
}

template <class T>
int count_hits_device(Tree<T>* tree, const void* d_rays, uint32_t fmt, size_t nrays, const T* d_tmax, uint32_t* d_front, uint32_t* d_back) {
    bvhgpu_ctx* ctx = tree->ctx;
    cudaStream_t st = ctx->stream;
    if (nrays > 0x7FFFFFFFull) { set_error("count_hits: too many rays"); return BVHGPU_ERR_INVALID; }
    if (fmt != BVHGPU_RAYS_FULL && fmt != BVHGPU_RAYS_OD) { set_error("count_hits: bad ray layout %u", fmt); return BVHGPU_ERR_INVALID; }
    bool nothing;
    BVH_TRY(crossings_checks(tree, nrays, "count_hits", &nothing));
    if (nothing) return BVHGPU_OK;
    if (tree->n == 0) {
        BVH_CUDA_TRY(cudaMemsetAsync(d_front, 0, sizeof(uint32_t) * nrays, st));
        BVH_CUDA_TRY(cudaMemsetAsync(d_back, 0, sizeof(uint32_t) * nrays, st));
        return BVHGPU_OK;
    }
    crossings_kernel<T, false><<<(unsigned)((nrays + 127) / 128), 128, 0, st>>>(
        tree->d_nodes, tree->n, tree->d_aabb, reinterpret_cast<const DTri<T>*>(tree->d_tris), reinterpret_cast<const T*>(d_rays),
        fmt == BVHGPU_RAYS_FULL ? 9u : 6u, (uint32_t)nrays, d_tmax, d_front, d_back, 0, nullptr);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}

static int check_rule(const char* who, int rule) {
    if (rule != BVHGPU_FILL_EVEN_ODD && rule != BVHGPU_FILL_NONZERO) { set_error("%s: unknown fill rule %d", who, rule); return BVHGPU_ERR_INVALID; }
    return BVHGPU_OK;
}

// The containment walk after the checks: out_inside[n] (device), all zero for an empty tree.
template <class T>
static int contains_launch(Tree<T>* tree, const T* d_points, size_t n, int rule, uint8_t* d_inside) {
    bvhgpu_ctx* ctx = tree->ctx;
    if (tree->n == 0) {
        BVH_CUDA_TRY(cudaMemsetAsync(d_inside, 0, n, ctx->stream));
        return BVHGPU_OK;
    }
    crossings_kernel<T, true><<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(
        tree->d_nodes, tree->n, tree->d_aabb, reinterpret_cast<const DTri<T>*>(tree->d_tris), d_points, 3u, (uint32_t)n, nullptr, nullptr,
        nullptr, rule, d_inside);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}

template <class T>
int contains_points_device(Tree<T>* tree, const T* d_points, size_t n, int rule, uint8_t* d_inside) {
    BVH_TRY(check_rule("contains_points", rule));
    bool nothing;
    BVH_TRY(crossings_checks(tree, n, "contains_points", &nothing));
    if (nothing) return BVHGPU_OK;
    return contains_launch(tree, d_points, n, rule, d_inside);
}

// knn_tri_device with k = 1 and no limit, the containment walk into scratch from the context's pool, apply_sign_kernel: three launches
// on the context's stream, nothing synchronises.
template <class T>
int signed_distance_device(Tree<T>* tree, const T* d_points, size_t n, int rule, uint32_t* d_shape, T* d_dist, T* d_closest) {
    BVH_TRY(check_rule("signed_distance", rule));
    bool nothing;
    BVH_TRY(crossings_checks(tree, n, "signed_distance", &nothing));
    if (nothing) return BVHGPU_OK;
    bvhgpu_ctx* ctx = tree->ctx;
    Scratch scratch(ctx);
    uint8_t* inside = nullptr;
    BVH_TRY(scratch.get(&inside, n));
    BVH_TRY(knn_tri_device<T>(tree, d_points, n, 1, nullptr, d_shape, d_dist, d_closest));
    BVH_TRY(contains_launch(tree, d_points, n, rule, inside));
    apply_sign_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>((uint32_t)n, inside, d_shape, d_dist);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}

template int count_hits_device<float>(Tree<float>*, const void*, uint32_t, size_t, const float*, uint32_t*, uint32_t*);
template int count_hits_device<double>(Tree<double>*, const void*, uint32_t, size_t, const double*, uint32_t*, uint32_t*);
template int contains_points_device<float>(Tree<float>*, const float*, size_t, int, uint8_t*);
template int contains_points_device<double>(Tree<double>*, const double*, size_t, int, uint8_t*);
template int signed_distance_device<float>(Tree<float>*, const float*, size_t, int, uint32_t*, float*, float*);
template int signed_distance_device<double>(Tree<double>*, const double*, size_t, int, uint32_t*, double*, double*);

template int set_triangles<float>(Tree<float>*, const float*, size_t, bool);
template int set_triangles<double>(Tree<double>*, const double*, size_t, bool);
template int closest_hit_device<float>(Tree<float>*, const void*, uint32_t, size_t, int, uint32_t*, float*, float*);
template int closest_hit_device<double>(Tree<double>*, const void*, uint32_t, size_t, int, uint32_t*, double*, double*);
template int closest_aabb_device<2, float>(bvhgpu_ctx*, const bvh_node3f*, uint32_t, const DAabbF*, const float*, size_t, uint32_t*, float*);
template int closest_aabb_device<2, double>(bvhgpu_ctx*, const bvh_node3d*, uint32_t, const DAabbD*, const double*, size_t, uint32_t*, double*);
template int closest_aabb_device<4, float>(bvhgpu_ctx*, const bvh_node4f*, uint32_t, const bvh_aabb4f*, const float*, size_t, uint32_t*, float*);
template int closest_aabb_device<4, double>(bvhgpu_ctx*, const bvh_node4d*, uint32_t, const bvh_aabb4d*, const double*, size_t, uint32_t*, double*);

template int any_hit_device<float>(Tree<float>*, const void*, uint32_t, size_t, const float*, int, uint32_t*);
template int any_hit_device<double>(Tree<double>*, const void*, uint32_t, size_t, const double*, int, uint32_t*);
template int any_hit_aabb_device<2, float>(bvhgpu_ctx*, const bvh_node3f*, uint32_t, const DAabbF*, const float*, size_t, const float*, uint32_t*);
template int any_hit_aabb_device<2, double>(bvhgpu_ctx*, const bvh_node3d*, uint32_t, const DAabbD*, const double*, size_t, const double*, uint32_t*);
template int any_hit_aabb_device<4, float>(bvhgpu_ctx*, const bvh_node4f*, uint32_t, const bvh_aabb4f*, const float*, size_t, const float*, uint32_t*);
template int any_hit_aabb_device<4, double>(bvhgpu_ctx*, const bvh_node4d*, uint32_t, const bvh_aabb4d*, const double*, size_t, const double*, uint32_t*);

template int multi_hit_device<float>(Tree<float>*, const void*, uint32_t, size_t, uint32_t, const float*, int, uint32_t*, float*, float*);
template int multi_hit_device<double>(Tree<double>*, const void*, uint32_t, size_t, uint32_t, const double*, int, uint32_t*, double*, double*);
template int multi_hit_aabb_device<2, float>(bvhgpu_ctx*, const bvh_node3f*, uint32_t, const DAabbF*, const float*, size_t, uint32_t, const float*, uint32_t*, float*);
template int multi_hit_aabb_device<2, double>(bvhgpu_ctx*, const bvh_node3d*, uint32_t, const DAabbD*, const double*, size_t, uint32_t, const double*, uint32_t*, double*);
template int multi_hit_aabb_device<4, float>(bvhgpu_ctx*, const bvh_node4f*, uint32_t, const bvh_aabb4f*, const float*, size_t, uint32_t, const float*, uint32_t*, float*);
template int multi_hit_aabb_device<4, double>(bvhgpu_ctx*, const bvh_node4d*, uint32_t, const bvh_aabb4d*, const double*, size_t, uint32_t, const double*, uint32_t*, double*);

}  // namespace bvhb200
