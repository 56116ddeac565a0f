// bvh_b200/csrc/flatten.cu -- Bvh::flatten (src/flat_bvh.rs:60-143, 240-251, 312-319) as a closed-form
// map over the preorder node array, the device-only traversal records, whole-tree SAH cost, optimize and the 3-D growth rebuild of
// update_shapes / add_shapes (the drivers of refit and the dynamic operations are in dynamic.cu).
//
// Closed form (DESIGN.md "flatten"): the reference's recursive flatten pushes, for every non-root
// Bvh node i, a navigator FlatNode and, for leaves, a leaf FlatNode right behind it.  Because
// Bvh.nodes is in preorder with child_l = i+1, the navigator of node i lands at
//     nav(i) = (i - 1) + start(i)          start(i) = number of leaves before i = first shape position
// with entry = nav+1 and exit = nav + 3*count(i) - 1.  One thread per node, no recursion, no scan.
#include "internal.h"
#include "update.cuh"

namespace bvhb200 {

template <class T>
__global__ void __launch_bounds__(256) flat_kernel(const typename Traits<T>::Node* __restrict__ nodes,
                                                   const uint32_t* __restrict__ node_start, uint32_t n_nodes,
                                                   typename Traits<T>::Flat* __restrict__ flat, const BuildStatus* __restrict__ status) {
    using Tr = Traits<T>;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_nodes) return;
    if (status->error | status->nan_found) return;      // the (asynchronous) build failed: the node array is garbage, map nothing
    const uint4 meta = *reinterpret_cast<const uint4*>(nodes + i);      // parent, child_l, child_r, shape/count
    const bool leaf = meta.y == BVH_INVALID;
    if (i == 0) {
        if (leaf) {                                                      // root leaf: flat_bvh.rs:129-141 only
            typename Tr::Flat f;
            for (int k = 0; k < 3; ++k) { f.aabb.min[k] = Tr::inf(); f.aabb.max[k] = -Tr::inf(); }
            f.entry_index = BVH_INVALID; f.exit_index = 1; f.shape_index = meta.w;
            flat[0] = f;
        }
        return;
    }
    const uint32_t nav = (i - 1) + node_start[i];
    const uint32_t count = leaf ? 1u : meta.w;
    const typename Tr::Node& par = nodes[meta.x];
    const bool is_left = par.child_l == i;
    typename Tr::Flat f;
    for (int k = 0; k < 3; ++k) {
        f.aabb.min[k] = is_left ? par.l_aabb.min[k] : par.r_aabb.min[k];
        f.aabb.max[k] = is_left ? par.l_aabb.max[k] : par.r_aabb.max[k];
    }
    f.entry_index = nav + 1; f.exit_index = nav + 3 * count - 1; f.shape_index = BVH_INVALID;   // flat_bvh.rs:80-88
    flat[nav] = f;
    if (leaf) {
        typename Tr::Flat g;
        for (int k = 0; k < 3; ++k) { g.aabb.min[k] = Tr::inf(); g.aabb.max[k] = -Tr::inf(); }
        g.entry_index = BVH_INVALID; g.exit_index = nav + 2; g.shape_index = meta.w;            // flat_bvh.rs:129-141
        flat[nav + 1] = g;
    }
}

// Traversal records: record r = node r+1 of the preorder array (the root has no AABB of its own).
//   hit  -> next record r+1 (left child / leaf reported)
//   miss -> skip = first record after the node's subtree
template <class T>
__global__ void __launch_bounds__(256) trec_kernel(const typename Traits<T>::Node* __restrict__ nodes, uint32_t n_nodes,
                                                   const typename Traits<T>::DAabb* __restrict__ aabb,
                                                   typename Traits<T>::TNode* __restrict__ trec, const BuildStatus* __restrict__ status, int dims) {
    using Tr = Traits<T>;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_nodes) return;
    if (status->error | status->nan_found) return;
    typename Tr::TNode r;
    if (n_nodes == 1) {                       // root leaf: the shape's own AABB is tested (bvh_node.rs:314)
        T mn[3], mx[3];
        load_aabb(aabb + nodes[0].shape, mn, mx);
        for (int k = 0; k < 3; ++k) { r.min[k] = mn[k]; r.max[k] = mx[k]; }
        r.skip = 1; r.shape = nodes[0].shape;
        if (dims == 2) { r.min[2] = T(-1); r.max[2] = T(1); }
        if constexpr (sizeof(T) == 8) { r.pad[0] = r.pad[1] = 0; }
        trec[0] = r;
        return;
    }
    if (i == 0) return;
    const uint4 meta = *reinterpret_cast<const uint4*>(nodes + i);
    const bool leaf = meta.y == BVH_INVALID;
    const typename Tr::Node& par = nodes[meta.x];
    const bool is_left = par.child_l == i;
    for (int k = 0; k < 3; ++k) {
        r.min[k] = is_left ? par.l_aabb.min[k] : par.r_aabb.min[k];
        r.max[k] = is_left ? par.l_aabb.max[k] : par.r_aabb.max[k];
    }
    const uint32_t count = leaf ? 1u : meta.w;
    r.skip = (i - 1) + (2 * count - 1);
    r.shape = leaf ? meta.w : BVH_INVALID;
    if (dims == 2) { r.min[2] = T(-1); r.max[2] = T(1); }          // 2-D tree: the z slab must not constrain (dim2.cu)
    if constexpr (sizeof(T) == 8) { r.pad[0] = r.pad[1] = 0; }
    trec[i - 1] = r;
}

template <class T> int build_traversal_records(Tree<T>* tree) {
    bvhgpu_ctx* ctx = tree->ctx;
    if (tree->n == 0) { tree->n_trec = 0; return BVHGPU_OK; }
    const uint32_t n_trec = tree->n == 1 ? 1u : tree->n_nodes - 1;
    if (!tree->d_tnodes) BVH_TRY(dalloc_t(ctx, &tree->d_tnodes, n_trec));
    tree->n_trec = n_trec;
    tree->top_valid = false;                                    // the shared-memory top records are rebuilt from these lazily
    trec_kernel<T><<<(tree->n_nodes + 255) / 256, 256, 0, ctx->stream>>>(tree->d_nodes, tree->n_nodes, tree->dims == 2 && tree->d_aabb_trav ? tree->d_aabb_trav : tree->d_aabb, tree->d_tnodes, tree->d_status, tree->dims);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}

// ---- top-of-tree records for the shared-memory walk (walk_top_kernel, f32) ---------------------------------------------------------
// P = {root} + all inner nodes with >= C shapes below them; T = the children of P's nodes, in preorder: the records a ray meets before it
// dives below the C-level.  An entry is the node's traversal record with other links:
//   node in P (top-internal) : w3 = index in T of the first entry behind its subtree, w7 = 0xFFFFFFFF       hit -> next entry
//   fringe leaf              : w7 = shape                                                               hit -> report, next entry
//   fringe inner node        : w3 = end of its subtree in the GLOBAL records, w7 = 0x80000000 | first global record of the subtree
//                                                                                   hit -> walk the global records [begin, end), then next
// C is chosen on the device (no host round trip: the records are rebuilt inside the asynchronous traversal call after every
// refit / update): a histogram of count(parent) over 8 bins per octave, then the smallest C whose entries fit the budget.
// d_top = header {n_top, C, 0, 0, ...} (32 B) followed by lo[n_top], hi[n_top].
constexpr uint32_t TOP_BINS = 256;
__device__ __forceinline__ uint32_t top_bin(uint32_t c) { const uint32_t k = 31 - __clz(c); return 8 * k + (((c << 3) >> k) & 7u); }
__global__ void __launch_bounds__(256) top_hist_kernel(const bvh_node3f* __restrict__ nodes, uint32_t n_nodes, uint32_t* __restrict__ hist) {
    __shared__ uint32_t sh[TOP_BINS];
    sh[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 1 && i < n_nodes) atomicAdd(sh + top_bin(nodes[nodes[i].parent].shape), 1u);      // an inner node stores the shapes below it
    __syncthreads();
    if (sh[threadIdx.x]) atomicAdd(hist + threadIdx.x, sh[threadIdx.x]);
}
__global__ void __launch_bounds__(32) top_choose_kernel(const uint32_t* __restrict__ hist, uint32_t budget, uint32_t* __restrict__ hdr) {
    // One warp, 8 bins per lane.  Bins are taken from the highest down while their running sum S(b) = sum of hist[b..] fits the budget;
    // S grows as b falls, so the bins taken are a suffix of the bin range: count them, and the last one's S is the number of entries.
    const uint32_t l = threadIdx.x & 31u, FULL = 0xffffffffu;
    uint32_t h[8], t = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) { h[k] = hist[8 * l + k]; t += h[k]; }
    uint32_t incl = t;                                                 // this lane's bins and all higher lanes'
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_down_sync(FULL, incl, o); if (l + o < 32) incl += v; }
    uint32_t run = incl - t, taken = 0, total = 0;
#pragma unroll
    for (int k = 7; k >= 0; --k) { run += h[k]; if (run <= budget) { ++taken; total = run; } }
    taken = __reduce_add_sync(FULL, taken);
    total = __reduce_max_sync(FULL, total);
    if (l) return;
    // the smallest count that falls into a taken bin (bins nb ..): ceil((8 + sub) * 2^k / 8); everything taken: C = 2
    uint32_t C = 2;
    if (taken == 0) C = 0xFFFFFFFFu;                                   // not even the highest bin fits: no node qualifies, n_top = 0 (the walk then stays below)
    else if (taken < TOP_BINS) { const uint32_t nb = TOP_BINS - taken, k = nb >> 3, sub = nb & 7u; C = (uint32_t)((((unsigned long long)(8 + sub) << k) + 7ull) >> 3); }
    hdr[0] = total; hdr[1] = C; hdr[2] = 0; hdr[3] = 0;
}
__global__ void __launch_bounds__(256) top_flag_kernel(const bvh_node3f* __restrict__ nodes, uint32_t n_nodes, const uint32_t* __restrict__ hdr, uint32_t* __restrict__ flags) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n_nodes) return;
    const uint32_t C = hdr[1];
    uint32_t f = 0;
    if (i >= 1 && i < n_nodes) f = nodes[nodes[i].parent].shape >= C ? 1u : 0u;
    flags[i] = f;
}
__global__ void __launch_bounds__(256) top_emit_kernel(const bvh_node3f* __restrict__ nodes, uint32_t n_nodes, const TNodeF* __restrict__ trec,
                                                       const uint32_t* __restrict__ flags, const uint32_t* __restrict__ pre, float4* __restrict__ top) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0 || i >= n_nodes || !flags[i]) return;
    const uint32_t n_top = reinterpret_cast<const uint32_t*>(top)[0], C = reinterpret_cast<const uint32_t*>(top)[1];
    float4* lo = top + 2;
    float4* hi = lo + n_top;
    const uint32_t k = pre[i];
    if (k >= n_top) return;                                             // (cannot happen: the flags are derived from the same C)
    const uint4 meta = *reinterpret_cast<const uint4*>(nodes + i);
    const bool leaf = meta.y == BVH_INVALID;
    const uint32_t cnt = leaf ? 1u : meta.w;
    const TNodeF r = trec[i - 1];
    uint32_t w3, w7;
    if (!leaf && cnt >= C) { const uint32_t end = i + 2 * cnt - 1; w3 = pre[end < n_nodes ? end : n_nodes]; w7 = 0xFFFFFFFFu; }
    else if (leaf)         { w3 = k + 1; w7 = meta.w; }
    else                   { w3 = r.skip; w7 = 0x80000000u | i; }        // global record of node i's left child = i (miss: next entry)
    lo[k] = make_float4(r.min[0], r.min[1], r.min[2], __uint_as_float(w3));
    hi[k] = make_float4(r.max[0], r.max[1], r.max[2], __uint_as_float(w7));
}
}  // namespace bvhb200
#include <cub/device/device_scan.cuh>
namespace bvhb200 {
// (Re)builds tree->d_top for at most `budget` entries; asynchronous on the context's stream.  n >= 2 only (n_top >= 2 then: the
// root's two children always fit).
int build_top_records(Tree<float>* tree, uint32_t budget) {
    bvhgpu_ctx* ctx = tree->ctx;
    cudaStream_t st = ctx->stream;
    const uint32_t nn = tree->n_nodes;
    Scratch scratch(ctx);
    uint32_t *hist = nullptr, *flags = nullptr, *pre = nullptr;
    BVH_TRY(scratch.get(&hist, TOP_BINS));
    BVH_TRY(scratch.get(&flags, (size_t)nn + 1));
    BVH_TRY(scratch.get(&pre, (size_t)nn + 1));
    if (tree->d_top && tree->top_cap < budget) { dfree(ctx, tree->d_top); tree->d_top = nullptr; }
    if (!tree->d_top) { BVH_TRY(dalloc(ctx, &tree->d_top, 32 * ((size_t)budget + 1))); tree->top_cap = budget; }
    BVH_CUDA_TRY(cudaMemsetAsync(hist, 0, TOP_BINS * sizeof(uint32_t), st));
    const unsigned g = (nn + 256) / 256;
    uint32_t* hdr = reinterpret_cast<uint32_t*>(tree->d_top);
    top_hist_kernel<<<g, 256, 0, st>>>(tree->d_nodes, nn, hist);
    top_choose_kernel<<<1, 32, 0, st>>>(hist, budget, hdr);
    top_flag_kernel<<<g, 256, 0, st>>>(tree->d_nodes, nn, hdr, flags);
    size_t tmp_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, flags, pre, (int)(nn + 1), st);
    unsigned char* tmp = nullptr;
    BVH_TRY(scratch.get(&tmp, tmp_bytes));
    cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, flags, pre, (int)(nn + 1), st);
    top_emit_kernel<<<g, 256, 0, st>>>(tree->d_nodes, nn, tree->d_tnodes, flags, pre, reinterpret_cast<float4*>(tree->d_top));
    ctx->launches += 5;
    BVH_CUDA_TRY(cudaGetLastError());
    tree->top_valid = true; tree->top_budget = budget;
    return BVHGPU_OK;
}

template <class T> int build_flat(Tree<T>* tree) {
    bvhgpu_ctx* ctx = tree->ctx;
    tree->n_flat = tree->n == 0 ? 0 : (tree->n == 1 ? 1 : 3 * (size_t)tree->n - 2);
    tree->have_flat = true;
    if (tree->n == 0) return BVHGPU_OK;
    if (!tree->d_flat) BVH_TRY(dalloc_t(ctx, &tree->d_flat, tree->n_flat));
    flat_kernel<T><<<(tree->n_nodes + 255) / 256, 256, 0, ctx->stream>>>(tree->d_nodes, tree->d_node_start, tree->n_nodes, tree->d_flat, tree->d_status);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}

// ---- whole-tree SAH cost (DESIGN.md): sum over non-root nodes of SA(aabb in parent) / SA(root) ----
template <class T>
__global__ void __launch_bounds__(256) sah_kernel(const typename Traits<T>::Node* __restrict__ nodes, uint32_t n_nodes, double* out2) {
    __shared__ double sp[8], sg[8];
    double p = 0.0, g = 0.0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_nodes; i += gridDim.x * blockDim.x) {
        const typename Traits<T>::Node& nd = nodes[i];
        if (nd.child_l == BVH_INVALID) continue;
        for (int side = 0; side < 2; ++side) {
            const auto& a = side ? nd.r_aabb : nd.l_aabb;
            const double x = (double)a.max[0] - (double)a.min[0], y = (double)a.max[1] - (double)a.min[1], z = (double)a.max[2] - (double)a.min[2];
            p += 2.0 * (x * x + y * y + z * z);
            g += 2.0 * (x * y + y * z + z * x);
        }
    }
    for (int o = 16; o > 0; o >>= 1) { p += __shfl_xor_sync(0xffffffffu, p, o); g += __shfl_xor_sync(0xffffffffu, g, o); }
    if (lane_id() == 0) { sp[threadIdx.x >> 5] = p; sg[threadIdx.x >> 5] = g; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double tp = 0, tg = 0;
        for (int w = 0; w < 8; ++w) { tp += sp[w]; tg += sg[w]; }
        atomicAdd(out2, tp);
        atomicAdd(out2 + 1, tg);
    }
}

template <class T> int sah_cost(Tree<T>* tree, double* out2) {
    bvhgpu_ctx* ctx = tree->ctx;
    out2[0] = out2[1] = 0.0;
    if (tree->n < 2) return BVHGPU_OK;
    double* d = nullptr;
    BVH_TRY(dalloc_t(ctx, &d, 2));
    BVH_CUDA_TRY(cudaMemsetAsync(d, 0, 2 * sizeof(double), ctx->stream));
    const int blocks = (int)std::min<uint64_t>((tree->n_nodes + 255) / 256, (uint64_t)ctx->sm_count * 4);
    sah_kernel<T><<<blocks, 256, 0, ctx->stream>>>(tree->d_nodes, tree->n_nodes, d);
    ctx->launches++;
    double h[2];
    typename Traits<T>::Node root;
    BVH_CUDA_TRY(cudaMemcpyAsync(h, d, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaMemcpyAsync(&root, tree->d_nodes, sizeof(root), cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    dfree(ctx, d);
    double s[3];
    for (int k = 0; k < 3; ++k) {
        const double mn = std::min((double)root.l_aabb.min[k], (double)root.r_aabb.min[k]);
        const double mx = std::max((double)root.l_aabb.max[k], (double)root.r_aabb.max[k]);
        s[k] = mx - mn;
    }
    out2[0] = h[0] / (2.0 * (s[0] * s[0] + s[1] * s[1] + s[2] * s[2]));
    out2[1] = h[1] / (2.0 * (s[0] * s[1] + s[1] * s[2] + s[2] * s[0]));
    return BVHGPU_OK;
}


// ---- optimize: refit + exact rebuild of the subtrees the motion degraded (replaces Bvh::update_shapes) --------------------
// The reference re-inserts every changed shape sequentially (optimization.rs:290-302).  The data-parallel counterpart:
//   1. remember SA(node) of every inner node, refit bottom-up (new AABBs and centroid bounds of every node);
//   2. a node is BAD when its surface area grew by more than `max_growth`; bad nodes form chains from the moved leaves
//      upwards, ending where the ancestor is big enough to have absorbed the motion;
//   3. rebuild roots = the outermost nodes that are not bad but have a bad child (or the tree root if it is bad itself):
//      the smallest subtrees inside which every moved shape can be placed properly again;
//   4. those subtrees are rebuilt IN PLACE by the exact builder (build_sah.cu: rebuild_subtrees): preorder layout makes
//      the subtree of a node with k shapes the contiguous node range [i, i + 2k - 1) over the contiguous leaf range
//      [start(i), start(i) + k), so a rebuild only rewrites its own ranges.
template <class T>
__global__ void __launch_bounds__(256) mark_bad_kernel(const typename Traits<T>::Node* __restrict__ nodes, uint32_t n_nodes,
                                                       const T* __restrict__ sa_old, T max_growth, uint8_t* __restrict__ bad) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_nodes) return;
    const typename Traits<T>::Node& nd = nodes[i];
    if (nd.child_l == BVH_INVALID) { bad[i] = 0; return; }
    T mn[3], mx[3];
    for (int k = 0; k < 3; ++k) { mn[k] = min_t(nd.l_aabb.min[k], nd.r_aabb.min[k]); mx[k] = max_t(nd.l_aabb.max[k], nd.r_aabb.max[k]); }
    bad[i] = surface_area(mn, mx) > mul_rn(max_growth, sa_old[i]) ? 1 : 0;
}
template <class T>
__global__ void __launch_bounds__(256) select_roots_kernel(const typename Traits<T>::Node* __restrict__ nodes, uint32_t n_nodes,
                                                           const uint8_t* __restrict__ bad, uint32_t* __restrict__ roots, uint32_t* n_roots) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_nodes) return;
    const uint4 meta = *reinterpret_cast<const uint4*>(nodes + i);      // parent, child_l, child_r, count
    if (!rebuild_candidate(i, meta.y, meta.z, bad)) return;
    uint32_t a = i;
    while (a != 0) {                                                   // an outer candidate takes this subtree with it
        a = nodes[a].parent;
        const uint4 m = *reinterpret_cast<const uint4*>(nodes + a);
        if (rebuild_candidate(a, m.y, m.z, bad)) return;
    }
    roots[atomicAdd(n_roots, 1u)] = i;
}
// shapes in leaf order: position of a leaf = its node_start
__global__ void __launch_bounds__(256) leaf_order_kernel(const uint32_t* __restrict__ node_index, const uint32_t* __restrict__ node_start,
                                                         uint32_t n, uint32_t* __restrict__ idx) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n) idx[node_start[node_index[s]]] = s;
}

template <class T> int optimize(Tree<T>* tree, double max_growth) {
    bvhgpu_ctx* ctx = tree->ctx;
    if (tree->n < 3) return refit(tree);                                // one or two shapes: nothing a rebuild could change
    cudaStream_t st = ctx->stream;
    const uint32_t n = tree->n, nn = tree->n_nodes;
    T* cb = nullptr;
    uint8_t* bad = nullptr;
    uint32_t *roots = nullptr, *n_roots = nullptr, *idx0 = nullptr, *arrivals = nullptr;
    BVH_TRY(ensure_sa_base(tree));                                      // first optimize on this tree: the baseline is the tree as built
    T* sa_old = tree->d_sa_base;
    Scratch scratch(ctx);                                               // released on every return path
    BVH_TRY(scratch.get(&cb, (size_t)nn * 6));
    BVH_TRY(scratch.get(&bad, nn));
    BVH_TRY(scratch.get(&roots, n));
    BVH_TRY(scratch.get(&n_roots, 1));
    BVH_TRY(scratch.get(&idx0, n));
    BVH_TRY(scratch.get(&arrivals, nn));
    BVH_CUDA_TRY(cudaMemsetAsync(arrivals, 0, sizeof(uint32_t) * nn, st));
    BVH_CUDA_TRY(cudaMemsetAsync(n_roots, 0, sizeof(uint32_t), st));
    const unsigned gn = (nn + 255) / 256, gs = (n + 255) / 256;
    refit_kernel<3, T, true><<<gs, 256, 0, st>>>(tree->d_nodes, tree->d_node_index, tree->d_aabb, n, arrivals, cb);
    mark_bad_kernel<T><<<gn, 256, 0, st>>>(tree->d_nodes, nn, sa_old, (T)max_growth, bad);
    select_roots_kernel<T><<<gn, 256, 0, st>>>(tree->d_nodes, nn, bad, roots, n_roots);
    leaf_order_kernel<<<gs, 256, 0, st>>>(tree->d_node_index, tree->d_node_start, n, idx0);
    ctx->launches += 4;
    BVH_CUDA_TRY(cudaGetLastError());
    BVH_TRY(rebuild_subtrees(ctx, tree, roots, n_roots, cb, idx0, false));
    rebase_kernel<3, T, typename Traits<T>::Node><<<std::max(1, std::min(ctx->sm_count * 4, (int)n)), 256, 0, st>>>(tree->d_nodes, roots, n_roots, sa_old);
    ctx->launches++;
    return refresh_caches(tree);
}

// one warp per rebuild root: the shapes of its subtree in leaf order (index buffer of the rebuild) and the bounds of their centres
template <class T>
__global__ void __launch_bounds__(256) root_prep_kernel(const typename Traits<T>::Node* __restrict__ nodes, const uint32_t* __restrict__ node_start,
                                                        const typename Traits<T>::DAabb* __restrict__ aabb, const uint32_t* __restrict__ roots,
                                                        const uint32_t* __restrict__ n_roots, uint32_t* __restrict__ idx0, T* __restrict__ cb_roots) {
    const uint32_t warps = gridDim.x * (blockDim.x >> 5), nr = *n_roots;
    for (uint32_t k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); k < nr; k += warps) {
        const uint32_t r = roots[k], cnt = nodes[r].shape;
        T cmn[3] = {Traits<T>::inf(), Traits<T>::inf(), Traits<T>::inf()}, cmx[3] = {-Traits<T>::inf(), -Traits<T>::inf(), -Traits<T>::inf()};
        for (uint32_t i = r + lane_id(); i < r + 2 * cnt - 1; i += 32) {
            const uint4 meta = *reinterpret_cast<const uint4*>(nodes + i);
            if (meta.y != BVH_INVALID) continue;
            idx0[node_start[i]] = meta.w;
            T mn[3], mx[3];
            load_aabb(aabb + meta.w, mn, mx);
            for (int c = 0; c < 3; ++c) { const T ctr = center1(mn[c], mx[c]); cmn[c] = min_t(cmn[c], ctr); cmx[c] = max_t(cmx[c], ctr); }
        }
        for (int c = 0; c < 3; ++c) {
            typename Traits<T>::Key a = f2key(cmn[c]), b = f2key(cmx[c]);
            a = warp_min_key(a); b = warp_max_key(b);
            if (lane_id() == 0) { cb_roots[6 * (size_t)k + c] = key2f(a); cb_roots[6 * (size_t)k + 3 + c] = key2f(b); }
        }
    }
}
// dirty[0 .. cnts[0]) = the nodes whose box changed, tree->d_bad = their growth flags.  Rebuilds in place the outermost degraded
// subtrees (cnts[1], zero on entry, counts them), gives them fresh baselines and clears the flags.  The builder counts the shapes it
// rebuilt in tree->d_status and reports its errors there.
template <class T> int rebuild_degraded(Tree<T>* tree, const uint32_t* dirty, uint32_t* cnts, size_t*, const char*) {
    bvhgpu_ctx* ctx = tree->ctx;
    cudaStream_t st = ctx->stream;
    const uint32_t n = tree->n, gn = (tree->n_nodes + 255) / 256;
    Scratch scratch(ctx);
    uint32_t *roots = nullptr, *idx0 = nullptr;
    T* cb_roots = nullptr;
    BVH_TRY(scratch.get(&roots, n));
    BVH_TRY(scratch.get(&idx0, n));
    BVH_TRY(scratch.get(&cb_roots, 6 * (size_t)n / 2 + 6));             // rebuild roots are inner nodes of disjoint subtrees: at most n / 2 of them
    select_roots_dirty_kernel<typename Traits<T>::Node><<<gn, 256, 0, st>>>(tree->d_nodes, tree->d_bad, dirty, cnts, roots, cnts + 1);
    root_prep_kernel<T><<<std::max(1, ctx->sm_count * 8), 256, 0, st>>>(tree->d_nodes, tree->d_node_start, tree->d_aabb, roots, cnts + 1, idx0, cb_roots);
    ctx->launches += 2;
    BVH_CUDA_TRY(cudaGetLastError());
    BVH_TRY(rebuild_subtrees(ctx, tree, roots, cnts + 1, cb_roots, idx0, true));
    rebase_kernel<3, T, typename Traits<T>::Node><<<std::max(1, ctx->sm_count * 8), 256, 0, st>>>(tree->d_nodes, roots, cnts + 1, tree->d_sa_base);
    clear_bad_kernel<<<gn, 256, 0, st>>>(dirty, cnts, tree->d_bad);
    ctx->launches += 2;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}

#define INST(T)                                           \
    template int rebuild_degraded<T>(Tree<T>*, const uint32_t*, uint32_t*, size_t*, const char*); \
    template int optimize<T>(Tree<T>*, double);           \
    template int build_traversal_records<T>(Tree<T>*);    \
    template int build_flat<T>(Tree<T>*);                 \
    template int sah_cost<T>(Tree<T>*, double*);
INST(float)
INST(double)

}  // namespace bvhb200
