// bvh_b200/csrc/dynamic.cu -- Bvh::add_shape / Bvh::remove_shape (src/bvh/optimization.rs:67-301) in batched, data-parallel form.
//
// The node array stays in Bvh::build's preorder layout (child_l = i + 1, the subtree of a node with c shapes is the node range
// [i, i + 2c - 1) over the leaf range [start(i), start(i) + c)), so both operations are a relocation of the whole array by prefix
// sums plus work on the touched root paths (DESIGN.md §4.10):
//
//   add    every new shape descends the tree as it was before the call (the reference's insertion test, one thread per shape);
//          at every insertion point p chosen by a_p shapes a graft node G takes p's place, its left child is the exact-SAH
//          subtree over those shapes (a leaf when a_p = 1), its right child is p's old subtree.  With S = inclusive scan of a:
//              G of node i          -> i + 2 (S(i) - a_i)            (= where links to i point)
//              old content of i     -> i + 2 S(i)
//              start(i)             += S(i)
//   remove removed leaves go, inner nodes left with one non-empty child are spliced out (the child takes their place); the new
//          index of a surviving node is the exclusive scan of the survive flags.  Shape indices are compacted by the swap rule.
//
// Then the boxes of the affected nodes (the ancestors of the insertion points / of the removed leaves) are recomputed bottom-up
// by one climb (climb_affected_kernel); an add also runs the growth test of bvhgpu_update_* on them and rebuilds the degraded
// subtrees in place.  The kernels that touch nodes or boxes are generic in D (dynamic.cuh, update.cuh).
//
// The host drivers of refit, update_shapes, add_shapes and remove_shapes are here too, one per operation for Tree<T> (D = 2, 3) and
// Tree4<T> (D = 4) alike (DESIGN.md sections 4.12, 4.13).  What the two tree types do differently is an overload on the tree type:
// building subtrees from seeded roots, the growth rebuild, the caches after boxes change in place and after a relocation, the
// per-shape geometry (triangles of a 3-D tree, segments of a 2-D tree) and the deferred build status.
#include "internal.h"
#include "dynamic.cuh"
#include <cub/device/device_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>
#include <type_traits>

namespace bvhb200 {

// ---- kernels that touch neither nodes nor boxes (the others are in dynamic.cuh) --------------------------------------------------
__global__ void __launch_bounds__(256) iota_kernel(uint32_t* __restrict__ v, uint32_t k) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < k) v[j] = j;
}
// one thread per group (= distinct insertion point): its size a_p, scattered onto the old node array
__global__ void __launch_bounds__(256) group_scatter_kernel(const uint32_t* __restrict__ uniq, const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ n_groups,
                                                            uint32_t* __restrict__ a) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g < *n_groups) a[uniq[g]] = cnt[g];
}
__global__ void __launch_bounds__(256) removed_positions_kernel(const uint32_t* __restrict__ rm, uint32_t n, const uint32_t* __restrict__ node_index,
                                                                const uint32_t* __restrict__ node_start, uint32_t* __restrict__ kpos) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n && rm[s]) kpos[node_start[node_index[s]]] = 1u;
}
// the vacated indices below m = n - k, in ascending order
__global__ void __launch_bounds__(256) holes_kernel(const uint32_t* __restrict__ rm, const uint32_t* __restrict__ Rm, uint32_t m, uint32_t* __restrict__ holes) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < m && rm[s]) holes[Rm[s]] = s;
}

// ---- host side -----------------------------------------------------------------------------------------------------------------
int exclusive_sum_u32(Scratch& scratch, const uint32_t* in, uint32_t* out, size_t len, cudaStream_t st) {
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, (int64_t)len, st);
    unsigned char* tmp = nullptr;
    BVH_TRY(scratch.get(&tmp, bytes));
    BVH_CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, bytes, in, out, (int64_t)len, st));
    return BVHGPU_OK;
}

int group_insertions(bvhgpu_ctx* ctx, Scratch& scratch, const uint32_t* point, uint32_t k, uint32_t nn, uint32_t* ng, Groups* G) {
    cudaStream_t st = ctx->stream;
    uint32_t *iota = nullptr, *spoint = nullptr;
    BVH_TRY(scratch.get(&iota, k));
    BVH_TRY(scratch.get(&spoint, k));
    BVH_TRY(scratch.get(&G->sshape, k));
    BVH_TRY(scratch.get(&G->uniq, k));
    BVH_TRY(scratch.get(&G->cnt, (size_t)k + 1));
    BVH_TRY(scratch.get(&G->goff, (size_t)k + 1));
    BVH_CUDA_TRY(cudaMemsetAsync(G->cnt, 0, ((size_t)k + 1) * sizeof(uint32_t), st));
    const unsigned gk = (k + 255) / 256;
    // group the new shapes by insertion point, ascending shape index inside a group (stable radix sort: deterministic)
    {
        int bits = 1;
        while (bits < 32 && (1ull << bits) < nn) ++bits;
        iota_kernel<<<gk, 256, 0, st>>>(iota, k);
        size_t b1 = 0, b2 = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, b1, point, spoint, iota, G->sshape, (int)k, 0, bits, st);
        cub::DeviceRunLengthEncode::Encode(nullptr, b2, spoint, G->uniq, G->cnt, ng, (int)k, st);
        unsigned char* tmp = nullptr;
        BVH_TRY(scratch.get(&tmp, std::max(b1, b2)));
        BVH_CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, b1, point, spoint, iota, G->sshape, (int)k, 0, bits, st));
        BVH_CUDA_TRY(cub::DeviceRunLengthEncode::Encode(tmp, b2, spoint, G->uniq, G->cnt, ng, (int)k, st));
    }
    BVH_TRY(exclusive_sum_u32(scratch, G->cnt, G->goff, (size_t)k + 1, st));
    BVH_TRY(scratch.get(&G->a, nn));
    BVH_TRY(scratch.get(&G->S, nn));
    BVH_CUDA_TRY(cudaMemsetAsync(G->a, 0, sizeof(uint32_t) * nn, st));
    group_scatter_kernel<<<gk, 256, 0, st>>>(G->uniq, G->cnt, ng, G->a);
    {
        size_t bytes = 0;
        cub::DeviceScan::InclusiveSum(nullptr, bytes, G->a, G->S, (int64_t)nn, st);
        unsigned char* tmp = nullptr;
        BVH_TRY(scratch.get(&tmp, bytes));
        BVH_CUDA_TRY(cub::DeviceScan::InclusiveSum(tmp, bytes, G->a, G->S, (int64_t)nn, st));
    }
    return BVHGPU_OK;
}

int remove_ranks(bvhgpu_ctx* ctx, Scratch& scratch, const uint32_t* rm, uint32_t n, uint32_t k, const uint32_t* node_index,
                 const uint32_t* node_start, Ranks* r) {
    cudaStream_t st = ctx->stream;
    const uint32_t m = n - k;
    uint32_t* kpos = nullptr;
    BVH_TRY(scratch.get(&kpos, (size_t)n + 1));
    BVH_TRY(scratch.get(&r->R, (size_t)n + 1));
    BVH_TRY(scratch.get(&r->Rm, (size_t)n + 1));
    BVH_TRY(scratch.get(&r->holes, k));
    BVH_CUDA_TRY(cudaMemsetAsync(kpos, 0, sizeof(uint32_t) * ((size_t)n + 1), st));
    const unsigned gs = (n + 255) / 256;
    removed_positions_kernel<<<gs, 256, 0, st>>>(rm, n, node_index, node_start, kpos);
    BVH_TRY(exclusive_sum_u32(scratch, kpos, r->R, (size_t)n + 1, st));
    BVH_TRY(exclusive_sum_u32(scratch, rm, r->Rm, (size_t)n + 1, st));
    holes_kernel<<<gs, 256, 0, st>>>(rm, r->Rm, m, r->holes);
    return BVHGPU_OK;
}

// ---- the steps that differ between Tree<T> (D = 2, 3) and Tree4<T> (D = 4) -------------------------------------------------------
// The 4-D overloads are in dim4.cu, the 3-D growth rebuild in flatten.cu.

// Caches after the boxes changed in place.  A 2-D tree's FLAT leaf boxes (z = [-1, +1]) are read by the records: they go first.
template <class T> int refresh_caches(Tree<T>* tree) {
    if (tree->dims == 2) BVH_TRY(dim2_finish_build(tree));
    BVH_TRY(build_traversal_records(tree));
    if (tree->have_flat) BVH_TRY(build_flat(tree));
    return BVHGPU_OK;
}

// Caches that depend on the node count or the shape numbering: dropped, rebuilt lazily (or here) for the new tree.
template <class T> int finish_relayout(Tree<T>* tree) {
    bvhgpu_ctx* ctx = tree->ctx;
    dfree(ctx, tree->d_arrive); tree->d_arrive = nullptr;                   // all-zero between calls: reallocated (zeroed) by the next update
    dfree(ctx, tree->d_bad); tree->d_bad = nullptr;
    dfree(ctx, tree->d_tnodes); tree->d_tnodes = nullptr; tree->n_trec = 0;
    dfree(ctx, tree->d_flat); tree->d_flat = nullptr; tree->n_flat = 0;
    tree->top_valid = false;
    tree->last_total = 0; tree->last_nrays = 0; tree->last_visits = 0;       // the retained traversal result refers to the old numbering
    if (tree->dims == 2) {                                                    // the FLAT leaf boxes (z = [-1, +1]), read by the records, at the new n
        dfree(ctx, tree->d_aabb_trav); tree->d_aabb_trav = nullptr;
        BVH_TRY(dim2_finish_build(tree));
    }
    BVH_TRY(build_traversal_records(tree));
    if (tree->have_flat) BVH_TRY(build_flat(tree));
    return BVHGPU_OK;
}

// The group subtrees of an add: the exact builder restarted from the group roots (centre bounds per root).  The status counts growth
// rebuilds only, so the count of this run is cleared.
template <class T> static int build_subtrees(Tree<T>* tree, const uint32_t* d_roots, const uint32_t* d_n_roots, uint32_t, const T* cb, uint32_t* idx,
                                             const char*) {
    BVH_TRY(rebuild_subtrees(tree->ctx, tree, d_roots, d_n_roots, cb, idx, true));
    BVH_CUDA_TRY(cudaMemsetAsync(&tree->d_status->rebuilt, 0, sizeof(uint32_t), tree->ctx->stream));
    return BVHGPU_OK;
}

// status->error of the first of two builder runs in one call survives the second run
__global__ void keep_error_kernel(BuildStatus* status, uint32_t* saved, int restore) {
    if (threadIdx.x) return;
    if (!restore) *saved = status->error;
    else if (*saved && !status->error) status->error = *saved;
}
// An add that runs the builder twice (group subtrees, growth rebuild) keeps the first run's error in a 3-D tree's deferred status.
// A 4-D build reports its errors synchronously.
template <class T> static int keep_build_error(Tree<T>* tree, uint32_t* saved, bool restore) {
    keep_error_kernel<<<1, 32, 0, tree->ctx->stream>>>(tree->d_status, saved, restore ? 1 : 0);
    tree->ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}
template <class T> static int keep_build_error(Tree4<T>*, uint32_t*, bool) { return BVHGPU_OK; }

// The per-shape geometry a tree carries: the triangles of a 3-D tree (bvhgpu_tree_set_triangles_*, DTri<T>) or the segments of a 2-D
// tree (bvhgpu_tree_set_segments_*, DSeg<T>).  A removal permutes it with the boxes (*words: its size in 16-byte words), an add drops
// it (the new shapes' geometry is unknown until it is set again).
template <class T> static const void* geometry(const Tree<T>* tree, uint32_t* words) {
    *words = (uint32_t)((tree->dims == 2 ? sizeof(DSeg<T>) : sizeof(DTri<T>)) / 16);
    return tree->dims == 2 ? tree->d_segs : tree->d_tris;
}
template <class T> static const void* geometry(const Tree4<T>*, uint32_t* words) { *words = 0; return nullptr; }
template <class T> static void swap_geometry(Tree<T>* tree, void* g) {
    void*& slot = tree->dims == 2 ? tree->d_segs : tree->d_tris;
    dfree(tree->ctx, slot);
    slot = g;
}
template <class T> static void swap_geometry(Tree4<T>*, void*) {}

// ---- refit and update_shapes (Bvh::update_shapes, src/bvh/optimization.rs:304-351; DESIGN.md section 4.12) ----------------------
template <class TreeT> int check_boxes(TreeT* tree, const uint32_t* d_changed, const typename TreeT::Aabb* d_fresh, uint32_t m, Scratch& scratch,
                                       const char* who) {
    bvhgpu_ctx* ctx = tree->ctx;
    uint32_t* flags = nullptr;
    BVH_TRY(scratch.get(&flags, 2));
    BVH_CUDA_TRY(cudaMemsetAsync(flags, 0, 2 * sizeof(uint32_t), ctx->stream));
    check_boxes_kernel<TreeT::D, typename TreeT::Scalar><<<(m + 255) / 256, 256, 0, ctx->stream>>>(d_changed, d_fresh, m, tree->n, flags);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    uint32_t* h = ctx->h_pinned + 208;
    BVH_CUDA_TRY(cudaMemcpyAsync(h, flags, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (h[1]) { set_error("%s: a changed shape index is >= %u; the tree was left unchanged", who, tree->n); return BVHGPU_ERR_INVALID; }
    if (h[0]) { set_error("%s: NaN coordinate in a new AABB; the tree was left unchanged", who); return BVHGPU_ERR_NAN; }
    return BVHGPU_OK;
}

template <class TreeT> int scatter_boxes(TreeT* tree, const uint32_t* d_changed, const typename TreeT::Aabb* d_fresh, uint32_t m) {
    bvhgpu_ctx* ctx = tree->ctx;
    scatter_boxes_kernel<<<(m + 255) / 256, 256, 0, ctx->stream>>>(d_changed, d_fresh, m, tree->d_aabb);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}

template <class TreeT> int ensure_sa_base(TreeT* tree) {
    if (tree->d_sa_base || tree->n_nodes == 0) return BVHGPU_OK;
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_TRY(dalloc_t(ctx, &tree->d_sa_base, tree->n_nodes));
    node_sa_kernel<TreeT::D><<<(tree->n_nodes + 255) / 256, 256, 0, ctx->stream>>>(tree->d_nodes, tree->n_nodes, tree->d_sa_base);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}

template <class TreeT> int refit(TreeT* tree) {
    using T = typename TreeT::Scalar;
    bvhgpu_ctx* ctx = tree->ctx;
    if (tree->n >= 2) {
        Scratch scratch(ctx);
        uint32_t* arrivals = nullptr;
        BVH_TRY(scratch.get(&arrivals, tree->n_nodes));
        BVH_CUDA_TRY(cudaMemsetAsync(arrivals, 0, sizeof(uint32_t) * tree->n_nodes, ctx->stream));
        refit_kernel<TreeT::D, T, false><<<(tree->n + 255) / 256, 256, 0, ctx->stream>>>(tree->d_nodes, tree->d_node_index, tree->d_aabb, tree->n,
                                                                                        arrivals, nullptr);
        ctx->launches++;
        BVH_CUDA_TRY(cudaGetLastError());
    }
    return refresh_caches(tree);                                               // n = 1: the root record holds the shape's own box
}

template <class TreeT> int update_incremental(TreeT* tree, const uint32_t* d_changed, uint32_t m, double max_growth, size_t* rebuilt) {
    using T = typename TreeT::Scalar;
    using Node = typename TreeT::Node;
    bvhgpu_ctx* ctx = tree->ctx;
    cudaStream_t st = ctx->stream;
    const uint32_t nn = tree->n_nodes;
    const bool rebuild = max_growth > 0.0;
    if (tree->n < 3) return refit(tree);                                      // one or two shapes: nothing a rebuild could change
    if (!tree->d_arrive) {
        BVH_TRY(dalloc_t(ctx, &tree->d_arrive, nn));
        BVH_CUDA_TRY(cudaMemsetAsync(tree->d_arrive, 0, sizeof(uint32_t) * nn, st));
    }
    if (rebuild && !tree->d_bad) {
        BVH_TRY(dalloc_t(ctx, &tree->d_bad, nn));
        BVH_CUDA_TRY(cudaMemsetAsync(tree->d_bad, 0, nn, st));
    }
    if (rebuild) BVH_TRY(ensure_sa_base(tree));                               // first update on this tree: the baseline is the tree before the motion
    Scratch scratch(ctx);
    uint32_t *dirty = nullptr, *cnts = nullptr;
    BVH_TRY(scratch.get(&dirty, nn));
    BVH_TRY(scratch.get(&cnts, 2));                                           // [0] dirty nodes, [1] rebuild roots
    BVH_CUDA_TRY(cudaMemsetAsync(cnts, 0, 2 * sizeof(uint32_t), st));
    const unsigned gm = (m + 255) / 256;
    mark_paths_kernel<Node><<<gm, 256, 0, st>>>(tree->d_nodes, tree->d_node_index, d_changed, m, tree->d_arrive);
    climb_paths_kernel<TreeT::D, T><<<gm, 256, 0, st>>>(tree->d_nodes, tree->d_node_index, tree->d_aabb, d_changed, m, tree->d_arrive,
                                                        tree->d_sa_base, (T)max_growth, rebuild ? tree->d_bad : nullptr, dirty, cnts);
    ctx->launches += 2;
    BVH_CUDA_TRY(cudaGetLastError());
    if (rebuild) BVH_TRY(rebuild_degraded(tree, dirty, cnts, rebuilt, "update"));
    return refresh_caches(tree);
}

// ---- add_shapes / remove_shapes (Bvh::add_shape / Bvh::remove_shape, src/bvh/optimization.rs:67-301; DESIGN.md section 4.13) ----
template <class TreeT> int add_shapes(TreeT* tree, typename TreeT::Box* aabb_all, uint32_t k, double max_growth, size_t* rebuilt) {
    using T = typename TreeT::Scalar;
    using Node = typename TreeT::Node;
    constexpr int D = TreeT::D;
    using CB = typename std::conditional<D == 4, typename Traits<T>::Key, T>::type;   // centre bounds of a group root, as its builder takes them
    bvhgpu_ctx* ctx = tree->ctx;
    cudaStream_t st = ctx->stream;
    const uint32_t n = tree->n, nn = tree->n_nodes, nn2 = nn + 2 * k, N = n + k;
    const bool rebuild = max_growth > 0.0;
    const int wave = std::max(ctx->sm_count, 1) * 8;
    if (rebuild) BVH_TRY(ensure_sa_base(tree));                               // baseline = the tree before the call
    T* sa_old = tree->d_sa_base;
    Scratch scratch(ctx);
    uint32_t *point = nullptr, *ng = nullptr;
    BVH_TRY(scratch.get(&point, k));
    // [0] groups, [1] group subtrees to build, [2] dirty nodes, [3] growth rebuild roots, [4] saved build error, [5] nodes that failed the growth test
    BVH_TRY(scratch.get(&ng, 6));
    BVH_CUDA_TRY(cudaMemsetAsync(ng, 0, 6 * sizeof(uint32_t), st));
    descend_kernel<D, T><<<(k + 255) / 256, 256, 0, st>>>(tree->d_nodes, aabb_all, n, k, point);
    ctx->launches++;
    Groups G;
    BVH_TRY(group_insertions(ctx, scratch, point, k, nn, ng, &G));
    // scratch of the relocation, then the new arrays (freed again if nothing can be launched)
    Scratch scratch2(ctx);
    uint32_t *idx = nullptr, *roots = nullptr, *gbase = nullptr, *arrive = nullptr, *dirty = nullptr;
    uint8_t* aff = nullptr;
    CB* cb = nullptr;
    BVH_TRY(scratch2.get(&aff, nn2));
    BVH_TRY(scratch2.get(&idx, (D == 4 ? 2 : 1) * (size_t)N));                // the groups' shapes in leaf order (the 4-D builder's two index buffers)
    BVH_TRY(scratch2.get(&roots, k));
    BVH_TRY(scratch2.get(&gbase, k));
    BVH_TRY(scratch2.get(&cb, 2 * D * (size_t)k));
    BVH_TRY(scratch2.get(&arrive, nn2));
    BVH_TRY(scratch2.get(&dirty, nn2));
    Node* nw = nullptr;
    uint32_t *nstart = nullptr, *nidx = nullptr;
    T* sa_new = nullptr;
    int rc = dalloc_t(ctx, &nw, nn2);
    if (rc == BVHGPU_OK) rc = dalloc_t(ctx, &nstart, nn2);
    if (rc == BVHGPU_OK) rc = dalloc_t(ctx, &nidx, N);
    if (rc == BVHGPU_OK && sa_old) rc = dalloc_t(ctx, &sa_new, nn2);
    if (rc == BVHGPU_OK && cudaMemsetAsync(aff, 0, nn2, st) != cudaSuccess) rc = BVHGPU_ERR_CUDA;
    if (rc == BVHGPU_OK) {
        graft_relayout_kernel<D, T><<<(nn + 255) / 256, 256, 0, st>>>(tree->d_nodes, tree->d_node_start, sa_old, nn, G.a, G.S, nw, nstart, nidx, aff, sa_new);
        graft_groups_kernel<D, T><<<wave, 256, 0, st>>>(G.uniq, G.cnt, G.goff, ng, G.sshape, tree->d_node_start, G.S, aabb_all, n,
                                                        nw, nstart, nidx, idx, roots, ng + 1, cb, gbase);
        ctx->launches += 2;
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) { set_error("add_shapes: %s", cudaGetErrorString(e)); rc = BVHGPU_ERR_CUDA; }
    }
    if (rc != BVHGPU_OK) { dfree(ctx, nw); dfree(ctx, nstart); dfree(ctx, nidx); dfree(ctx, sa_new); return rc; }
    // the tree now is the new one (its boxes on the affected paths are still to be recomputed); from here on a failure leaves it
    // half-done, and the caller marks it failed
    dfree(ctx, tree->d_nodes); dfree(ctx, tree->d_node_start); dfree(ctx, tree->d_node_index); dfree(ctx, tree->d_aabb); dfree(ctx, tree->d_sa_base);
    swap_geometry(tree, nullptr);
    tree->d_nodes = nw; tree->d_node_start = nstart; tree->d_node_index = nidx; tree->d_aabb = aabb_all; tree->d_sa_base = sa_new;
    tree->n = N; tree->n_nodes = nn2;
    uint32_t* h = ctx->h_pinned + 220;
    BVH_CUDA_TRY(cudaMemcpyAsync(h, ng + 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    BVH_CUDA_TRY(cudaStreamSynchronize(st));
    if (*h) BVH_TRY(build_subtrees(tree, roots, ng + 1, k, cb, idx, "add_shapes"));   // exact-SAH subtrees of the groups with >= 2 shapes
    // boxes of the affected paths (+ the growth test)
    BVH_CUDA_TRY(cudaMemsetAsync(arrive, 0, sizeof(uint32_t) * nn2, st));
    if (rebuild) {
        dfree(ctx, tree->d_bad);                                               // (an earlier update's flags, sized for the old tree)
        tree->d_bad = nullptr;
        BVH_TRY(dalloc_t(ctx, &tree->d_bad, nn2));
        BVH_CUDA_TRY(cudaMemsetAsync(tree->d_bad, 0, nn2, st));
    }
    climb_affected_kernel<D, T><<<(nn2 + 255) / 256, 256, 0, st>>>(tree->d_nodes, nn2, aff, tree->d_aabb, arrive, sa_new, (T)max_growth,
                                                                 rebuild ? tree->d_bad : nullptr, ng + 5, dirty, ng + 2);
    ctx->launches++;
    if (sa_new) { graft_rebase_kernel<D, T><<<wave, 256, 0, st>>>(tree->d_nodes, gbase, G.cnt, ng, sa_new); ctx->launches++; }
    BVH_CUDA_TRY(cudaGetLastError());
    if (rebuild) {
        BVH_CUDA_TRY(cudaMemcpyAsync(h, ng + 5, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        BVH_CUDA_TRY(cudaStreamSynchronize(st));
        if (*h) {                                                              // a node failed the growth test
            BVH_TRY(keep_build_error(tree, ng + 4, false));
            BVH_TRY(rebuild_degraded(tree, dirty, ng + 2, rebuilt, "add_shapes"));
            BVH_TRY(keep_build_error(tree, ng + 4, true));
        }
    }
    return finish_relayout(tree);                                              // (the growth flags: all clear again, dropped with the counters)
}

template <class TreeT> int remove_shapes(TreeT* tree, const uint32_t* d_rm, uint32_t k) {
    using T = typename TreeT::Scalar;
    using Node = typename TreeT::Node;
    using Box = typename TreeT::Box;
    bvhgpu_ctx* ctx = tree->ctx;
    cudaStream_t st = ctx->stream;
    const uint32_t n = tree->n, nn = tree->n_nodes, m = n - k, nn2 = m ? 2 * m - 1 : 0;
    if (m == 0) {                                                              // everything goes: the tree of an n == 0 build
        dfree(ctx, tree->d_nodes); dfree(ctx, tree->d_node_start); dfree(ctx, tree->d_node_index); dfree(ctx, tree->d_aabb); dfree(ctx, tree->d_sa_base);
        swap_geometry(tree, nullptr);
        tree->d_nodes = nullptr; tree->d_node_start = nullptr; tree->d_node_index = nullptr; tree->d_aabb = nullptr; tree->d_sa_base = nullptr;
        tree->n = 0; tree->n_nodes = 0;
        return finish_relayout(tree);
    }
    Scratch scratch(ctx);
    uint32_t *flag = nullptr, *newidx = nullptr, *arrive = nullptr;
    uint8_t* aff = nullptr;
    Ranks rk;
    BVH_TRY(remove_ranks(ctx, scratch, d_rm, n, k, tree->d_node_index, tree->d_node_start, &rk));
    BVH_TRY(scratch.get(&flag, (size_t)nn + 1));
    BVH_TRY(scratch.get(&newidx, (size_t)nn + 1));
    BVH_TRY(scratch.get(&aff, nn2));
    BVH_TRY(scratch.get(&arrive, nn2));
    BVH_CUDA_TRY(cudaMemsetAsync(arrive, 0, sizeof(uint32_t) * nn2, st));
    survive_kernel<<<(nn + 256) / 256, 256, 0, st>>>(tree->d_nodes, tree->d_node_start, nn, rk.R, flag);
    ctx->launches++;
    BVH_TRY(exclusive_sum_u32(scratch, flag, newidx, (size_t)nn + 1, st));
    uint32_t t_words = 0;
    const void* tris = geometry(tree, &t_words);
    Node* nw = nullptr;
    uint32_t *nstart = nullptr, *nidx = nullptr;
    Box* a_new = nullptr;
    T* sa_new = nullptr;
    void* t_new = nullptr;
    int rc = dalloc_t(ctx, &nw, nn2);
    if (rc == BVHGPU_OK) rc = dalloc_t(ctx, &nstart, nn2);
    if (rc == BVHGPU_OK) rc = dalloc_t(ctx, &nidx, m);
    if (rc == BVHGPU_OK) rc = dalloc_t(ctx, &a_new, m);
    if (rc == BVHGPU_OK && tree->d_sa_base) rc = dalloc_t(ctx, &sa_new, nn2);
    if (rc == BVHGPU_OK && tris) rc = dalloc(ctx, &t_new, 16 * (size_t)t_words * m);
    if (rc != BVHGPU_OK) { dfree(ctx, nw); dfree(ctx, nstart); dfree(ctx, nidx); dfree(ctx, a_new); dfree(ctx, sa_new); dfree(ctx, t_new); return rc; }
    contract_kernel<T><<<(nn + 255) / 256, 256, 0, st>>>(tree->d_nodes, tree->d_node_start, nn, rk.R, newidx, m, rk.Rm, rk.holes,
                                                          tree->d_sa_base, nw, nstart, nidx, aff, sa_new);
    permute_shapes_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_rm, n, m, rk.Rm, rk.holes, tree->d_aabb, a_new, static_cast<const uint4*>(tris),
                                                           static_cast<uint4*>(t_new), t_words);
    ctx->launches += 2;
    dfree(ctx, tree->d_nodes); dfree(ctx, tree->d_node_start); dfree(ctx, tree->d_node_index); dfree(ctx, tree->d_aabb); dfree(ctx, tree->d_sa_base);
    swap_geometry(tree, t_new);
    tree->d_nodes = nw; tree->d_node_start = nstart; tree->d_node_index = nidx; tree->d_aabb = a_new; tree->d_sa_base = sa_new;
    tree->n = m; tree->n_nodes = nn2;
    if (nn2 > 1) {
        climb_affected_kernel<TreeT::D, T><<<(nn2 + 255) / 256, 256, 0, st>>>(tree->d_nodes, nn2, aff, tree->d_aabb, arrive, nullptr, T(0), nullptr,
                                                                            nullptr, nullptr, nullptr);
        ctx->launches++;
    }
    BVH_CUDA_TRY(cudaGetLastError());
    return finish_relayout(tree);
}

// ---- validation (before the tree is touched) -------------------------------------------------------------------------------------
// flags[0]: an index >= n, flags[1]: an index listed twice.  rm[n + 1] (zeroed by the caller) = removed flag of every shape.
__global__ void __launch_bounds__(256) remove_check_kernel(const uint32_t* __restrict__ idx, uint32_t k, uint32_t n, uint32_t* __restrict__ rm, uint32_t* __restrict__ flags) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= k) return;
    const uint32_t s = idx[i];
    if (s >= n) { atomicExch(flags, 1u); return; }
    if (atomicExch(rm + s, 1u) != 0u) atomicExch(flags + 1, 1u);
}
int remove_check(bvhgpu_ctx* ctx, const uint32_t* d_idx, uint32_t k, uint32_t n, uint32_t* d_rm, uint32_t* d_flags) {
    remove_check_kernel<<<(k + 255) / 256, 256, 0, ctx->stream>>>(d_idx, k, n, d_rm, d_flags);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}

#define INST(TREE)                                                                                                              \
    template int check_boxes<TREE>(TREE*, const uint32_t*, const TREE::Aabb*, uint32_t, Scratch&, const char*);                   \
    template int scatter_boxes<TREE>(TREE*, const uint32_t*, const TREE::Aabb*, uint32_t);                                          \
    template int ensure_sa_base<TREE>(TREE*);                                                                                       \
    template int refit<TREE>(TREE*);                                                                                                \
    template int update_incremental<TREE>(TREE*, const uint32_t*, uint32_t, double, size_t*);                                       \
    template int add_shapes<TREE>(TREE*, TREE::Box*, uint32_t, double, size_t*);                                                   \
    template int remove_shapes<TREE>(TREE*, const uint32_t*, uint32_t);
INST(Tree<float>)
INST(Tree<double>)
INST(Tree4<float>)
INST(Tree4<double>)
#undef INST
template int refresh_caches<float>(Tree<float>*);
template int refresh_caches<double>(Tree<double>*);

}  // namespace bvhb200
