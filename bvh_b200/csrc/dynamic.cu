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
// subtrees in place.  The kernels that touch nodes or boxes are generic in D (dynamic.cuh); the drivers here instantiate D = 3, the
// 4-D drivers are in dim4.cu.
#include "internal.h"
#include "dynamic.cuh"
#include <cub/device/device_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>

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

// Caches that depend on the node count or the shape numbering: dropped, rebuilt lazily (or here) for the new tree.
template <class T> static int finish_relayout(Tree<T>* tree) {
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

// status->error of the first of two builder runs in one call survives the second run
__global__ void keep_error_kernel(BuildStatus* status, uint32_t* saved, int restore) {
    if (threadIdx.x) return;
    if (!restore) *saved = status->error;
    else if (*saved && !status->error) status->error = *saved;
}

template <class T>
int add_shapes(Tree<T>* tree, typename Traits<T>::DAabb* aabb_all, uint32_t k, double max_growth) {
    using Node = typename Traits<T>::Node;
    bvhgpu_ctx* ctx = tree->ctx;
    cudaStream_t st = ctx->stream;
    const uint32_t n = tree->n, nn = tree->n_nodes, nn2 = nn + 2 * k;
    const bool rebuild = max_growth > 0.0;
    if (rebuild) BVH_TRY(ensure_sa_base(tree));                                // baseline = the tree before the call
    T* sa_old = reinterpret_cast<T*>(tree->d_sa_base);
    Scratch scratch(ctx);
    uint32_t *point = nullptr, *ng = nullptr;
    BVH_TRY(scratch.get(&point, k));
    // [0] groups, [1] group subtrees to build, [2] dirty nodes, [3] growth rebuild roots, [4] saved status, [5] nodes that failed the growth test
    BVH_TRY(scratch.get(&ng, 6));
    BVH_CUDA_TRY(cudaMemsetAsync(ng, 0, 6 * sizeof(uint32_t), st));
    const unsigned gk = (k + 255) / 256, gn = (nn + 255) / 256, gn2 = (nn2 + 255) / 256;
    descend_kernel<3, T><<<gk, 256, 0, st>>>(tree->d_nodes, aabb_all, n, k, point);
    ctx->launches++;
    Groups G;
    BVH_TRY(group_insertions(ctx, scratch, point, k, nn, ng, &G));
    uint32_t *sshape = G.sshape, *uniq = G.uniq, *cnt = G.cnt, *goff = G.goff, *a = G.a, *S = G.S;
    // scratch of the relocation, then the new arrays (freed again if nothing can be launched)
    Scratch scratch2(ctx);
    uint32_t *idx0 = nullptr, *roots = nullptr, *gbase = nullptr, *arrive = nullptr, *dirty = nullptr;
    uint8_t* aff = nullptr;
    T* cb_roots = nullptr;
    BVH_TRY(scratch2.get(&aff, nn2));
    BVH_TRY(scratch2.get(&idx0, (size_t)n + k));
    BVH_TRY(scratch2.get(&roots, k));
    BVH_TRY(scratch2.get(&gbase, k));
    BVH_TRY(scratch2.get(&cb_roots, 6 * (size_t)k));
    BVH_TRY(scratch2.get(&arrive, nn2));
    BVH_TRY(scratch2.get(&dirty, nn2));
    Node* nw = nullptr;
    uint32_t *nstart = nullptr, *nidx = nullptr;
    T* sa_new = nullptr;
    int rc = dalloc_t(ctx, &nw, nn2);
    if (rc == BVHGPU_OK) rc = dalloc_t(ctx, &nstart, nn2);
    if (rc == BVHGPU_OK) rc = dalloc_t(ctx, &nidx, (size_t)n + k);
    if (rc == BVHGPU_OK && sa_old) rc = dalloc(ctx, (void**)&sa_new, sizeof(T) * nn2);
    if (rc == BVHGPU_OK && cudaMemsetAsync(aff, 0, nn2, st) != cudaSuccess) rc = BVHGPU_ERR_CUDA;
    if (rc == BVHGPU_OK) {
        graft_relayout_kernel<3, T><<<gn, 256, 0, st>>>(tree->d_nodes, tree->d_node_start, sa_old, nn, a, S, nw, nstart, nidx, aff, sa_new);
        graft_groups_kernel<3, T><<<std::max(1, ctx->sm_count * 8), 256, 0, st>>>(uniq, cnt, goff, ng, sshape, tree->d_node_start, S, aabb_all, n,
                                                                                nw, nstart, nidx, idx0, roots, ng + 1, cb_roots, gbase);
        ctx->launches += 3;
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) { set_error("add_shapes: %s", cudaGetErrorString(e)); rc = BVHGPU_ERR_CUDA; }
    }
    if (rc != BVHGPU_OK) { dfree(ctx, nw); dfree(ctx, nstart); dfree(ctx, nidx); dfree(ctx, sa_new); return rc; }
    // the tree now is the new one (its boxes on the affected paths are still to be recomputed); from here on a failure leaves it
    // half-done, and the caller marks it failed
    dfree(ctx, tree->d_nodes); dfree(ctx, tree->d_node_start); dfree(ctx, tree->d_node_index); dfree(ctx, tree->d_aabb); dfree(ctx, tree->d_sa_base);
    dfree(ctx, tree->d_tris); tree->d_tris = nullptr;                          // triangles of the new shapes are unknown: set them again
    tree->d_nodes = nw; tree->d_node_start = nstart; tree->d_node_index = nidx; tree->d_aabb = aabb_all; tree->d_sa_base = sa_new;
    tree->n = n + k; tree->n_nodes = nn2;
    uint32_t* h = ctx->h_pinned + 220;
    BVH_CUDA_TRY(cudaMemcpyAsync(h, ng + 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    BVH_CUDA_TRY(cudaStreamSynchronize(st));
    const bool groups = *h != 0;
    if (groups) BVH_TRY(rebuild_subtrees(ctx, tree, roots, ng + 1, cb_roots, idx0, true));     // exact-SAH subtrees of the groups with >= 2 shapes
    // boxes of the affected paths (+ the growth test)
    BVH_CUDA_TRY(cudaMemsetAsync(arrive, 0, sizeof(uint32_t) * nn2, st));
    if (rebuild) {
        dfree(ctx, tree->d_bad);                                               // (an earlier update's flags, sized for the old tree)
        tree->d_bad = nullptr;
        BVH_TRY(dalloc_t(ctx, &tree->d_bad, nn2));
        BVH_CUDA_TRY(cudaMemsetAsync(tree->d_bad, 0, nn2, st));
    }
    climb_affected_kernel<3, T><<<gn2, 256, 0, st>>>(tree->d_nodes, nn2, aff, tree->d_aabb, arrive, sa_new, (T)max_growth, rebuild ? tree->d_bad : nullptr,
                                                  ng + 5, dirty, ng + 2);
    ctx->launches++;
    if (sa_new) { graft_rebase_kernel<3, T><<<std::max(1, ctx->sm_count * 8), 256, 0, st>>>(tree->d_nodes, gbase, cnt, ng, sa_new); ctx->launches++; }
    BVH_CUDA_TRY(cudaGetLastError());
    bool grow = false;
    if (rebuild) {
        BVH_CUDA_TRY(cudaMemcpyAsync(h, ng + 5, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        BVH_CUDA_TRY(cudaStreamSynchronize(st));
        grow = *h != 0;                                                        // a node failed the growth test
    }
    if (grow) {
        keep_error_kernel<<<1, 32, 0, st>>>(tree->d_status, ng + 4, 0);
        BVH_TRY(rebuild_degraded(tree, dirty, ng + 2));
        keep_error_kernel<<<1, 32, 0, st>>>(tree->d_status, ng + 4, 1);
        ctx->launches += 2;
    } else if (groups) {                                                       // status->rebuilt counts growth rebuilds only
        BVH_CUDA_TRY(cudaMemsetAsync(&tree->d_status->rebuilt, 0, sizeof(uint32_t), st));
    }
    BVH_CUDA_TRY(cudaGetLastError());
    return finish_relayout(tree);
}

template <class T>
int remove_shapes(Tree<T>* tree, const uint32_t* d_rm, uint32_t k) {
    using Node = typename Traits<T>::Node;
    using DAabb = typename Traits<T>::DAabb;
    bvhgpu_ctx* ctx = tree->ctx;
    cudaStream_t st = ctx->stream;
    const uint32_t n = tree->n, nn = tree->n_nodes, m = n - k, nn2 = m ? 2 * m - 1 : 0;
    const size_t t_words = sizeof(T) == 4 ? 3 : 6;                            // DTri<T> (closest.cu) in 16-byte words
    if (m == 0) {                                                              // everything goes: the tree of an n == 0 build
        dfree(ctx, tree->d_nodes); dfree(ctx, tree->d_node_start); dfree(ctx, tree->d_node_index); dfree(ctx, tree->d_aabb);
        dfree(ctx, tree->d_sa_base); dfree(ctx, tree->d_tris);
        tree->d_nodes = nullptr; tree->d_node_start = nullptr; tree->d_node_index = nullptr; tree->d_aabb = nullptr;
        tree->d_sa_base = nullptr; tree->d_tris = nullptr;
        tree->n = 0; tree->n_nodes = 0;
        return finish_relayout(tree);
    }
    Scratch scratch(ctx);
    uint32_t *flag = nullptr, *newidx = nullptr, *arrive = nullptr;
    uint8_t* aff = nullptr;
    Ranks rk;
    BVH_TRY(remove_ranks(ctx, scratch, d_rm, n, k, tree->d_node_index, tree->d_node_start, &rk));
    const uint32_t *R = rk.R, *Rm = rk.Rm, *holes = rk.holes;
    BVH_TRY(scratch.get(&flag, (size_t)nn + 1));
    BVH_TRY(scratch.get(&newidx, (size_t)nn + 1));
    BVH_TRY(scratch.get(&aff, nn2));
    BVH_TRY(scratch.get(&arrive, nn2));
    BVH_CUDA_TRY(cudaMemsetAsync(arrive, 0, sizeof(uint32_t) * nn2, st));
    const unsigned gs = (n + 255) / 256, gn = (nn + 256) / 256, gn2 = (nn2 + 255) / 256;
    survive_kernel<<<gn, 256, 0, st>>>(tree->d_nodes, tree->d_node_start, nn, R, flag);
    BVH_TRY(exclusive_sum_u32(scratch, flag, newidx, (size_t)nn + 1, st));
    Node* nw = nullptr;
    uint32_t *nstart = nullptr, *nidx = nullptr;
    DAabb* a_new = nullptr;
    T* sa_new = nullptr;
    void* t_new = nullptr;
    int rc = dalloc_t(ctx, &nw, nn2);
    if (rc == BVHGPU_OK) rc = dalloc_t(ctx, &nstart, nn2);
    if (rc == BVHGPU_OK) rc = dalloc_t(ctx, &nidx, m);
    if (rc == BVHGPU_OK) rc = dalloc_t(ctx, &a_new, m);
    if (rc == BVHGPU_OK && tree->d_sa_base) rc = dalloc(ctx, (void**)&sa_new, sizeof(T) * nn2);
    if (rc == BVHGPU_OK && tree->d_tris) rc = dalloc(ctx, &t_new, 16 * t_words * m);
    if (rc != BVHGPU_OK) { dfree(ctx, nw); dfree(ctx, nstart); dfree(ctx, nidx); dfree(ctx, a_new); dfree(ctx, sa_new); dfree(ctx, t_new); return rc; }
    contract_kernel<T><<<(nn + 255) / 256, 256, 0, st>>>(tree->d_nodes, tree->d_node_start, nn, R, newidx, m, Rm, holes,
                                                          reinterpret_cast<const T*>(tree->d_sa_base), nw, nstart, nidx, aff, sa_new);
    permute_shapes_kernel<<<gs, 256, 0, st>>>(d_rm, n, m, Rm, holes, tree->d_aabb, a_new, reinterpret_cast<const uint4*>(tree->d_tris),
                                                 reinterpret_cast<uint4*>(t_new), (uint32_t)t_words);
    ctx->launches += 5;
    dfree(ctx, tree->d_nodes); dfree(ctx, tree->d_node_start); dfree(ctx, tree->d_node_index); dfree(ctx, tree->d_aabb);
    dfree(ctx, tree->d_sa_base); dfree(ctx, tree->d_tris);
    tree->d_nodes = nw; tree->d_node_start = nstart; tree->d_node_index = nidx; tree->d_aabb = a_new; tree->d_sa_base = sa_new; tree->d_tris = t_new;
    tree->n = m; tree->n_nodes = nn2;
    if (nn2 > 1) {
        climb_affected_kernel<3, T><<<gn2, 256, 0, st>>>(tree->d_nodes, nn2, aff, tree->d_aabb, arrive, nullptr, T(0), nullptr, nullptr, nullptr, nullptr);
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

template int add_shapes<float>(Tree<float>*, DAabbF*, uint32_t, double);
template int add_shapes<double>(Tree<double>*, DAabbD*, uint32_t, double);
template int remove_shapes<float>(Tree<float>*, const uint32_t*, uint32_t);
template int remove_shapes<double>(Tree<double>*, const uint32_t*, uint32_t);

}  // namespace bvhb200
