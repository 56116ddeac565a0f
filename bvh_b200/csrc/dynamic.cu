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
// subtrees in place.
#include "internal.h"
#include <cub/device/device_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>

namespace bvhb200 {

template <class T> __device__ __forceinline__ void join3(T mn[3], T mx[3], const T amn[3], const T amx[3]) {
    for (int c = 0; c < 3; ++c) { mn[c] = min_t(mn[c], amn[c]); mx[c] = max_t(mx[c], amx[c]); }
}
template <class A, class T> __device__ __forceinline__ void box_of(const A& a, T mn[3], T mx[3]) {
    for (int c = 0; c < 3; ++c) { mn[c] = a.min[c]; mx[c] = a.max[c]; }
}
template <class A, class T> __device__ __forceinline__ void set_box(A& a, const T mn[3], const T mx[3]) {
    for (int c = 0; c < 3; ++c) { a.min[c] = mn[c]; a.max[c] = mx[c]; }
}
template <class T, class A> __device__ __forceinline__ void set_empty(A& a) {
    for (int c = 0; c < 3; ++c) { a.min[c] = Traits<T>::inf(); a.max[c] = -Traits<T>::inf(); }
}

// ---- add: insertion point of every new shape (optimization.rs:88-207, evaluated against the tree before the call) -------------
template <class T>
__global__ void __launch_bounds__(256) descend_kernel(const typename Traits<T>::Node* __restrict__ nodes, const typename Traits<T>::DAabb* __restrict__ aabb,
                                                      uint32_t n, uint32_t k, uint32_t* __restrict__ point) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= k) return;
    T smn[3], smx[3];
    load_aabb(aabb + n + j, smn, smx);
    const T shape_sa = surface_area(smn, smx);
    uint32_t i = 0;
    for (;;) {
        const typename Traits<T>::Node& nd = nodes[i];
        if (nd.child_l == BVH_INVALID) break;                                  // a leaf: split it
        T lmn[3], lmx[3], rmn[3], rmx[3], le_mn[3], le_mx[3], re_mn[3], re_mx[3], m_mn[3], m_mx[3];
        box_of(nd.l_aabb, lmn, lmx); box_of(nd.r_aabb, rmn, rmx);
        for (int c = 0; c < 3; ++c) {
            le_mn[c] = min_t(lmn[c], smn[c]); le_mx[c] = max_t(lmx[c], smx[c]);
            re_mn[c] = min_t(rmn[c], smn[c]); re_mx[c] = max_t(rmx[c], smx[c]);
            m_mn[c] = min_t(rmn[c], lmn[c]);  m_mx[c] = max_t(rmx[c], lmx[c]);
        }
        const T send_left = add_rn(surface_area(rmn, rmx), surface_area(le_mn, le_mx));
        const T send_right = add_rn(surface_area(lmn, lmx), surface_area(re_mn, re_mx));
        const T merged = add_rn(surface_area(m_mn, m_mx), shape_sa);
        const T min_send = send_left < send_right ? send_left : send_right;
        if (merged < div_rn(mul_rn(min_send, T(3)), T(10))) break;             // merge here: the new shape becomes this node's sibling
        i = send_left < send_right ? nd.child_l : nd.child_r;
    }
    point[j] = i;
}

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

// every old node: its content moves to i + 2 S(i); a graft node is written in front of it when new shapes chose it
template <class T>
__global__ void __launch_bounds__(256) graft_relayout_kernel(const typename Traits<T>::Node* __restrict__ old, const uint32_t* __restrict__ old_start,
                                                             const T* __restrict__ sa_old, uint32_t nn, const uint32_t* __restrict__ a, const uint32_t* __restrict__ S,
                                                             typename Traits<T>::Node* __restrict__ nw, uint32_t* __restrict__ nstart, uint32_t* __restrict__ nidx,
                                                             uint8_t* __restrict__ aff, T* __restrict__ sa_new) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nn) return;
    typename Traits<T>::Node o = old[i];
    const uint32_t ai = a[i], si = S[i], base = i + 2 * (si - ai), pos = base + 2 * ai;
    const bool leaf = o.child_l == BVH_INVALID;
    const uint32_t par = i ? o.parent + 2 * S[o.parent] : 0u;
    uint32_t below = 0, cnt = 1;                                               // new shapes strictly inside the subtree / new shape count
    o.parent = ai ? base : par;
    if (!leaf) {
        const uint32_t c = o.shape, cr = o.child_r;
        below = S[i + 2 * c - 2] - si;
        cnt = c + below;
        o.child_l = pos + 1;
        o.child_r = cr + 2 * (S[cr] - a[cr]);
        o.shape = cnt;
    } else {
        nidx[o.shape] = pos;
    }
    nw[pos] = o;
    nstart[pos] = old_start[i] + si;
    aff[pos] = below ? 1 : 0;
    if (sa_new) sa_new[pos] = sa_old[i];
    if (ai) {
        typename Traits<T>::Node g;
        g.parent = par; g.child_l = base + 1; g.child_r = pos; g.shape = ai + cnt;
        set_empty<T>(g.l_aabb); set_empty<T>(g.r_aabb);                             // written by the climb
        nw[base] = g;
        nstart[base] = old_start[i] + si - ai;
        aff[base] = 1;
        if (sa_new) sa_new[base] = Traits<T>::inf();                          // fresh node: never "degraded"; its baseline is set after the climb
    }
}

// warp-wide bounds of the group's AABBs (centres = false) or of their centres (centres = true)
template <class T>
__device__ __noinline__ void group_bounds(const typename Traits<T>::DAabb* __restrict__ aabb, uint32_t n, const uint32_t* __restrict__ shapes, uint32_t ap,
                                          bool centres, T mn[3], T mx[3]) {
    typename Traits<T>::Key kmn[3] = {Traits<T>::KEY_POS_INF, Traits<T>::KEY_POS_INF, Traits<T>::KEY_POS_INF};
    typename Traits<T>::Key kmx[3] = {Traits<T>::KEY_NEG_INF, Traits<T>::KEY_NEG_INF, Traits<T>::KEY_NEG_INF};
    for (uint32_t j = lane_id(); j < ap; j += 32) {
        T a[3], b[3];
        load_aabb(aabb + n + shapes[j], a, b);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const T lo = centres ? center1(a[c], b[c]) : a[c], hi = centres ? lo : b[c];
            const auto klo = f2key(lo), khi = f2key(hi);
            kmn[c] = klo < kmn[c] ? klo : kmn[c];
            kmx[c] = khi > kmx[c] ? khi : kmx[c];
        }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) { mn[c] = key2f(warp_min_key(kmn[c])); mx[c] = key2f(warp_max_key(kmx[c])); }
}

// one warp per group: the left child of its graft node -- a leaf (a_p = 1) or the root placeholder of an exact-SAH rebuild over the
// group's shapes in ascending index order (count, box, parent and start are what rebuild_subtrees reads from it)
template <class T>
__global__ void __launch_bounds__(256) graft_groups_kernel(const uint32_t* __restrict__ uniq, const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ goff,
                                                           const uint32_t* __restrict__ n_groups, const uint32_t* __restrict__ sorted_shape,
                                                           const uint32_t* __restrict__ old_start, const uint32_t* __restrict__ S,
                                                           const typename Traits<T>::DAabb* __restrict__ aabb, uint32_t n,
                                                           typename Traits<T>::Node* __restrict__ nw, uint32_t* __restrict__ nstart, uint32_t* __restrict__ nidx,
                                                           uint32_t* __restrict__ idx0, uint32_t* __restrict__ roots, uint32_t* __restrict__ n_roots,
                                                           T* __restrict__ cb_roots, uint32_t* __restrict__ gbase) {
    using Tr = Traits<T>;
    const uint32_t warps = gridDim.x * (blockDim.x >> 5), ng = *n_groups;
    for (uint32_t g = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); g < ng; g += warps) {
        const uint32_t p = uniq[g], ap = cnt[g], off = goff[g];
        const uint32_t base = p + 2 * (S[p] - ap), L = base + 1, start = old_start[p] + S[p] - ap;
        T bmn[3], bmx[3], cmn[3], cmx[3];
        group_bounds<T>(aabb, n, sorted_shape + off, ap, false, bmn, bmx);     // the group's box, then the bounds of its centres
        group_bounds<T>(aabb, n, sorted_shape + off, ap, true, cmn, cmx);
        if (ap > 1) for (uint32_t j = lane_id(); j < ap; j += 32) idx0[start + j] = n + sorted_shape[off + j];
        if (lane_id() != 0) continue;
        gbase[g] = base;
        typename Tr::Node& l = nw[L];                                         // written field by field: no 112-byte node in registers
        l.parent = base;
        l.child_r = BVH_INVALID;
        set_empty<T>(l.r_aabb);
        nstart[L] = start;
        if (ap == 1) {
            const uint32_t s = n + sorted_shape[off];
            l.child_l = BVH_INVALID; l.shape = s;
            set_empty<T>(l.l_aabb);
            nidx[s] = L;
        } else {
            l.child_l = L + 1; l.shape = ap;
            set_box(l.l_aabb, bmn, bmx);
            const uint32_t slot = atomicAdd(n_roots, 1u);
            roots[slot] = L;
            #pragma unroll
            for (int c = 0; c < 3; ++c) { cb_roots[6 * (size_t)slot + c] = cmn[c]; cb_roots[6 * (size_t)slot + 3 + c] = cmx[c]; }
        }
    }
}

// Fresh surface-area baselines of the graft ranges [G, G + 2 a_p): the graft node and the new subtree below its left side.
template <class T>
__global__ void __launch_bounds__(256) graft_rebase_kernel(const typename Traits<T>::Node* __restrict__ nodes, const uint32_t* __restrict__ gbase,
                                                           const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ n_groups, T* __restrict__ sa) {
    const uint32_t warps = gridDim.x * (blockDim.x >> 5), ng = *n_groups;
    for (uint32_t g = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); g < ng; g += warps) {
        const uint32_t b = gbase[g], e = b + 2 * cnt[g];
        for (uint32_t i = b + lane_id(); i < e; i += 32) {
            const typename Traits<T>::Node& nd = nodes[i];
            if (nd.child_l == BVH_INVALID) { sa[i] = T(0); continue; }
            T mn[3], mx[3], bmn[3], bmx[3];
            box_of(nd.l_aabb, mn, mx); box_of(nd.r_aabb, bmn, bmx);
            join3(mn, mx, bmn, bmx);
            sa[i] = surface_area(mn, mx);
        }
    }
}

// ---- the climb over the affected nodes ------------------------------------------------------------------------------------------
// Affected nodes (aff = 1) are closed under "parent of": every ancestor of an affected node is affected.  Both child slots of an
// affected node are rewritten.  The climbs start at the unaffected children of affected nodes, whose box is known (a leaf: its shape's
// AABB; an inner node: the join of its own child slots, as get_node_aabb, bvh_node.rs:616-625); every climb writes its box into the
// parent's slot, and the second arrival at a node joins both slots and carries on.  bad != nullptr: growth test against sa_base as
// bvhgpu_update_* does (n_bad counts the failures); every affected node is logged in `dirty`.
template <class T>
__global__ void __launch_bounds__(256) climb_affected_kernel(typename Traits<T>::Node* nodes, uint32_t nn, const uint8_t* __restrict__ aff,
                                                             const typename Traits<T>::DAabb* __restrict__ aabb, uint32_t* __restrict__ arrive,
                                                             const T* __restrict__ sa_base, T max_growth, uint8_t* __restrict__ bad, uint32_t* __restrict__ n_bad,
                                                             uint32_t* __restrict__ dirty, uint32_t* __restrict__ n_dirty) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j == 0 || j >= nn || aff[j]) return;
    if (!aff[nodes[j].parent]) return;
    T mn[3], mx[3];
    {
        const typename Traits<T>::Node& nd = nodes[j];                     // not affected: nothing writes it during this kernel
        if (nd.child_l == BVH_INVALID) load_aabb(aabb + nd.shape, mn, mx);
        else { T bmn[3], bmx[3]; box_of(nd.l_aabb, mn, mx); box_of(nd.r_aabb, bmn, bmx); join3(mn, mx, bmn, bmx); }
    }
    uint32_t node = j;
    for (;;) {
        const uint32_t p = __ldcg(&nodes[node].parent);
        typename Traits<T>::Node* pn = nodes + p;
        const bool is_left = __ldcg(&pn->child_l) == node;
        auto* dst = is_left ? &pn->l_aabb : &pn->r_aabb;
        for (int c = 0; c < 3; ++c) { __stcg(&dst->min[c], mn[c]); __stcg(&dst->max[c], mx[c]); }
        __threadfence();
        if (atomicAdd(arrive + p, 1u) == 0u) return;                          // the other side is not finished yet
        __threadfence();
        const auto* sib = is_left ? &pn->r_aabb : &pn->l_aabb;
        for (int c = 0; c < 3; ++c) { mn[c] = min_t(__ldcg(&sib->min[c]), mn[c]); mx[c] = max_t(__ldcg(&sib->max[c]), mx[c]); }
        if (bad && surface_area(mn, mx) > mul_rn(max_growth, sa_base[p])) { bad[p] = 1; atomicAdd(n_bad, 1u); }
        if (dirty) dirty[atomicAdd(n_dirty, 1u)] = p;
        if (p == 0) return;
        node = p;
    }
}

// ---- remove ------------------------------------------------------------------------------------------------------------------------
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
// swap rule: a survivor >= m takes the hole of the same rank among the holes (ascending), the others keep their index
__device__ __forceinline__ uint32_t relabel(uint32_t s, uint32_t m, const uint32_t* Rm, const uint32_t* holes) {
    return s < m ? s : holes[(s - m) - (Rm[s] - Rm[m])];
}
// shapes removed below a node: R = exclusive scan of the removed flags by leaf position
template <class T> struct Shrink { uint32_t c, cl, ncl, nc; bool leaf; };
template <class T>
__device__ __forceinline__ Shrink<T> shrink(const typename Traits<T>::Node* nodes, const uint32_t* node_start, const uint32_t* R, uint32_t i) {
    Shrink<T> r;
    const typename Traits<T>::Node& nd = nodes[i];
    const uint32_t s = node_start[i];
    r.leaf = nd.child_l == BVH_INVALID;
    r.c = r.leaf ? 1u : nd.shape;
    r.nc = r.c - (R[s + r.c] - R[s]);
    r.cl = r.ncl = 0;
    if (!r.leaf) {
        r.cl = nodes[i + 1].child_l == BVH_INVALID ? 1u : nodes[i + 1].shape;
        r.ncl = r.cl - (R[s + r.cl] - R[s]);
    }
    return r;
}
template <class T>
__global__ void __launch_bounds__(256) survive_kernel(const typename Traits<T>::Node* __restrict__ nodes, const uint32_t* __restrict__ node_start, uint32_t nn,
                                                      const uint32_t* __restrict__ R, uint32_t* __restrict__ flag) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > nn) return;
    if (i == nn) { flag[i] = 0; return; }
    const Shrink<T> r = shrink<T>(nodes, node_start, R, i);
    flag[i] = r.leaf ? (r.nc == 1u) : (r.ncl > 0 && r.nc > r.ncl);            // an inner node survives when both sides keep a shape
}
// every surviving node writes its own fields at its new index and the parent links of its two new children
template <class T>
__global__ void __launch_bounds__(256) contract_kernel(const typename Traits<T>::Node* __restrict__ old, const uint32_t* __restrict__ old_start, uint32_t nn,
                                                       const uint32_t* __restrict__ R, const uint32_t* __restrict__ newidx,
                                                       uint32_t m, const uint32_t* __restrict__ Rm, const uint32_t* __restrict__ holes,
                                                       const T* __restrict__ sa_old, typename Traits<T>::Node* __restrict__ nw, uint32_t* __restrict__ nstart,
                                                       uint32_t* __restrict__ nidx, uint8_t* __restrict__ aff, T* __restrict__ sa_new) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nn) return;
    const uint32_t j = newidx[i];
    if (newidx[i + 1] == j) return;                                           // removed or spliced out
    const typename Traits<T>::Node& nd = old[i];
    const Shrink<T> r = shrink<T>(old, old_start, R, i);
    typename Traits<T>::Node& o = nw[j];
    o.l_aabb = nd.l_aabb; o.r_aabb = nd.r_aabb;                               // the affected sides are rewritten by the climb
    if (r.leaf) {
        const uint32_t s = relabel(nd.shape, m, Rm, holes);
        o.child_l = BVH_INVALID; o.child_r = BVH_INVALID; o.shape = s;
        nidx[s] = j;
        aff[j] = 0;
    } else {
        o.child_l = j + 1; o.child_r = j + 2 * r.ncl; o.shape = r.nc;
        nw[j + 1].parent = j;
        nw[j + 2 * r.ncl].parent = j;
        aff[j] = r.nc != r.c ? 1 : 0;
    }
    if (j == 0) o.parent = 0;
    nstart[j] = old_start[i] - R[old_start[i]];
    if (sa_new) sa_new[j] = sa_old[i];
}
template <class T>
__global__ void __launch_bounds__(256) permute_shapes_kernel(const uint32_t* __restrict__ rm, uint32_t n, uint32_t m, const uint32_t* __restrict__ Rm,
                                                             const uint32_t* __restrict__ holes, const typename Traits<T>::DAabb* __restrict__ a_old,
                                                             typename Traits<T>::DAabb* __restrict__ a_new, const uint4* __restrict__ t_old,
                                                             uint4* __restrict__ t_new, uint32_t t_words) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n || rm[s]) return;
    const uint32_t d = relabel(s, m, Rm, holes);
    a_new[d] = a_old[s];
    if (t_old) for (uint32_t w = 0; w < t_words; ++w) t_new[(size_t)d * t_words + w] = t_old[(size_t)s * t_words + w];
}

// ---- host side -----------------------------------------------------------------------------------------------------------------
template <class P> static int cub_exclusive_sum(Scratch& scratch, const P* in, P* out, size_t len, cudaStream_t st) {
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, (int64_t)len, st);
    unsigned char* tmp = nullptr;
    BVH_TRY(scratch.get(&tmp, bytes));
    BVH_CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, bytes, in, out, (int64_t)len, st));
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
    uint32_t *point = nullptr, *iota = nullptr, *spoint = nullptr, *sshape = nullptr, *uniq = nullptr, *cnt = nullptr, *goff = nullptr, *ng = nullptr;
    BVH_TRY(scratch.get(&point, k));
    BVH_TRY(scratch.get(&iota, k));
    BVH_TRY(scratch.get(&spoint, k));
    BVH_TRY(scratch.get(&sshape, k));
    BVH_TRY(scratch.get(&uniq, k));
    BVH_TRY(scratch.get(&cnt, (size_t)k + 1));
    BVH_TRY(scratch.get(&goff, (size_t)k + 1));
    // [0] groups, [1] group subtrees to build, [2] dirty nodes, [3] growth rebuild roots, [4] saved status, [5] nodes that failed the growth test
    BVH_TRY(scratch.get(&ng, 6));
    BVH_CUDA_TRY(cudaMemsetAsync(ng, 0, 6 * sizeof(uint32_t), st));
    BVH_CUDA_TRY(cudaMemsetAsync(cnt, 0, ((size_t)k + 1) * sizeof(uint32_t), st));
    const unsigned gk = (k + 255) / 256, gn = (nn + 255) / 256, gn2 = (nn2 + 255) / 256;
    descend_kernel<T><<<gk, 256, 0, st>>>(tree->d_nodes, aabb_all, n, k, point);
    ctx->launches++;
    // group the new shapes by insertion point, ascending shape index inside a group (stable radix sort: deterministic)
    {
        int bits = 1;
        while (bits < 32 && (1ull << bits) < nn) ++bits;
        iota_kernel<<<gk, 256, 0, st>>>(iota, k);
        size_t b1 = 0, b2 = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, b1, point, spoint, iota, sshape, (int)k, 0, bits, st);
        cub::DeviceRunLengthEncode::Encode(nullptr, b2, spoint, uniq, cnt, ng, (int)k, st);
        unsigned char* tmp = nullptr;
        BVH_TRY(scratch.get(&tmp, std::max(b1, b2)));
        BVH_CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, b1, point, spoint, iota, sshape, (int)k, 0, bits, st));
        BVH_CUDA_TRY(cub::DeviceRunLengthEncode::Encode(tmp, b2, spoint, uniq, cnt, ng, (int)k, st));
    }
    BVH_TRY(cub_exclusive_sum(scratch, cnt, goff, (size_t)k + 1, st));
    uint32_t *a = nullptr, *S = nullptr;
    BVH_TRY(scratch.get(&a, nn));
    BVH_TRY(scratch.get(&S, nn));
    BVH_CUDA_TRY(cudaMemsetAsync(a, 0, sizeof(uint32_t) * nn, st));
    group_scatter_kernel<<<gk, 256, 0, st>>>(uniq, cnt, ng, a);
    {
        size_t bytes = 0;
        cub::DeviceScan::InclusiveSum(nullptr, bytes, a, S, (int64_t)nn, st);
        unsigned char* tmp = nullptr;
        BVH_TRY(scratch.get(&tmp, bytes));
        BVH_CUDA_TRY(cub::DeviceScan::InclusiveSum(tmp, bytes, a, S, (int64_t)nn, st));
    }
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
        graft_relayout_kernel<T><<<gn, 256, 0, st>>>(tree->d_nodes, tree->d_node_start, sa_old, nn, a, S, nw, nstart, nidx, aff, sa_new);
        graft_groups_kernel<T><<<std::max(1, ctx->sm_count * 8), 256, 0, st>>>(uniq, cnt, goff, ng, sshape, tree->d_node_start, S, aabb_all, n,
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
    climb_affected_kernel<T><<<gn2, 256, 0, st>>>(tree->d_nodes, nn2, aff, tree->d_aabb, arrive, sa_new, (T)max_growth, rebuild ? tree->d_bad : nullptr,
                                                  ng + 5, dirty, ng + 2);
    ctx->launches++;
    if (sa_new) { graft_rebase_kernel<T><<<std::max(1, ctx->sm_count * 8), 256, 0, st>>>(tree->d_nodes, gbase, cnt, ng, sa_new); ctx->launches++; }
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
    uint32_t *kpos = nullptr, *R = nullptr, *Rm = nullptr, *holes = nullptr, *flag = nullptr, *newidx = nullptr, *arrive = nullptr;
    uint8_t* aff = nullptr;
    BVH_TRY(scratch.get(&kpos, (size_t)n + 1));
    BVH_TRY(scratch.get(&R, (size_t)n + 1));
    BVH_TRY(scratch.get(&Rm, (size_t)n + 1));
    BVH_TRY(scratch.get(&holes, k));
    BVH_TRY(scratch.get(&flag, (size_t)nn + 1));
    BVH_TRY(scratch.get(&newidx, (size_t)nn + 1));
    BVH_TRY(scratch.get(&aff, nn2));
    BVH_TRY(scratch.get(&arrive, nn2));
    BVH_CUDA_TRY(cudaMemsetAsync(kpos, 0, sizeof(uint32_t) * ((size_t)n + 1), st));
    BVH_CUDA_TRY(cudaMemsetAsync(arrive, 0, sizeof(uint32_t) * nn2, st));
    const unsigned gs = (n + 255) / 256, gn = (nn + 256) / 256, gn2 = (nn2 + 255) / 256;
    removed_positions_kernel<<<gs, 256, 0, st>>>(d_rm, n, tree->d_node_index, tree->d_node_start, kpos);
    BVH_TRY(cub_exclusive_sum(scratch, kpos, R, (size_t)n + 1, st));
    BVH_TRY(cub_exclusive_sum(scratch, d_rm, Rm, (size_t)n + 1, st));
    holes_kernel<<<gs, 256, 0, st>>>(d_rm, Rm, m, holes);
    survive_kernel<T><<<gn, 256, 0, st>>>(tree->d_nodes, tree->d_node_start, nn, R, flag);
    BVH_TRY(cub_exclusive_sum(scratch, flag, newidx, (size_t)nn + 1, st));
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
    permute_shapes_kernel<T><<<gs, 256, 0, st>>>(d_rm, n, m, Rm, holes, tree->d_aabb, a_new, reinterpret_cast<const uint4*>(tree->d_tris),
                                                 reinterpret_cast<uint4*>(t_new), (uint32_t)t_words);
    ctx->launches += 5;
    dfree(ctx, tree->d_nodes); dfree(ctx, tree->d_node_start); dfree(ctx, tree->d_node_index); dfree(ctx, tree->d_aabb);
    dfree(ctx, tree->d_sa_base); dfree(ctx, tree->d_tris);
    tree->d_nodes = nw; tree->d_node_start = nstart; tree->d_node_index = nidx; tree->d_aabb = a_new; tree->d_sa_base = sa_new; tree->d_tris = t_new;
    tree->n = m; tree->n_nodes = nn2;
    if (nn2 > 1) {
        climb_affected_kernel<T><<<gn2, 256, 0, st>>>(tree->d_nodes, nn2, aff, tree->d_aabb, arrive, nullptr, T(0), nullptr, nullptr, nullptr, nullptr);
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
