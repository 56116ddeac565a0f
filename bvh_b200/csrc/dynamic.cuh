// bvh_b200/csrc/dynamic.cuh -- the kernels of batched add_shape / remove_shape (dynamic.cu, DESIGN.md section 4.10) that D = 3
// (dynamic.cu, and D = 2 through the z = 0 embedding of dim2.cu) and D = 4 (dim4.cu) share.
//
// The relocation, the contraction and the climb are index arithmetic on the preorder layout; only box loads, joins and surface areas
// depend on D.  The kernels are templated on D, T, the node type and the shape-box type, as update.cuh is: a shape box is loaded with
// load_box of csr.cuh (the padded 3-D device layout or the 4-D ABI layout) and surface areas are taken with surface_area_d<D>, so
// the D = 3 instantiations perform exactly the operations the 3-D kernels always did.
//
// The kernels that do not touch nodes or boxes (grouping by insertion point, removed positions, holes) stay in dynamic.cu; the host
// helpers at the end of this file launch them for both drivers.
#pragma once
#include "update.cuh"

namespace bvhb200 {

#ifdef __CUDACC__
template <int D, class T> __device__ __forceinline__ void join_d(T mn[D], T mx[D], const T amn[D], const T amx[D]) {
    for (int c = 0; c < D; ++c) { mn[c] = min_t(mn[c], amn[c]); mx[c] = max_t(mx[c], amx[c]); }
}
template <int D, class A, class T> __device__ __forceinline__ void box_of(const A& a, T mn[D], T mx[D]) {
    for (int c = 0; c < D; ++c) { mn[c] = a.min[c]; mx[c] = a.max[c]; }
}
template <int D, class A, class T> __device__ __forceinline__ void set_box(A& a, const T mn[D], const T mx[D]) {
    for (int c = 0; c < D; ++c) { a.min[c] = mn[c]; a.max[c] = mx[c]; }
}
template <int D, class T, class A> __device__ __forceinline__ void set_empty(A& a) {
    for (int c = 0; c < D; ++c) { a.min[c] = Traits<T>::inf(); a.max[c] = -Traits<T>::inf(); }
}
// the centre bounds of a group root: T values for rebuild_subtrees (D = 3), order-preserving keys for root_seed4_kernel (D = 4)
__device__ __forceinline__ void store_cb(float* p, float v) { *p = v; }
__device__ __forceinline__ void store_cb(double* p, double v) { *p = v; }
__device__ __forceinline__ void store_cb(uint32_t* p, float v) { *p = f2key(v); }
__device__ __forceinline__ void store_cb(unsigned long long* p, double v) { *p = f2key(v); }

// ---- add: insertion point of every new shape (optimization.rs:88-207, evaluated against the tree before the call) -------------
template <int D, class T, class Node, class Box>
__global__ void __launch_bounds__(256) descend_kernel(const Node* __restrict__ nodes, const Box* __restrict__ aabb,
                                                      uint32_t n, uint32_t k, uint32_t* __restrict__ point) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= k) return;
    T smn[D], smx[D];
    load_box(aabb + n + j, smn, smx);
    const T shape_sa = surface_area_d<D>(smn, smx);
    uint32_t i = 0;
    for (;;) {
        const Node& nd = nodes[i];
        if (nd.child_l == BVH_INVALID) break;                                  // a leaf: split it
        T lmn[D], lmx[D], rmn[D], rmx[D], le_mn[D], le_mx[D], re_mn[D], re_mx[D], m_mn[D], m_mx[D];
        box_of<D>(nd.l_aabb, lmn, lmx); box_of<D>(nd.r_aabb, rmn, rmx);
        for (int c = 0; c < D; ++c) {
            le_mn[c] = min_t(lmn[c], smn[c]); le_mx[c] = max_t(lmx[c], smx[c]);
            re_mn[c] = min_t(rmn[c], smn[c]); re_mx[c] = max_t(rmx[c], smx[c]);
            m_mn[c] = min_t(rmn[c], lmn[c]);  m_mx[c] = max_t(rmx[c], lmx[c]);
        }
        const T send_left = add_rn(surface_area_d<D>(rmn, rmx), surface_area_d<D>(le_mn, le_mx));
        const T send_right = add_rn(surface_area_d<D>(lmn, lmx), surface_area_d<D>(re_mn, re_mx));
        const T merged = add_rn(surface_area_d<D>(m_mn, m_mx), shape_sa);
        const T min_send = send_left < send_right ? send_left : send_right;
        if (merged < div_rn(mul_rn(min_send, T(3)), T(10))) break;             // merge here: the new shape becomes this node's sibling
        i = send_left < send_right ? nd.child_l : nd.child_r;
    }
    point[j] = i;
}

// every old node: its content moves to i + 2 S(i); a graft node is written in front of it when new shapes chose it
template <int D, class T, class Node>
__global__ void __launch_bounds__(256) graft_relayout_kernel(const Node* __restrict__ old, const uint32_t* __restrict__ old_start,
                                                             const T* __restrict__ sa_old, uint32_t nn, const uint32_t* __restrict__ a, const uint32_t* __restrict__ S,
                                                             Node* __restrict__ nw, uint32_t* __restrict__ nstart, uint32_t* __restrict__ nidx,
                                                             uint8_t* __restrict__ aff, T* __restrict__ sa_new) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nn) return;
    Node o = old[i];
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
        Node g;
        g.parent = par; g.child_l = base + 1; g.child_r = pos; g.shape = ai + cnt;
        set_empty<D, T>(g.l_aabb); set_empty<D, T>(g.r_aabb);                   // written by the climb
        nw[base] = g;
        nstart[base] = old_start[i] + si - ai;
        aff[base] = 1;
        if (sa_new) sa_new[base] = Traits<T>::inf();                          // fresh node: never "degraded"; its baseline is set after the climb
    }
}

// warp-wide bounds of the group's AABBs (centres = false) or of their centres (centres = true)
template <int D, class T, class Box>
__device__ __noinline__ void group_bounds(const Box* __restrict__ aabb, uint32_t n, const uint32_t* __restrict__ shapes, uint32_t ap,
                                          bool centres, T mn[D], T mx[D]) {
    typename Traits<T>::Key kmn[D], kmx[D];
#pragma unroll
    for (int c = 0; c < D; ++c) { kmn[c] = Traits<T>::KEY_POS_INF; kmx[c] = Traits<T>::KEY_NEG_INF; }
    for (uint32_t j = lane_id(); j < ap; j += 32) {
        T a[D], b[D];
        load_box(aabb + n + shapes[j], a, b);
#pragma unroll
        for (int c = 0; c < D; ++c) {
            const T lo = centres ? center1(a[c], b[c]) : a[c], hi = centres ? lo : b[c];
            const auto klo = f2key(lo), khi = f2key(hi);
            kmn[c] = klo < kmn[c] ? klo : kmn[c];
            kmx[c] = khi > kmx[c] ? khi : kmx[c];
        }
    }
#pragma unroll
    for (int c = 0; c < D; ++c) { mn[c] = key2f(warp_min_key(kmn[c])); mx[c] = key2f(warp_max_key(kmx[c])); }
}

// one warp per group: the left child of its graft node -- a leaf (a_p = 1) or the root placeholder of an exact-SAH rebuild over the
// group's shapes in ascending index order.  Count, box, parent and start are what rebuild_subtrees (D = 3) and root_seed4_kernel
// (D = 4) read from it; the group's shapes go to their leaf positions of idx0 and its centre bounds to cb_roots[2 D slot ..] (CB = T
// for D = 3, the key type for D = 4).
template <int D, class T, class Node, class Box, class CB>
__global__ void __launch_bounds__(256) graft_groups_kernel(const uint32_t* __restrict__ uniq, const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ goff,
                                                           const uint32_t* __restrict__ n_groups, const uint32_t* __restrict__ sorted_shape,
                                                           const uint32_t* __restrict__ old_start, const uint32_t* __restrict__ S,
                                                           const Box* __restrict__ aabb, uint32_t n,
                                                           Node* __restrict__ nw, uint32_t* __restrict__ nstart, uint32_t* __restrict__ nidx,
                                                           uint32_t* __restrict__ idx0, uint32_t* __restrict__ roots, uint32_t* __restrict__ n_roots,
                                                           CB* __restrict__ cb_roots, uint32_t* __restrict__ gbase) {
    const uint32_t warps = gridDim.x * (blockDim.x >> 5), ng = *n_groups;
    for (uint32_t g = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); g < ng; g += warps) {
        const uint32_t p = uniq[g], ap = cnt[g], off = goff[g];
        const uint32_t base = p + 2 * (S[p] - ap), L = base + 1, start = old_start[p] + S[p] - ap;
        T bmn[D], bmx[D], cmn[D], cmx[D];
        group_bounds<D, T>(aabb, n, sorted_shape + off, ap, false, bmn, bmx);  // the group's box, then the bounds of its centres
        group_bounds<D, T>(aabb, n, sorted_shape + off, ap, true, cmn, cmx);
        if (ap > 1) for (uint32_t j = lane_id(); j < ap; j += 32) idx0[start + j] = n + sorted_shape[off + j];
        if (lane_id() != 0) continue;
        gbase[g] = base;
        Node& l = nw[L];                                                      // written field by field: no whole node in registers
        l.parent = base;
        l.child_r = BVH_INVALID;
        set_empty<D, T>(l.r_aabb);
        nstart[L] = start;
        if (ap == 1) {
            const uint32_t s = n + sorted_shape[off];
            l.child_l = BVH_INVALID; l.shape = s;
            set_empty<D, T>(l.l_aabb);
            nidx[s] = L;
        } else {
            l.child_l = L + 1; l.shape = ap;
            set_box<D>(l.l_aabb, bmn, bmx);
            const uint32_t slot = atomicAdd(n_roots, 1u);
            roots[slot] = L;
            #pragma unroll
            for (int c = 0; c < D; ++c) { store_cb(cb_roots + 2 * D * (size_t)slot + c, cmn[c]); store_cb(cb_roots + 2 * D * (size_t)slot + D + c, cmx[c]); }
        }
    }
}

// Fresh surface-area baselines of the graft ranges [G, G + 2 a_p): the graft node and the new subtree below its left side.
template <int D, class T, class Node>
__global__ void __launch_bounds__(256) graft_rebase_kernel(const Node* __restrict__ nodes, const uint32_t* __restrict__ gbase,
                                                           const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ n_groups, T* __restrict__ sa) {
    const uint32_t warps = gridDim.x * (blockDim.x >> 5), ng = *n_groups;
    for (uint32_t g = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); g < ng; g += warps) {
        const uint32_t b = gbase[g], e = b + 2 * cnt[g];
        for (uint32_t i = b + lane_id(); i < e; i += 32) {
            const Node& nd = nodes[i];
            if (nd.child_l == BVH_INVALID) { sa[i] = T(0); continue; }
            T mn[D], mx[D], bmn[D], bmx[D];
            box_of<D>(nd.l_aabb, mn, mx); box_of<D>(nd.r_aabb, bmn, bmx);
            join_d<D>(mn, mx, bmn, bmx);
            sa[i] = surface_area_d<D>(mn, mx);
        }
    }
}

// ---- the climb over the affected nodes ------------------------------------------------------------------------------------------
// Affected nodes (aff = 1) are closed under "parent of": every ancestor of an affected node is affected.  Both child slots of an
// affected node are rewritten.  The climbs start at the unaffected children of affected nodes, whose box is known (a leaf: its shape's
// AABB; an inner node: the join of its own child slots, as get_node_aabb, bvh_node.rs:616-625); every climb writes its box into the
// parent's slot, and the second arrival at a node joins both slots and carries on.  bad != nullptr: growth test against sa_base as
// bvhgpu_update_* does (n_bad counts the failures); every affected node is logged in `dirty`.
template <int D, class T, class Node, class Box>
__global__ void __launch_bounds__(256) climb_affected_kernel(Node* nodes, uint32_t nn, const uint8_t* __restrict__ aff,
                                                             const Box* __restrict__ aabb, uint32_t* __restrict__ arrive,
                                                             const T* __restrict__ sa_base, T max_growth, uint8_t* __restrict__ bad, uint32_t* __restrict__ n_bad,
                                                             uint32_t* __restrict__ dirty, uint32_t* __restrict__ n_dirty) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j == 0 || j >= nn || aff[j]) return;
    if (!aff[nodes[j].parent]) return;
    T mn[D], mx[D];
    {
        const Node& nd = nodes[j];                                          // not affected: nothing writes it during this kernel
        if (nd.child_l == BVH_INVALID) load_box(aabb + nd.shape, mn, mx);
        else { T bmn[D], bmx[D]; box_of<D>(nd.l_aabb, mn, mx); box_of<D>(nd.r_aabb, bmn, bmx); join_d<D>(mn, mx, bmn, bmx); }
    }
    uint32_t node = j;
    for (;;) {
        const uint32_t p = __ldcg(&nodes[node].parent);
        Node* pn = nodes + p;
        const bool is_left = __ldcg(&pn->child_l) == node;
        auto* dst = is_left ? &pn->l_aabb : &pn->r_aabb;
        for (int c = 0; c < D; ++c) { __stcg(&dst->min[c], mn[c]); __stcg(&dst->max[c], mx[c]); }
        __threadfence();
        if (atomicAdd(arrive + p, 1u) == 0u) return;                          // the other side is not finished yet
        __threadfence();
        const auto* sib = is_left ? &pn->r_aabb : &pn->l_aabb;
        for (int c = 0; c < D; ++c) { mn[c] = min_t(__ldcg(&sib->min[c]), mn[c]); mx[c] = max_t(__ldcg(&sib->max[c]), mx[c]); }
        if (bad && surface_area_d<D>(mn, mx) > mul_rn(max_growth, sa_base[p])) { bad[p] = 1; atomicAdd(n_bad, 1u); }
        if (dirty) dirty[atomicAdd(n_dirty, 1u)] = p;
        if (p == 0) return;
        node = p;
    }
}

// ---- remove ------------------------------------------------------------------------------------------------------------------------
// swap rule: a survivor >= m takes the hole of the same rank among the holes (ascending), the others keep their index
__device__ __forceinline__ uint32_t relabel(uint32_t s, uint32_t m, const uint32_t* Rm, const uint32_t* holes) {
    return s < m ? s : holes[(s - m) - (Rm[s] - Rm[m])];
}
// shapes removed below a node: R = exclusive scan of the removed flags by leaf position
struct Shrink { uint32_t c, cl, ncl, nc; bool leaf; };
template <class Node>
__device__ __forceinline__ Shrink shrink(const Node* nodes, const uint32_t* node_start, const uint32_t* R, uint32_t i) {
    Shrink r;
    const Node& nd = nodes[i];
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
template <class Node>
__global__ void __launch_bounds__(256) survive_kernel(const Node* __restrict__ nodes, const uint32_t* __restrict__ node_start, uint32_t nn,
                                                      const uint32_t* __restrict__ R, uint32_t* __restrict__ flag) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > nn) return;
    if (i == nn) { flag[i] = 0; return; }
    const Shrink r = shrink(nodes, node_start, R, i);
    flag[i] = r.leaf ? (r.nc == 1u) : (r.ncl > 0 && r.nc > r.ncl);            // an inner node survives when both sides keep a shape
}
// every surviving node writes its own fields at its new index and the parent links of its two new children
template <class T, class Node>
__global__ void __launch_bounds__(256) contract_kernel(const Node* __restrict__ old, const uint32_t* __restrict__ old_start, uint32_t nn,
                                                       const uint32_t* __restrict__ R, const uint32_t* __restrict__ newidx,
                                                       uint32_t m, const uint32_t* __restrict__ Rm, const uint32_t* __restrict__ holes,
                                                       const T* __restrict__ sa_old, Node* __restrict__ nw, uint32_t* __restrict__ nstart,
                                                       uint32_t* __restrict__ nidx, uint8_t* __restrict__ aff, T* __restrict__ sa_new) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nn) return;
    const uint32_t j = newidx[i];
    if (newidx[i + 1] == j) return;                                           // removed or spliced out
    const Node& nd = old[i];
    const Shrink r = shrink(old, old_start, R, i);
    Node& o = nw[j];
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
// the surviving shapes' boxes (and triangles, t_old != nullptr) at their new indices
template <class Box>
__global__ void __launch_bounds__(256) permute_shapes_kernel(const uint32_t* __restrict__ rm, uint32_t n, uint32_t m, const uint32_t* __restrict__ Rm,
                                                             const uint32_t* __restrict__ holes, const Box* __restrict__ a_old,
                                                             Box* __restrict__ a_new, const uint4* __restrict__ t_old,
                                                             uint4* __restrict__ t_new, uint32_t t_words) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n || rm[s]) return;
    const uint32_t d = relabel(s, m, Rm, holes);
    a_new[d] = a_old[s];
    if (t_old) for (uint32_t w = 0; w < t_words; ++w) t_new[(size_t)d * t_words + w] = t_old[(size_t)s * t_words + w];
}
#endif  // __CUDACC__

// ---- host helpers (dynamic.cu), shared by the D = 3 and D = 4 drivers --------------------------------------------------------------
// out = exclusive scan of in[0 .. len)
int exclusive_sum_u32(Scratch& scratch, const uint32_t* in, uint32_t* out, size_t len, cudaStream_t st);
// The k insertion points point[0 .. k) (node indices < nn) grouped: sshape = the new shapes (0 .. k-1) sorted by insertion point,
// ascending shape index inside a group (stable: deterministic); uniq / cnt = the distinct points and their group sizes, *ng (device) =
// the number of groups; goff = exclusive scan of cnt; a = group size scattered onto the old node array, S = its inclusive scan.
// Everything but ng comes from `scratch` (8 entries).
struct Groups { uint32_t *sshape, *uniq, *cnt, *goff, *a, *S; };
int group_insertions(bvhgpu_ctx* ctx, Scratch& scratch, const uint32_t* point, uint32_t k, uint32_t nn, uint32_t* ng, Groups* g);
// The ranks of a removal: R = exclusive scan by leaf position of the removed flags (node_start / node_index of the tree), Rm = exclusive
// scan of rm by shape index, holes = the vacated indices below n - k, ascending.  From `scratch` (5 entries).
struct Ranks { uint32_t *R, *Rm, *holes; };
int remove_ranks(bvhgpu_ctx* ctx, Scratch& scratch, const uint32_t* rm, uint32_t n, uint32_t k, const uint32_t* node_index,
                 const uint32_t* node_start, Ranks* r);

}  // namespace bvhb200
