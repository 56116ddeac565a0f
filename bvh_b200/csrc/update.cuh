// bvh_b200/csrc/update.cuh -- the kernels of refit and the incremental update (Bvh::update_shapes, src/bvh/optimization.rs:304-351)
// that D = 3 (and D = 2 through the z = 0 embedding of dim2.cu) and D = 4 share; the host drivers are in dynamic.cu.
//
// Every node POD starts with the same 16 bytes {parent, child_l, child_r, shape}, so the kernels that only follow links are
// templated on the node type.  The kernels that touch boxes are templated on D as well: they load a shape box with load_box of
// csr.cuh (the padded 3-D device layout or the 4-D ABI layout) and take surface areas with surface_area_d<D>, which is the 3-D
// surface_area for D = 3 and surface_area4 for D = 4.  Both sum the squared extents left to right without FMA, so the D = 3
// instantiations perform exactly the operations the 3-D kernels always did.
#pragma once
#include "csr.cuh"

namespace bvhb200 {

#ifdef __CUDACC__
// ---- Aabb::surface_area for D = 4: 2 * (((sx*sx + sy*sy) + sz*sz) + sw*sw), left to right, no FMA ----
template <class T> __device__ __forceinline__ T surface_area4(const T mn[4], const T mx[4]) {
    T acc = add_rn(mul_rn(sub_rn(mx[0], mn[0]), sub_rn(mx[0], mn[0])), mul_rn(sub_rn(mx[1], mn[1]), sub_rn(mx[1], mn[1])));
    acc = add_rn(acc, mul_rn(sub_rn(mx[2], mn[2]), sub_rn(mx[2], mn[2])));
    acc = add_rn(acc, mul_rn(sub_rn(mx[3], mn[3]), sub_rn(mx[3], mn[3])));
    return mul_rn(T(2), acc);
}

template <int D, class T> __device__ __forceinline__ T surface_area_d(const T mn[D], const T mx[D]) {
    static_assert(D == 3 || D == 4, "surface_area_d: D = 3 or 4");
    if constexpr (D == 3) return surface_area(mn, mx);
    else return surface_area4(mn, mx);
}

// ---- refit: bottom-up recomputation of the child boxes from the (new) shape boxes ----
// (the data-parallel part of Bvh::update_shapes: fix_aabbs_ascending, src/bvh/optimization.rs:317-351).  One thread per shape climbs
// from its leaf and writes its box into the parent's child slot; the second thread to reach a node joins the two slots and carries on.
// Topology, node_index and node_start are kept; leaves keep their Aabb::empty() child boxes.
// WITH_CB (bvhgpu_optimize, D = 3 only): the climb also carries the bounds of the shape CENTRES below every node into cb[node][6]
// (min xyz, max xyz) -- what the builder needs, next to the box, to restart from an inner node.
template <int D, class T, bool WITH_CB, class Node, class Box>
__global__ void __launch_bounds__(256) refit_kernel(Node* nodes, const uint32_t* __restrict__ node_index,
                                                    const Box* __restrict__ aabb, uint32_t n, uint32_t* arrivals, T* cb) {
    static_assert(D == 3 || !WITH_CB, "refit_kernel: centre bounds for D = 3 only");
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    T mn[D], mx[D], cmn[D], cmx[D];
    load_box(aabb + s, mn, mx);
    for (int k = 0; k < D; ++k) cmn[k] = cmx[k] = center1(mn[k], mx[k]);
    uint32_t node = node_index[s];
    while (node != 0) {
        const uint32_t p = __ldcg(&nodes[node].parent);
        Node* pn = nodes + p;
        const uint32_t pl = __ldcg(&pn->child_l);
        const bool is_left = pl == node;
        auto* dst = is_left ? &pn->l_aabb : &pn->r_aabb;
        for (int k = 0; k < D; ++k) { __stcg(&dst->min[k], mn[k]); __stcg(&dst->max[k], mx[k]); }
        if (WITH_CB) for (int k = 0; k < D; ++k) { __stcg(cb + 2 * D * (size_t)node + k, cmn[k]); __stcg(cb + 2 * D * (size_t)node + D + k, cmx[k]); }
        __threadfence();
        if (atomicAdd(arrivals + p, 1u) == 0u) return;      // sibling subtree not finished yet
        __threadfence();
        const auto* sib = is_left ? &pn->r_aabb : &pn->l_aabb;
        for (int k = 0; k < D; ++k) {
            const T smn = __ldcg(&sib->min[k]), smx = __ldcg(&sib->max[k]);
            mn[k] = min_t(smn, mn[k]);
            mx[k] = max_t(smx, mx[k]);
        }
        if (WITH_CB) {
            const uint32_t sn = is_left ? __ldcg(&pn->child_r) : pl;
            for (int k = 0; k < D; ++k) {
                cmn[k] = min_t(__ldcg(cb + 2 * D * (size_t)sn + k), cmn[k]);
                cmx[k] = max_t(__ldcg(cb + 2 * D * (size_t)sn + D + k), cmx[k]);
            }
        }
        node = p;
    }
    if (WITH_CB) for (int k = 0; k < D; ++k) { __stcg(cb + k, cmn[k]); __stcg(cb + D + k, cmx[k]); }     // the root's
}

// ---- new shape boxes of refit / update_shapes / add_shapes, checked before anything is written ----
// flags[0]: a NaN coordinate, flags[1]: an index >= n.  Box = the ABI box of D (2 D scalars); changed == nullptr: box i belongs to
// shape i (no index to check).
template <int D, class T, class Box>
__global__ void __launch_bounds__(256) check_boxes_kernel(const uint32_t* __restrict__ changed, const Box* __restrict__ fresh,
                                                          uint32_t m, uint32_t n, uint32_t* __restrict__ flags) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    if (changed && changed[i] >= n) atomicExch(flags + 1, 1u);
    const T* p = reinterpret_cast<const T*>(fresh + i);
    bool nan = false;
#pragma unroll
    for (int c = 0; c < 2 * D; ++c) nan |= p[c] != p[c];
    if (nan) atomicExch(flags, 1u);
}
// a checked ABI box into the tree's array: converted to the padded 3-D device layout, or copied (the 4-D ABI box is the device layout)
template <class T> __device__ __forceinline__ void store_padded(typename Traits<T>::DAabb* dst, const T* p) {
    typename Traits<T>::DAabb d;
#pragma unroll
    for (int c = 0; c < 3; ++c) { d.min[c] = p[c]; d.max[c] = p[3 + c]; }
    if constexpr (sizeof(T) == 4) { d.pad0 = 0; d.pad1 = 0; }
    *dst = d;
}
__device__ __forceinline__ void store_box(DAabbF* dst, const bvh_aabb3f* src) { store_padded<float>(dst, reinterpret_cast<const float*>(src)); }
__device__ __forceinline__ void store_box(DAabbD* dst, const bvh_aabb3d* src) { store_padded<double>(dst, reinterpret_cast<const double*>(src)); }
__device__ __forceinline__ void store_box(bvh_aabb4f* dst, const bvh_aabb4f* src) { *dst = *src; }
__device__ __forceinline__ void store_box(bvh_aabb4d* dst, const bvh_aabb4d* src) { *dst = *src; }
template <class Box, class DBox>
__global__ void __launch_bounds__(256) scatter_boxes_kernel(const uint32_t* __restrict__ changed, const Box* __restrict__ fresh, uint32_t m,
                                                            DBox* __restrict__ aabb) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    store_box(aabb + changed[i], fresh + i);            // an index listed twice: one of its boxes wins (the reference would use shapes[i] for both)
}

// ---- rebuild roots ----
// A node is a rebuild candidate when it is not degraded itself but a child is (the smallest subtree in which the moved shapes can
// be placed properly again), or when it is the degraded root.
__device__ __forceinline__ bool rebuild_candidate(uint32_t i, uint32_t child_l, uint32_t child_r, const uint8_t* bad) {
    if (child_l == BVH_INVALID) return false;
    if (bad[i]) return i == 0;
    return bad[child_l] || bad[child_r];
}

// ---- incremental form: only the root paths of the changed leaves are touched ----------------------------------------------------
// mark: every changed leaf walks up and counts, in arrive[p], how many of p's children lie on a changed path (the first walker through
// a node carries on, later ones stop).  climb: every changed leaf writes its box into its parent and decrements; the LAST arrival at a
// node joins the two stored child boxes (both final by then), tests the growth against the node's baseline, logs the node as dirty and
// carries on.  Work = number of nodes on the changed paths, not n.  Both leave arrive[] all zero.
template <class Node>
__global__ void __launch_bounds__(256) mark_paths_kernel(const Node* __restrict__ nodes, const uint32_t* __restrict__ node_index,
                                                         const uint32_t* __restrict__ changed, uint32_t m, uint32_t* __restrict__ arrive) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    uint32_t node = node_index[changed[i]];
    while (node != 0) {
        const uint32_t p = nodes[node].parent;
        if (atomicAdd(arrive + p, 1u) != 0u) break;
        node = p;
    }
}
template <int D, class T, class Node, class Box>
__global__ void __launch_bounds__(256) climb_paths_kernel(Node* nodes, const uint32_t* __restrict__ node_index,
                                                          const Box* __restrict__ aabb, const uint32_t* __restrict__ changed, uint32_t m,
                                                          uint32_t* __restrict__ arrive, const T* __restrict__ sa_base, T max_growth, uint8_t* __restrict__ bad,
                                                          uint32_t* __restrict__ dirty, uint32_t* __restrict__ n_dirty) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const uint32_t s = changed[i];
    T mn[D], mx[D];
    load_box(aabb + s, mn, mx);
    uint32_t node = node_index[s];
    while (node != 0) {
        const uint32_t p = __ldcg(&nodes[node].parent);
        Node* pn = nodes + p;
        const bool is_left = __ldcg(&pn->child_l) == node;
        auto* dst = is_left ? &pn->l_aabb : &pn->r_aabb;
        for (int k = 0; k < D; ++k) { __stcg(&dst->min[k], mn[k]); __stcg(&dst->max[k], mx[k]); }
        __threadfence();
        if (atomicSub(arrive + p, 1u) != 1u) return;        // another changed path still has to come through p
        __threadfence();
        const auto* sib = is_left ? &pn->r_aabb : &pn->l_aabb;
        for (int k = 0; k < D; ++k) { mn[k] = min_t(__ldcg(&sib->min[k]), mn[k]); mx[k] = max_t(__ldcg(&sib->max[k]), mx[k]); }
        if (bad && surface_area_d<D>(mn, mx) > mul_rn(max_growth, sa_base[p])) bad[p] = 1;
        dirty[atomicAdd(n_dirty, 1u)] = p;
        node = p;
    }
}
template <class Node>
__global__ void __launch_bounds__(256) select_roots_dirty_kernel(const Node* __restrict__ nodes, const uint8_t* __restrict__ bad,
                                                                 const uint32_t* __restrict__ dirty, const uint32_t* __restrict__ n_dirty,
                                                                 uint32_t* __restrict__ roots, uint32_t* n_roots) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= *n_dirty) return;
    const uint32_t i = dirty[k];
    const uint4 meta = *reinterpret_cast<const uint4*>(nodes + i);
    if (!rebuild_candidate(i, meta.y, meta.z, bad)) return;
    uint32_t a = i;
    while (a != 0) {                                                   // an outer candidate takes this subtree with it
        a = nodes[a].parent;
        const uint4 mm = *reinterpret_cast<const uint4*>(nodes + a);
        if (rebuild_candidate(a, mm.y, mm.z, bad)) return;
    }
    roots[atomicAdd(n_roots, 1u)] = i;
}
static __global__ void __launch_bounds__(256) clear_bad_kernel(const uint32_t* __restrict__ dirty, const uint32_t* __restrict__ n_dirty, uint8_t* __restrict__ bad) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < *n_dirty) bad[dirty[k]] = 0;
}

// ---- surface-area baseline of the growth test ----
// SA of the join of an inner node's two child boxes (0 for leaves).
template <int D, class T, class Node>
__global__ void __launch_bounds__(256) node_sa_kernel(const Node* __restrict__ nodes, uint32_t n_nodes, T* __restrict__ sa) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_nodes) return;
    const Node& nd = nodes[i];
    if (nd.child_l == BVH_INVALID) { sa[i] = T(0); return; }
    T mn[D], mx[D];
    for (int k = 0; k < D; ++k) { mn[k] = min_t(nd.l_aabb.min[k], nd.r_aabb.min[k]); mx[k] = max_t(nd.l_aabb.max[k], nd.r_aabb.max[k]); }
    sa[i] = surface_area_d<D>(mn, mx);
}
// After a rebuild the nodes of the rebuilt subtrees get a new surface-area baseline; every other node keeps the one it had when
// it was last built (so slow drift accumulates against it instead of being forgiven at every call).
template <int D, class T, class Node>
__global__ void __launch_bounds__(256) rebase_kernel(const Node* __restrict__ nodes, const uint32_t* __restrict__ roots,
                                                     const uint32_t* __restrict__ n_roots, T* __restrict__ sa_base) {
    const uint32_t warps = gridDim.x * (blockDim.x >> 5), nr = *n_roots;
    for (uint32_t k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); k < nr; k += warps) {
        const uint32_t r = roots[k];
        const uint32_t cnt = __ldcg(&nodes[r].shape);                        // shapes below the root: its subtree is the node range [r, r + 2 cnt - 1)
        for (uint32_t i = r + lane_id(); i < r + 2 * cnt - 1; i += 32) {
            const Node& nd = nodes[i];
            if (__ldcg(&nd.child_l) == BVH_INVALID) { sa_base[i] = T(0); continue; }
            T mn[D], mx[D];
            for (int c = 0; c < D; ++c) { mn[c] = min_t(__ldcg(&nd.l_aabb.min[c]), __ldcg(&nd.r_aabb.min[c])); mx[c] = max_t(__ldcg(&nd.l_aabb.max[c]), __ldcg(&nd.r_aabb.max[c])); }
            sa_base[i] = surface_area_d<D>(mn, mx);
        }
    }
}
#endif  // __CUDACC__

}  // namespace bvhb200
