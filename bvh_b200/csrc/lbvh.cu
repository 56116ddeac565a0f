// bvh_b200/csrc/lbvh.cu -- BVHGPU_BUILD_LBVH: Morton / Karras linear BVH emitted in the reference's node layout.
//
// Not a restatement of anything in the reference (the crate has one builder, the top-down 6-bucket SAH):
// this is the throughput builder BASELINE.json's north_star asks for.  Pipeline:
//   1. morton_kernel     63-bit Morton code of every shape centroid (Aabb::center, aabb_impl.rs:501-504)
//                        inside the scene's centroid bounds; key = code, value = shape index
//   2. cub::DeviceRadixSort::SortPairs   (library radix sort, 64-bit keys)
//   3. karras_kernel     one thread per internal node: range + split from common-prefix lengths, ties broken
//                        by position so duplicate codes still give a strict binary tree (Karras 2012)
//   4. path_kernel x7    pointer jumping: L(v) = number of left edges on the root path, needed for ...
//   5. box_kernel        bottom-up subtree AABBs with arrival counters
//   5b. (BVHGPU_BUILD_LBVH_TREELET) every subtree of <= 512 shapes is handed to the persistent SAH build kernel as a SEG
//       task: binned-SAH re-optimisation of the treelets, staged in shared memory, same preorder index range
//   6. emit_kernel       ... the reference's indexing rule  index(v) = 2*first(v) + L(v)  which is exactly
//                        child_l = i+1, child_r = i + 2*n_l (bvh_node.rs:138-142): the output is a valid
//                        preorder `Bvh.nodes`, so flatten / traversal / refit run on it unchanged.
// Hit sets are identical to the reference tree's for rays without an exactly-zero direction component
// (every valid BVH yields the same set; DESIGN.md); topology, node indices and SAH cost differ.
#include "internal.h"
#include "build_types.cuh"
#include <cub/device/device_radix_sort.cuh>

namespace bvhb200 {

__device__ __forceinline__ unsigned long long expand21(unsigned long long v) {     // 21 bits -> every third bit
    v &= 0x1FFFFFull;
    v = (v | (v << 32)) & 0x1F00000000FFFFull;
    v = (v | (v << 16)) & 0x1F0000FF0000FFull;
    v = (v | (v << 8)) & 0x100F00F00F00F00Full;
    v = (v | (v << 4)) & 0x10C30C30C30C30C3ull;
    v = (v | (v << 2)) & 0x1249249249249249ull;
    return v;
}

template <class T>
__global__ void __launch_bounds__(256) morton_kernel(const typename Traits<T>::DAabb* __restrict__ aabb, uint32_t n,
                                                     const typename Traits<T>::Key* __restrict__ rootkeys,
                                                     unsigned long long* __restrict__ keys, uint32_t* __restrict__ vals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    T mn[3], mx[3];
    load_aabb(aabb + i, mn, mx);
    unsigned long long code = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double lo = (double)key2f(rootkeys[6 + k]), hi = (double)key2f(rootkeys[9 + k]);
        const double c = (double)center1(mn[k], mx[k]);
        double num = c - lo, den = hi - lo;
        if (den == __longlong_as_double(0x7ff0000000000000ll)) {    // f64 extent beyond DBL_MAX: quantise with both operands halved
            num = c * 0.5 - lo * 0.5;
            den = hi * 0.5 - lo * 0.5;
        }
        double u = hi > lo ? num / den : 0.0;
        u = u >= 0.0 ? (u > 1.0 ? 1.0 : u) : 0.0;                  // NaN -> 0: never convert a NaN to an integer
        unsigned long long q = (unsigned long long)(u * 2097151.0);
        if (q > 2097151ull) q = 2097151ull;
        code |= expand21(q) << (2 - k);
    }
    keys[i] = code;
    vals[i] = i;
}

// Common prefix of sorted positions i and j (63-bit codes, ties broken by position).
__device__ __forceinline__ int delta(const unsigned long long* __restrict__ keys, int n, int i, int j) {
    if (j < 0 || j >= n) return -1;
    const unsigned long long a = keys[i], b = keys[j];
    if (a == b) return 64 + __clz((unsigned)i ^ (unsigned)j);
    return __clzll(a ^ b);
}

// Node numbering inside this file: internal nodes 0..n-2, leaves n-1+p (p = sorted position).
__global__ void __launch_bounds__(256) karras_kernel(const unsigned long long* __restrict__ keys, int n,
                                                     uint32_t* __restrict__ left, uint32_t* __restrict__ right,
                                                     uint32_t* __restrict__ first, uint32_t* __restrict__ count,
                                                     uint32_t* __restrict__ parent, uint8_t* __restrict__ isleft) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n - 1) return;
    const int d = (delta(keys, n, i, i + 1) - delta(keys, n, i, i - 1)) >= 0 ? 1 : -1;
    const int dmin = delta(keys, n, i, i - d);
    int lmax = 2;
    while (delta(keys, n, i, i + lmax * d) > dmin) lmax <<= 1;
    int l = 0;
    for (int t = lmax >> 1; t >= 1; t >>= 1)
        if (delta(keys, n, i, i + (l + t) * d) > dmin) l += t;
    const int j = i + l * d;
    const int dnode = delta(keys, n, i, j);
    int s = 0;
    for (int t = (l + 1) >> 1;; t = (t + 1) >> 1) {
        if (delta(keys, n, i, i + (s + t) * d) > dnode) s += t;
        if (t == 1) break;
    }
    const int gamma = i + s * d + (d < 0 ? -1 : 0);
    const int lo = i < j ? i : j, hi = i < j ? j : i;
    const uint32_t cl = (lo == gamma) ? (uint32_t)(n - 1 + gamma) : (uint32_t)gamma;
    const uint32_t cr = (hi == gamma + 1) ? (uint32_t)(n - 1 + gamma + 1) : (uint32_t)(gamma + 1);
    left[i] = cl; right[i] = cr; first[i] = (uint32_t)lo; count[i] = (uint32_t)(hi - lo + 1);
    parent[cl] = (uint32_t)i; isleft[cl] = 1;
    parent[cr] = (uint32_t)i; isleft[cr] = 0;
    if (i == 0) { parent[0] = 0; isleft[0] = 0; }
}

// Pointer jumping: after r rounds val[v] = number of left edges on the 2^r nearest edges towards the root.
__global__ void __launch_bounds__(256) path_init_kernel(const uint32_t* __restrict__ parent, const uint8_t* __restrict__ isleft, uint32_t total,
                                                        uint32_t* __restrict__ up, uint32_t* __restrict__ val) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= total) return;
    up[v] = parent[v];
    val[v] = v == 0 ? 0u : (uint32_t)isleft[v];
}
__global__ void __launch_bounds__(256) path_kernel(const uint32_t* __restrict__ up_in, const uint32_t* __restrict__ val_in, uint32_t total,
                                                   uint32_t* __restrict__ up_out, uint32_t* __restrict__ val_out, uint32_t* __restrict__ not_done) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= total) return;
    const uint32_t u = up_in[v];
    val_out[v] = val_in[v] + (u != v ? val_in[u] : 0u);       // the root (up == self, val 0) absorbs
    const uint32_t uu = up_in[u];
    up_out[v] = uu;
    if (not_done && uu != 0u) *not_done = (uint32_t)BVHGPU_ERR_INTERNAL;   // root path longer than 2^rounds edges
}

// Bottom-up subtree bounds: one thread per leaf climbs; the second arrival at a node merges and carries on.
// boxes[v][0..5] = AABB of the subtree, boxes[v][6..11] = bounds of its shapes' centroids (needed as centroid_bounds by
// the SAH re-optimisation of the treelets).
template <class T>
__global__ void __launch_bounds__(256) box_up_kernel(const typename Traits<T>::DAabb* __restrict__ aabb, const uint32_t* __restrict__ vals, uint32_t n,
                                                     const uint32_t* __restrict__ parent, const uint32_t* __restrict__ left, const uint32_t* __restrict__ right,
                                                     T* __restrict__ boxes, uint32_t* arrivals) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    T b[12];
    load_aabb(aabb + vals[p], b, b + 3);
#pragma unroll
    for (int k = 0; k < 3; ++k) b[6 + k] = b[9 + k] = center1(b[k], b[3 + k]);
    uint32_t v = n - 1 + p;
    {
        T* d = boxes + 12ull * v;
#pragma unroll
        for (int k = 0; k < 12; ++k) __stcg(d + k, b[k]);
    }
    while (v != 0) {
        const uint32_t par = parent[v];
        __threadfence();
        if (atomicAdd(arrivals + par, 1u) == 0u) return;       // sibling subtree not finished yet
        __threadfence();
        const uint32_t sib = left[par] == v ? right[par] : left[par];
        const T* sb = boxes + 12ull * sib;
#pragma unroll
        for (int k = 0; k < 12; ++k) {                         // min_t / max_t: order-free, -0 below +0 (whichever thread arrives second)
            const T o = __ldcg(sb + k);
            const bool isMin = (k % 6) < 3;
            b[k] = isMin ? min_t(o, b[k]) : max_t(o, b[k]);
        }
        v = par;
        T* d = boxes + 12ull * v;
#pragma unroll
        for (int k = 0; k < 12; ++k) __stcg(d + k, b[k]);
    }
}

// Emits the reference-layout nodes.  treelets: subtrees of <= TILE shapes are NOT emitted; their root becomes a SEG task of
// the persistent SAH build kernel (queue slot written here, consumed by the next launch), which rebuilds that range with the
// reference's 6-bucket SAH in shared memory and writes its nodes / leaves into the same preorder index range.
template <class T>
__global__ void __launch_bounds__(256) lbvh_emit_kernel(uint32_t n, const uint32_t* __restrict__ vals, const uint32_t* __restrict__ left,
                                                        const uint32_t* __restrict__ right, const uint32_t* __restrict__ first,
                                                        const uint32_t* __restrict__ count, const uint32_t* __restrict__ parent,
                                                        const uint32_t* __restrict__ L, const T* __restrict__ boxes,
                                                        typename Traits<T>::Node* __restrict__ nodes, uint32_t* __restrict__ node_index,
                                                        uint32_t* __restrict__ node_start,
                                                        bool treelets, QSlot<T>* q, uint32_t* qseq, uint32_t qmask, BuildCtl* ctl,
                                                        const BuildStatus* __restrict__ status) {
    using Tr = Traits<T>;
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= 2 * n - 1) return;
    if (status->nan_found) return;          // NaN shapes: no nodes, no treelet tasks -- the build reports BVHGPU_ERR_NAN (the reference panics)
    const bool leaf = v >= n - 1;
    const uint32_t f = leaf ? v - (n - 1) : first[v];
    const uint32_t idx = 2 * f + L[v];
    const uint32_t par = parent[v];
    const uint32_t pidx = v == 0 ? 0u : 2 * first[par] + L[par];
    const uint32_t cnt = leaf ? 1u : count[v];
    if (treelets) {
        if (v != 0 && count[par] <= (uint32_t)TILE) return;           // strictly inside a treelet: the SAH kernel writes it
        if (!leaf && cnt <= (uint32_t)TILE) {                          // treelet root -> SEG task
            const uint32_t tk = atomicAdd(&ctl->tail, 1u);
            QSlot<T>& s = q[tk & qmask];
            s.t.start = f; s.t.count = cnt; s.t.node = idx; s.t.parent_buf = pidx;          // range lives in index buffer 0
            const T* b = boxes + 12ull * v;
#pragma unroll
            for (int k = 0; k < 6; ++k) { s.t.ab[k] = b[k]; s.t.cb[k] = b[6 + k]; }
            s.kind = KIND_SEG; s.a = s.b = s.pad = 0;
            qseq[tk & qmask] = tk + 1u;
            return;
        }
    }
    typename Tr::Node nd;
    nd.parent = pidx;
    if (leaf) {
        const uint32_t shape = vals[f];
        nd.child_l = BVH_INVALID; nd.child_r = BVH_INVALID; nd.shape = shape;
#pragma unroll
        for (int k = 0; k < 3; ++k) { nd.l_aabb.min[k] = nd.r_aabb.min[k] = Tr::inf(); nd.l_aabb.max[k] = nd.r_aabb.max[k] = -Tr::inf(); }
        node_index[shape] = idx;
        if (treelets) atomicAdd(&ctl->leaves_done, 1u);
    } else {
        const uint32_t cl = left[v], cr = right[v];
        const uint32_t nl = cl >= n - 1 ? 1u : count[cl];
        nd.child_l = idx + 1; nd.child_r = idx + 2 * nl; nd.shape = cnt;
        const T* bl = boxes + 12ull * cl;
        const T* br = boxes + 12ull * cr;
#pragma unroll
        for (int k = 0; k < 3; ++k) { nd.l_aabb.min[k] = bl[k]; nd.l_aabb.max[k] = bl[3 + k]; nd.r_aabb.min[k] = br[k]; nd.r_aabb.max[k] = br[3 + k]; }
    }
    nodes[idx] = nd;
    node_start[idx] = f;
}

template <class T> __global__ void lbvh_single_leaf_kernel(typename Traits<T>::Node* nodes, uint32_t* node_index, uint32_t* node_start) {
    using Tr = Traits<T>;
    if (threadIdx.x != 0) return;
    typename Tr::Node nd;
    nd.parent = 0; nd.child_l = BVH_INVALID; nd.child_r = BVH_INVALID; nd.shape = 0;
    for (int k = 0; k < 3; ++k) { nd.l_aabb.min[k] = nd.r_aabb.min[k] = Tr::inf(); nd.l_aabb.max[k] = nd.r_aabb.max[k] = -Tr::inf(); }
    nodes[0] = nd; node_index[0] = 0; node_start[0] = 0;
}

// defined in build_sah.cu
template <class T> int prep_only(bvhgpu_ctx* ctx, const typename Traits<T>::Aabb* in_aabbs, uint32_t n, typename Traits<T>::DAabb* out,
                                 typename Traits<T>::Key* rootkeys, BuildStatus* status);

template <class T>
int build_lbvh(bvhgpu_ctx* ctx, const typename Traits<T>::Aabb* in_aabbs, uint32_t n, Tree<T>* tree, bool treelets) {
    using Tr = Traits<T>;
    cudaStream_t st = ctx->stream;
    tree->ctx = ctx; tree->n = n; tree->n_nodes = n ? 2 * n - 1 : 0;
    BVH_TRY(dalloc_t(ctx, &tree->d_status, 1));
    BVH_CUDA_TRY(cudaMemsetAsync(tree->d_status, 0, sizeof(BuildStatus), st));
    if (n == 0) return BVHGPU_OK;
    BVH_TRY(dalloc_t(ctx, &tree->d_aabb, n));
    BVH_TRY(dalloc_t(ctx, &tree->d_nodes, tree->n_nodes));
    BVH_TRY(dalloc_t(ctx, &tree->d_node_index, n));
    BVH_TRY(dalloc_t(ctx, &tree->d_node_start, tree->n_nodes));
    typename Tr::Key* rootkeys = nullptr;
    BVH_TRY(dalloc_t(ctx, &rootkeys, 12));
    BVH_TRY(prep_only<T>(ctx, in_aabbs, n, tree->d_aabb, rootkeys, tree->d_status));
    tree->status_pending = true;
    if (n == 1) {
        lbvh_single_leaf_kernel<T><<<1, 32, 0, st>>>(tree->d_nodes, tree->d_node_index, tree->d_node_start);
        ctx->launches++;
        dfree(ctx, rootkeys);
        return BVHGPU_OK;
    }
    const uint32_t total = 2 * n - 1;
    unsigned long long *keys = nullptr, *keys2 = nullptr;
    uint32_t *vals = nullptr, *vals2 = nullptr, *left = nullptr, *right = nullptr, *first = nullptr, *count = nullptr, *parent = nullptr;
    uint32_t *upA = nullptr, *upB = nullptr, *valA = nullptr, *valB = nullptr, *arrivals = nullptr;
    uint8_t* isleft = nullptr;
    T* boxes = nullptr;
    BVH_TRY(dalloc_t(ctx, &keys, n)); BVH_TRY(dalloc_t(ctx, &keys2, n));
    BVH_TRY(dalloc_t(ctx, &vals, n)); BVH_TRY(dalloc_t(ctx, &vals2, n));
    BVH_TRY(dalloc_t(ctx, &left, n)); BVH_TRY(dalloc_t(ctx, &right, n)); BVH_TRY(dalloc_t(ctx, &first, n)); BVH_TRY(dalloc_t(ctx, &count, n));
    BVH_TRY(dalloc_t(ctx, &parent, total)); BVH_TRY(dalloc_t(ctx, &isleft, total));
    BVH_TRY(dalloc_t(ctx, &upA, total)); BVH_TRY(dalloc_t(ctx, &upB, total)); BVH_TRY(dalloc_t(ctx, &valA, total)); BVH_TRY(dalloc_t(ctx, &valB, total));
    BVH_TRY(dalloc_t(ctx, &arrivals, n)); BVH_TRY(dalloc_t(ctx, &boxes, 12ull * total));
    const unsigned gn = (n + 255) / 256, gt = (total + 255) / 256;
    morton_kernel<T><<<gn, 256, 0, st>>>(tree->d_aabb, n, rootkeys, keys, vals);
    size_t tmp_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys, keys2, vals, vals2, (int)n, 0, 63, st);
    void* tmp = nullptr;
    BVH_TRY(dalloc(ctx, &tmp, tmp_bytes));
    cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys, keys2, vals, vals2, (int)n, 0, 63, st);
    karras_kernel<<<gn, 256, 0, st>>>(keys2, (int)n, left, right, first, count, parent, isleft);
    path_init_kernel<<<gt, 256, 0, st>>>(parent, isleft, total, upA, valA);
    uint32_t *ui = upA, *uo = upB, *vi = valA, *vo = valB;
    for (int r = 0; r < 7; ++r) {                       // covers root paths of up to 128 edges
        path_kernel<<<gt, 256, 0, st>>>(ui, vi, total, uo, vo, r == 6 ? &tree->d_status->error : nullptr);
        std::swap(ui, uo); std::swap(vi, vo);
    }
    BVH_CUDA_TRY(cudaMemsetAsync(arrivals, 0, sizeof(uint32_t) * n, st));
    box_up_kernel<T><<<gn, 256, 0, st>>>(tree->d_aabb, vals2, n, parent, left, right, boxes, arrivals);
    TreeletSession<T> S;
    if (treelets) BVH_TRY(treelet_begin<T>(ctx, tree, vals2, &S));
    lbvh_emit_kernel<T><<<gt, 256, 0, st>>>(n, vals2, left, right, first, count, parent, vi, boxes, tree->d_nodes, tree->d_node_index, tree->d_node_start,
                                            treelets, S.q, S.qseq, S.qmask, S.ctl, tree->d_status);
    ctx->launches += 14;
    BVH_CUDA_TRY(cudaGetLastError());
    if (treelets) BVH_TRY(treelet_finish<T>(ctx, tree, &S));
    dfree(ctx, keys); dfree(ctx, keys2); dfree(ctx, vals); dfree(ctx, vals2); dfree(ctx, left); dfree(ctx, right); dfree(ctx, first); dfree(ctx, count);
    dfree(ctx, parent); dfree(ctx, isleft); dfree(ctx, upA); dfree(ctx, upB); dfree(ctx, valA); dfree(ctx, valB); dfree(ctx, arrivals); dfree(ctx, boxes);
    dfree(ctx, tmp); dfree(ctx, rootkeys);
    return BVHGPU_OK;
}

template int build_lbvh<float>(bvhgpu_ctx*, const bvh_aabb3f*, uint32_t, Tree<float>*, bool);
template int build_lbvh<double>(bvhgpu_ctx*, const bvh_aabb3d*, uint32_t, Tree<double>*, bool);

}  // namespace bvhb200
