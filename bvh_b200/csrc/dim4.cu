// bvh_b200/csrc/dim4.cu -- D = 4: Bvh<T,4>::build (exact 6-bucket SAH), flatten and batched ray traversal, f32 and f64.
//
// The reference is generic in D (src/bvh/bvh_node.rs:81-279, src/flat_bvh.rs:60-143, src/ray/intersect_default.rs:16-37) and ships
// 4-wide slab tests for Ray<f32,4> / Ray<f64,4> (src/ray/intersect_simd.rs).  A fourth axis cannot hide in the 3-D kernels the way
// D = 2 hides in z = 0 (dim2.cu): surface areas, largest_axis and the slab test all see it.  So D = 4 has its own pipeline here, with
// its own node types and its own Tree4<T>; it shares the exact-arithmetic helpers and keys of common.cuh, Scratch, the records,
// walk, count -> scan -> fill driver and CSR drivers of csr.cuh, and the predicates of queries.cuh.  DESIGN.md section 4.11
// describes the design.  This file holds the kernels, the Tree4<T> instances of the CSR drivers with the 4-D steps they call
// (ensure_records, nearest_bound, the ray probe), and the other device-side drivers declared in internal.h; the bvhgpu_*_f32x4 / _f64x4 entry points are the
// D = 4 instances of the host layer in capi.cu, which checks the arguments and the tree's status and stages the batch.  Refit,
// update_shapes, add_shapes and remove_shapes run the drivers of dynamic.cu; the 4-D steps they call (the builder seeded from
// subtree roots, the growth rebuild, the caches) are at the end of this file.
//
// Builder (bit-identical to Bvh::build in the sense of DESIGN.md section 2):
//   ranges of more than SMALL4 shapes: level-synchronous.  Per level: prep (tile numbering, bucket identities), bin (one warp per
//     TILE4 shapes: bucket counts + min/max keys of boxes and centres, folded with warp REDUX, flushed with global atomics), split
//     (one warp per range: the 5 candidate costs in exact arithmetic, the node, the child ranges, the stable per-tile destinations),
//     scatter (one warp per tile, stable by ballots).  The host reads back one word per level: the number of ranges left.
//   ranges of at most SMALL4 shapes: one warp each, depth-first with an explicit stack in shared memory.  The smaller child is
//     split first and the larger one is pushed, so the stack never holds more than log2(SMALL4) + 1 entries, however skewed the range.
// Node positions depend only on counts (cl = me + 1, cr = me + 2 nl) and every reduction is a min / max / sum of integers, so the
// order in which warps run never shows in the result: two builds of the same input are byte-identical.
#include "internal.h"
#include "csr.cuh"
#include "queries.cuh"
#include "update.cuh"
#include <algorithm>
#include <new>

namespace bvhb200 {

// The node / record types D4<T>, the tree Tree4<T> and the records TRec4F / TRec4D are in internal.h.

constexpr uint32_t SMALL4 = 256;     // ranges this small are finished by one warp (depth-first, shared-memory stack)
constexpr uint32_t TILE4 = 512;      // shapes per warp tile of a large range
constexpr int STACK4 = 12;           // > log2(SMALL4) + 1: the smaller-child-first order bounds the stack
constexpr uint32_t CTL_NEXT = 0, CTL_SMALL = 1, CTL_ERROR = 2, CTL_NAN = 3, CTL_REBUILT = 4;

template <class T> struct __align__(16) Task4 {
    uint32_t start, count, node, parent;
    uint32_t buf, pad[3];              // index buffer that holds the range
    T ab[8];                           // aabb_bounds      (min xyzw, max xyzw)
    T cb[8];                           // centroid_bounds
};

// key slot k of a bucket: 0..3 box min, 4..7 box max, 8..11 centre min, 12..15 centre max
__device__ __forceinline__ bool kmin4(int k) { return ((k >> 2) & 1) == 0; }
template <class Key> __device__ __forceinline__ Key fold_key(int k, Key acc, Key v) { return kmin4(k) ? (v < acc ? v : acc) : (v > acc ? v : acc); }

// How a range is split: largest_axis (first strict maximum) of the centroid extent, halving below T::EPSILON (bvh_node.rs:114-124).
template <class T> struct Plan4 { int axis; T cmin, ext; bool halve; uint32_t half; };
template <class T> __device__ __forceinline__ Plan4<T> plan4(const T cb[8], uint32_t count) {
    Plan4<T> p;
    T size[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) size[k] = sub_rn(cb[4 + k], cb[k]);
    p.axis = 0; p.ext = size[0]; p.cmin = cb[0];
#pragma unroll
    for (int k = 1; k < 4; ++k) if (size[k] > p.ext) { p.axis = k; p.ext = size[k]; p.cmin = cb[k]; }
    p.halve = p.ext < Traits<T>::eps();
    p.half = count / 2;
    return p;
}
// bucket of a shape (bvh_node.rs:204-222) or its half of a halved range
template <class T> __device__ __forceinline__ int bucket4(const Plan4<T>& p, const T c[4], uint32_t rel_pos) {
    if (p.halve) return rel_pos < p.half ? 0 : 1;
    const T ca = p.axis == 0 ? c[0] : (p.axis == 1 ? c[1] : (p.axis == 2 ? c[2] : c[3]));
    const T K = sub_rn(T(6), T(0.01));                       // T::from(NUM_BUCKETS) - T::from(0.01), bvh_node.rs:214-215
    int b = (int)mul_rn(div_rn(sub_rn(ca, p.cmin), p.ext), K);   // to_usize(): truncation toward zero
    return b < 0 ? 0 : (b > 5 ? 5 : b);                       // inert for tight bounds; keeps memory safe
}

// Bins positions [p0, p1) of src (range starting at r0).  Lane k < 16 folds key k of every bucket into acc[]; cnt[] is warp-uniform.
// The bucket of every position is kept in bkt[] for the scatter.
template <class T>
__device__ __forceinline__ void bin4(const typename D4<T>::Aabb* __restrict__ aabb, const uint32_t* src, uint8_t* bkt, uint32_t r0,
                                     uint32_t p0, uint32_t p1, const Plan4<T>& pl, typename Traits<T>::Key acc[6], uint32_t cnt[6]) {
    using Tr = Traits<T>;
    using Key = typename Tr::Key;
    const int lane = (int)lane_id();
#pragma unroll
    for (int bb = 0; bb < 6; ++bb) { acc[bb] = kmin4(lane & 15) ? Tr::KEY_POS_INF : Tr::KEY_NEG_INF; cnt[bb] = 0; }
    for (uint32_t base = p0; base < p1; base += 32) {
        const uint32_t pos = base + lane;
        T mn[4], mx[4], c[4];
        int b = -1;
        if (pos < p1) {
            load4(aabb + __ldcg(src + pos), mn, mx);
#pragma unroll
            for (int k = 0; k < 4; ++k) c[k] = center1(mn[k], mx[k]);
            b = bucket4(pl, c, pos - r0);
            bkt[pos] = (uint8_t)b;
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) mn[k] = mx[k] = c[k] = T(0);
        }
#pragma unroll
        for (int bb = 0; bb < 6; ++bb) {
            const uint32_t m = __ballot_sync(0xffffffffu, b == bb);
            if (!m) continue;                                      // warp-uniform
            cnt[bb] += __popc(m);
            const bool in = b == bb;
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                const T val = k < 4 ? mn[k & 3] : (k < 8 ? mx[k & 3] : c[k & 3]);
                const bool is_min = kmin4(k);
                const Key v = in ? f2key(val) : (is_min ? Tr::KEY_POS_INF : Tr::KEY_NEG_INF);
                const Key r = is_min ? warp_min_key(v) : warp_max_key(v);
                if (lane == k) acc[bb] = is_min ? (r < acc[bb] ? r : acc[bb]) : (r > acc[bb] ? r : acc[bb]);
            }
        }
    }
}

// Stable 6-way partition of positions [p0, p1) of src into dst; dest[b] = next free position of bucket b (warp-uniform, advanced).
__device__ __forceinline__ void scatter4(const uint32_t* src, uint32_t* dst, const uint8_t* bkt, uint32_t p0, uint32_t p1, uint32_t dest[6]) {
    const uint32_t lane = lane_id(), lt = lanemask_lt();
    for (uint32_t base = p0; base < p1; base += 32) {
        const uint32_t pos = base + lane;
        const bool valid = pos < p1;
        const uint32_t id = valid ? __ldcg(src + pos) : 0u;
        const int b = valid ? (int)bkt[pos] : -1;
        uint32_t d = 0;
#pragma unroll
        for (int bb = 0; bb < 6; ++bb) {
            const uint32_t m = __ballot_sync(0xffffffffu, b == bb);
            if (b == bb) d = dest[bb] + __popc(m & lt);
            dest[bb] += __popc(m);
        }
        if (valid) __stcg(dst + d, id);
    }
}

// The split (bvh_node.rs:225-279) from the six buckets: keys[b * 16 + k], cnt[b].  One thread.  child = lab, lcb, rab, rcb (8 T each);
// Aabb::empty() for all four when no candidate cost is < +inf.  Returns the left count.
template <class T>
__device__ uint32_t split4(const typename Traits<T>::Key* keys, const uint32_t cnt[6], const T ab[8], const Plan4<T>& pl, T child[32]) {
    using Tr = Traits<T>;
    using Key = typename Tr::Key;
    if (pl.halve) {                                          // children = the two halves, bounds recomputed (joint_aabb / centroid)
        for (int k = 0; k < 8; ++k) {
            child[k] = key2f(keys[k]); child[8 + k] = key2f(keys[8 + k]);
            child[16 + k] = key2f(keys[16 + k]); child[24 + k] = key2f(keys[16 + 8 + k]);
        }
        return pl.half;
    }
    int best = 0;
    bool found = false;
    T min_cost = Tr::inf();
    const T sa_parent = surface_area4(ab, ab + 4);
    for (int s = 0; s < 5; ++s) {
        Key L[16], R[16];
        uint32_t nL = 0, nR = 0;
        for (int k = 0; k < 16; ++k) L[k] = R[k] = kmin4(k) ? Tr::KEY_POS_INF : Tr::KEY_NEG_INF;
        for (int b = 0; b <= s; ++b) {
            nL += cnt[b];
            for (int k = 0; k < 16; ++k) L[k] = fold_key(k, L[k], keys[b * 16 + k]);
        }
        for (int b = s + 1; b < 6; ++b) {
            nR += cnt[b];
            for (int k = 0; k < 16; ++k) R[k] = fold_key(k, R[k], keys[b * 16 + k]);
        }
        T lmn[4], lmx[4], rmn[4], rmx[4];
        for (int k = 0; k < 4; ++k) { lmn[k] = key2f(L[k]); lmx[k] = key2f(L[4 + k]); rmn[k] = key2f(R[k]); rmx[k] = key2f(R[4 + k]); }
        // cost = (T(nL) * SA(L) + T(nR) * SA(R)) / SA(aabb_bounds), bvh_node.rs:236-238
        const T cost = div_rn(add_rn(mul_rn((T)nL, surface_area4(lmn, lmx)), mul_rn((T)nR, surface_area4(rmn, rmx))), sa_parent);
        if (cost < min_cost) {
            best = s; min_cost = cost; found = true;
            for (int k = 0; k < 8; ++k) { child[k] = key2f(L[k]); child[8 + k] = key2f(L[8 + k]); child[16 + k] = key2f(R[k]); child[24 + k] = key2f(R[8 + k]); }
        }
    }
    if (!found)                                              // overflowing surface areas: bucket 0 left, empty child bounds
        for (int q = 0; q < 4; ++q) for (int k = 0; k < 8; ++k) child[q * 8 + k] = k < 4 ? Tr::inf() : -Tr::inf();
    uint32_t nl = 0;
    for (int b = 0; b <= best; ++b) nl += cnt[b];
    return nl;
}

template <class T> __device__ __forceinline__ void write_leaf4(typename D4<T>::Node* nodes, uint32_t* node_index, uint32_t* node_start,
                                                               uint32_t node, uint32_t parent, uint32_t shape, uint32_t start) {
    typename D4<T>::Node nd;
    nd.parent = parent; nd.child_l = BVH_INVALID; nd.child_r = BVH_INVALID; nd.shape = shape;
    for (int k = 0; k < 4; ++k) { nd.l_aabb.min[k] = nd.r_aabb.min[k] = Traits<T>::inf(); nd.l_aabb.max[k] = nd.r_aabb.max[k] = -Traits<T>::inf(); }
    nodes[node] = nd;
    node_index[shape] = node;                                // Shapes::set_node_index, bvh_node.rs:103
    node_start[node] = start;
}
template <class T> __device__ __forceinline__ void write_inner4(typename D4<T>::Node* nodes, uint32_t* node_start, const Task4<T>& t,
                                                                uint32_t nl, const T child[32]) {
    typename D4<T>::Node nd;
    nd.parent = t.parent; nd.child_l = t.node + 1; nd.child_r = t.node + 2 * nl; nd.shape = t.count;
    for (int k = 0; k < 4; ++k) {
        nd.l_aabb.min[k] = child[k]; nd.l_aabb.max[k] = child[4 + k];
        nd.r_aabb.min[k] = child[16 + k]; nd.r_aabb.max[k] = child[20 + k];
    }
    nodes[t.node] = nd;
    node_start[t.node] = t.start;
}
template <class T> __device__ __forceinline__ Task4<T> child_task(const Task4<T>& t, int side, uint32_t nl, const T child[32]) {
    Task4<T> c;
    c.start = side ? t.start + nl : t.start;
    c.count = side ? t.count - nl : nl;
    c.node = side ? t.node + 2 * nl : t.node + 1;
    c.parent = t.node;
    c.buf = t.buf ^ 1u;                                      // the split moved the range into the other index buffer
    c.pad[0] = c.pad[1] = c.pad[2] = 0;
    for (int k = 0; k < 8; ++k) { c.ab[k] = child[side * 16 + k]; c.cb[k] = child[side * 16 + 8 + k]; }
    return c;
}

struct BuildArgs4 {
    uint32_t* idx[2];          // index buffers
    uint8_t* bkt;              // bucket of every position (bin -> scatter)
    uint32_t* ctl;             // CTL_* words
    void* small;               // Task4[]: ranges of <= SMALL4 shapes
};

// ---- upload pass: NaN check, root bounds (keys), identity permutation ----
template <class T>
__global__ void __launch_bounds__(256) upload4_kernel(const typename D4<T>::Aabb* __restrict__ aabb, uint32_t n, uint32_t* __restrict__ idx,
                                                      typename Traits<T>::Key* __restrict__ root_keys, uint32_t* __restrict__ ctl) {
    using Tr = Traits<T>;
    using Key = typename Tr::Key;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    T mn[4], mx[4];
    bool nan = false;
    if (i < n) {
        load4(aabb + i, mn, mx);
        idx[i] = i;
#pragma unroll
        for (int k = 0; k < 4; ++k) nan |= (mn[k] != mn[k]) | (mx[k] != mx[k]);
    }
    if (__any_sync(0xffffffffu, nan) && lane_id() == 0) atomicOr(ctl + CTL_NAN, 1u);
    const int lane = (int)lane_id();
    Key mine = 0;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        const bool is_min = kmin4(k);
        Key v = is_min ? Tr::KEY_POS_INF : Tr::KEY_NEG_INF;
        if (i < n && !nan) v = f2key(k < 4 ? mn[k & 3] : (k < 8 ? mx[k & 3] : center1(mn[k & 3], mx[k & 3])));
        const Key r = is_min ? warp_min_key(v) : warp_max_key(v);
        if (lane == k) mine = r;
    }
    if (lane < 16) { if (kmin4(lane)) atomicMin(root_keys + lane, mine); else atomicMax(root_keys + lane, mine); }
}
template <class T> __global__ void keys_init_kernel(typename Traits<T>::Key* keys, uint32_t groups) {
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < 16 * groups; j += gridDim.x * blockDim.x)
        keys[j] = kmin4((int)(j & 15)) ? Traits<T>::KEY_POS_INF : Traits<T>::KEY_NEG_INF;
}
template <class T> __global__ void root_task4_kernel(const typename Traits<T>::Key* __restrict__ root_keys, uint32_t n, Task4<T>* __restrict__ dst) {
    Task4<T> t;
    t.start = 0; t.count = n; t.node = 0; t.parent = 0; t.buf = 0; t.pad[0] = t.pad[1] = t.pad[2] = 0;
    for (int k = 0; k < 8; ++k) { t.ab[k] = key2f(root_keys[k]); t.cb[k] = key2f(root_keys[8 + k]); }
    *dst = t;
}

// One block of 1024 threads: tile0[j] = first tile of item j (exclusive scan of tiles(j) over j < m), total in tile0[m].
template <class F> __device__ __forceinline__ void tile_scan1024(uint32_t m, F tiles, uint32_t* __restrict__ tile0) {
    __shared__ uint32_t wsum[32];
    __shared__ uint32_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint32_t j0 = 0; j0 < m; j0 += 1024) {
        const uint32_t j = j0 + threadIdx.x;
        const uint32_t v = j < m ? tiles(j) : 0u;
        uint32_t incl = v;
        for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o); if ((int)lane_id() >= o) incl += t; }
        if (lane_id() == 31) wsum[threadIdx.x >> 5] = incl;
        __syncthreads();
        uint32_t woff = 0;
        for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) woff += wsum[w];
        const uint32_t c = carry;
        if (j < m) tile0[j] = c + woff + incl - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry = c + woff + incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) tile0[m] = carry;
}

// ---- large ranges, one level ----
// prep: first tile of every range (exclusive scan of ceil(count / TILE4)), total in tile0[m]; bucket identities; next-level counter.
template <class T>
__global__ void __launch_bounds__(1024) level_prep4_kernel(const Task4<T>* __restrict__ tasks, uint32_t m, uint32_t* __restrict__ tile0,
                                                           typename Traits<T>::Key* __restrict__ acc, uint32_t* __restrict__ acnt, uint32_t* __restrict__ ctl) {
    if (threadIdx.x == 0) ctl[CTL_NEXT] = 0;
    tile_scan1024(m, [&](uint32_t j) { return (tasks[j].count + TILE4 - 1) / TILE4; }, tile0);
    for (uint32_t j = threadIdx.x; j < 96 * m; j += 1024) acc[j] = kmin4((int)(j & 15)) ? Traits<T>::KEY_POS_INF : Traits<T>::KEY_NEG_INF;
    for (uint32_t j = threadIdx.x; j < 6 * m; j += 1024) acnt[j] = 0;
}

__device__ __forceinline__ uint32_t tile_owner(const uint32_t* tile0, uint32_t m, uint32_t t) {   // last j with tile0[j] <= t
    uint32_t lo = 0, hi = m - 1;
    while (lo < hi) { const uint32_t mid = (lo + hi + 1) >> 1; if (tile0[mid] <= t) lo = mid; else hi = mid - 1; }
    return lo;
}

template <class T>
__global__ void __launch_bounds__(256) level_bin4_kernel(const typename D4<T>::Aabb* __restrict__ aabb, const Task4<T>* __restrict__ tasks, uint32_t m,
                                                         const uint32_t* __restrict__ tile0, BuildArgs4 A, typename Traits<T>::Key* __restrict__ acc,
                                                         uint32_t* __restrict__ acnt, uint32_t* __restrict__ tilecnt) {
    using Key = typename Traits<T>::Key;
    const uint32_t ntiles = tile0[m];
    const int lane = (int)lane_id();
    for (uint32_t t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < ntiles; t += (gridDim.x * blockDim.x) >> 5) {
        const uint32_t j = tile_owner(tile0, m, t);
        const Task4<T>& tk = tasks[j];
        const uint32_t p0 = tk.start + (t - tile0[j]) * TILE4, p1 = min(p0 + TILE4, tk.start + tk.count);
        const Plan4<T> pl = plan4<T>(tk.cb, tk.count);
        Key a[6];
        uint32_t cnt[6];
        bin4<T>(aabb, A.idx[tk.buf], A.bkt, tk.start, p0, p1, pl, a, cnt);
#pragma unroll
        for (int bb = 0; bb < 6; ++bb) {
            if (!cnt[bb]) continue;
            if (lane < 16) { if (kmin4(lane)) atomicMin(acc + 96 * (size_t)j + 16 * bb + lane, a[bb]); else atomicMax(acc + 96 * (size_t)j + 16 * bb + lane, a[bb]); }
            if (lane == 0) atomicAdd(acnt + 6 * (size_t)j + bb, cnt[bb]);
        }
        if (lane < 6) {
            uint32_t c = cnt[0];
#pragma unroll
            for (int bb = 1; bb < 6; ++bb) c = lane == bb ? cnt[bb] : c;
            tilecnt[6 * (size_t)t + lane] = c;
        }
    }
}

// one warp per range: the split, the node, the children, and the stable destination of every (tile, bucket)
template <class T>
__global__ void __launch_bounds__(256) level_split4_kernel(const Task4<T>* __restrict__ tasks, uint32_t m, const uint32_t* __restrict__ tile0,
                                                           const typename Traits<T>::Key* __restrict__ acc, const uint32_t* __restrict__ acnt,
                                                           uint32_t* __restrict__ tiledest, Task4<T>* __restrict__ next, BuildArgs4 A,
                                                           typename D4<T>::Node* __restrict__ nodes, uint32_t* __restrict__ node_index, uint32_t* __restrict__ node_start) {
    const uint32_t j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (j >= m) return;
    const uint32_t lane = lane_id();
    const Task4<T> t = tasks[j];
    uint32_t cnt[6], dest[6], run = t.start;
    for (int b = 0; b < 6; ++b) { cnt[b] = acnt[6 * (size_t)j + b]; dest[b] = run; run += cnt[b]; }
    for (uint32_t q0 = tile0[j]; q0 < tile0[j + 1]; q0 += 32) {
        const uint32_t q = q0 + lane;
        const bool in = q < tile0[j + 1];
        for (int b = 0; b < 6; ++b) {
            const uint32_t v = in ? tiledest[6 * (size_t)q + b] : 0u;
            uint32_t incl = v;
            for (int o = 1; o < 32; o <<= 1) { const uint32_t x = __shfl_up_sync(0xffffffffu, incl, o); if ((int)lane >= o) incl += x; }
            if (in) tiledest[6 * (size_t)q + b] = dest[b] + incl - v;
            dest[b] += __shfl_sync(0xffffffffu, incl, 31);
        }
    }
    if (lane != 0) return;
    const Plan4<T> pl = plan4<T>(t.cb, t.count);
    T child[32];
    const uint32_t nl = split4<T>(acc + 96 * (size_t)j, cnt, t.ab, pl, child);
    if (nl == 0 || nl >= t.count) { atomicCAS(A.ctl + CTL_ERROR, 0u, (uint32_t)BVHGPU_ERR_INTERNAL); return; }
    write_inner4<T>(nodes, node_start, t, nl, child);
    Task4<T>* small = reinterpret_cast<Task4<T>*>(A.small);
    for (int side = 0; side < 2; ++side) {
        const Task4<T> c = child_task<T>(t, side, nl, child);
        if (c.count > SMALL4) next[atomicAdd(A.ctl + CTL_NEXT, 1u)] = c;
        else small[atomicAdd(A.ctl + CTL_SMALL, 1u)] = c;
    }
}

template <class T>
__global__ void __launch_bounds__(256) level_scatter4_kernel(const Task4<T>* __restrict__ tasks, uint32_t m, const uint32_t* __restrict__ tile0,
                                                             const uint32_t* __restrict__ tiledest, BuildArgs4 A) {
    const uint32_t ntiles = tile0[m];
    for (uint32_t t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < ntiles; t += (gridDim.x * blockDim.x) >> 5) {
        const uint32_t j = tile_owner(tile0, m, t);
        const Task4<T>& tk = tasks[j];
        const uint32_t p0 = tk.start + (t - tile0[j]) * TILE4, p1 = min(p0 + TILE4, tk.start + tk.count);
        uint32_t dest[6];
        for (int b = 0; b < 6; ++b) dest[b] = tiledest[6 * (size_t)t + b];
        scatter4(A.idx[tk.buf], A.idx[tk.buf ^ 1u], A.bkt, p0, p1, dest);
    }
}

// ---- small ranges: one warp each, depth-first ----
template <class T> struct __align__(16) WarpState4 {
    typename Traits<T>::Key keys[96];
    T child[32];
    uint32_t nl;
    uint32_t pad[3];
    Task4<T> stack[STACK4];
};

template <class T>
__global__ void __launch_bounds__(256) small4_kernel(const typename D4<T>::Aabb* __restrict__ aabb, uint32_t count, BuildArgs4 A,
                                                     typename D4<T>::Node* __restrict__ nodes, uint32_t* __restrict__ node_index, uint32_t* __restrict__ node_start) {
    using Key = typename Traits<T>::Key;
    __shared__ WarpState4<T> st[8];
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= count) return;
    WarpState4<T>& ws = st[threadIdx.x >> 5];
    const int lane = (int)lane_id();
    Task4<T> t = reinterpret_cast<const Task4<T>*>(A.small)[w];
    int top = 0;
    for (;;) {
        if (t.count == 1) {
            if (lane == 0) write_leaf4<T>(nodes, node_index, node_start, t.node, t.parent, __ldcg(A.idx[t.buf] + t.start), t.start);
        } else {
            const Plan4<T> pl = plan4<T>(t.cb, t.count);
            Key a[6];
            uint32_t cnt[6];
            bin4<T>(aabb, A.idx[t.buf], A.bkt, t.start, t.start, t.start + t.count, pl, a, cnt);
            if (lane < 16) {
#pragma unroll
                for (int bb = 0; bb < 6; ++bb) ws.keys[16 * bb + lane] = a[bb];
            }
            __syncwarp();
            if (lane == 0) {
                ws.nl = split4<T>(ws.keys, cnt, t.ab, pl, ws.child);
                if (ws.nl == 0 || ws.nl >= t.count) atomicCAS(A.ctl + CTL_ERROR, 0u, (uint32_t)BVHGPU_ERR_INTERNAL);
                else write_inner4<T>(nodes, node_start, t, ws.nl, ws.child);
            }
            __syncwarp();
            const uint32_t nl = ws.nl;
            if (nl == 0 || nl >= t.count) return;
            uint32_t dest[6], run = t.start;
#pragma unroll
            for (int b = 0; b < 6; ++b) { dest[b] = run; run += cnt[b]; }
            scatter4(A.idx[t.buf], A.idx[t.buf ^ 1u], A.bkt, t.start, t.start + t.count, dest);
            __syncwarp();
            const Task4<T> l = child_task<T>(t, 0, nl, ws.child), r = child_task<T>(t, 1, nl, ws.child);
            const bool left_first = l.count <= r.count;           // continue with the smaller child, push the larger
            if (top == STACK4) { if (lane == 0) atomicCAS(A.ctl + CTL_ERROR, 0u, (uint32_t)BVHGPU_ERR_INTERNAL); return; }
            if (lane == 0) ws.stack[top] = left_first ? r : l;
            ++top;
            t = left_first ? l : r;
            __syncwarp();
            continue;
        }
        if (top == 0) break;
        __syncwarp();
        t = ws.stack[--top];
        __syncwarp();
    }
}

// ---- flatten and traversal records: closed forms over the preorder node array (as flatten.cu) ----
template <class T>
__global__ void __launch_bounds__(256) flat4_kernel(const typename D4<T>::Node* __restrict__ nodes, const uint32_t* __restrict__ node_start,
                                                    uint32_t n_nodes, typename D4<T>::Flat* __restrict__ flat) {
    using Flat = typename D4<T>::Flat;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_nodes) return;
    const typename D4<T>::Node& nd = nodes[i];
    const bool leaf = nd.child_l == BVH_INVALID;
    Flat g;
    for (int k = 0; k < 4; ++k) { g.aabb.min[k] = Traits<T>::inf(); g.aabb.max[k] = -Traits<T>::inf(); }
    if constexpr (sizeof(T) == 8) g._pad = 0;
    if (i == 0) {
        if (leaf) { g.entry_index = BVH_INVALID; g.exit_index = 1; g.shape_index = nd.shape; flat[0] = g; }   // flat_bvh.rs:129-141 only
        return;
    }
    const uint32_t nav = (i - 1) + node_start[i];
    const uint32_t count = leaf ? 1u : nd.shape;
    const typename D4<T>::Node& par = nodes[nd.parent];
    const bool is_left = par.child_l == i;
    Flat f = g;
    for (int k = 0; k < 4; ++k) {
        f.aabb.min[k] = is_left ? par.l_aabb.min[k] : par.r_aabb.min[k];
        f.aabb.max[k] = is_left ? par.l_aabb.max[k] : par.r_aabb.max[k];
    }
    f.entry_index = nav + 1; f.exit_index = nav + 3 * count - 1; f.shape_index = BVH_INVALID;   // flat_bvh.rs:80-88
    flat[nav] = f;
    if (leaf) { g.entry_index = BVH_INVALID; g.exit_index = nav + 2; g.shape_index = nd.shape; flat[nav + 1] = g; }
}

// record r = node r+1 (the root has no box of its own); a root leaf gets the shape's own box (bvh_node.rs:314)
template <class T>
__global__ void __launch_bounds__(256) trec4_kernel(const typename D4<T>::Node* __restrict__ nodes, uint32_t n_nodes,
                                                    const typename D4<T>::Aabb* __restrict__ aabb, typename D4<T>::Rec* __restrict__ trec) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_nodes) return;
    typename D4<T>::Rec r;
    r.pad[0] = r.pad[1] = 0;
    if (n_nodes == 1) {
        const uint32_t s = nodes[0].shape;
        for (int k = 0; k < 4; ++k) { r.min[k] = aabb[s].min[k]; r.max[k] = aabb[s].max[k]; }
        r.skip = 1; r.shape = s;
        trec[0] = r;
        return;
    }
    if (i == 0) return;
    const typename D4<T>::Node& nd = nodes[i];
    const bool leaf = nd.child_l == BVH_INVALID;
    const typename D4<T>::Node& par = nodes[nd.parent];
    const bool is_left = par.child_l == i;
    for (int k = 0; k < 4; ++k) {
        r.min[k] = is_left ? par.l_aabb.min[k] : par.r_aabb.min[k];
        r.max[k] = is_left ? par.l_aabb.max[k] : par.r_aabb.max[k];
    }
    r.skip = (i - 1) + (2 * (leaf ? 1u : nd.shape) - 1);
    r.shape = leaf ? nd.shape : BVH_INVALID;
    trec[i - 1] = r;
}

// ---- walk: one ray per thread over the records, the 4-wide slab test (intersect_default.rs:16-37, intersect_simd.rs) ----
template <class T>
__device__ __forceinline__ bool slab4(const T o[4], const T inv[4], const T mn[4], const T mx[4]) {
    T lo[4], hi[4];
    bool nan = false;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const T l = mul_rn(sub_rn(mn[k], o[k]), inv[k]), r = mul_rn(sub_rn(mx[k], o[k]), inv[k]);
        nan |= (l != l) | (r != r);                            // any NaN rejects the box
        lo[k] = min_t(l, r); hi[k] = max_t(l, r);
    }
    const T tmin = max_t(max_t(lo[0], lo[1]), max_t(lo[2], lo[3]));
    const T tmax = min_t(min_t(hi[0], hi[1]), min_t(hi[2], hi[3]));
    return !nan && tmax >= (tmin > T(0) ? tmin : T(0));
}

// The probe of a ray batch for csr_walk_kernel (csr.cuh): load(src, r) reads ray r, hit(mn, mx) is the 4-wide slab test.  Queries
// use Query<T, KIND, 4> of queries.cuh (query_csr).
template <class T> struct RayProbe4 {
    T o[4], inv[4];
    __device__ __forceinline__ void load(const void* src, uint32_t r) { load_ray_full(reinterpret_cast<const typename D4<T>::Ray*>(src) + r, o, inv); }
    __device__ __forceinline__ bool hit(const T mn[4], const T mx[4]) const { return slab4(o, inv, mn, mx); }
};

// ---- nearest_to: the walks of queries.cuh over the 4-D nodes / flat array; the leaf value is the shape AABB's distance ----
template <class T, bool FLAT>
__global__ void __launch_bounds__(128) nearest4_kernel(const typename D4<T>::Node* __restrict__ nodes, const typename D4<T>::Flat* __restrict__ flat,
                                                       uint32_t n_flat, const typename D4<T>::Aabb* __restrict__ aabb, const T* __restrict__ points,
                                                       uint32_t nq, uint32_t* __restrict__ out_shape, T* __restrict__ out_dist) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    T p[4];
    for (int k = 0; k < 4; ++k) p[k] = points[4 * (size_t)i + k];
    uint32_t best = BVH_INVALID;
    T best_d = T(0);
    auto leaf = [&](uint32_t shape) { T mn[4], mx[4]; load4(aabb + shape, mn, mx); return aabb_min_d2<4>(p, mn, mx); };
    if (!FLAT) nearest_walk<4, T, true>(nodes, p, best, best_d, leaf);
    else       nearest_flat<4, T>(flat, n_flat, p, best, best_d, leaf);
    out_shape[i] = best;
    out_dist[i] = sqrt_rn(best_d);                          // bvh_impl.rs:237
}
// k nearest shapes: knn_walk<4, T, K> (queries.cuh) over the 4-D nodes, keys from the shapes' own boxes; one thread per point
template <class T, int K>
__global__ void __launch_bounds__(128) knn4_kernel(const typename D4<T>::Node* __restrict__ nodes, uint32_t n_shapes, const typename D4<T>::Aabb* __restrict__ aabb,
                                                   const T* __restrict__ points, const T* __restrict__ max_dist, uint32_t nq, uint32_t k,
                                                   uint32_t* __restrict__ out_shape, T* __restrict__ out_dist) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    T p[4];
    for (int c = 0; c < 4; ++c) p[c] = points[4 * (size_t)i + c];
    auto leaf = [&](uint32_t shape) { T mn[4], mx[4]; load4(aabb + shape, mn, mx); return aabb_min_d2<4>(p, mn, mx); };
    knn_point<4, T, K>(nodes, n_shapes, p, max_dist != nullptr, max_dist ? max_dist[i] : T(0), k, out_shape + (size_t)i * k,
                       out_dist + (size_t)i * k, leaf);
}
// nearest_candidates, first pass: the farthest-corner bound U of every point (as nearest_bound_kernel), records {p, U} for QUERY_WITHIN
template <class T>
__global__ void __launch_bounds__(128) nearest_bound4_kernel(const typename D4<T>::Node* __restrict__ nodes, const typename D4<T>::Aabb* __restrict__ aabb,
                                                             const T* __restrict__ points, uint32_t nq, T* __restrict__ records) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    T p[4];
    for (int k = 0; k < 4; ++k) p[k] = points[4 * (size_t)i + k];
    uint32_t best;
    T u, g[4];
    root_magnitude<4>(nodes, p, g);
    nearest_walk<4, T, false>(nodes, p, best, u, [&](uint32_t shape) { T mn[4], mx[4]; load4(aabb + shape, mn, mx); return box_upper_d2<4>(p, mn, mx, g); });
    u = mul_rn(u, add_rn(T(1), mul_rn(T(16), Traits<T>::eps())));      // the bound itself is a rounded sum: keep it an upper bound
    for (int k = 0; k < 4; ++k) records[5 * (size_t)i + k] = p[k];
    records[5 * (size_t)i + 4] = u;
}

// ---- the growth rebuild of update_shapes / add_shapes and the group subtrees of add_shapes (DESIGN.md sections 4.12, 4.13) ----
// Seeding the builder from the rebuild roots roots[0 .. *n_roots) (disjoint inner nodes).  The subtree of root r with c shapes is the
// node range [r, r + 2c - 1) over the leaf positions [node_start[r], node_start[r] + c).  Its nodes are cut into tiles of TILE4, so
// that a root that holds every shape (global motion) is reduced by many warps, as level_bin4 does.
// prep (one block): first tile of every root, total in tile0[nr]; centre-bound keys (min xyzw, max xyzw per root) at their identities.
template <class T>
__global__ void __launch_bounds__(1024) root_tiles4_kernel(const typename D4<T>::Node* __restrict__ nodes, const uint32_t* __restrict__ roots,
                                                           const uint32_t* __restrict__ n_roots, uint32_t* __restrict__ tile0,
                                                           typename Traits<T>::Key* __restrict__ keys) {
    const uint32_t nr = *n_roots;
    tile_scan1024(nr, [&](uint32_t j) { return (2 * nodes[roots[j]].shape - 1 + TILE4 - 1) / TILE4; }, tile0);
    for (uint32_t j = threadIdx.x; j < 8 * nr; j += 1024) keys[j] = (j & 7) < 4 ? Traits<T>::KEY_POS_INF : Traits<T>::KEY_NEG_INF;
}
// bin (one warp per tile): every leaf of the tile puts its shape at its leaf position of index buffer 0 and folds its centre into the
// root's keys
template <class T>
__global__ void __launch_bounds__(256) root_bin4_kernel(const typename D4<T>::Node* __restrict__ nodes, const uint32_t* __restrict__ node_start,
                                                        const typename D4<T>::Aabb* __restrict__ aabb, const uint32_t* __restrict__ roots,
                                                        const uint32_t* __restrict__ n_roots, const uint32_t* __restrict__ tile0, uint32_t* __restrict__ idx0,
                                                        typename Traits<T>::Key* __restrict__ keys) {
    const uint32_t nr = *n_roots;
    if (nr == 0) return;
    const uint32_t ntiles = tile0[nr];
    for (uint32_t t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < ntiles; t += (gridDim.x * blockDim.x) >> 5) {
        const uint32_t j = tile_owner(tile0, nr, t), r = roots[j];
        const uint32_t end = r + 2 * nodes[r].shape - 1, i0 = r + (t - tile0[j]) * TILE4, i1 = min(i0 + TILE4, end);
        T cmn[4], cmx[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) { cmn[k] = Traits<T>::inf(); cmx[k] = -Traits<T>::inf(); }
        for (uint32_t i = i0 + lane_id(); i < i1; i += 32) {
            const uint4 meta = *reinterpret_cast<const uint4*>(nodes + i);    // parent, child_l, child_r, shape
            if (meta.y != BVH_INVALID) continue;
            idx0[node_start[i]] = meta.w;
            T mn[4], mx[4];
            load4(aabb + meta.w, mn, mx);
#pragma unroll
            for (int k = 0; k < 4; ++k) { const T c = center1(mn[k], mx[k]); cmn[k] = min_t(cmn[k], c); cmx[k] = max_t(cmx[k], c); }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const typename Traits<T>::Key a = warp_min_key(f2key(cmn[k])), b = warp_max_key(f2key(cmx[k]));
            if (lane_id() == 0) { atomicMin(keys + 8 * (size_t)j + k, a); atomicMax(keys + 8 * (size_t)j + 4 + k, b); }
        }
    }
}
// rebase (one warp per tile of root_tiles4): the nodes of the rebuilt subtrees get their new surface area as the growth baseline.  The
// tiles matter when a root holds every shape: rebase_kernel (update.cuh) gives each root a single warp.
template <class T>
__global__ void __launch_bounds__(256) rebase4_kernel(const typename D4<T>::Node* __restrict__ nodes, const uint32_t* __restrict__ roots,
                                                      const uint32_t* __restrict__ n_roots, const uint32_t* __restrict__ tile0, T* __restrict__ sa_base) {
    const uint32_t nr = *n_roots;
    if (nr == 0) return;
    const uint32_t ntiles = tile0[nr];
    for (uint32_t t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < ntiles; t += (gridDim.x * blockDim.x) >> 5) {
        const uint32_t j = tile_owner(tile0, nr, t), r = roots[j];
        const uint32_t end = r + 2 * __ldcg(&nodes[r].shape) - 1, i0 = r + (t - tile0[j]) * TILE4, i1 = min(i0 + TILE4, end);
        for (uint32_t i = i0 + lane_id(); i < i1; i += 32) {
            const typename D4<T>::Node& nd = nodes[i];
            if (__ldcg(&nd.child_l) == BVH_INVALID) { sa_base[i] = T(0); continue; }
            T mn[4], mx[4];
            for (int c = 0; c < 4; ++c) { mn[c] = min_t(__ldcg(&nd.l_aabb.min[c]), __ldcg(&nd.r_aabb.min[c])); mx[c] = max_t(__ldcg(&nd.l_aabb.max[c]), __ldcg(&nd.r_aabb.max[c])); }
            sa_base[i] = surface_area4(mn, mx);
        }
    }
}
// seed (one thread per root): the root's task -- its leaf range, node, parent, box (the join of its two child boxes, as the 3-D
// rebuild takes it: tight after the climb) and centre bounds -- into the level list (> SMALL4 shapes) or the small list
template <class T>
__global__ void __launch_bounds__(256) root_seed4_kernel(const typename D4<T>::Node* __restrict__ nodes, const uint32_t* __restrict__ node_start,
                                                         const uint32_t* __restrict__ roots, const uint32_t* __restrict__ n_roots,
                                                         const typename Traits<T>::Key* __restrict__ keys, Task4<T>* __restrict__ tasks, BuildArgs4 A) {
    const uint32_t nr = *n_roots;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < nr; j += gridDim.x * blockDim.x) {
        const uint32_t r = roots[j];
        const typename D4<T>::Node& nd = nodes[r];
        Task4<T> t;
        t.start = node_start[r]; t.count = nd.shape; t.node = r; t.parent = nd.parent;
        t.buf = 0; t.pad[0] = t.pad[1] = t.pad[2] = 0;
        for (int k = 0; k < 4; ++k) {
            t.ab[k] = min_t(nd.l_aabb.min[k], nd.r_aabb.min[k]); t.ab[4 + k] = max_t(nd.l_aabb.max[k], nd.r_aabb.max[k]);
            t.cb[k] = key2f(keys[8 * (size_t)j + k]); t.cb[4 + k] = key2f(keys[8 * (size_t)j + 4 + k]);
        }
        atomicAdd(A.ctl + CTL_REBUILT, t.count);
        if (t.count > SMALL4) tasks[atomicAdd(A.ctl + CTL_NEXT, 1u)] = t;
        else reinterpret_cast<Task4<T>*>(A.small)[atomicAdd(A.ctl + CTL_SMALL, 1u)] = t;
    }
}

// ================================================================================================================================
// host side
// ================================================================================================================================
#define LAUNCHED(ctx, k) do { (ctx)->launches += (k); BVH_CUDA_TRY(cudaGetLastError()); } while (0)

// Buffers of the level loop, sized for n shapes: at most max_tasks disjoint ranges of > SMALL4 shapes on one level.
template <class T> struct Levels4 {
    Task4<T>* tasks = nullptr;                   // [2 max_tasks]: this level's ranges, the next level's
    typename Traits<T>::Key* acc = nullptr;      // [96 max_tasks] bucket keys
    uint32_t *acnt = nullptr, *tile0 = nullptr, *tilecnt = nullptr;
    uint32_t max_tasks = 0;
};
template <class T> static int levels4_alloc(Scratch& scratch, uint32_t n, Levels4<T>* L) {
    L->max_tasks = n / (SMALL4 + 1) + 1;
    const uint32_t max_tiles = n / TILE4 + L->max_tasks;
    BVH_TRY(scratch.get(&L->tasks, 2 * (size_t)L->max_tasks));
    BVH_TRY(scratch.get(&L->acc, 96 * (size_t)L->max_tasks));
    BVH_TRY(scratch.get(&L->acnt, 6 * (size_t)L->max_tasks));
    BVH_TRY(scratch.get(&L->tile0, (size_t)L->max_tasks + 1));
    BVH_TRY(scratch.get(&L->tilecnt, 6 * (size_t)max_tiles));
    return BVHGPU_OK;
}

// The builder from seeded tasks: the ranges of more than SMALL4 shapes in L.tasks[0 .. m) go through the level loop, then the n_small
// ranges in A.small (the seeds' and the loop's) are finished by small4_kernel.  Build and rebuild run this same code.  Synchronous: the
// host reads the range count of every level.  `who` names the caller in error messages.
template <class T> static int run_levels4(Tree4<T>* tree, const BuildArgs4& A, const Levels4<T>& L, uint32_t m, uint32_t n_small, const char* who) {
    bvhgpu_ctx* ctx = tree->ctx;
    cudaStream_t st = ctx->stream;
    const uint32_t n = tree->n;
    uint32_t* h = ctx->h_pinned + 232;
    const std::string err = std::string(who) + ": the device reported an empty split (non-finite input?); the tree is unusable";
    const int wave = std::max(ctx->sm_count, 1) * 8;           // blocks of the grid-stride tile kernels
    int cur = 0;
    while (m) {
        Task4<T>* tc = L.tasks + (size_t)cur * L.max_tasks;
        Task4<T>* tn = L.tasks + (size_t)(cur ^ 1) * L.max_tasks;
        const uint32_t tiles_bound = n / TILE4 + m;
        const int grid = (int)std::min<uint32_t>((tiles_bound + 7) / 8, (uint32_t)wave);
        level_prep4_kernel<T><<<1, 1024, 0, st>>>(tc, m, L.tile0, L.acc, L.acnt, A.ctl);
        level_bin4_kernel<T><<<grid, 256, 0, st>>>(tree->d_aabb, tc, m, L.tile0, A, L.acc, L.acnt, L.tilecnt);
        level_split4_kernel<T><<<(m + 7) / 8, 256, 0, st>>>(tc, m, L.tile0, L.acc, L.acnt, L.tilecnt, tn, A, tree->d_nodes, tree->d_node_index, tree->d_node_start);
        level_scatter4_kernel<T><<<grid, 256, 0, st>>>(tc, m, L.tile0, L.tilecnt, A);
        LAUNCHED(ctx, 4);
        BVH_CUDA_TRY(cudaMemcpyAsync(h, A.ctl, 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        BVH_CUDA_TRY(cudaStreamSynchronize(st));
        if (h[CTL_ERROR]) return mark_failed(tree, (int)h[CTL_ERROR], who, err.c_str());
        m = h[CTL_NEXT];
        n_small = h[CTL_SMALL];
        cur ^= 1;
    }
    if (n_small) {
        small4_kernel<T><<<(n_small + 7) / 8, 256, 0, st>>>(tree->d_aabb, n_small, A, tree->d_nodes, tree->d_node_index, tree->d_node_start);
        LAUNCHED(ctx, 1);
    }
    BVH_CUDA_TRY(cudaMemcpyAsync(h, A.ctl, 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    BVH_CUDA_TRY(cudaStreamSynchronize(st));
    if (h[CTL_ERROR]) return mark_failed(tree, (int)h[CTL_ERROR], who, err.c_str());
    return BVHGPU_OK;
}

// The exact SAH build.  h_aabbs: host pointer (device pointer with kind = cudaMemcpyDeviceToDevice).  Synchronous (the host learns the range count of every level anyway).
template <class T> int build4(Tree4<T>* tree, const typename D4<T>::Aabb* h_aabbs, cudaMemcpyKind kind) {
    using Key = typename Traits<T>::Key;
    bvhgpu_ctx* ctx = tree->ctx;
    cudaStream_t st = ctx->stream;
    const uint32_t n = tree->n;
    BVH_TRY(dalloc_t(ctx, &tree->d_aabb, n));
    BVH_TRY(dalloc_t(ctx, &tree->d_nodes, tree->n_nodes));
    BVH_TRY(dalloc_t(ctx, &tree->d_node_index, n));
    BVH_TRY(dalloc_t(ctx, &tree->d_node_start, tree->n_nodes));
    BVH_CUDA_TRY(cudaMemcpyAsync(tree->d_aabb, h_aabbs, sizeof(*h_aabbs) * n, kind, st));

    Scratch scratch(ctx);
    BuildArgs4 A{};
    uint32_t* idx = nullptr;
    Key* root_keys = nullptr;
    Task4<T>* small = nullptr;
    BVH_TRY(scratch.get(&idx, 2 * (size_t)n));
    BVH_TRY(scratch.get(&A.bkt, n));
    BVH_TRY(scratch.get(&A.ctl, 8));
    BVH_TRY(scratch.get(&root_keys, 16));
    BVH_TRY(scratch.get(&small, n));
    A.idx[0] = idx; A.idx[1] = idx + n; A.small = small;
    BVH_CUDA_TRY(cudaMemsetAsync(A.ctl, 0, 8 * sizeof(uint32_t), st));
    keys_init_kernel<T><<<1, 32, 0, st>>>(root_keys, 1);
    upload4_kernel<T><<<(n + 255) / 256, 256, 0, st>>>(tree->d_aabb, n, idx, root_keys, A.ctl);
    LAUNCHED(ctx, 2);
    uint32_t* h = ctx->h_pinned + 232;
    BVH_CUDA_TRY(cudaMemcpyAsync(h, A.ctl, 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    BVH_CUDA_TRY(cudaStreamSynchronize(st));
    if (h[CTL_NAN]) return mark_failed(tree, BVHGPU_ERR_NAN, "build", "build: NaN coordinate in an input AABB (the reference panics here, src/bvh/bvh_node.rs:214-217)");

    Levels4<T> L;
    if (n > SMALL4) {                                          // one root task: the level list, or the small list
        BVH_TRY(levels4_alloc(scratch, n, &L));
        root_task4_kernel<T><<<1, 1, 0, st>>>(root_keys, n, L.tasks);
    } else {
        root_task4_kernel<T><<<1, 1, 0, st>>>(root_keys, n, small);
    }
    LAUNCHED(ctx, 1);
    return run_levels4(tree, A, L, n > SMALL4 ? 1u : 0u, n > SMALL4 ? 0u : 1u, "build");
}

// The FlatBvh, built once (3n - 2 nodes for n >= 2, 1 for n == 1, 0 for n == 0).
template <class T> int build_flat4(Tree4<T>* tree) {
    bvhgpu_ctx* ctx = tree->ctx;
    tree->n_flat = tree->n == 0 ? 0 : (tree->n == 1 ? 1 : 3 * (size_t)tree->n - 2);
    if (tree->n && !tree->d_flat) {
        BVH_TRY(dalloc_t(ctx, &tree->d_flat, tree->n_flat));
        flat4_kernel<T><<<(tree->n_nodes + 255) / 256, 256, 0, ctx->stream>>>(tree->d_nodes, tree->d_node_start, tree->n_nodes, tree->d_flat);
        LAUNCHED(ctx, 1);
    }
    return BVHGPU_OK;
}

// The traversal records of the CSR walks, built on first use.
template <class T> int ensure_records(Tree4<T>* tree) {
    bvhgpu_ctx* ctx = tree->ctx;
    if (tree->d_tnodes) return BVHGPU_OK;
    tree->n_trec = tree->n == 1 ? 1u : tree->n_nodes - 1;
    BVH_TRY(dalloc_t(ctx, &tree->d_tnodes, tree->n_trec));
    trec4_kernel<T><<<(tree->n_nodes + 255) / 256, 256, 0, ctx->stream>>>(tree->d_nodes, tree->n_nodes, tree->d_aabb, tree->d_tnodes);
    LAUNCHED(ctx, 1);
    return BVHGPU_OK;
}

// ---- the CSR walks of csr.cuh: the 4-D ray traversal is the query walk with RayProbe4 ----
template <class T> int traverse_csr(Tree4<T>* tree, int mode, const void* rays, size_t n, const CsrOut& out, const char* what) {
    BVH_TRY(check_walk(what, n, mode));
    return probe_csr<RayProbe4<T>>(tree, mode == BVHGPU_TRAVERSE_FLAT, rays, n, out, what);
}
template <class T> int nearest_bound(Tree4<T>* tree, const T* d_points, uint32_t n, T* d_records) {
    bvhgpu_ctx* ctx = tree->ctx;
    nearest_bound4_kernel<T><<<(n + 127) / 128, 128, 0, ctx->stream>>>(tree->d_nodes, tree->d_aabb, d_points, n, d_records);
    LAUNCHED(ctx, 1);
    return BVHGPU_OK;
}

// ---- nearest_to: 4 T per point ----
template <class T> int nearest4_device(Tree4<T>* tree, int mode, const T* d_points, size_t n, uint32_t* d_shape, T* d_dist) {
    bvhgpu_ctx* ctx = tree->ctx;
    cudaStream_t st = ctx->stream;
    if (n == 0) return BVHGPU_OK;
    if (tree->n == 0) {                                            // empty tree: None (bvh_impl.rs:229-231)
        BVH_CUDA_TRY(cudaMemsetAsync(d_shape, 0xFF, sizeof(uint32_t) * n, st));
        BVH_CUDA_TRY(cudaMemsetAsync(d_dist, 0, sizeof(T) * n, st));
        return BVHGPU_OK;
    }
    const unsigned grid = (unsigned)((n + 127) / 128);
    if (mode == BVHGPU_TRAVERSE_FLAT) {
        BVH_TRY(build_flat4(tree));
        nearest4_kernel<T, true><<<grid, 128, 0, st>>>(tree->d_nodes, tree->d_flat, (uint32_t)tree->n_flat, tree->d_aabb, d_points, (uint32_t)n, d_shape, d_dist);
    } else {
        nearest4_kernel<T, false><<<grid, 128, 0, st>>>(tree->d_nodes, nullptr, 0u, tree->d_aabb, d_points, (uint32_t)n, d_shape, d_dist);
    }
    LAUNCHED(ctx, 1);
    return BVHGPU_OK;
}
// ---- k nearest shapes: 4 T per point, n limits (nullptr: none), n * k results ----
template <class T> int knn4_device(Tree4<T>* tree, const T* d_points, size_t n, uint32_t k, const T* d_max_dist, uint32_t* d_shape, T* d_dist) {
    if (n > 0x7FFFFFFFull) { set_error("knn: n = %zu exceeds 2^31-1", n); return BVHGPU_ERR_INVALID; }
    if (k < 1 || k > BVHGPU_KNN_MAX_K) { set_error("knn: k = %u outside 1 .. %d", k, BVHGPU_KNN_MAX_K); return BVHGPU_ERR_INVALID; }
    BVH_TRY(resolve_status(tree));
    if (n == 0) return BVHGPU_OK;
    bvhgpu_ctx* ctx = tree->ctx;
    const unsigned grid = (unsigned)((n + 127) / 128);
    knn_bucket(k, [&](auto kb) {
        knn4_kernel<T, decltype(kb)::value><<<grid, 128, 0, ctx->stream>>>(tree->d_nodes, tree->n, tree->d_aabb, d_points, d_max_dist, (uint32_t)n, k, d_shape, d_dist);
    });
    LAUNCHED(ctx, 1);
    return BVHGPU_OK;
}

// ---- the 4-D steps of the dynamic drivers (dynamic.cu) ----
// The traversal records and the flat array, if they were built, are rewritten in place from the new boxes (their sizes do not change);
// otherwise traverse, query, flatten and FLAT nearest_to would keep using the old boxes.
template <class T> int refresh_caches(Tree4<T>* tree) {
    bvhgpu_ctx* ctx = tree->ctx;
    const unsigned g = (tree->n_nodes + 255) / 256;
    if (tree->d_tnodes) { trec4_kernel<T><<<g, 256, 0, ctx->stream>>>(tree->d_nodes, tree->n_nodes, tree->d_aabb, tree->d_tnodes); LAUNCHED(ctx, 1); }
    if (tree->d_flat) { flat4_kernel<T><<<g, 256, 0, ctx->stream>>>(tree->d_nodes, tree->d_node_start, tree->n_nodes, tree->d_flat); LAUNCHED(ctx, 1); }
    return BVHGPU_OK;
}

// Arrays that depend on the node count or the shape numbering, after a relocation: the traversal records and the flat array are
// rebuilt at the new size on first use (refresh_caches rewrites them in place and assumes the node count did not change); the
// update's arrival counters and growth flags are reallocated by the next update.
template <class T> int finish_relayout(Tree4<T>* tree) {
    bvhgpu_ctx* ctx = tree->ctx;
    dfree(ctx, tree->d_tnodes); tree->d_tnodes = nullptr;
    dfree(ctx, tree->d_flat); tree->d_flat = nullptr;
    dfree(ctx, tree->d_arrive); tree->d_arrive = nullptr;
    dfree(ctx, tree->d_bad); tree->d_bad = nullptr;
    tree->n_trec = tree->n == 0 ? 0u : (tree->n == 1 ? 1u : tree->n_nodes - 1);
    tree->n_flat = tree->n == 0 ? 0 : (tree->n == 1 ? 1 : 3 * (size_t)tree->n - 2);
    return BVHGPU_OK;
}

// dirty[0 .. cnts[0]) = the nodes whose box changed, tree->d_bad = their growth flags.  Rebuilds in place, with the level loop and
// small4_kernel of the build, the outermost degraded subtrees (cnts[1], zero on entry, counts them), gives their nodes fresh baselines
// and clears the flags.  *rebuilt = shapes in the rebuilt subtrees.  `who` names the caller in error messages.
template <class T> int rebuild_degraded(Tree4<T>* tree, const uint32_t* dirty, uint32_t* cnts, size_t* rebuilt, const char* who) {
    using Key = typename Traits<T>::Key;
    using Node = typename D4<T>::Node;
    bvhgpu_ctx* ctx = tree->ctx;
    cudaStream_t st = ctx->stream;
    const uint32_t n = tree->n, gn = (tree->n_nodes + 255) / 256;
    const uint32_t max_roots = n / 2 + 1;                       // rebuild roots are inner nodes of disjoint subtrees
    const int wave = std::max(ctx->sm_count, 1) * 8;
    Scratch scratch(ctx);
    BuildArgs4 A{};
    uint32_t *roots = nullptr, *idx = nullptr, *tile0 = nullptr;
    Key* keys = nullptr;
    Task4<T>* small = nullptr;
    Levels4<T> L;
    BVH_TRY(scratch.get(&roots, max_roots));
    BVH_TRY(scratch.get(&tile0, (size_t)max_roots + 1));
    BVH_TRY(scratch.get(&keys, 8 * (size_t)max_roots));
    BVH_TRY(scratch.get(&idx, 2 * (size_t)n));
    BVH_TRY(scratch.get(&A.bkt, n));
    BVH_TRY(scratch.get(&A.ctl, 8));
    BVH_TRY(scratch.get(&small, n));
    BVH_TRY(levels4_alloc(scratch, n, &L));
    A.idx[0] = idx; A.idx[1] = idx + n; A.small = small;
    BVH_CUDA_TRY(cudaMemsetAsync(A.ctl, 0, 8 * sizeof(uint32_t), st));
    select_roots_dirty_kernel<Node><<<gn, 256, 0, st>>>(tree->d_nodes, tree->d_bad, dirty, cnts, roots, cnts + 1);
    root_tiles4_kernel<T><<<1, 1024, 0, st>>>(tree->d_nodes, roots, cnts + 1, tile0, keys);
    root_bin4_kernel<T><<<wave, 256, 0, st>>>(tree->d_nodes, tree->d_node_start, tree->d_aabb, roots, cnts + 1, tile0, idx, keys);
    root_seed4_kernel<T><<<std::min<uint32_t>((max_roots + 255) / 256, (uint32_t)wave), 256, 0, st>>>(tree->d_nodes, tree->d_node_start, roots, cnts + 1,
                                                                                                       keys, L.tasks, A);
    LAUNCHED(ctx, 4);
    uint32_t* h = ctx->h_pinned + 244;
    BVH_CUDA_TRY(cudaMemcpyAsync(h, A.ctl, 5 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    BVH_CUDA_TRY(cudaStreamSynchronize(st));
    const uint32_t m = h[CTL_NEXT], n_small = h[CTL_SMALL], shapes = h[CTL_REBUILT];
    if (m || n_small) BVH_TRY(run_levels4(tree, A, L, m, n_small, who));
    rebase4_kernel<T><<<wave, 256, 0, st>>>(tree->d_nodes, roots, cnts + 1, tile0, tree->d_sa_base);
    clear_bad_kernel<<<gn, 256, 0, st>>>(dirty, cnts, tree->d_bad);
    LAUNCHED(ctx, 2);
    if (rebuilt) *rebuilt = shapes;
    return BVHGPU_OK;
}

// The group subtrees of an add: one task per root (root_seed4_kernel) into the level loop and small4_kernel of the build.
template <class T> int build_subtrees(Tree4<T>* tree, const uint32_t* roots, const uint32_t* n_roots, uint32_t max_roots,
                                      const typename Traits<T>::Key* keys, uint32_t* idx, const char* who) {
    bvhgpu_ctx* ctx = tree->ctx;
    cudaStream_t st = ctx->stream;
    const uint32_t N = tree->n;
    const int wave = std::max(ctx->sm_count, 1) * 8;
    Scratch scratch(ctx);
    BuildArgs4 A{};
    Task4<T>* small = nullptr;
    Levels4<T> L;
    BVH_TRY(scratch.get(&A.bkt, N));
    BVH_TRY(scratch.get(&A.ctl, 8));
    BVH_TRY(scratch.get(&small, N));
    BVH_TRY(levels4_alloc(scratch, N, &L));
    A.idx[0] = idx; A.idx[1] = idx + N; A.small = small;
    BVH_CUDA_TRY(cudaMemsetAsync(A.ctl, 0, 8 * sizeof(uint32_t), st));
    root_seed4_kernel<T><<<std::min<uint32_t>((max_roots + 255) / 256, (uint32_t)wave), 256, 0, st>>>(tree->d_nodes, tree->d_node_start, roots, n_roots,
                                                                                                       keys, L.tasks, A);
    LAUNCHED(ctx, 1);
    uint32_t* h = ctx->h_pinned + 224;
    BVH_CUDA_TRY(cudaMemcpyAsync(h, A.ctl, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    BVH_CUDA_TRY(cudaStreamSynchronize(st));
    return run_levels4(tree, A, L, h[CTL_NEXT], h[CTL_SMALL], who);
}

#define INSTANTIATE4(T)                                                                                                              \
    template int build4<T>(Tree4<T>*, const D4<T>::Aabb*, cudaMemcpyKind);                                                          \
    template int build_flat4<T>(Tree4<T>*);                                                                                         \
    template int traverse_csr<T>(Tree4<T>*, int, const void*, size_t, const CsrOut&, const char*);                                  \
    template int nearest4_device<T>(Tree4<T>*, int, const T*, size_t, uint32_t*, T*);                                               \
    template int knn4_device<T>(Tree4<T>*, const T*, size_t, uint32_t, const T*, uint32_t*, T*);                                    \
    template int refresh_caches<T>(Tree4<T>*);                                                                                    \
    template int finish_relayout<T>(Tree4<T>*);                                                                                     \
    template int rebuild_degraded<T>(Tree4<T>*, const uint32_t*, uint32_t*, size_t*, const char*);                                  \
    template int build_subtrees<T>(Tree4<T>*, const uint32_t*, const uint32_t*, uint32_t, const Traits<T>::Key*, uint32_t*, const char*);
INSTANTIATE4(float)
INSTANTIATE4(double)
#undef INSTANTIATE4
BVH_INSTANTIATE_CSR(Tree4<float>, float)
BVH_INSTANTIATE_CSR(Tree4<double>, double)

}  // namespace bvhb200
