// bvh_b200/csrc/traverse.cu -- batched Ray traversal: Bvh::traverse (src/bvh/bvh_impl.rs:104-119,
// src/bvh/bvh_node.rs:288-319) and FlatBvh::traverse (src/flat_bvh.rs:396-431) for whole ray batches,
// with the crate's slab test (src/ray/intersect_default.rs:16-37) reproduced operation for operation.
//
// One ray per thread walks the preorder traversal records without a stack: a record holds the AABB
// the node has in its parent, `skip` (first record behind the node's subtree) and the shape index of
// a leaf.  hit -> next record, miss -> skip.  The visiting order is exactly the reference's
// left-first DFS, so per-ray hit lists come out in the reference's order.
//
// Output is CSR (offsets[nrays+1], hits[total]).  Single-pass scheme: the walk stores the first K
// hits of every ray in slot-major scratch ([K][nrays], coalesced across a warp) and counts all of
// them; an exclusive scan turns counts into offsets; the emit kernel copies the slots into place and
// re-walks only rays with more than K hits.  K = 0 degenerates to the classic count / scan / fill.
#include "internal.h"
#include "csr.cuh"
#include "queries.cuh"
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <chrono>

namespace bvhb200 {

// Per-ray hit slots of the single-pass scheme: "traverse_slots" option, or (-1, default) as many as a 4 GB
// scratch budget allows, between 4 and 64 -- rays with more hits than slots are walked a second time by the emit pass
// (with few slots the re-walks of a hit-heavy batch cost more than the walk itself).
// The budget is additionally capped at a quarter of the device memory that was free at the context's first traversal (a multi-GB
// scratch request must not be what runs a nearly full device out of memory); below 4 slots' worth the path degrades to fewer slots, down to the two-pass scheme.
static inline uint32_t pick_slots(bvhgpu_ctx* ctx, uint32_t nrays) {
    if (ctx->traverse_slots >= 0) return (uint32_t)std::min<int64_t>(ctx->traverse_slots, 64);
    uint64_t budget_words = 1ull << 30;               // 4 GB of slot scratch at most (64 slots for a 16 M-ray batch)
    if (ctx->slot_budget_words == 0) {                // cudaMemGetInfo is slow: asked once per context, not per traversal
        size_t free_b = 0, total_b = 0;
        ctx->slot_budget_words = cudaMemGetInfo(&free_b, &total_b) == cudaSuccess ? std::max<uint64_t>((uint64_t)free_b / 16, 1) : budget_words;
    }
    budget_words = std::min<uint64_t>(budget_words, ctx->slot_budget_words);
    const uint64_t k = budget_words / std::max<uint32_t>(nrays, 1u);
    if (k < 4) return (uint32_t)k;                   // 0..3 slots: memory is tight
    uint32_t p = 4;
    while (p * 2 <= k && p < 64) p *= 2;
    return p;
}

constexpr int SCAN_ITEMS = 8;
constexpr int SCAN_THREADS = 256;
constexpr int SCAN_TILE = SCAN_ITEMS * SCAN_THREADS;     // 2048 counts per block
static_assert(SCAN_THREADS == CSR_SCAN_THREADS && SCAN_TILE == CSR_SCAN_TILE, "scan geometry declared in internal.h");

// ---- slab test: intersect_default.rs:16-37 --------------------------------------------------------
template <class T> __device__ __forceinline__ T tmin2(T a, T b);
template <> __device__ __forceinline__ float tmin2(float a, float b) { return fminf(a, b); }
template <> __device__ __forceinline__ double tmin2(double a, double b) { return fmin(a, b); }
template <class T> __device__ __forceinline__ T tmax2(T a, T b);
template <> __device__ __forceinline__ float tmax2(float a, float b) { return fmaxf(a, b); }
template <> __device__ __forceinline__ double tmax2(double a, double b) { return fmax(a, b); }

template <class T>
__device__ __forceinline__ bool slab_hit(const T o[3], const T inv[3], const T mn[3], const T mx[3]) {
    // lbr = (aabb.min - origin) * inv_direction ; rtr = (aabb.max - origin) * inv_direction   (:19-20)
    const T l0 = mul_rn(sub_rn(mn[0], o[0]), inv[0]), r0 = mul_rn(sub_rn(mx[0], o[0]), inv[0]);
    const T l1 = mul_rn(sub_rn(mn[1], o[1]), inv[1]), r1 = mul_rn(sub_rn(mx[1], o[1]), inv[1]);
    const T l2 = mul_rn(sub_rn(mn[2], o[2]), inv[2]), r2 = mul_rn(sub_rn(mx[2], o[2]), inv[2]);
    // has_nan(lbr) | has_nan(rtr) => no intersection (:22-28).  (x != y is true iff unordered or different;
    // the pairwise isnan tests compile to 3 unordered-compare instructions.)
    const bool nan = (l0 != l0) | (r0 != r0) | (l1 != l1) | (r1 != r1) | (l2 != l2) | (r2 != r2);
    // NaN-free from here on, so fmin/fmax are the plain component-wise inf/sup (:30-33).
    const T tmin = tmax2(tmax2(tmin2(l0, r0), tmin2(l1, r1)), tmin2(l2, r2));
    const T tmax = tmin2(tmin2(tmax2(l0, r0), tmax2(l1, r1)), tmax2(l2, r2));
    const T lo = tmin > T(0) ? tmin : T(0);                     // fast_max(tmin, 0), utils.rs:52-54
    return !nan && tmax >= lo;                                  // :35
}
// f32: the folds propagate NaN (min.NaN / max.NaN, one FMNMX.NAN each) and the six NaN tests go.  Every product enters both the
// tmin and the tmax fold, so a NaN anywhere makes tmax NaN and `tmax >= lo` false: a miss, as above.  Without a NaN both forms
// give the same values up to the sign of a zero, which neither the clamp nor the comparison can see (DESIGN §2).
__device__ __forceinline__ float fmin_nan(float a, float b) { float r; asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ float fmax_nan(float a, float b) { float r; asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
template <>
__device__ __forceinline__ bool slab_hit<float>(const float o[3], const float inv[3], const float mn[3], const float mx[3]) {
    const float l0 = mul_rn(sub_rn(mn[0], o[0]), inv[0]), r0 = mul_rn(sub_rn(mx[0], o[0]), inv[0]);
    const float l1 = mul_rn(sub_rn(mn[1], o[1]), inv[1]), r1 = mul_rn(sub_rn(mx[1], o[1]), inv[1]);
    const float l2 = mul_rn(sub_rn(mn[2], o[2]), inv[2]), r2 = mul_rn(sub_rn(mx[2], o[2]), inv[2]);
    const float tmin = fmax_nan(fmax_nan(fmin_nan(l0, r0), fmin_nan(l1, r1)), fmin_nan(l2, r2));
    const float tmax = fmin_nan(fmin_nan(fmax_nan(l0, r0), fmax_nan(l1, r1)), fmax_nan(l2, r2));
    const float lo = tmin > 0.f ? tmin : 0.f;
    return tmax >= lo;
}

// The walk.  `emit(shape)` is called for every reported shape in reference order.
template <class T, bool FLAT, class Emit>
__device__ __forceinline__ uint32_t walk(const typename Traits<T>::TNode* __restrict__ trec, uint32_t n_rec,
                                         const typename Traits<T>::DAabb* __restrict__ aabb,
                                         const T o[3], const T inv[3], Emit emit) {
    uint32_t i = 0, visits = 0;
    while (i < n_rec) {
        T mn[3], mx[3];
        uint32_t skip, shape;
        fetch(trec + i, mn, mx, skip, shape);
        ++visits;
        if (slab_hit(o, inv, mn, mx)) {
            if (shape != BVH_INVALID) {
                bool report = true;
                if (FLAT) {                       // flat_bvh.rs:412-416: the leaf re-tests shapes[shape].aabb()
                    T smn[3], smx[3];
                    load_aabb(aabb + shape, smn, smx);
                    report = slab_hit(o, inv, smn, smx);
                }
                if (report) emit(shape);
            }
            i = i + 1;
        } else {
            i = skip;
        }
    }
    return visits;
}

// Ray batches come in two layouts.  RAYS_FULL: the 9-scalar Ray of the C ABI {origin, direction, inv_direction}.
// RAYS_OD: 6 scalars {origin, direction} with the direction as Ray stores it (already normalised by Ray::new); the
// inverse direction is recomputed here with the same IEEE division Ray::new performs (src/ray/ray_impl.rs:76-78), so
// both layouts give bit-identical traversals while the compact one moves a third fewer bytes across PCIe.
// L2 = true: the batch is still arriving by DMA while the kernel runs (streaming host path): bypass the non-coherent path.
template <class T> struct RaySrc { const T* base; uint32_t fmt; };
constexpr uint32_t RAYS_FULL = 0, RAYS_OD = 1;
template <class T, bool L2>
__device__ __forceinline__ void load_ray(const RaySrc<T>& src, size_t r, T o[3], T inv[3]) {
    if (src.fmt == RAYS_FULL) {
        const T* p = src.base + 9 * r;
#pragma unroll
        for (int k = 0; k < 3; ++k) { o[k] = L2 ? __ldcg(p + k) : __ldg(p + k); inv[k] = L2 ? __ldcg(p + 6 + k) : __ldg(p + 6 + k); }
    } else {
        const T* p = src.base + 6 * r;
#pragma unroll
        for (int k = 0; k < 3; ++k) { o[k] = L2 ? __ldcg(p + k) : __ldg(p + k); inv[k] = div_rn(T(1), L2 ? __ldcg(p + 3 + k) : __ldg(p + 3 + k)); }
    }
}

// Coherence probe: neighbouring rays of a coherent batch (camera rays) point the same way, and then the static
// one-ray-per-thread mapping wins (adjacent lanes walk the same nodes: one L1 wavefront serves many lanes); on
// incoherent batches the persistent refill kernel wins.  The probe samples 1024 neighbour pairs and leaves its
// verdict in *flag; BOTH pass-1 kernels are launched and the one the verdict rules out returns immediately, so
// the choice costs no host synchronisation.  (Rejected alternative: one persistent kernel that refills whole warps with
// 32 consecutive rays on coherent batches was slower than the static kernel on Sponza camera rays: the
// static mapping also keeps neighbouring warps of a CTA on neighbouring pixels, which is what feeds the L1.)
template <class T>
__global__ void __launch_bounds__(256) coherence_probe_kernel(RaySrc<T> rays, uint32_t nrays, uint32_t* flag) {
    __shared__ float acc[8];
    float sum = 0.f;
    const uint32_t samples = 1024, stride = nrays > 2 * samples ? nrays / samples : 1;
    const uint32_t rstride = rays.fmt == RAYS_FULL ? 9u : 6u;       // the direction sits at scalar 3 in both layouts
    uint32_t n = 0;
    for (uint32_t k = threadIdx.x; k < samples; k += 256) {
        const uint32_t i = k * stride;
        if (i + 1 >= nrays) break;
        const T* a = rays.base + (size_t)rstride * i + 3;
        const T* b = rays.base + (size_t)rstride * (i + 1) + 3;
        sum += (float)(a[0] * b[0] + a[1] * b[1] + a[2] * b[2]);
        ++n;
    }
    for (int o = 16; o > 0; o >>= 1) { sum += __shfl_xor_sync(0xffffffffu, sum, o); n += __shfl_xor_sync(0xffffffffu, n, o); }
    __shared__ uint32_t cnt[8];
    if (lane_id() == 0) { acc[threadIdx.x >> 5] = sum; cnt[threadIdx.x >> 5] = n; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f; uint32_t c = 0;
        for (int w = 0; w < 8; ++w) { s += acc[w]; c += cnt[w]; }
        *flag = (c > 0 && s / (float)c > 0.9f) ? 1u : 0u;          // 1 = coherent
    }
}

// Pass 1: count all hits of every ray, keep the first K in slot-major scratch.
template <class T, bool FLAT>
__global__ void __launch_bounds__(256) walk_count_kernel(const typename Traits<T>::TNode* __restrict__ trec, uint32_t n_rec,
                                                         const typename Traits<T>::DAabb* __restrict__ aabb,
                                                         RaySrc<T> rays, uint32_t nrays,
                                                         uint32_t first, uint32_t count,
                                                         uint32_t* __restrict__ counts, uint32_t* __restrict__ slots, uint32_t K,
                                                         unsigned long long* __restrict__ visit_total, const uint32_t* __restrict__ gate, uint32_t run_if) {
    if (gate && *gate != run_if) return;             // the coherence probe chose the other pass-1 kernel
    const uint32_t r = first + blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t visits = 0;
    if (r < first + count) {
        T o[3], inv[3];
        load_ray<T, false>(rays, r, o, inv);
        uint32_t cnt = 0;
        visits = walk<T, FLAT>(trec, n_rec, aabb, o, inv, [&](uint32_t shape) {
            if (cnt < K) slots[(size_t)cnt * nrays + r] = shape;
            ++cnt;
        });
        counts[r] = cnt;
    }
    visits = __reduce_add_sync(0xffffffffu, visits);
    if (lane_id() == 0 && visits) atomicAdd(visit_total, (unsigned long long)visits);
}

// Pass 1, persistent form.  A fixed grid of warps pulls rays from a global ticket counter; a lane that finishes
// its ray is refilled as soon as REFILL lanes of its warp are idle, so warps stay populated although rays take
// 10..400 visits (the one-ray-per-thread kernel above averages 12 of 32 active lanes on random rays).
// STREAM: the rays are still arriving from the host (chunked H2D on the copy stream, enqueued BEFORE this kernel is
// launched); `ready` counts the rays whose bytes are resident (bumped by a 4-byte DMA after every chunk), lanes wait
// for their ray to arrive, and ray loads bypass the non-coherent path.  Copy and walk overlap without any per-chunk
// kernel tail.  The wait carries a %globaltimer watchdog: if the copies never come (failed DMA, a tool that replays
// the kernel against a restored `ready` word) the kernel raises BVHGPU_ERR_TIMEOUT in *err and drains instead of
// spinning forever.
template <class T, bool FLAT, bool STREAM>
__global__ void __launch_bounds__(256) walk_persistent_kernel(const typename Traits<T>::TNode* __restrict__ trec, uint32_t n_rec,
                                                              const typename Traits<T>::DAabb* __restrict__ aabb,
                                                              RaySrc<T> rays, uint32_t nrays,
                                                              uint32_t* __restrict__ ticket, const uint32_t* ready,
                                                              uint32_t* __restrict__ counts, uint32_t* __restrict__ slots, uint32_t K,
                                                              unsigned long long* __restrict__ visit_total, const uint32_t* __restrict__ gate, uint32_t run_if,
                                                              uint32_t* err, unsigned long long timeout_ns) {
    if (gate && *gate != run_if) return;
    constexpr uint32_t NONE = 0xFFFFFFFFu;
    constexpr int REFILL = 8;
    const uint32_t FULL = 0xffffffffu;
    const uint32_t lane = lane_id(), lt = lanemask_lt();
    uint32_t r = NONE, i = 0, cnt = 0, visits = 0;
    bool loaded = false;                 // STREAM: a lane may hold a ticket whose ray has not arrived yet (pending)
    T o[3] = {T(0), T(0), T(0)}, inv[3] = {T(0), T(0), T(0)};
    bool exhausted = false;
    for (;;) {
        // ---- refill idle lanes -------------------------------------------------------------------------
        const uint32_t need = __ballot_sync(FULL, r == NONE);
        if (need && !exhausted) {
            uint32_t base = 0;
            if (lane == 0) base = atomicAdd(ticket, (uint32_t)__popc(need));
            base = __shfl_sync(FULL, base, 0);
            if (base >= nrays) exhausted = true;
            const uint32_t mine = base + __popc(need & lt);
            if (r == NONE && mine < nrays) {
                r = mine; i = 0; cnt = 0;
                if (STREAM) loaded = false;
                else load_ray<T, false>(rays, mine, o, inv);
            }
        }
        if (STREAM) {
            // Pending lanes never block the lanes that are walking: the arrival counter is polled, and only a warp with nothing
            // to walk waits for it (with the watchdog).  Tickets and copies are both in ray order, so the wait is for the next chunk.
            const uint32_t pend = __ballot_sync(FULL, r != NONE && !loaded);
            if (pend) {
                const bool any_active = __ballot_sync(FULL, r != NONE && loaded) != 0u;
                const uint32_t lowest = __reduce_min_sync(FULL, (r != NONE && !loaded) ? r : NONE);
                uint32_t rd = 0, ok = 1;
                if (lane == 0) {
                    rd = *(volatile const uint32_t*)ready;
                    if (!any_active && rd <= lowest) {
                        uint32_t ns = 100;
                        const unsigned long long t0 = global_timer_ns();
                        while (rd <= lowest) {
                            if (*(volatile const uint32_t*)err != 0u) { ok = 0; break; }          // another warp gave up already
                            if (global_timer_ns() - t0 > timeout_ns) { ok = 0; atomicExch(err, (uint32_t)BVHGPU_ERR_TIMEOUT); break; }
                            __nanosleep(ns);
                            if (ns < 2000) ns <<= 1;
                            rd = *(volatile const uint32_t*)ready;
                        }
                    }
                }
                rd = __shfl_sync(FULL, rd, 0);
                ok = __shfl_sync(FULL, ok, 0);
                if (!ok) {                                           // the copies never came: the call fails, drain what is walking
                    exhausted = true;
                    if (r != NONE && !loaded) r = NONE;
                } else if (__ballot_sync(FULL, r != NONE && !loaded && r < rd)) {
                    __threadfence();
                    if (r != NONE && !loaded && r < rd) { load_ray<T, true>(rays, r, o, inv); loaded = true; }
                }
            }
        }
        if (__ballot_sync(FULL, r != NONE) == 0) break;
        // ---- walk until enough lanes have gone idle ----------------------------------------------------
        uint32_t rounds = 0;
        for (;;) {
            if (r != NONE && (!STREAM || loaded)) {
                T mn[3], mx[3];
                uint32_t skip, shape;
                fetch(trec + i, mn, mx, skip, shape);
                ++visits;
                if (slab_hit(o, inv, mn, mx)) {
                    if (shape != BVH_INVALID) {
                        bool report = true;
                        if (FLAT) {
                            T smn[3], smx[3];
                            load_aabb(aabb + shape, smn, smx);
                            report = slab_hit(o, inv, smn, smx);
                        }
                        if (report) { if (cnt < K) slots[(size_t)cnt * nrays + r] = shape; ++cnt; }
                    }
                    i = i + 1;
                } else {
                    i = skip;
                }
                if (i >= n_rec) { counts[r] = cnt; r = NONE; }
            }
            const uint32_t idle_mask = __ballot_sync(FULL, r == NONE);
            const int idle = __popc(idle_mask);
            if (idle == 32 || (idle >= REFILL && !exhausted)) break;
            if (STREAM) {                                            // look for arrivals every 16 visits, at once if nobody walks
                const uint32_t pend = __ballot_sync(FULL, r != NONE && !loaded);
                if (pend && (((++rounds) & 15u) == 0u || (pend | idle_mask) == FULL)) break;
            }
        }
    }
    visits = __reduce_add_sync(FULL, visits);
    if (lane == 0 && visits) atomicAdd(visit_total, (unsigned long long)visits);
}

// Shared-memory top-of-tree variant of the persistent walk (f32; automatic from 5 MB of records, option traverse_top; STREAM as
// above).  Every CTA (one per SM, 1024 threads)
// keeps the top records (flatten.cu: build_top_records) in shared memory; a lane walks them with two LDS.128 per visit and drops
// to the global records (two LDG.128, as above) only inside a fringe subtree.  Visit order and tests are exactly the preorder walk's,
// so counts and hit lists are bit-identical.  Lane state: j = next top entry (also the resume point while g walks [g, gend)).
// VPC: visits per lane between two votes on the idle lanes (see the walk loop).
template <bool FLAT, bool STREAM, int VPC>
__global__ void __launch_bounds__(1024, 1) walk_top_kernel(const TNodeF* __restrict__ trec, const DAabbF* __restrict__ aabb,
                                                           uint32_t n_rec, const float4* __restrict__ top,
                                                           RaySrc<float> rays, uint32_t nrays, uint32_t* __restrict__ ticket, const uint32_t* ready,
                                                           uint32_t* __restrict__ counts, uint32_t* __restrict__ slots, uint32_t K,
                                                           unsigned long long* __restrict__ visit_total, const uint32_t* __restrict__ gate, uint32_t run_if,
                                                           uint32_t* err, unsigned long long timeout_ns, int refill) {
    extern __shared__ float4 s_top[];
    if (gate && *gate != run_if) return;
    const uint32_t n_top = reinterpret_cast<const uint32_t*>(top)[0];      // header {n_top, C}, then lo[n_top], hi[n_top]
    for (uint32_t k = threadIdx.x; k < 2 * n_top; k += blockDim.x) s_top[k] = top[2 + k];
    __syncthreads();
    uint32_t s_lo, s_hi;                                             // opaque: keeps ptxas from re-deriving the window addresses every visit
    asm volatile("mov.u32 %0, %1;" : "=r"(s_lo) : "r"((uint32_t)__cvta_generic_to_shared(s_top)));
    asm volatile("mov.u32 %0, %1;" : "=r"(s_hi) : "r"(s_lo + 16u * n_top));
    constexpr uint32_t NONE = 0xFFFFFFFFu;
    const uint32_t FULL = 0xffffffffu;
    const uint32_t lane = lane_id(), lt = lanemask_lt();
    // Lane state: r ray, j next top entry (the resume point while below the top), [g, gend) global records left to walk in the
    // current fringe subtree -- empty (g >= gend) while the lane is in the top.  The lane walks while g < gend || j < n_top: a
    // lane without a ray, with a ray still in flight (STREAM: `loaded` as in walk_persistent_kernel) or with a finished ray has
    // j = NONE or j >= n_top and an empty range, so the visit needs no other test of the lane.
    uint32_t r = NONE, j = NONE, g = 0, gend = 0, cnt = 0, visits = 0;
    bool loaded = false;
    float o[3] = {0.f, 0.f, 0.f}, inv[3] = {0.f, 0.f, 0.f};
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;              // the record being visited: {min, w3}, {max, w7}
    bool exhausted = false;
    for (;;) {
        const uint32_t need = __ballot_sync(FULL, r == NONE);
        if (need && !exhausted) {
            uint32_t base = 0;
            if (lane == 0) base = atomicAdd(ticket, (uint32_t)__popc(need));
            base = __shfl_sync(FULL, base, 0);
            if (base >= nrays) exhausted = true;
            const uint32_t mine = base + __popc(need & lt);
            // (no top records -- a degenerate tree whose first histogram bin already exceeds the budget: everything is "below")
            if (r == NONE && mine < nrays) {
                r = mine; cnt = 0; g = 0;
                if (STREAM) { loaded = false; j = NONE; gend = 0; }         // pending: does not walk until its ray is loaded
                else { j = 0; gend = n_top ? 0u : n_rec; load_ray<float, false>(rays, mine, o, inv); }
            }
        }
        if (STREAM) {                                                // see walk_persistent_kernel: pending lanes never block walking lanes
            const uint32_t pend = __ballot_sync(FULL, r != NONE && !loaded);
            if (pend) {
                const bool any_active = __ballot_sync(FULL, r != NONE && loaded) != 0u;
                const uint32_t lowest = __reduce_min_sync(FULL, (r != NONE && !loaded) ? r : NONE);
                uint32_t rd = 0, ok = 1;
                if (lane == 0) {
                    rd = *(volatile const uint32_t*)ready;
                    if (!any_active && rd <= lowest) {
                        uint32_t ns = 100;
                        const unsigned long long t0 = global_timer_ns();
                        while (rd <= lowest) {
                            if (*(volatile const uint32_t*)err != 0u) { ok = 0; break; }
                            if (global_timer_ns() - t0 > timeout_ns) { ok = 0; atomicExch(err, (uint32_t)BVHGPU_ERR_TIMEOUT); break; }
                            __nanosleep(ns);
                            if (ns < 2000) ns <<= 1;
                            rd = *(volatile const uint32_t*)ready;
                        }
                    }
                }
                rd = __shfl_sync(FULL, rd, 0);
                ok = __shfl_sync(FULL, ok, 0);
                if (!ok) {
                    exhausted = true;
                    if (r != NONE && !loaded) r = NONE;
                } else if (__ballot_sync(FULL, r != NONE && !loaded && r < rd)) {
                    __threadfence();
                    if (r != NONE && !loaded && r < rd) {
                        load_ray<float, true>(rays, r, o, inv); loaded = true;
                        j = 0; gend = n_top ? 0u : n_rec;
                    }
                }
            }
        }
        if (__ballot_sync(FULL, r != NONE) == 0) break;
        const int leave = exhausted ? 32 : refill;                   // idle lanes at which the warp goes back for tickets
        // One warp step = VPC visits per lane, then one vote on the idle lanes: the vote, its population count and the loop branch
        // are paid once per VPC visits.  A lane whose ray ends inside a step idles for the rest of it, and the warp goes back for
        // tickets up to VPC - 1 visits later: cheap where a visit is a shared-memory or L1/L2 hit, not where visits wait on DRAM.
        // VPC = 1 (trees beyond L2, visits wait on DRAM): the visit branches between the top and the global records and ends the
        // ray itself; the predicated visit below was 2 % slower there (DESIGN §4.3).
        auto visit_branchy = [&]() {
            if (r != NONE && (!STREAM || loaded)) {
                float mn[3], mx[3];
                uint32_t w3, w7;
                const bool below = g < gend;
                if (!below) {
                    float4 lo4, hi4;                                  // explicit shared-window addresses: two LDS.128, no per-visit cvta
                    asm("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(lo4.x), "=f"(lo4.y), "=f"(lo4.z), "=f"(lo4.w) : "r"(s_lo + 16u * j));
                    asm("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(hi4.x), "=f"(hi4.y), "=f"(hi4.z), "=f"(hi4.w) : "r"(s_hi + 16u * j));
                    mn[0] = lo4.x; mn[1] = lo4.y; mn[2] = lo4.z; w3 = __float_as_uint(lo4.w);
                    mx[0] = hi4.x; mx[1] = hi4.y; mx[2] = hi4.z; w7 = __float_as_uint(hi4.w);
                } else {
                    fetch(trec + g, mn, mx, w3, w7);
                }
                ++visits;
                // One select chain for both index spaces (no divergence between lanes in the top and lanes below it).
                const bool hit = slab_hit(o, inv, mn, mx);
                const bool fringe = !below && (w7 + 0x80000000u) < 0x7FFFFFFFu;
                const uint32_t cur = below ? g : j;
                const uint32_t nxt = (hit || fringe) ? cur + 1 : w3;
                if (hit && (int32_t)w7 >= 0) {                       // a leaf
                    bool report = true;
                    if (FLAT) {
                        float smn[3], smx[3];
                        load_aabb(aabb + w7, smn, smx);
                        report = slab_hit(o, inv, smn, smx);
                    }
                    if (report) { if (cnt < K) slots[(size_t)cnt * nrays + r] = w7; ++cnt; }
                }
                j = below ? j : nxt;
                gend = below ? gend : ((hit && fringe) ? w3 : 0u);
                g = below ? nxt : (w7 & 0x7FFFFFFFu);
                if (g >= gend && j >= n_top) { counts[r] = cnt; r = NONE; }
            }
        };
        // VPC > 1: a visit is straight-line code for every lane: the record comes from a predicated LDS pair (top) or LDG pair
        // (below) into the same registers, and the lane state moves by predicated selects.  Only a reached leaf branches.
        auto visit = [&]() {
            const bool below = g < gend;
            const bool top = !below && j < n_top;
            const bool walking = below || top;
            const TNodeF* gp = trec + g;
            asm("{\n\t.reg .pred pt, pb;\n\t"
                "setp.ne.u32 pt, %10, 0;\n\tsetp.ne.u32 pb, %11, 0;\n\t"
                "@pt ld.shared.v4.f32 {%0,%1,%2,%3}, [%8];\n\t"
                "@pt ld.shared.v4.f32 {%4,%5,%6,%7}, [%9];\n\t"
                "@pb ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%12];\n\t"
                "@pb ld.global.nc.v4.f32 {%4,%5,%6,%7}, [%12+16];\n\t}"
                : "+f"(a.x), "+f"(a.y), "+f"(a.z), "+f"(a.w), "+f"(b.x), "+f"(b.y), "+f"(b.z), "+f"(b.w)
                : "r"(s_lo + 16u * j), "r"(s_hi + 16u * j), "r"((uint32_t)top), "r"((uint32_t)below), "l"(gp));
            const float mn[3] = {a.x, a.y, a.z}, mx[3] = {b.x, b.y, b.z};
            const uint32_t w3 = __float_as_uint(a.w), w7 = __float_as_uint(b.w);
            visits += walking;
            //   top entry: w7 = ~0 top-internal | 0x80000000+first global record (fringe inner, w3 = end of that range) | shape;
            //   global record: w7 = shape | ~0, never in the fringe range, so `fringe` needs no test of `below`.
            const bool hit = walking & slab_hit(o, inv, mn, mx);      // `&`: no branch around the test
            const bool fringe = (int32_t)w7 < -1;
            const bool adv = hit || fringe;                           // next record, else the skip link w3
            if (hit && (int32_t)w7 >= 0) {                           // a leaf
                bool report = true;
                if (FLAT) {
                    float smn[3], smx[3];
                    load_aabb(aabb + w7, smn, smx);
                    report = slab_hit(o, inv, smn, smx);
                }
                if (report) { if (cnt < K) slots[(size_t)cnt * nrays + r] = w7; ++cnt; }
            }
            if (top) j = adv ? j + 1 : w3;
            if (below) g = adv ? g + 1 : w3;
            if (hit && fringe) { g = w7 & 0x7FFFFFFFu; gend = w3; }     // enter the subtree's global records [g, gend)
        };
        uint32_t rounds = 0;
        for (;;) {
            if constexpr (VPC == 1) {
                visit_branchy();
            } else {
#pragma unroll
                for (int u = 0; u < VPC; ++u) visit();
                if (r != NONE && (!STREAM || loaded) && g >= gend && j >= n_top) { counts[r] = cnt; r = NONE; }   // the ray ended in this step
            }
            const uint32_t idle_mask = __ballot_sync(FULL, r == NONE);
            if (__popc(idle_mask) >= leave) break;
            if (STREAM) {                                            // look for arrivals every 16 visits, at once if nobody walks
                const uint32_t pend = __ballot_sync(FULL, r != NONE && !loaded);
                if (pend && ((rounds += VPC) >= 16u || (pend | idle_mask) == FULL)) break;
            }
        }
    }
    visits = __reduce_add_sync(FULL, visits);
    if (lane == 0 && visits) atomicAdd(visit_total, (unsigned long long)visits);
}

// A tile of SCAN_TILE counts can sum past 2^32 (2048 rays through 2^21 + 1 boxes), so the scans below add in 64 bits.  The in-tile
// offsets they leave in `local` (u32) are saturated at 0xFFFFFFFF: every reader adds the tile's 64-bit offset and clamps the sum to
// 0xFFFFFFFF, and a clamped offset means a total past 2^32, which the call reports as BVHGPU_ERR_CAPACITY.
__device__ __forceinline__ uint32_t sat_u32(unsigned long long x) { return x > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)x; }

// Exclusive scan of counts, phase A: per-block local exclusive offsets + block totals (+ the largest count, if asked for).
__global__ void __launch_bounds__(SCAN_THREADS) scan_local_kernel(const uint32_t* __restrict__ counts, uint32_t n,
                                                                  uint32_t* __restrict__ local, unsigned long long* __restrict__ blocksum,
                                                                  uint32_t* __restrict__ maxcount) {
    __shared__ unsigned long long wsum[SCAN_THREADS / 32];
    const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
    uint32_t v[SCAN_ITEMS], m = 0;
    unsigned long long s = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) { v[k] = (base + k < n) ? counts[base + k] : 0u; s += v[k]; m = v[k] > m ? v[k] : m; }
    unsigned long long incl = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o); if ((int)lane_id() >= o) incl += t; }
    if (lane_id() == 31) wsum[threadIdx.x >> 5] = incl;
    if (maxcount) { m = __reduce_max_sync(0xffffffffu, m); if (lane_id() == 0 && m) atomicMax(maxcount, m); }
    __syncthreads();
    unsigned long long woff = 0;
    for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) woff += wsum[w];
    unsigned long long run = woff + incl - s;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) { if (base + k < n) local[base + k] = sat_u32(run); run += v[k]; }
    if (threadIdx.x == SCAN_THREADS - 1) blocksum[blockIdx.x] = woff + incl;
}
// Phase B: one block turns block totals into exclusive block offsets (64-bit) and the grand total.
__global__ void __launch_bounds__(1024) scan_blocks_kernel(unsigned long long* __restrict__ blocksum, uint32_t nblocks,
                                                           unsigned long long* __restrict__ total) {
    __shared__ unsigned long long wsum[32];
    __shared__ unsigned long long carry_s;
    if (threadIdx.x == 0) carry_s = *total;          // running total of the chunks scanned before this one (0 for the first)
    __syncthreads();
    for (uint32_t b0 = 0; b0 < nblocks; b0 += 1024) {
        const uint32_t b = b0 + threadIdx.x;
        const unsigned long long v = b < nblocks ? blocksum[b] : 0ull;
        unsigned long long incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o); if ((int)lane_id() >= o) incl += t; }
        if (lane_id() == 31) wsum[threadIdx.x >> 5] = incl;
        __syncthreads();
        unsigned long long woff = 0;
        for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) woff += wsum[w];
        const unsigned long long carry = carry_s;
        if (b < nblocks) blocksum[b] = carry + woff + incl - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry_s = carry + woff + incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = carry_s;
}

// ---- exchange over peer memory (multi-GPU ray sharding) -------------------------------------------------------------------
// Every rank ends the step with its own copy of the GLOBAL CSR (offsets u32[NG+1], hit lists) in original ray order.
// Mailbox (u64 words; BVHGPU_MAILBOX_BYTES per rank, zero-initialised):
//   [ (par*8 + src)*4 + {0,1} ]      = {seq, hit total} published by rank `src`
//   [ 64 + par*8 + src ]             = seq of the step whose hit lists of rank `src` have landed ("done")
//   [ 128 + (seq % 1024)*4 + {0..3} ] = trace of this rank: {seq, %globaltimer when the peers' posts were all in, ns waited for
//                                       the posts, ns waited for the done flags}   (diagnostics, bench.py)
// Staging (2 x BVHGPU_SHARD_STAGE_BYTES per rank, the halves alternate with the parity of seq).  Rays are handled in TILES of
// SCAN_TILE = 2048 (per source rank, counted from its first ray); a tile of source s with tile index t has the global tile
// number g = tiles_before[s] + t.
//   counts of tile g : 8192 bytes at 8192*g -- the per-ray hit counts in the tile's own width (1, 2 or 4 bytes, from the tile's
//                      largest count): 1 byte per ray crosses NVLink on ordinary batches, not a 4-byte offset
//   table entry g    : u64 at table_off + 8*g = exclusive hit offset of the tile inside its source's list | width << 56
// The step is the SAME number of launches as on one GPU (after the walk: scan_post, then emit with the goffsets blocks appended):
//   scan_post  per tile: local scan, counts pushed to all ranks; the last block scans the tile sums, pushes the tile table,
//              publishes the total (a peer that sees the seq also sees counts and table) and then waits for the peers' posts
//              (LOCAL polling), which fixes every source's hit base
//   emit       hit lists into the local copy of the global hit buffer at hit base + local offset, then the block copies its
//              contiguous piece to every peer (16-byte P2P stores); last block: done flags
//   goffsets   (extra blocks of the emit launch) per tile of every source: offsets = hit base of the source + tile offset + prefix of
//              the staged counts; block 0 ends the step by waiting for the peers' done flags
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
constexpr int MB_TOT = 0, MB_DONE = 64, MB_TRACE = 128, MB_TRACE_LEN = 1024;
constexpr unsigned long long TILE_BYTES = 4ull * SCAN_TILE;
constexpr unsigned long long OFF_MASK = (1ull << 56) - 1ull;
struct PeerBoxes {
    int rank, world;                                   // world == 0: single GPU, nothing below is used
    unsigned long long* box[BVHGPU_MAX_PEERS];
    unsigned char* stage[BVHGPU_MAX_PEERS];            // staging of every rank (the half of this step's parity)
    uint32_t* hits[BVHGPU_MAX_PEERS];                  // global hit buffer of every rank
    unsigned long long seq;
    unsigned long long rays_before[BVHGPU_MAX_PEERS + 1];    // prefix sums of the shard sizes
    unsigned long long tiles_before[BVHGPU_MAX_PEERS + 1];   // prefix sums of ceil(shard size / SCAN_TILE)
    unsigned long long table_off;                            // byte offset of the tile table inside a staging half
    uint32_t* err;                                           // sticky error word of the context
    unsigned long long timeout_ns;
};

// Wait (threads 0..31 of the calling block) until every peer has posted step pb.seq; hit bases of all sources + the grand total.
struct XInfo { unsigned long long base[BVHGPU_MAX_PEERS], grand, waited; };
__device__ __forceinline__ void wait_posts(const PeerBoxes& pb, XInfo* xs) {
    const int lane = threadIdx.x;
    const unsigned long long par = pb.seq & 1ull;
    unsigned long long tot = 0, waited = 0;
    if (lane < pb.world) {
        const unsigned long long* slot = pb.box[pb.rank] + MB_TOT + (par * BVHGPU_MAX_PEERS + lane) * 4;
        const unsigned long long t0 = global_timer_ns();
        uint32_t spins = 0;
        while (ld_acquire_sys(slot) != pb.seq) {
            if (((++spins) & 63u) == 0u && global_timer_ns() - t0 > pb.timeout_ns) { atomicExch(pb.err, (uint32_t)BVHGPU_ERR_TIMEOUT); break; }
            __nanosleep(100);
        }
        tot = slot[1];
        waited = global_timer_ns() - t0;
    }
    unsigned long long run = 0, wmax = 0, mine = 0;
    for (int r = 0; r < pb.world; ++r) {
        const unsigned long long v = __shfl_sync(0xffffffffu, tot, r), w = __shfl_sync(0xffffffffu, waited, r);
        if (lane == r) mine = run;
        run += v;
        wmax = w > wmax ? w : wmax;
    }
    if (lane < BVHGPU_MAX_PEERS) xs->base[lane] = mine;
    if (lane == 0) { xs->grand = run; xs->waited = wmax; }
}

// Exclusive scan of the per-ray counts: per-tile local offsets + (last block) exclusive tile offsets and the total -- one kernel
// (the last block to arrive scans the tile sums).  SHARDED: the tile's counts, then the tile table and the total, go to all ranks.
template <bool SHARDED>
__global__ void __launch_bounds__(SCAN_THREADS) scan_post_kernel(const uint32_t* __restrict__ counts, uint32_t n, uint32_t* __restrict__ local,
                                                                 unsigned long long* __restrict__ blocksum, unsigned long long* __restrict__ total,
                                                                 uint32_t* __restrict__ arrival, PeerBoxes pb, unsigned long long* __restrict__ xinfo) {
    __shared__ uint32_t wmax[SCAN_THREADS / 32];
    __shared__ XInfo xs;
    __shared__ unsigned long long wsum[SCAN_THREADS / 32], wsum64[SCAN_THREADS / 32];
    __shared__ unsigned long long carry_s;
    __shared__ bool last;
    const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
    uint32_t v[SCAN_ITEMS], m = 0;
    unsigned long long s = 0;                                             // 64-bit sums: see sat_u32
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) { v[k] = (base + k < n) ? counts[base + k] : 0u; s += v[k]; m = v[k] > m ? v[k] : m; }
    unsigned long long incl = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o); if ((int)lane_id() >= o) incl += t; }
    m = __reduce_max_sync(0xffffffffu, m);
    if (lane_id() == 31) wsum[threadIdx.x >> 5] = incl;
    if (lane_id() == 0) wmax[threadIdx.x >> 5] = m;
    __syncthreads();
    unsigned long long woff = 0, tsum = 0;                                // tsum < 2^43 (2048 counts < 2^32): fits below the width byte
    uint32_t tmax = 0;
#pragma unroll
    for (int w = 0; w < SCAN_THREADS / 32; ++w) { if (w < (int)(threadIdx.x >> 5)) woff += wsum[w]; tsum += wsum[w]; tmax = wmax[w] > tmax ? wmax[w] : tmax; }
    unsigned long long run = woff + incl - s;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) { if (base + k < n) local[base + k] = sat_u32(run); run += v[k]; }
    const unsigned long long width = tmax <= 0xFFu ? 1ull : (tmax <= 0xFFFFu ? 2ull : 4ull);
    if (SHARDED) {
        unsigned long long tb_mine = 0;
#pragma unroll
        for (int k = 1; k < BVHGPU_MAX_PEERS; ++k) if (k == pb.rank) tb_mine = pb.tiles_before[k];
        const unsigned long long at = TILE_BYTES * (tb_mine + blockIdx.x) + (unsigned long long)threadIdx.x * SCAN_ITEMS * width;
        if (width == 1) {
            const uint2 q = make_uint2(v[0] | v[1] << 8 | v[2] << 16 | v[3] << 24, v[4] | v[5] << 8 | v[6] << 16 | v[7] << 24);
#pragma unroll
            for (int d = 0; d < BVHGPU_MAX_PEERS; ++d) if (d < pb.world) *reinterpret_cast<uint2*>(pb.stage[d] + at) = q;
        } else if (width == 2) {
            const uint4 q = make_uint4(v[0] | v[1] << 16, v[2] | v[3] << 16, v[4] | v[5] << 16, v[6] | v[7] << 16);
#pragma unroll
            for (int d = 0; d < BVHGPU_MAX_PEERS; ++d) if (d < pb.world) *reinterpret_cast<uint4*>(pb.stage[d] + at) = q;
        } else {
            const uint4 q0 = make_uint4(v[0], v[1], v[2], v[3]), q1 = make_uint4(v[4], v[5], v[6], v[7]);
#pragma unroll
            for (int d = 0; d < BVHGPU_MAX_PEERS; ++d) if (d < pb.world) { *reinterpret_cast<uint4*>(pb.stage[d] + at) = q0; *reinterpret_cast<uint4*>(pb.stage[d] + at + 16) = q1; }
        }
    }
    if (threadIdx.x == 0) blocksum[blockIdx.x] = tsum | (width << 56);
    // the block's stores -> barrier -> ONE fence (cumulative over what the barrier ordered) -> arrival counter
    __syncthreads();
    if (threadIdx.x == 0) {
        if (SHARDED && pb.world > 1) __threadfence_system(); else __threadfence();
        last = atomicAdd(arrival, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    if (threadIdx.x == 0) { __threadfence(); carry_s = 0ull; }
    __syncthreads();
    unsigned long long tb_mine = 0;
    if (SHARDED) {
#pragma unroll
        for (int k = 1; k < BVHGPU_MAX_PEERS; ++k) if (k == pb.rank) tb_mine = pb.tiles_before[k];
    }
    for (uint32_t b0 = 0; b0 < gridDim.x; b0 += SCAN_THREADS) {           // exclusive scan of the tile sums by this (last) block
        const uint32_t bb = b0 + threadIdx.x;
        const unsigned long long e = bb < gridDim.x ? __ldcg(blocksum + bb) : 0ull;
        const unsigned long long val = e & OFF_MASK;
        unsigned long long in64 = val;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const unsigned long long t = __shfl_up_sync(0xffffffffu, in64, o); if ((int)lane_id() >= o) in64 += t; }
        if (lane_id() == 31) wsum64[threadIdx.x >> 5] = in64;
        __syncthreads();
        unsigned long long wo = 0;
        for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) wo += wsum64[w];
        const unsigned long long carry = carry_s;
        const unsigned long long excl = carry + wo + in64 - val;
        if (bb < gridDim.x) {
            blocksum[bb] = excl;
            if (SHARDED) {
                const unsigned long long entry = (excl & OFF_MASK) | (e & ~OFF_MASK);
#pragma unroll
                for (int d = 0; d < BVHGPU_MAX_PEERS; ++d) if (d < pb.world) *reinterpret_cast<unsigned long long*>(pb.stage[d] + pb.table_off + 8ull * (tb_mine + bb)) = entry;
            }
        }
        __syncthreads();
        if (threadIdx.x == SCAN_THREADS - 1) carry_s = carry + wo + in64;
        __syncthreads();
    }
    if (threadIdx.x == 0) { *total = carry_s; *arrival = 0u; }
    if (SHARDED) {
        if (threadIdx.x == 0) __threadfence_system();
        __syncthreads();
        if (threadIdx.x < (unsigned)pb.world) {
            unsigned long long* slot = pb.box[threadIdx.x] + MB_TOT + ((pb.seq & 1ull) * BVHGPU_MAX_PEERS + pb.rank) * 4;
            slot[1] = carry_s;
            __threadfence_system();
            st_release_sys(slot, pb.seq);
        }
        // ... and the same (last) block waits for the peers' posts and leaves {hit base of every source, grand total, ns waited} in
        // xinfo[0..9] for the two kernels behind it: no kernel of its own, and no polling from every block of emit / goffsets
        // (polling from every block costs time on every step)
        __syncthreads();
        if (threadIdx.x < 32) {
            wait_posts(pb, &xs);
            __syncwarp();
            if (threadIdx.x < BVHGPU_MAX_PEERS) xinfo[threadIdx.x] = xs.base[threadIdx.x];
            if (threadIdx.x == 0) { xinfo[8] = xs.grand; xinfo[9] = xs.waited; }
        }
    }
}

// Global offsets: one block per tile of every source rank.
__device__ __forceinline__ void goffsets_body(const PeerBoxes& pb, const unsigned long long* __restrict__ xinfo, uint32_t* __restrict__ offsets,
                                              uint32_t bid, uint32_t ntiles) {
    __shared__ unsigned long long wsum[SCAN_THREADS / 32];
    __shared__ uint32_t failed;
    if (threadIdx.x == 0) failed = *(volatile uint32_t*)pb.err;
    __syncthreads();
    const unsigned long long g = bid;
    if (failed == 0u) {
        int sg = 0;
        unsigned long long tb = 0, rb = 0, re = pb.rays_before[1];
#pragma unroll
        for (int k = 1; k < BVHGPU_MAX_PEERS; ++k) if (k < pb.world && g >= pb.tiles_before[k]) { sg = k; tb = pb.tiles_before[k]; rb = pb.rays_before[k]; re = pb.rays_before[k + 1]; }
        const unsigned long long hb = xinfo[sg];
        const unsigned char* stage = nullptr;
#pragma unroll
        for (int d = 0; d < BVHGPU_MAX_PEERS; ++d) if (d == pb.rank) stage = pb.stage[d];
        const unsigned long long entry = __ldcg(reinterpret_cast<const unsigned long long*>(stage + pb.table_off + 8ull * g));
        const unsigned long long width = entry >> 56;
        const unsigned char* p = stage + TILE_BYTES * g + (unsigned long long)threadIdx.x * SCAN_ITEMS * width;
        uint32_t v[SCAN_ITEMS];
        unsigned long long s = 0;                                  // 64-bit sums: see sat_u32
        static_assert(SCAN_ITEMS == 8, "8 counts per thread");
        if (width == 1) {
            const uint2 q = __ldcg(reinterpret_cast<const uint2*>(p));
            v[0] = q.x & 0xFFu; v[1] = (q.x >> 8) & 0xFFu; v[2] = (q.x >> 16) & 0xFFu; v[3] = q.x >> 24; v[4] = q.y & 0xFFu; v[5] = (q.y >> 8) & 0xFFu; v[6] = (q.y >> 16) & 0xFFu; v[7] = q.y >> 24;
        } else if (width == 2) {
            const uint4 q = __ldcg(reinterpret_cast<const uint4*>(p));
            v[0] = q.x & 0xFFFFu; v[1] = q.x >> 16; v[2] = q.y & 0xFFFFu; v[3] = q.y >> 16; v[4] = q.z & 0xFFFFu; v[5] = q.z >> 16; v[6] = q.w & 0xFFFFu; v[7] = q.w >> 16;
        } else {
            const uint4 q0 = __ldcg(reinterpret_cast<const uint4*>(p)), q1 = __ldcg(reinterpret_cast<const uint4*>(p) + 1);
            v[0] = q0.x; v[1] = q0.y; v[2] = q0.z; v[3] = q0.w; v[4] = q1.x; v[5] = q1.y; v[6] = q1.z; v[7] = q1.w;
        }
#pragma unroll
        for (int k = 0; k < SCAN_ITEMS; ++k) s += v[k];
        unsigned long long incl = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o); if ((int)lane_id() >= o) incl += t; }
        if (lane_id() == 31) wsum[threadIdx.x >> 5] = incl;
        __syncthreads();
        unsigned long long woff = 0;
        for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) woff += wsum[w];
        unsigned long long run = hb + (entry & OFF_MASK) + woff + incl - s;
        const unsigned long long j0 = rb + (g - tb) * SCAN_TILE + (unsigned long long)threadIdx.x * SCAN_ITEMS;
        uint32_t ov[SCAN_ITEMS];
#pragma unroll
        for (int k = 0; k < SCAN_ITEMS; ++k) { ov[k] = sat_u32(run); run += v[k]; }
        if (j0 + SCAN_ITEMS <= re && (j0 & 3ull) == 0ull) {
            uint4* o4 = reinterpret_cast<uint4*>(offsets + j0);
            o4[0] = make_uint4(ov[0], ov[1], ov[2], ov[3]);
            o4[1] = make_uint4(ov[4], ov[5], ov[6], ov[7]);
        } else {
#pragma unroll
            for (int k = 0; k < SCAN_ITEMS; ++k) if (j0 + k < re) offsets[j0 + k] = ov[k];
        }
        if (g == ntiles - 1 && threadIdx.x == 0) {
            unsigned long long ng = 0;
#pragma unroll
            for (int k = 1; k <= BVHGPU_MAX_PEERS; ++k) if (k == pb.world) ng = pb.rays_before[k];
            const unsigned long long grand = xinfo[8];
            offsets[ng] = grand > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)grand;
        }
    }
    if (bid == 0 && threadIdx.x < 32) {                        // the step ends when every peer's hit lists have landed here
        const int lane = threadIdx.x;
        const unsigned long long par = pb.seq & 1ull;
        unsigned long long waited = 0;
        if (lane < pb.world) {
            const unsigned long long* slot = pb.box[pb.rank] + MB_DONE + par * BVHGPU_MAX_PEERS + lane;
            const unsigned long long t0 = global_timer_ns();
            uint32_t spins = 0;
            while (ld_acquire_sys(slot) != pb.seq) {
                if (((++spins) & 63u) == 0u && global_timer_ns() - t0 > pb.timeout_ns) { atomicExch(pb.err, (uint32_t)BVHGPU_ERR_TIMEOUT); break; }
                __nanosleep(100);
            }
            waited = global_timer_ns() - t0;
        }
        for (int o = 16; o > 0; o >>= 1) { const unsigned long long w = __shfl_xor_sync(0xffffffffu, waited, o); waited = w > waited ? w : waited; }
        if (lane == 0) {
            unsigned long long* tr = pb.box[pb.rank] + MB_TRACE + (pb.seq % MB_TRACE_LEN) * 4;
            tr[0] = pb.seq; tr[1] = global_timer_ns(); tr[2] = xinfo[9]; tr[3] = waited;
        }
    }
}

// Destination of the emit pass.  Single GPU: the caller's buffers.  Sharded (pb.world > 0): the local copy of the global hit buffer
// at hit base + local offset; the offsets are not written here (goffsets_kernel rebuilds them on every rank).
struct EmitDst {
    uint32_t* offsets;                       // single GPU: the caller's offsets; sharded: nullptr
    uint32_t* hits;
    unsigned long long nrays_out;            // single GPU: index of the closing offsets entry
};

// Pass 2: final offsets + hit lists.  Rays with <= K hits copy their slots, the rest walk again.  Sharded: the block then ships
// its piece of the hit lists -- contiguous, because the block's rays are -- to every peer.
template <class T, bool FLAT>
__device__ __forceinline__ void emit_body(const typename Traits<T>::TNode* __restrict__ trec, uint32_t n_rec,
                                          const typename Traits<T>::DAabb* __restrict__ aabb,
                                          const RaySrc<T>& rays, uint32_t nrays,
                                          const uint32_t* __restrict__ counts, const uint32_t* __restrict__ slots, uint32_t K,
                                          const uint32_t* __restrict__ local, const unsigned long long* __restrict__ blocksum,
                                          const unsigned long long* __restrict__ total,
                                          const EmitDst& dst, unsigned long long cap, uint32_t first, uint32_t count,
                                          const PeerBoxes& pb, const unsigned long long* __restrict__ xinfo, uint32_t* __restrict__ arrival,
                                          uint32_t bid, uint32_t nblocks) {
    __shared__ unsigned long long rng[2];
    __shared__ uint32_t failed;
    __shared__ bool last;
    const bool sharded = pb.world > 0;
    unsigned long long hbase = 0;
    if (sharded) {
        if (threadIdx.x == 0) failed = *(volatile uint32_t*)pb.err;
        __syncthreads();
        hbase = xinfo[pb.rank];
    }
    const uint32_t r = first + bid * blockDim.x + threadIdx.x;
    if (!sharded || failed == 0u) {
        if (r == first && dst.offsets) {          // (sliced host path: the last slice's write is the final total)
            const unsigned long long t = *total;
            dst.offsets[dst.nrays_out] = t > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)t;
        }
        if (r < first + count) {
            const unsigned long long off = hbase + blocksum[r / SCAN_TILE] + local[r];
            if (dst.offsets) dst.offsets[r] = off > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)off;
            const uint32_t c = counts[r];
            if (c != 0 && dst.hits != nullptr) {
                if (c <= K) {
                    // 8 slot loads in flight per lane before the first store (one load per iteration leaves the lane waiting on every
                    // single slot)
                    for (uint32_t k0 = 0; k0 < c; k0 += 8) {
                        uint32_t h[8];
#pragma unroll
                        for (uint32_t j = 0; j < 8; ++j) if (k0 + j < c) h[j] = __ldcs(slots + (size_t)(k0 + j) * nrays + r);
#pragma unroll
                        for (uint32_t j = 0; j < 8; ++j) if (k0 + j < c && off + k0 + j < cap) dst.hits[off + k0 + j] = h[j];
                    }
                } else {
                    T o[3], inv[3];
                    load_ray<T, false>(rays, r, o, inv);
                    unsigned long long w = off;
                    walk<T, FLAT>(trec, n_rec, aabb, o, inv, [&](uint32_t shape) { if (w < cap) dst.hits[w] = shape; ++w; });
                }
            }
        }
    }
    if (!sharded) return;
    bool pushed = false;
    if (failed == 0u && pb.world > 1) {
        if (threadIdx.x == 0) {
            const uint32_t r0 = first + bid * blockDim.x;
            const uint32_t r1 = min(r0 + blockDim.x, first + count) - 1u;
            rng[0] = hbase + blocksum[r0 / SCAN_TILE] + local[r0];
            rng[1] = hbase + blocksum[r1 / SCAN_TILE] + local[r1] + counts[r1];
        }
        __syncthreads();                                              // also: the block's own hit stores are visible to the block
        const unsigned long long begin = rng[0], end = rng[1] < cap ? rng[1] : cap;
        if (begin < end) {
            pushed = true;
            const uint32_t* src = dst.hits;
            const unsigned long long q0 = (begin + 3ull) & ~3ull, q1 = end & ~3ull;
            if (q0 < q1) {
                for (unsigned long long q = (q0 >> 2) + threadIdx.x; q < (q1 >> 2); q += blockDim.x) {
                    const uint4 v = __ldcg(reinterpret_cast<const uint4*>(src) + q);
#pragma unroll
                    for (int d = 0; d < BVHGPU_MAX_PEERS; ++d) if (d < pb.world && d != pb.rank) reinterpret_cast<uint4*>(pb.hits[d])[q] = v;
                }
            }
            if (threadIdx.x < 8) {                                     // up to 3 words in front of q0 and 3 behind q1; or a short piece (< 7 words) as a whole
                unsigned long long w;
                bool ok;
                if (q0 < q1) { w = threadIdx.x < 4 ? begin + threadIdx.x : q1 + (threadIdx.x - 4); ok = threadIdx.x < 4 ? w < q0 : w < end; }
                else         { w = begin + threadIdx.x; ok = w < end; }
                if (ok) {
                    const uint32_t v = __ldcg(src + w);
#pragma unroll
                    for (int d = 0; d < BVHGPU_MAX_PEERS; ++d) if (d < pb.world && d != pb.rank) pb.hits[d][w] = v;
                }
            }
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        if (pushed) __threadfence_system();                           // only a block that stored to peers has something to order
        last = atomicAdd(arrival, 1u) == nblocks - 1;
    }
    __syncthreads();
    if (!last) return;
    if (threadIdx.x == 0) { __threadfence_system(); *arrival = 0u; }
    __syncthreads();
    if (threadIdx.x < (unsigned)pb.world) st_release_sys(pb.box[threadIdx.x] + MB_DONE + (pb.seq & 1ull) * BVHGPU_MAX_PEERS + pb.rank, pb.seq);
}
template <class T, bool FLAT>
__global__ void __launch_bounds__(256) emit_kernel(const typename Traits<T>::TNode* __restrict__ trec, uint32_t n_rec,
                                                   const typename Traits<T>::DAabb* __restrict__ aabb,
                                                   RaySrc<T> rays, uint32_t nrays,
                                                   const uint32_t* __restrict__ counts, const uint32_t* __restrict__ slots, uint32_t K,
                                                   const uint32_t* __restrict__ local, const unsigned long long* __restrict__ blocksum,
                                                   const unsigned long long* __restrict__ total,
                                                   EmitDst dst, unsigned long long cap, uint32_t first, uint32_t count,
                                                   PeerBoxes pb, const unsigned long long* __restrict__ xinfo, uint32_t* __restrict__ arrival) {
    emit_body<T, FLAT>(trec, n_rec, aabb, rays, nrays, counts, slots, K, local, blocksum, total, dst, cap, first, count, pb, xinfo, arrival, blockIdx.x, gridDim.x);
}
// Sharded step: the emit blocks and the global-offsets blocks are independent of each other (both only need the posts), so they are
// ONE launch: blocks [0, emit_blocks) emit and ship hit lists, the rest rebuild the offsets -- one kernel boundary less, and the
// offsets pass overlaps the emit.
template <class T, bool FLAT>
__global__ void __launch_bounds__(256) emit_goffsets_kernel(const typename Traits<T>::TNode* __restrict__ trec, uint32_t n_rec,
                                                            const typename Traits<T>::DAabb* __restrict__ aabb,
                                                            RaySrc<T> rays, uint32_t nrays,
                                                            const uint32_t* __restrict__ counts, const uint32_t* __restrict__ slots, uint32_t K,
                                                            const uint32_t* __restrict__ local, const unsigned long long* __restrict__ blocksum,
                                                            const unsigned long long* __restrict__ total,
                                                            EmitDst dst, unsigned long long cap, uint32_t count,
                                                            PeerBoxes pb, const unsigned long long* __restrict__ xinfo, uint32_t* __restrict__ arrival,
                                                            uint32_t emit_blocks, uint32_t* __restrict__ offsets) {
    if (blockIdx.x < emit_blocks) emit_body<T, FLAT>(trec, n_rec, aabb, rays, nrays, counts, slots, K, local, blocksum, total, dst, cap, 0u, count, pb, xinfo, arrival, blockIdx.x, emit_blocks);
    else goffsets_body(pb, xinfo, offsets, blockIdx.x - emit_blocks, gridDim.x - emit_blocks);
}

// Launch pass 1 over rays [first, first+count): persistent refill kernel (default) or one ray per thread.
// sums layout (u64 words): [nblk] total, [nblk+1] visits, [nblk+2 .. nblk+11] exchange info, [nblk+12] error, [nblk+13] ticket,
// [nblk+14] ready, [nblk+15] probe verdict, [nblk+16] largest count, [nblk+17] block counter of the exchange post.
constexpr uint32_t SUMS_TAIL = 20;
constexpr uint32_t S_TOTAL = 0, S_VISITS = 1, S_XINFO = 2, S_ERR = 12, S_TICKET = 13, S_READY = 14, S_GATE = 15, S_MAXC = 16, S_BLKDONE = 17;
constexpr unsigned long long STREAM_TIMEOUT_NS = 4ull * 1000ull * 1000ull * 1000ull;
// The shared-memory top-tree walk: f32 trees only; false = not applicable (the caller launches the plain persistent kernel).
constexpr uint32_t TOP_BUDGET = 7000;                               // entries: 224 000 B of the 227 KB a CTA may own
constexpr size_t TOP_UNROLL_MAX_BYTES = (size_t)32 << 20;           // traversal records that count as L2-resident (H100: 50 MB of L2)
constexpr int TOP_VPC_L2 = 5;                                       // visits per vote on those trees (see launch_top)
template <class T> static bool launch_top(Tree<T>*, bool, RaySrc<T>, uint32_t, uint32_t*, uint32_t*, uint32_t, unsigned long long*, uint32_t*, bool) { return false; }
template <> bool launch_top<float>(Tree<float>* tree, bool flat, RaySrc<float> rays, uint32_t R, uint32_t* counts, uint32_t* slots, uint32_t K,
                                   unsigned long long* tail, uint32_t* gate, bool stream_mode) {
    bvhgpu_ctx* ctx = tree->ctx;
    if (tree->n < 2) return false;
    const uint32_t budget = ctx->traverse_top > 1 ? (uint32_t)std::min<int64_t>(std::max<int64_t>(ctx->traverse_top, 8), TOP_BUDGET) : TOP_BUDGET;
    if ((!tree->top_valid || tree->top_budget != budget) && build_top_records(tree, budget) != BVHGPU_OK) return false;
    if (!ctx->top_attr_set) {                                           // a per-device function attribute: once per context
        const int bytes = (int)(TOP_BUDGET * 32);
        auto raise = [&](const void* f) { return cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) == cudaSuccess; };
        if (!raise((const void*)walk_top_kernel<false, false, 1>) || !raise((const void*)walk_top_kernel<true, false, 1>) ||
            !raise((const void*)walk_top_kernel<false, true, 1>) || !raise((const void*)walk_top_kernel<true, true, 1>) ||
            !raise((const void*)walk_top_kernel<false, false, TOP_VPC_L2>) || !raise((const void*)walk_top_kernel<true, false, TOP_VPC_L2>) ||
            !raise((const void*)walk_top_kernel<false, true, TOP_VPC_L2>) || !raise((const void*)walk_top_kernel<true, true, TOP_VPC_L2>)) { cudaGetLastError(); return false; }
        ctx->top_attr_set = true;
    }
    const size_t smem = (size_t)budget * 32;                            // n_top <= budget lives on the device: reserve for the budget
    const int grid = (int)std::min<uint64_t>((uint64_t)ctx->sm_count, ((uint64_t)R + 1023) / 1024);
    uint32_t* ticket = reinterpret_cast<uint32_t*>(tail + S_TICKET);
    uint32_t* err = reinterpret_cast<uint32_t*>(tail + S_ERR);
    const float4* top = reinterpret_cast<const float4*>(tree->d_top);
    static const int top_refill = getenv("BVHGPU_TOP_REFILL") ? std::max(1, std::min(32, atoi(getenv("BVHGPU_TOP_REFILL")))) : 8;   // dev knob: idle lanes per refill
    // Visits per vote: TOP_VPC_L2 = 5 where the records stay L2-resident, 1 for trees beyond L2 (hbm_bound, 640 MB: 4 was 2 % slower
    // there, its visits wait on DRAM).  On config 2 (7.7 MB, H100) the walk kernel took 0.316 ms at 5 visits per vote, 0.327 at 3,
    // 0.317-0.322 at 7, but 0.361 at 2, 0.352 at 4 (the previous choice), 0.350 at 6 and 0.351 at 8 (DESIGN §4.3).
    const bool l2_tree = (size_t)tree->n_trec * sizeof(TNodeF) <= TOP_UNROLL_MAX_BYTES;
#define BVH_TOP_LAUNCH(F, S, V, TMO) walk_top_kernel<F, S, V><<<grid, 1024, smem, ctx->stream>>>(tree->d_tnodes, walk_aabbs(tree), tree->n_trec, top, rays, R, ticket, \
                                                                    ctx->d_ready, counts, slots, K, tail + S_VISITS, gate, 0u, err, TMO, top_refill)
#define BVH_TOP_FORMS(V) do { if (stream_mode) { if (flat) BVH_TOP_LAUNCH(true, true, V, STREAM_TIMEOUT_NS); else BVH_TOP_LAUNCH(false, true, V, STREAM_TIMEOUT_NS); } \
                              else             { if (flat) BVH_TOP_LAUNCH(true, false, V, 0ull); else BVH_TOP_LAUNCH(false, false, V, 0ull); } } while (0)
    if (l2_tree) BVH_TOP_FORMS(TOP_VPC_L2); else BVH_TOP_FORMS(1);
#undef BVH_TOP_FORMS
#undef BVH_TOP_LAUNCH
    ctx->launches++;
    return true;
}

template <class T>
static int launch_pass1(Tree<T>* tree, bool flat, RaySrc<T> rays, uint32_t R, uint32_t first, uint32_t count,
                        uint32_t* counts, uint32_t* slots, uint32_t K, unsigned long long* sums, uint32_t nblk, bool stream_mode) {
    bvhgpu_ctx* ctx = tree->ctx;
    cudaStream_t st = ctx->stream;
    unsigned long long* tail = sums + nblk;
    // traverse_persistent: 0 = one ray per thread, 1 = persistent refill, 2 (default) = probe decides on the device
    const int64_t pmode = stream_mode ? 1 : ctx->traverse_persistent;
    uint32_t* gate = nullptr;
    if (pmode >= 2) {
        gate = reinterpret_cast<uint32_t*>(tail + S_GATE);
        coherence_probe_kernel<T><<<1, 256, 0, st>>>(rays, R, gate);
        ctx->launches++;
    }
    if (pmode == 0 || pmode >= 2) {
        const int grid = (count + 255) / 256;
        if (flat) walk_count_kernel<T, true><<<grid, 256, 0, st>>>(tree->d_tnodes, tree->n_trec, walk_aabbs(tree), rays, R, first, count, counts, slots, K, tail + S_VISITS, gate, 1u);
        else      walk_count_kernel<T, false><<<grid, 256, 0, st>>>(tree->d_tnodes, tree->n_trec, walk_aabbs(tree), rays, R, first, count, counts, slots, K, tail + S_VISITS, gate, 1u);
        ctx->launches++;
        if (pmode == 0) return BVHGPU_OK;
    }
    if (first != 0 || count != R) { set_error("internal: persistent walk covers whole batches only"); return BVHGPU_ERR_INTERNAL; }
    // Shared-memory top of the tree: pays off on large trees; on small ones (Sponza's 133 k records) the global fetches still hit
    // L1 well.  Automatic from 5 MB of records (threshold from the previous target, not re-swept on H100), forced by option
    // traverse_top >= 1.
    const bool want_top = ctx->traverse_top >= 1 || (ctx->traverse_top < 0 && (size_t)tree->n_trec * sizeof(typename Traits<T>::TNode) >= ((size_t)5 << 20));
    if (want_top && launch_top(tree, flat, rays, R, counts, slots, K, tail, gate, stream_mode)) return BVHGPU_OK;
    if (ctx->walk_grid == 0) {
        int occ = 1;
        BVH_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, walk_persistent_kernel<float, false, false>, 256, 0));
        ctx->walk_grid = ctx->sm_count * (occ < 1 ? 1 : occ);
    }
    // A lane should see ~6 rays or more: with fewer, the last ray of every lane (the drain phase, where warps run half empty) is a
    // large part of the kernel.  Hence fewer CTAs per SM for small batches (at least 4), the full wave for large ones.
    const uint64_t sms = (uint64_t)ctx->sm_count;
    const uint64_t per_sm = std::min<uint64_t>((uint64_t)ctx->walk_grid / sms, std::max<uint64_t>(4, (uint64_t)R / (6ull * 256ull * sms)));
    const int grid = (int)std::min<uint64_t>(ctx->walk_grid_forced ? (uint64_t)ctx->walk_grid : std::max<uint64_t>(1, per_sm) * sms, ((uint64_t)R + 255) / 256);
    uint32_t* ticket = reinterpret_cast<uint32_t*>(tail + S_TICKET);
    const uint32_t* ready = ctx->d_ready;                    // only read by the streamed form
    uint32_t* err = reinterpret_cast<uint32_t*>(tail + S_ERR);
    if (stream_mode) {
        if (flat) walk_persistent_kernel<T, true, true><<<grid, 256, 0, st>>>(tree->d_tnodes, tree->n_trec, walk_aabbs(tree), rays, R, ticket, ready, counts, slots, K, tail + S_VISITS, nullptr, 0u, err, STREAM_TIMEOUT_NS);
        else      walk_persistent_kernel<T, false, true><<<grid, 256, 0, st>>>(tree->d_tnodes, tree->n_trec, walk_aabbs(tree), rays, R, ticket, ready, counts, slots, K, tail + S_VISITS, nullptr, 0u, err, STREAM_TIMEOUT_NS);
    } else {
        if (flat) walk_persistent_kernel<T, true, false><<<grid, 256, 0, st>>>(tree->d_tnodes, tree->n_trec, walk_aabbs(tree), rays, R, ticket, ready, counts, slots, K, tail + S_VISITS, gate, 0u, err, 0ull);
        else      walk_persistent_kernel<T, false, false><<<grid, 256, 0, st>>>(tree->d_tnodes, tree->n_trec, walk_aabbs(tree), rays, R, ticket, ready, counts, slots, K, tail + S_VISITS, gate, 0u, err, 0ull);
    }
    ctx->launches++;
    return BVHGPU_OK;
}

// Loads the kernels of the sharded step into the current device's context.  Under lazy module loading the first launch of a kernel
// loads it, and a load can wait for kernels already running -- such as a scan kernel spinning on a peer whose own launch is held up
// behind the load (ranks of one process share the device's context).  bvhgpu_peer_alloc, which every rank calls before its first
// step, loads them up front.
int preload_shard_kernels() {
    cudaFuncAttributes a;
    BVH_CUDA_TRY(cudaFuncGetAttributes(&a, scan_post_kernel<true>));
    BVH_CUDA_TRY(cudaFuncGetAttributes(&a, emit_goffsets_kernel<float, false>));
    BVH_CUDA_TRY(cudaFuncGetAttributes(&a, emit_goffsets_kernel<float, true>));
    BVH_CUDA_TRY(cudaFuncGetAttributes(&a, emit_goffsets_kernel<double, false>));
    BVH_CUDA_TRY(cudaFuncGetAttributes(&a, emit_goffsets_kernel<double, true>));
    return BVHGPU_OK;
}

// Every check of a sharded step's arguments, made before the call enqueues anything: a bad shard must not leave a walk (or a scan
// that stores through a null peer pointer) behind on the stream.  The mailbox starts zeroed, so seq 0 would let every wait pass at once.
int check_shard(const bvhgpu_shard* shard, size_t nrays) {
    const int W = shard->world;
    if (W < 1 || W > BVHGPU_MAX_PEERS || shard->rank < 0 || shard->rank >= W) { set_error("traverse_sharded: bad rank/world %d/%d", shard->rank, W); return BVHGPU_ERR_INVALID; }
    if (shard->seq == 0) { set_error("traverse_sharded: seq must start at 1 (the zeroed mailbox already holds 0)"); return BVHGPU_ERR_INVALID; }
    if (shard->ray_layout != BVHGPU_RAYS_FULL && shard->ray_layout != BVHGPU_RAYS_OD) { set_error("traverse_sharded: bad ray layout %d", shard->ray_layout); return BVHGPU_ERR_INVALID; }
    if (!shard->offsets) { set_error("traverse_sharded: shard->offsets is null"); return BVHGPU_ERR_INVALID; }
    unsigned long long NG = 0, NT = 0;
    for (int d = 0; d < W; ++d) {
        if (!shard->peer_counts[d] || !shard->peer_hits[d] || !shard->peer_mailbox[d]) { set_error("traverse_sharded: a peer buffer of rank %d is null", d); return BVHGPU_ERR_INVALID; }
        if (shard->shard_rays[d] == 0) { set_error("traverse_sharded: rank %d has an empty shard (every rank needs rays)", d); return BVHGPU_ERR_INVALID; }
        if (shard->shard_rays[d] > 0x7FFFFFFFull) { set_error("traverse_sharded: shard_rays[%d] = %zu exceeds 2^31-1", d, shard->shard_rays[d]); return BVHGPU_ERR_INVALID; }
        NG += shard->shard_rays[d];
        NT += (shard->shard_rays[d] + SCAN_TILE - 1) / SCAN_TILE;
    }
    if (shard->shard_rays[shard->rank] != nrays) { set_error("traverse_sharded: shard_rays[rank] = %zu but nrays = %zu", shard->shard_rays[shard->rank], nrays); return BVHGPU_ERR_INVALID; }
    if (NG > 0x7FFFFFFFull) { set_error("traverse_sharded: %llu rays in total exceed 2^31-1", NG); return BVHGPU_ERR_INVALID; }
    if (TILE_BYTES * NT + 8ull * NT > BVHGPU_SHARD_STAGE_BYTES(NG)) { set_error("internal: staging layout exceeds BVHGPU_SHARD_STAGE_BYTES"); return BVHGPU_ERR_INTERNAL; }
    return BVHGPU_OK;
}

template <class T>
int traverse_device(Tree<T>* tree, int mode, const void* d_rays, uint32_t fmt, size_t nrays,
                    uint32_t* d_offsets, uint32_t* d_hits, size_t cap, size_t* total, const bvhgpu_shard* shard) {
    bvhgpu_ctx* ctx = tree->ctx;
    cudaStream_t st = ctx->stream;
    if (nrays > 0x7FFFFFFFull) { set_error("traverse: nrays %zu exceeds 2^31-1", nrays); return BVHGPU_ERR_INVALID; }
    if (mode != BVHGPU_TRAVERSE_BVH && mode != BVHGPU_TRAVERSE_FLAT) { set_error("traverse: bad mode %d", mode); return BVHGPU_ERR_INVALID; }
    if (fmt != RAYS_FULL && fmt != RAYS_OD) { set_error("traverse: bad ray layout %u", fmt); return BVHGPU_ERR_INVALID; }
    tree->last_nrays = nrays;
    if (nrays == 0) {
        if (d_offsets) BVH_CUDA_TRY(cudaMemsetAsync(d_offsets, 0, sizeof(uint32_t), st));
        if (total) *total = 0;
        tree->last_total = 0;
        return BVHGPU_OK;
    }
    if (tree->n == 0) {                                          // empty Bvh: no hits (bvh_impl.rs:109-112)
        BVH_CUDA_TRY(cudaMemsetAsync(d_offsets, 0, sizeof(uint32_t) * (nrays + 1), st));
        if (total) *total = 0;
        tree->last_total = 0;
        return BVHGPU_OK;
    }
    BVH_TRY(resolve_status(tree));                               // never walk a tree whose build failed
    if (!tree->d_tnodes) BVH_TRY(build_traversal_records(tree));
    const RaySrc<T> rays{reinterpret_cast<const T*>(d_rays), fmt};
    const uint32_t R = (uint32_t)nrays;
    const uint32_t K = pick_slots(ctx, R);
    const uint32_t nblk = (R + SCAN_TILE - 1) / SCAN_TILE;
    Scratch scratch(ctx);
    uint32_t *counts = nullptr, *slots = nullptr, *local = nullptr;
    unsigned long long* sums = nullptr;       // [nblk] block offsets, then the tail words (see launch_pass1)
    BVH_TRY(scratch.get(&counts, R));
    BVH_TRY(scratch.get(&local, R));
    if (K) BVH_TRY(scratch.get(&slots, (size_t)K * R));
    BVH_TRY(scratch.get(&sums, (size_t)nblk + SUMS_TAIL));
    unsigned long long* tail = sums + nblk;
    BVH_CUDA_TRY(cudaMemsetAsync(tail, 0, SUMS_TAIL * sizeof(unsigned long long), st));
    const bool flat = mode == BVHGPU_TRAVERSE_FLAT;
    {
        if (ctx->profile) cudaEventRecord(ctx->ev_walk[0], st);
        BVH_TRY(launch_pass1<T>(tree, flat, rays, R, 0, R, counts, slots, K, sums, nblk, false));
        if (ctx->profile) { cudaEventRecord(ctx->ev_walk[1], st); ctx->have_walk = true; }
    }
    const int grid = (R + 255) / 256;
    EmitDst dst{};
    PeerBoxes pb{};                                                   // world == 0: single GPU
    uint32_t* arrival = reinterpret_cast<uint32_t*>(tail + S_BLKDONE);
    if (shard) {
        const int W = shard->world;
        pb.rank = shard->rank; pb.world = W; pb.seq = shard->seq;
        pb.err = ctx->d_async_err; pb.timeout_ns = 10ull * 1000ull * 1000ull * 1000ull;
        pb.rays_before[0] = 0; pb.tiles_before[0] = 0;
        for (int d = 0; d < BVHGPU_MAX_PEERS; ++d) {
            const unsigned long long nd = d < W ? (unsigned long long)shard->shard_rays[d] : 0ull;
            pb.rays_before[d + 1] = pb.rays_before[d] + nd;
            pb.tiles_before[d + 1] = pb.tiles_before[d] + (nd + SCAN_TILE - 1) / SCAN_TILE;
        }
        const unsigned long long NG = pb.rays_before[W], NT = pb.tiles_before[W];
        pb.table_off = TILE_BYTES * NT;
        const size_t half = BVHGPU_SHARD_STAGE_BYTES(NG);                // the staging alternates between two halves (parity of seq)
        for (int d = 0; d < W; ++d) {                                    // (check_shard has vetted the shard before anything ran)
            pb.box[d] = (unsigned long long*)shard->peer_mailbox[d];
            pb.stage[d] = (unsigned char*)shard->peer_counts[d] + (shard->seq & 1ull) * half;
            pb.hits[d] = (uint32_t*)shard->peer_hits[d];
        }
        cap = shard->cap;
        dst.offsets = nullptr; dst.hits = pb.hits[pb.rank];
        scan_post_kernel<true><<<nblk, SCAN_THREADS, 0, st>>>(counts, R, local, sums, tail + S_TOTAL, arrival, pb, tail + S_XINFO);
    } else {
        dst.offsets = d_offsets; dst.hits = d_hits; dst.nrays_out = R;
        scan_post_kernel<false><<<nblk, SCAN_THREADS, 0, st>>>(counts, R, local, sums, tail + S_TOTAL, arrival, pb, tail + S_XINFO);
    }
    ctx->launches++;
    unsigned long long* h = reinterpret_cast<unsigned long long*>(ctx->h_pinned);
    if (total) {                                                  // the total is known before the hit lists are written
        BVH_CUDA_TRY(cudaMemcpyAsync(h, tail, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
        BVH_CUDA_TRY(cudaEventRecord(ctx->ev_total, st));
    }
    if (shard) {
        const unsigned g2 = (unsigned)grid + (unsigned)pb.tiles_before[pb.world];
        if (flat) emit_goffsets_kernel<T, true><<<g2, 256, 0, st>>>(tree->d_tnodes, tree->n_trec, walk_aabbs(tree), rays, R, counts, slots, K, local, sums, tail + S_TOTAL, dst, (unsigned long long)cap, R, pb, tail + S_XINFO, arrival, (uint32_t)grid, (uint32_t*)shard->offsets);
        else      emit_goffsets_kernel<T, false><<<g2, 256, 0, st>>>(tree->d_tnodes, tree->n_trec, walk_aabbs(tree), rays, R, counts, slots, K, local, sums, tail + S_TOTAL, dst, (unsigned long long)cap, R, pb, tail + S_XINFO, arrival, (uint32_t)grid, (uint32_t*)shard->offsets);
    } else {
        if (flat) emit_kernel<T, true><<<grid, 256, 0, st>>>(tree->d_tnodes, tree->n_trec, walk_aabbs(tree), rays, R, counts, slots, K, local, sums, tail + S_TOTAL, dst, (unsigned long long)cap, 0u, R, pb, tail + S_XINFO, arrival);
        else      emit_kernel<T, false><<<grid, 256, 0, st>>>(tree->d_tnodes, tree->n_trec, walk_aabbs(tree), rays, R, counts, slots, K, local, sums, tail + S_TOTAL, dst, (unsigned long long)cap, 0u, R, pb, tail + S_XINFO, arrival);
    }
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    int rc = BVHGPU_OK;
    if (total) {
        BVH_CUDA_TRY(cudaEventSynchronize(ctx->ev_total));        // emit_kernel keeps running while the host reads the total
        *total = (size_t)h[0];
        tree->last_total = (size_t)h[0];
        tree->last_visits = h[1];
        if (h[0] > 0xFFFFFFFFull) { set_error("traverse: %llu hits overflow the u32 CSR offsets", h[0]); rc = BVHGPU_ERR_CAPACITY; }
        else if (d_hits && h[0] > cap) { set_error("traverse: %llu hits do not fit capacity %zu", h[0], cap); rc = BVHGPU_ERR_CAPACITY; }
    }
    return rc;
}

// ---- may the host path stream rays into a running kernel? ------------------------------------------------------------------
// The streaming form needs (a) kernel launches that return to the host while the kernel runs and (b) nobody replaying or
// serialising kernels.  Neither holds under CUDA_LAUNCH_BLOCKING=1, cuda-gdb, compute-sanitizer or Nsight Compute (which
// replays a kernel several times against restored memory: the DMA-bumped `ready` word would be rolled back).  Those are
// recognised from the environment / the injected libraries; in addition a one-off probe checks property (a) directly: a
// kernel that waits (bounded) for a flag which only a LATER-enqueued copy on another stream sets.
__global__ void overlap_probe_kernel(const volatile uint32_t* flag, uint32_t* saw, unsigned long long timeout_ns) {
    const unsigned long long t0 = global_timer_ns();
    uint32_t ok = 0;
    for (;;) {
        if (*flag) { ok = 1; break; }
        if (global_timer_ns() - t0 > timeout_ns) break;
        __nanosleep(200);
    }
    *saw = ok;
}
static bool tooling_detected() {
    const char* lb = getenv("CUDA_LAUNCH_BLOCKING");
    if (lb && lb[0] && strcmp(lb, "0") != 0) return true;
    // (as observed: under ncu the process carries NV_CUDA_START_SUSPENDED / NVIDIA_PROCESS_INJECTION_* and maps
    //  .../nsight-compute/.../libTreeLauncherTargetInjection.so; compute-sanitizer injects through CUDA_INJECTION64_PATH)
    static const char* vars[] = {"CUDA_INJECTION64_PATH", "CUDA_INJECTION32_PATH", "NV_CUDA_START_SUSPENDED", "NVIDIA_PROCESS_INJECTION_CRASH_REPORTING",
                                 "NVIDIA_PROCESS_INJECTION_XML_TARGET_SETTINGS", "CUDBG_USE_LEGACY_DEBUGGER", "NV_NSIGHT_INJECTION_TRANSPORT_TYPE",
                                 "NSIGHT_CUDA_DEBUGGER", "CUDA_DEBUGGER_SOFTWARE_PREEMPTION"};
    for (const char* v : vars) { const char* e = getenv(v); if (e && e[0]) return true; }
    // injected libraries: scanned ONCE per process (a python + torch process maps thousands of regions: reading /proc/self/maps
    // on every call would cost a noticeable part of a traversal); the environment above is checked every time
    static int mapped = -1;
    if (mapped < 0) {
        int found = 0;
        if (FILE* f = fopen("/proc/self/maps", "r")) {
            char line[1024];
            while (!found && fgets(line, sizeof line, f))
                if (strstr(line, "nsight") || strstr(line, "libcuda-injection") || strstr(line, "libsanitizer-collection") || strstr(line, "libInterceptorInjection") || strstr(line, "libTreeLauncher"))
                    found = 1;
            fclose(f);
        }
        mapped = found;
    }
    return mapped == 1;
}
static int stream_capable(bvhgpu_ctx* ctx) {
    if (ctx->traverse_stream == 0) return 0;
    if (ctx->traverse_stream == 1) return 1;
    if (tooling_detected()) return 0;                           // re-checked every call: cheap, and a tool can attach later
    if (ctx->stream_ok >= 0) return ctx->stream_ok;
    ctx->stream_ok = 0;
    uint32_t* d = nullptr;
    if (dalloc_t(ctx, &d, 2) != BVHGPU_OK) return 0;
    uint32_t* h = ctx->h_pinned + 128;
    bool ok = cudaMemsetAsync(d, 0, 2 * sizeof(uint32_t), ctx->stream) == cudaSuccess;
    ok = ok && cudaEventRecord(ctx->ev_order, ctx->stream) == cudaSuccess && cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_order, 0) == cudaSuccess;
    if (ok) {
        overlap_probe_kernel<<<1, 1, 0, ctx->stream>>>(d, d + 1, 20ull * 1000ull * 1000ull);      // gives up after 20 ms
        h[0] = 1u;
        ok = cudaMemcpyAsync(d, h, sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->copy_stream) == cudaSuccess;
        ok = ok && cudaMemcpyAsync(h + 1, d + 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream) == cudaSuccess;
        ok = (cudaStreamSynchronize(ctx->copy_stream) == cudaSuccess) && ok;
        ok = (cudaStreamSynchronize(ctx->stream) == cudaSuccess) && ok;
        ctx->launches++;
        if (ok && h[1] == 1u) ctx->stream_ok = 1;
    }
    dfree(ctx, d);
    return ctx->stream_ok;
}

// cuStreamWriteValue32 (driver API, resolved through the runtime: no libcuda link dependency): the arrival counter is bumped by a
// stream memory operation behind every chunk copy instead of a 4-byte DMA (each tiny copy costs copy-engine latency of its own,
// which adds up over the chunks of a transfer).  Falls back to the 4-byte copy where the entry point is missing.
typedef int (*WriteValue32Fn)(cudaStream_t, unsigned long long, uint32_t, unsigned int);
static WriteValue32Fn stream_write_value32() {
    static WriteValue32Fn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuStreamWriteValue32", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = (WriteValue32Fn)p;
        else (void)cudaGetLastError();
    }
    return fn;
}

// Host-pointer entry point.  Large batches on an undisturbed device are STREAMED: the batch is copied in chunks on the copy
// stream, each followed by a 4-byte DMA that bumps a device-side `ready` counter, and ONE persistent walk kernel -- launched
// AFTER all copies are enqueued, so it never depends on work the host has yet to submit -- consumes the rays as they arrive.
// Small batches, and any process in which launches are serialised or replayed (see stream_capable), take the plain form:
// one copy, then the same kernels as the device-pointer path.  The emit pass runs in slices whose offsets travel back on the
// D2H stream while the next slice is emitted.  Results are retained in tree->d_offsets / d_hits (bvhgpu_traverse_fetch_*).
template <class T>
int traverse_host_pipelined(Tree<T>* tree, int mode, const void* h_rays, uint32_t fmt, size_t nrays,
                            uint32_t* h_offsets, uint32_t* h_hits, size_t h_cap, size_t* total) {
    bvhgpu_ctx* ctx = tree->ctx;
    cudaStream_t st = ctx->stream;
    const uint32_t R = (uint32_t)nrays;
    const auto t_entry = std::chrono::steady_clock::now();
    auto stamp = [&](int k) { if (ctx->profile) ctx->host_us[k] = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t_entry).count(); };
    BVH_TRY(resolve_status(tree));
    if (fmt != RAYS_FULL && fmt != RAYS_OD) { set_error("traverse: bad ray layout %u", fmt); return BVHGPU_ERR_INVALID; }
    if (!tree->d_tnodes) BVH_TRY(build_traversal_records(tree));
    const size_t ray_bytes = (fmt == RAYS_FULL ? 9 : 6) * sizeof(T);
    const uint32_t K = pick_slots(ctx, R);
    const uint32_t nblk = (R + SCAN_TILE - 1) / SCAN_TILE;
    Scratch scratch(ctx);
    uint32_t *counts = nullptr, *slots = nullptr, *local = nullptr;
    unsigned long long* sums = nullptr;
    unsigned char* staged = nullptr;
    BVH_TRY(scratch.get(&counts, R));
    BVH_TRY(scratch.get(&local, R));
    if (K) BVH_TRY(scratch.get(&slots, (size_t)K * R));
    BVH_TRY(scratch.get(&sums, (size_t)nblk + SUMS_TAIL));
    BVH_TRY(scratch.get(&staged, ray_bytes * R));
    unsigned long long* tail = sums + nblk;
    BVH_CUDA_TRY(cudaMemsetAsync(tail, 0, SUMS_TAIL * sizeof(unsigned long long), st));
    const bool flat = mode == BVHGPU_TRAVERSE_FLAT;
    const RaySrc<T> rays{reinterpret_cast<const T*>(staged), fmt};
    EmitDst dst{};
    dst.offsets = tree->d_offsets; dst.hits = tree->d_hits; dst.nrays_out = R;
    const PeerBoxes nopeers{};
    uint32_t* arrival = reinterpret_cast<uint32_t*>(tail + S_BLKDONE);
    static const int force_chunks = getenv("BVHGPU_CHUNKS") ? atoi(getenv("BVHGPU_CHUNKS")) : 0;           // dev knob
    const uint32_t nchunks = force_chunks > 0 ? std::min<uint32_t>(BVH_MAX_CHUNKS, (uint32_t)force_chunks)
                                              : (R < 240000u ? 1u : std::max<uint32_t>(2, std::min<uint32_t>(BVH_MAX_CHUNKS, R / 250000)));   // 4 chunks per million rays
    const bool streaming = nchunks > 1 && stream_capable(ctx) == 1;
    ctx->last_streamed = streaming ? 1 : 0;
    stamp(0);                                                     // scratch allocated
    BVH_CUDA_TRY(cudaMemsetAsync(ctx->d_ready, 0, sizeof(uint32_t), st));
    BVH_CUDA_TRY(cudaEventRecord(ctx->ev_order, st));             // the scratch (and its zeroed tail) exists from here on
    BVH_CUDA_TRY(cudaStreamWaitEvent(ctx->d2h_stream, ctx->ev_order, 0));
    if (ctx->profile) cudaEventRecord(ctx->ev_e2e[0], st);
    if (streaming) {
        BVH_CUDA_TRY(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_order, 0));
        uint32_t* h_ready = ctx->h_pinned + 64;                  // pinned: one value per chunk, alive until the final sync
        uint32_t* d_ready = ctx->d_ready;                        // plain cudaMalloc memory: the stream memory operation refuses pool memory
        ctx->wv_ok = 1;
        static const int sched = getenv("BVHGPU_CHUNK_SCHEDULE") ? atoi(getenv("BVHGPU_CHUNK_SCHEDULE")) : 1;     // dev knob
        // Schedule 1 (default): the first half of the chunks carries two thirds of the rays.  Every chunk costs copy-engine
        // latency (copy + counter update), and the call ends one longest-ray latency behind the LAST chunk whatever its size:
        // few, large copies early and small ones at the end (tools/e2e_probe.py compares schedules).
        const uint32_t nhalf = nchunks / 2, units = sched == 1 ? nchunks + nhalf : nchunks;
        auto bound = [&](uint32_t c) -> uint32_t {
            const uint32_t u = sched == 1 ? (c <= nhalf ? 2 * c : nhalf + c) : c;
            return (uint32_t)((uint64_t)R * u / units);
        };
        for (uint32_t c = 0; c < nchunks; ++c) {
            const uint32_t lo = bound(c), hi = bound(c + 1);
            cudaError_t e = cudaMemcpyAsync(staged + ray_bytes * lo, (const unsigned char*)h_rays + ray_bytes * lo, ray_bytes * (hi - lo), cudaMemcpyHostToDevice, ctx->copy_stream);
            h_ready[c] = hi;
            if (e == cudaSuccess) {
                WriteValue32Fn wv = stream_write_value32();
                if (!wv || wv(ctx->copy_stream, (unsigned long long)(uintptr_t)d_ready, hi, 0u) != 0) {
                    ctx->wv_ok = 0;
                    e = cudaMemcpyAsync(d_ready, h_ready + c, sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->copy_stream);
                }
            }
            if (e != cudaSuccess) {                               // nothing waits on `ready` yet (the kernel is launched below): just report
                set_error("traverse: H2D copy of chunk %u failed: %s", c, cudaGetErrorString(e));
                cudaStreamSynchronize(ctx->copy_stream);
                return BVHGPU_ERR_CUDA;
            }
        }
        if (ctx->profile) cudaEventRecord(ctx->ev_e2e[2], ctx->copy_stream);
        stamp(1);                                                 // copies enqueued
        const int rc1 = launch_pass1<T>(tree, flat, rays, R, 0, R, counts, slots, K, sums, nblk, true);
        if (rc1 != BVHGPU_OK) { cudaStreamSynchronize(ctx->copy_stream); return rc1; }      // the copies still target the scratch
        if (ctx->profile) cudaEventRecord(ctx->ev_e2e[1], st);
    } else {
        BVH_CUDA_TRY(cudaMemcpyAsync(staged, h_rays, ray_bytes * R, cudaMemcpyHostToDevice, st));
        if (ctx->profile) cudaEventRecord(ctx->ev_e2e[2], st);
        BVH_TRY(launch_pass1<T>(tree, flat, rays, R, 0, R, counts, slots, K, sums, nblk, false));
        if (ctx->profile) cudaEventRecord(ctx->ev_e2e[1], st);
    }
    stamp(2);                                                     // walk launched
    {
        scan_post_kernel<false><<<nblk, SCAN_THREADS, 0, st>>>(counts, R, local, sums, tail + S_TOTAL, arrival, nopeers, tail + S_XINFO);
        // emit + D2H of the offsets in 4 slices so that the copy back overlaps the rest of the emit
        const uint32_t nsl = R >= 400000 ? 4 : 1;
        for (uint32_t c = 0; c < nsl; ++c) {
            const uint32_t lo = (uint32_t)((uint64_t)R * c / nsl), hi = (uint32_t)((uint64_t)R * (c + 1) / nsl), cnt = hi - lo;
            const int g = (cnt + 255) / 256;
            if (flat) emit_kernel<T, true><<<g, 256, 0, st>>>(tree->d_tnodes, tree->n_trec, walk_aabbs(tree), rays, R, counts, slots, K, local, sums, tail + S_TOTAL, dst, (unsigned long long)tree->hits_cap, lo, cnt, nopeers, tail + S_XINFO, arrival);
            else      emit_kernel<T, false><<<g, 256, 0, st>>>(tree->d_tnodes, tree->n_trec, walk_aabbs(tree), rays, R, counts, slots, K, local, sums, tail + S_TOTAL, dst, (unsigned long long)tree->hits_cap, lo, cnt, nopeers, tail + S_XINFO, arrival);
            BVH_CUDA_TRY(cudaEventRecord(ctx->ev_emit[c], st));
            BVH_CUDA_TRY(cudaStreamWaitEvent(ctx->d2h_stream, ctx->ev_emit[c], 0));
            const uint32_t ncopy = cnt + (c + 1 == nsl ? 1u : 0u);
            BVH_CUDA_TRY(cudaMemcpyAsync(h_offsets + lo, tree->d_offsets + lo, sizeof(uint32_t) * ncopy, cudaMemcpyDeviceToHost, ctx->d2h_stream));
        }
        if (ctx->profile) { cudaEventRecord(ctx->ev_e2e[3], st); cudaEventRecord(ctx->ev_e2e[4], ctx->d2h_stream); ctx->have_e2e = true; }
        ctx->launches += 1 + nsl;
    }
    BVH_CUDA_TRY(cudaGetLastError());
    unsigned long long* h = reinterpret_cast<unsigned long long*>(ctx->h_pinned);
    BVH_CUDA_TRY(cudaMemcpyAsync(h, tail, (S_ERR + 1) * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    stamp(3);                                                     // everything enqueued
    BVH_CUDA_TRY(cudaStreamSynchronize(st));
    stamp(4);                                                     // compute stream drained
    const unsigned long long tot = h[S_TOTAL];
    tree->last_total = (size_t)tot; tree->last_visits = h[S_VISITS]; tree->last_nrays = nrays;
    if (total) *total = (size_t)tot;
    if ((uint32_t)h[S_ERR] != 0u) {
        cudaStreamSynchronize(ctx->d2h_stream);
        if (streaming) ctx->stream_ok = 0;                        // whatever starved the kernel: do not stream again on this context
        set_error("traverse: the streamed rays did not arrive within %.1f s (device watchdog); the result is invalid", (double)STREAM_TIMEOUT_NS * 1e-9);
        return BVHGPU_ERR_TIMEOUT;
    }
    int rc = BVHGPU_OK;
    if (tot > 0xFFFFFFFFull) { set_error("traverse: %llu hits overflow the u32 CSR offsets", tot); rc = BVHGPU_ERR_CAPACITY; }
    else if (tot > tree->hits_cap) { set_error("traverse: %llu hits exceed the retained buffer (%zu)", tot, tree->hits_cap); rc = BVHGPU_ERR_CAPACITY; }
    else if (h_hits && tot <= h_cap) {
        if (tot) BVH_CUDA_TRY(cudaMemcpyAsync(h_hits, tree->d_hits, sizeof(uint32_t) * tot, cudaMemcpyDeviceToHost, ctx->d2h_stream));
    }
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->d2h_stream));
    stamp(5);                                                     // results in host memory
    return rc;
}
template int traverse_host_pipelined<float>(Tree<float>*, int, const void*, uint32_t, size_t, uint32_t*, uint32_t*, size_t, size_t*);
template int traverse_host_pipelined<double>(Tree<double>*, int, const void*, uint32_t, size_t, uint32_t*, uint32_t*, size_t, size_t*);

// ---- nearest_to (SURVEY 8f N4): Bvh::nearest_to (src/bvh/bvh_impl.rs:221-238, src/bvh/bvh_node.rs:327-372) and
// FlatBvh::nearest_to (src/flat_bvh.rs:513-562) for a batch of points ---------------------------------------------------
// The reference calls the shape's own PointDistance::distance_squared at the leaves -- user code.  Two device forms:
//   nearest_kernel        : shapes whose distance IS their AABB distance (the reference's UnitBox, testbase.rs:101-105):
//                           the reference's walk replayed exactly -- children ordered by Aabb::min_distance_squared
//                           (aabb_impl.rs:618-629, same operation order), strict `<` pruning, first minimum kept.
//                           The recursion becomes a stackless walk over parent links: on the way back up the two child
//                           distances are recomputed (same bits), so any tree depth works without a stack.
//   nearest_bound_kernel  : any shape inside its AABB: U = min over shapes of the squared distance to the FARTHEST
//                           corner of the shape's AABB bounds the true nearest distance from above; the candidates
//                           {s : lower(AABB_s) <= U} (QUERY_WITHIN) contain the nearest shape, and the caller evaluates its
//                           own distance on that short list.
// Both walks (nearest_walk, nearest_flat) are generic in the dimension and live in queries.cuh, shared with dim4.cu.
// Triangle::distance_squared of the reference's test shape (src/testbase.rs:353-443: closest_point_segment, closest_point_triangle),
// operation for operation -- the PointDistance every benchmark scene of the reference uses.  tri: {a.xyz,-, b.xyz,-, c.xyz,-}.
template <class T> __device__ __forceinline__ T dot3_rn(const T a[3], const T b[3]) { return add_rn(add_rn(mul_rn(a[0], b[0]), mul_rn(a[1], b[1])), mul_rn(a[2], b[2])); }
template <class T> __device__ __forceinline__ void closest_on_segment(const T p[3], const T a[3], const T b[3], T out[3]) {
    T ab[3], ap[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { ab[k] = sub_rn(b[k], a[k]); ap[k] = sub_rn(p[k], a[k]); }
    T s = div_rn(dot3_rn(ab, ap), dot3_rn(ab, ab));
    s = s < T(0) ? T(0) : (s > T(1) ? T(1) : s);
#pragma unroll
    for (int k = 0; k < 3; ++k) out[k] = add_rn(a[k], mul_rn(s, ab[k]));
}
// closest_point_triangle: the point q of triangle tri that the reference's Triangle::distance_squared measures p against.
template <class T> __device__ __forceinline__ void triangle_closest_point(const T p[3], const T* __restrict__ tri, T q[3]) {
    T a[3], b[3], c[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { a[k] = __ldg(tri + k); b[k] = __ldg(tri + 4 + k); c[k] = __ldg(tri + 8 + k); }
    const bool e_ab = a[0] == b[0] && a[1] == b[1] && a[2] == b[2], e_bc = b[0] == c[0] && b[1] == c[1] && b[2] == c[2], e_ac = a[0] == c[0] && a[1] == c[1] && a[2] == c[2];
    bool done = false;
    if (e_ab && e_bc && e_ac) { for (int k = 0; k < 3; ++k) q[k] = a[k]; done = true; }
    else if (e_ab) { closest_on_segment(p, a, c, q); done = true; }
    else if (e_bc) { closest_on_segment(p, a, b, q); done = true; }
    else if (e_ac) { closest_on_segment(p, a, b, q); done = true; }
    if (!done) {
        T ab[3], ac[3], ap[3], bp[3], cp[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) { ab[k] = sub_rn(b[k], a[k]); ac[k] = sub_rn(c[k], a[k]); ap[k] = sub_rn(p[k], a[k]); bp[k] = sub_rn(p[k], b[k]); cp[k] = sub_rn(p[k], c[k]); }
        const T d1 = dot3_rn(ab, ap), d2 = dot3_rn(ac, ap), d3 = dot3_rn(ab, bp), d4 = dot3_rn(ac, bp), d5 = dot3_rn(ab, cp), d6 = dot3_rn(ac, cp);
        const T vc = sub_rn(mul_rn(d1, d4), mul_rn(d3, d2)), vb = sub_rn(mul_rn(d5, d2), mul_rn(d1, d6)), va = sub_rn(mul_rn(d3, d6), mul_rn(d5, d4));
        if (d1 <= T(0) && d2 <= T(0)) { for (int k = 0; k < 3; ++k) q[k] = a[k]; }
        else if (d3 >= T(0) && d4 <= d3) { for (int k = 0; k < 3; ++k) q[k] = b[k]; }
        else if (d6 >= T(0) && d5 <= d6) { for (int k = 0; k < 3; ++k) q[k] = c[k]; }
        else if (vc <= T(0) && d1 >= T(0) && d3 <= T(0)) { const T v = div_rn(d1, sub_rn(d1, d3)); for (int k = 0; k < 3; ++k) q[k] = add_rn(a[k], mul_rn(v, ab[k])); }
        else if (vb <= T(0) && d2 >= T(0) && d6 <= T(0)) { const T v = div_rn(d2, sub_rn(d2, d6)); for (int k = 0; k < 3; ++k) q[k] = add_rn(a[k], mul_rn(v, ac[k])); }
        else if (va <= T(0) && sub_rn(d4, d3) >= T(0) && sub_rn(d5, d6) >= T(0)) {
            const T v = div_rn(sub_rn(d4, d3), add_rn(sub_rn(d4, d3), sub_rn(d5, d6)));
            for (int k = 0; k < 3; ++k) q[k] = add_rn(b[k], mul_rn(v, sub_rn(c[k], b[k])));
        } else {
            const T denom = div_rn(T(1), add_rn(add_rn(va, vb), vc));
            const T v = mul_rn(vb, denom), w = mul_rn(vc, denom);
            for (int k = 0; k < 3; ++k) q[k] = add_rn(add_rn(a[k], mul_rn(v, ab[k])), mul_rn(w, ac[k]));
        }
    }
}
template <class T> __device__ __forceinline__ T triangle_distance_squared(const T p[3], const T* __restrict__ tri) {
    T q[3];
    triangle_closest_point(p, tri, q);
    T d[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) d[k] = sub_rn(p[k], q[k]);
    return dot3_rn(d, d);
}

template <class T, bool FLAT>
__global__ void __launch_bounds__(128) nearest_kernel(const typename Traits<T>::Node* __restrict__ nodes, const typename Traits<T>::Flat* __restrict__ flat,
                                                      uint32_t n_flat, const typename Traits<T>::DAabb* __restrict__ aabb,
                                                      const T* __restrict__ points, uint32_t nq, uint32_t* __restrict__ out_shape, T* __restrict__ out_dist,
                                                      const T* __restrict__ tris) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    T p[3];
    for (int k = 0; k < 3; ++k) p[k] = points[3 * (size_t)i + k];
    uint32_t best = BVH_INVALID;
    T best_d = T(0);
    auto leaf = [&](uint32_t shape) -> T {                  // tris != nullptr: the triangle's own distance (Triangle::distance_squared)
        if (tris) return triangle_distance_squared(p, tris + 12 * (size_t)shape);
        T mn[3], mx[3];
        load_aabb(aabb + shape, mn, mx);
        return aabb_min_d2<3>(p, mn, mx);
    };
    if (!FLAT) nearest_walk<3, T, true>(nodes, p, best, best_d, leaf);
    else       nearest_flat<3, T>(flat, n_flat, p, best, best_d, leaf);
    out_shape[i] = best;
    out_dist[i] = sqrt_rn(best_d);                          // bvh_impl.rs:237
}
template <class T>
__global__ void __launch_bounds__(128) nearest_bound_kernel(const typename Traits<T>::Node* __restrict__ nodes, const typename Traits<T>::DAabb* __restrict__ aabb,
                                                            const T* __restrict__ points, uint32_t nq, T* __restrict__ records) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    T p[3];
    for (int k = 0; k < 3; ++k) p[k] = points[3 * (size_t)i + k];
    uint32_t best;
    T u, g[3];
    root_magnitude<3>(nodes, p, g);
    nearest_walk<3, T, false>(nodes, p, best, u, [&](uint32_t shape) { T mn[3], mx[3]; load_aabb(aabb + shape, mn, mx); return box_upper_d2<3>(p, mn, mx, g); });
    u = mul_rn(u, add_rn(T(1), mul_rn(T(16), Traits<T>::eps())));      // the bound itself is a rounded sum: keep it an upper bound
    for (int k = 0; k < 3; ++k) records[4 * (size_t)i + k] = p[k];
    records[4 * (size_t)i + 3] = u;
}

template <class T>
int nearest_device(Tree<T>* tree, int mode, const T* d_points, size_t nq, uint32_t* d_shape, T* d_dist, int use_triangles) {
    bvhgpu_ctx* ctx = tree->ctx;
    if (use_triangles && !tree->d_tris && tree->n) { set_error("nearest: triangle distances need bvhgpu_tree_set_triangles_* first"); return BVHGPU_ERR_INVALID; }
    const T* tris = use_triangles ? reinterpret_cast<const T*>(tree->d_tris) : nullptr;
    cudaStream_t st = ctx->stream;
    if (nq > 0x7FFFFFFFull) { set_error("nearest: too many points"); return BVHGPU_ERR_INVALID; }
    if (mode != BVHGPU_TRAVERSE_BVH && mode != BVHGPU_TRAVERSE_FLAT) { set_error("nearest: bad mode %d", mode); return BVHGPU_ERR_INVALID; }
    if (nq == 0) return BVHGPU_OK;
    BVH_TRY(resolve_status(tree));
    if (tree->n == 0) {                                     // empty tree: None (bvh_impl.rs:229-231)
        BVH_CUDA_TRY(cudaMemsetAsync(d_shape, 0xFF, sizeof(uint32_t) * nq, st));
        BVH_CUDA_TRY(cudaMemsetAsync(d_dist, 0, sizeof(T) * nq, st));
        return BVHGPU_OK;
    }
    const unsigned grid = (unsigned)((nq + 127) / 128);
    if (mode == BVHGPU_TRAVERSE_FLAT) {
        if (!tree->have_flat) BVH_TRY(build_flat(tree));
        nearest_kernel<T, true><<<grid, 128, 0, st>>>(tree->d_nodes, tree->d_flat, (uint32_t)tree->n_flat, tree->d_aabb, d_points, (uint32_t)nq, d_shape, d_dist, tris);
    } else {
        nearest_kernel<T, false><<<grid, 128, 0, st>>>(tree->d_nodes, nullptr, 0u, tree->d_aabb, d_points, (uint32_t)nq, d_shape, d_dist, tris);
    }
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}
template <class T> int nearest_bound(Tree<T>* tree, const T* d_points, uint32_t n, T* d_records) {
    bvhgpu_ctx* ctx = tree->ctx;
    nearest_bound_kernel<T><<<(n + 127) / 128, 128, 0, ctx->stream>>>(tree->d_nodes, tree->d_aabb, d_points, n, d_records);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}
template int nearest_device<float>(Tree<float>*, int, const float*, size_t, uint32_t*, float*, int);
template int nearest_device<double>(Tree<double>*, int, const double*, size_t, uint32_t*, double*, int);

// ---- k nearest shapes: knn_walk<3, T, K> (queries.cuh) over the node array, keys from the shapes' own boxes (d_aabb); one thread per
// point.  A 2-D tree runs here on points lifted to z = 0 (dim2.cu). ----
template <class T, int K>
__global__ void __launch_bounds__(128) knn_kernel(const typename Traits<T>::Node* __restrict__ nodes, uint32_t n_shapes,
                                                  const typename Traits<T>::DAabb* __restrict__ aabb, const T* __restrict__ points,
                                                  const T* __restrict__ max_dist, uint32_t nq, uint32_t k, uint32_t* __restrict__ out_shape,
                                                  T* __restrict__ out_dist) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    T p[3];
    for (int c = 0; c < 3; ++c) p[c] = points[3 * (size_t)i + c];
    auto leaf = [&](uint32_t shape) { T mn[3], mx[3]; load_aabb(aabb + shape, mn, mx); return aabb_min_d2<3>(p, mn, mx); };
    knn_point<3, T, K>(nodes, n_shapes, p, max_dist != nullptr, max_dist ? max_dist[i] : T(0), k, out_shape + (size_t)i * k,
                       out_dist + (size_t)i * k, leaf);
}
template <class T>
int knn_device(Tree<T>* tree, const T* d_points, size_t nq, uint32_t k, const T* d_max_dist, uint32_t* d_shape, T* d_dist) {
    if (nq > 0x7FFFFFFFull) { set_error("knn: n = %zu exceeds 2^31-1", nq); return BVHGPU_ERR_INVALID; }
    if (k < 1 || k > BVHGPU_KNN_MAX_K) { set_error("knn: k = %u outside 1 .. %d", k, BVHGPU_KNN_MAX_K); return BVHGPU_ERR_INVALID; }
    BVH_TRY(resolve_status(tree));
    if (nq == 0) return BVHGPU_OK;
    bvhgpu_ctx* ctx = tree->ctx;
    const unsigned grid = (unsigned)((nq + 127) / 128);
    knn_bucket(k, [&](auto kb) {
        knn_kernel<T, decltype(kb)::value><<<grid, 128, 0, ctx->stream>>>(tree->d_nodes, tree->n, tree->d_aabb, d_points, d_max_dist, (uint32_t)nq, k, d_shape, d_dist);
    });
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}
template int knn_device<float>(Tree<float>*, const float*, size_t, uint32_t, const float*, uint32_t*, float*);
template int knn_device<double>(Tree<double>*, const double*, size_t, uint32_t, const double*, uint32_t*, double*);

// ---- k nearest triangles: the same walk with Triangle::distance_squared (triangle_distance_squared, bit for bit the key of
// nearest_kernel's triangle mode) at the leaves.  A NaN key fails knn_walk's `key <= r2` and never enters the list.  The closest points
// are recomputed for the k final slots after the walk, in a loop of their own as the square roots are: the list carries no 3 K extra
// values, and the recomputation performs the same operations on the same inputs, so q is the point the key was measured against. ----
template <class T, int K>
__global__ void __launch_bounds__(128) knn_tri_kernel(const typename Traits<T>::Node* __restrict__ nodes, uint32_t n_shapes,
                                                      const T* __restrict__ tris, const T* __restrict__ points, const T* __restrict__ max_dist,
                                                      uint32_t nq, uint32_t k, uint32_t* __restrict__ out_shape, T* __restrict__ out_dist,
                                                      T* __restrict__ out_closest) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    T p[3];
    for (int c = 0; c < 3; ++c) p[c] = points[3 * (size_t)i + c];
    auto leaf = [&](uint32_t shape) { return triangle_distance_squared(p, tris + 12 * (size_t)shape); };
    knn_point<3, T, K>(nodes, n_shapes, p, max_dist != nullptr, max_dist ? max_dist[i] : T(0), k, out_shape + (size_t)i * k,
                       out_dist + (size_t)i * k, leaf);
    if (!out_closest) return;
#pragma unroll 1
    for (uint32_t j = 0; j < k; ++j) {
        const uint32_t s = out_shape[(size_t)i * k + j];
        T q[3] = {quiet_nan<T>(), quiet_nan<T>(), quiet_nan<T>()};
        if (s != BVH_INVALID) triangle_closest_point(p, tris + 12 * (size_t)s, q);
        T* o = out_closest + 3 * ((size_t)i * k + j);
        for (int c = 0; c < 3; ++c) o[c] = q[c];
    }
}
template <class T>
int knn_tri_device(Tree<T>* tree, const T* d_points, size_t nq, uint32_t k, const T* d_max_dist, uint32_t* d_shape, T* d_dist, T* d_closest) {
    if (nq > 0x7FFFFFFFull) { set_error("knn_triangles: n = %zu exceeds 2^31-1", nq); return BVHGPU_ERR_INVALID; }
    if (k < 1 || k > BVHGPU_KNN_MAX_K) { set_error("knn_triangles: k = %u outside 1 .. %d", k, BVHGPU_KNN_MAX_K); return BVHGPU_ERR_INVALID; }
    BVH_TRY(resolve_status(tree));
    if (!tree->d_tris && tree->n) { set_error("knn_triangles: triangle distances need bvhgpu_tree_set_triangles_* first"); return BVHGPU_ERR_INVALID; }
    if (nq == 0) return BVHGPU_OK;
    bvhgpu_ctx* ctx = tree->ctx;
    const unsigned grid = (unsigned)((nq + 127) / 128);
    const T* tris = reinterpret_cast<const T*>(tree->d_tris);
    knn_bucket(k, [&](auto kb) {
        knn_tri_kernel<T, decltype(kb)::value><<<grid, 128, 0, ctx->stream>>>(tree->d_nodes, tree->n, tris, d_points, d_max_dist, (uint32_t)nq, k,
                                                                            d_shape, d_dist, d_closest);
    });
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}
template int knn_tri_device<float>(Tree<float>*, const float*, size_t, uint32_t, const float*, uint32_t*, float*, float*);
template int knn_tri_device<double>(Tree<double>*, const double*, size_t, uint32_t, const double*, uint32_t*, double*, double*);

// ---- the CSR walks of csr.cuh (queries, nearest_candidates, ordered traversal, overlap, overlap between two trees) over Tree<T> ----
BVH_INSTANTIATE_CSR(Tree<float>, float)
BVH_INSTANTIATE_CSR(Tree<double>, double)

// ---- Ray::new for a batch (src/ray/ray_impl.rs:70-80) -------------------------------------------------
template <class T> __device__ __forceinline__ T sqrt_rn(T x);
template <> __device__ __forceinline__ float sqrt_rn(float x) { return __fsqrt_rn(x); }
template <> __device__ __forceinline__ double sqrt_rn(double x) { return __dsqrt_rn(x); }

template <class T>
__global__ void __launch_bounds__(256) rays_new_kernel(const T* __restrict__ origins, const T* __restrict__ dirs, size_t n,
                                                       typename Traits<T>::Ray* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const T dx = dirs[3 * i], dy = dirs[3 * i + 1], dz = dirs[3 * i + 2];
    const T nrm = sqrt_rn(add_rn(add_rn(mul_rn(dx, dx), mul_rn(dy, dy)), mul_rn(dz, dz)));   // [3p] nalgebra normalize
    typename Traits<T>::Ray r;
    const T d[3] = {div_rn(dx, nrm), div_rn(dy, nrm), div_rn(dz, nrm)};
#pragma unroll
    for (int k = 0; k < 3; ++k) { r.origin[k] = origins[3 * i + k]; r.direction[k] = d[k]; r.inv_direction[k] = div_rn(T(1), d[k]); }
    out[i] = r;
}

template <class T>
int rays_new_device(bvhgpu_ctx* ctx, const T* d_origins, const T* d_dirs, size_t n, typename Traits<T>::Ray* d_rays) {
    if (n == 0) return BVHGPU_OK;
    rays_new_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(d_origins, d_dirs, n, d_rays);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}

template int traverse_device<float>(Tree<float>*, int, const void*, uint32_t, size_t, uint32_t*, uint32_t*, size_t, size_t*, const bvhgpu_shard*);
template int traverse_device<double>(Tree<double>*, int, const void*, uint32_t, size_t, uint32_t*, uint32_t*, size_t, size_t*, const bvhgpu_shard*);
template int rays_new_device<float>(bvhgpu_ctx*, const float*, const float*, size_t, bvh_ray3f*);
template int rays_new_device<double>(bvhgpu_ctx*, const double*, const double*, size_t, bvh_ray3d*);

}  // namespace bvhb200
