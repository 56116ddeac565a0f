// bvh_b200/csrc/common.cuh -- shared device/host helpers for libbvh_b200.so (sm_90a only).
//
// Numerics contract (DESIGN.md "bit parity"): every arithmetic step of the reference's build
// and slab test is reproduced in T with round-to-nearest and WITHOUT fused multiply-add.  The
// library is compiled with -fmad=false and the parity-critical expressions additionally use the
// explicit *_rn intrinsics, so a stray compiler flag cannot contract them.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include "../../include/bvh_b200.h"

#define BVH_INVALID 0xFFFFFFFFu

namespace bvhb200 {

// ------------------------------------------------------------------------------------------
// Per-precision traits: PODs of the C ABI, device AABB layout, order-preserving integer keys.
// ------------------------------------------------------------------------------------------
template <class T> struct Traits;

// Device-resident shape AABB.  f32: padded to one 32-byte sector so that a random gather costs
// exactly one sector and two LDG.128 (the 24-byte ABI layout straddles sectors half of the time).
struct __align__(16) DAabbF { float min[3]; uint32_t pad0; float max[3]; uint32_t pad1; };  // 32 B
// f64: 48 B at 48-B stride always touches exactly two sectors; no padding needed.
struct __align__(16) DAabbD { double min[3]; double max[3]; };                              // 48 B

// Traversal record (device only): the AABB a node has in its parent, the index to jump to when
// the slab test fails (first record after the subtree) and the shape index for leaves.
//   f32: {min.xyz, skip} {max.xyz, shape}  = 32 B = one sector.
struct __align__(16) TNodeF { float min[3]; uint32_t skip; float max[3]; uint32_t shape; };
struct __align__(16) TNodeD { double min[3]; double max[3]; uint32_t skip; uint32_t shape; uint32_t pad[2]; };  // 64 B

template <> struct Traits<float> {
    using Aabb = bvh_aabb3f; using Ray = bvh_ray3f; using Node = bvh_node3f; using Flat = bvh_flat3f;
    using DAabb = DAabbF; using TNode = TNodeF;
    using Key = uint32_t;
    static constexpr Key KEY_POS_INF = 0xFF800000u;   // key(+inf): identity of min
    static constexpr Key KEY_NEG_INF = 0x007FFFFFu;   // key(-inf): identity of max
    __host__ __device__ static inline float eps() { return 1.1920928955078125e-7f; }   // f32::EPSILON
    __host__ __device__ static inline float inf() {
#ifdef __CUDA_ARCH__
        return __int_as_float(0x7f800000);
#else
        return __builtin_inff();
#endif
    }
};
template <> struct Traits<double> {
    using Aabb = bvh_aabb3d; using Ray = bvh_ray3d; using Node = bvh_node3d; using Flat = bvh_flat3d;
    using DAabb = DAabbD; using TNode = TNodeD;
    using Key = unsigned long long;
    static constexpr Key KEY_POS_INF = 0xFFF0000000000000ull;
    static constexpr Key KEY_NEG_INF = 0x000FFFFFFFFFFFFFull;
    __host__ __device__ static inline double eps() { return 2.220446049250313e-16; }     // f64::EPSILON
    __host__ __device__ static inline double inf() {
#ifdef __CUDA_ARCH__
        return __longlong_as_double(0x7ff0000000000000ll);
#else
        return __builtin_inf();
#endif
    }
};

static_assert(sizeof(bvh_node3f) == 64 && sizeof(bvh_node3d) == 112, "node POD size");
static_assert(sizeof(bvh_flat3f) == 36 && sizeof(bvh_flat3d) == 64, "flat POD size");
static_assert(sizeof(TNodeF) == 32 && sizeof(TNodeD) == 64 && sizeof(DAabbF) == 32 && sizeof(DAabbD) == 48, "device layouts");

#ifdef __CUDACC__
// ---- order-preserving float <-> unsigned keys (min/max of keys == min/max of floats, -0 < +0) ----
__device__ __forceinline__ uint32_t f2key(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key2f(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}
__device__ __forceinline__ unsigned long long f2key(double f) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(f);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double key2f(unsigned long long k) {
    return __longlong_as_double((long long)((k >> 63) ? (k & 0x7FFFFFFFFFFFFFFFull) : ~k));
}

// min / max in T.  On non-NaN inputs (NaN shapes are rejected up front) FMNMX / DMNMX agree bit for bit with min / max
// of the order-preserving keys, including -0 < +0 (PTX: min(+0, -0) = -0).
__device__ __forceinline__ float min_t(float a, float b) { return fminf(a, b); }
__device__ __forceinline__ float max_t(float a, float b) { return fmaxf(a, b); }
__device__ __forceinline__ double min_t(double a, double b) { return fmin(a, b); }
__device__ __forceinline__ double max_t(double a, double b) { return fmax(a, b); }

// ---- exact (non-contracted) arithmetic in T ----
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }

// Aabb::center (src/aabb/aabb_impl.rs:501-504): min*0.5 + max*0.5, two multiplies and one add.
template <class T> __device__ __forceinline__ T center1(T mn, T mx) { return add_rn(mul_rn(mn, T(0.5)), mul_rn(mx, T(0.5))); }
// Aabb::surface_area (src/aabb/aabb_impl.rs:459-461, 551-554): 2 * ((sx*sx + sy*sy) + sz*sz).
template <class T> __device__ __forceinline__ T surface_area(const T mn[3], const T mx[3]) {
    const T sx = sub_rn(mx[0], mn[0]), sy = sub_rn(mx[1], mn[1]), sz = sub_rn(mx[2], mn[2]);
    return mul_rn(T(2), add_rn(add_rn(mul_rn(sx, sx), mul_rn(sy, sy)), mul_rn(sz, sz)));
}

// Ray::intersection_slice_for_aabb (src/ray/ray_impl.rs:118-145) over D axes: (entry clamped at 0, exit), false = no intersection.
// Per axis l = (min - o) * inv, r = (max - o) * inv; any NaN rejects.  The axes are folded left to right, in the order of the
// reference's inf / sup over the vector: tmin = max(..max(min(l0, r0), min(l1, r1)).., min(l_{D-1}, r_{D-1})), tmax the
// same with min / max exchanged.  The distance-ordered traversal and the AABB-mode closest hit of every dimension use this one slice.
template <int D, class T>
__device__ __forceinline__ bool slab_slice(const T o[D], const T inv[D], const T mn[D], const T mx[D], T& tmin_out, T& tmax_out) {
    T l[D], r[D];
#pragma unroll
    for (int k = 0; k < D; ++k) { l[k] = mul_rn(sub_rn(mn[k], o[k]), inv[k]); r[k] = mul_rn(sub_rn(mx[k], o[k]), inv[k]); }
    bool nan = (l[0] != l[0]) | (r[0] != r[0]);
#pragma unroll
    for (int k = 1; k < D; ++k) nan = nan | (l[k] != l[k]) | (r[k] != r[k]);
    T tmin = min_t(l[0], r[0]), tmax = max_t(l[0], r[0]);
#pragma unroll
    for (int k = 1; k < D; ++k) tmin = max_t(tmin, min_t(l[k], r[k]));
#pragma unroll
    for (int k = 1; k < D; ++k) tmax = min_t(tmax, max_t(l[k], r[k]));
    tmin_out = tmin > T(0) ? tmin : T(0);                       // fast_max(inf.max(), 0)
    tmax_out = tmax;
    return !nan && !(tmin_out > tmax);                          // None iff tmin > tmax or NaN
}

// ---- coherent (L2) loads/stores for data that other SMs produce during the same kernel ----
template <class V> __device__ __forceinline__ V ld_cg(const V* p) { return __ldcg(p); }
template <class V> __device__ __forceinline__ void st_cg(V* p, V v) { __stcg(p, v); }
__device__ __forceinline__ uint32_t ld_acquire(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(uint32_t* p, uint32_t v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_relaxed(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long global_timer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }
__device__ __forceinline__ uint32_t lanemask_lt() {
    uint32_t m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}

// ---- shape AABB loads (immutable while kernels run: read-only path) ----
__device__ __forceinline__ void load_aabb(const DAabbF* p, float mn[3], float mx[3]) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(p));
    const float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
    mn[0] = a.x; mn[1] = a.y; mn[2] = a.z; mx[0] = b.x; mx[1] = b.y; mx[2] = b.z;
}
__device__ __forceinline__ void load_aabb(const DAabbD* p, double mn[3], double mx[3]) {
    const double2 a = __ldg(reinterpret_cast<const double2*>(p));
    const double2 b = __ldg(reinterpret_cast<const double2*>(p) + 1);
    const double2 c = __ldg(reinterpret_cast<const double2*>(p) + 2);
    mn[0] = a.x; mn[1] = a.y; mn[2] = b.x; mx[0] = b.y; mx[1] = c.x; mx[2] = c.y;
}

// warp-wide min / max of keys (u32: one REDUX instruction; u64: shuffles)
__device__ __forceinline__ uint32_t warp_min_key(uint32_t k) { return __reduce_min_sync(0xffffffffu, k); }
__device__ __forceinline__ uint32_t warp_max_key(uint32_t k) { return __reduce_max_sync(0xffffffffu, k); }
// u64: two REDUX passes -- the high words, then the low words of the lanes that hold the winning high word
__device__ __forceinline__ unsigned long long warp_min_key(unsigned long long k) {
    const uint32_t hi = (uint32_t)(k >> 32);
    const uint32_t mh = __reduce_min_sync(0xffffffffu, hi);
    const uint32_t ml = __reduce_min_sync(0xffffffffu, hi == mh ? (uint32_t)k : 0xFFFFFFFFu);
    return ((unsigned long long)mh << 32) | ml;
}
__device__ __forceinline__ unsigned long long warp_max_key(unsigned long long k) {
    const uint32_t hi = (uint32_t)(k >> 32);
    const uint32_t mh = __reduce_max_sync(0xffffffffu, hi);
    const uint32_t ml = __reduce_max_sync(0xffffffffu, hi == mh ? (uint32_t)k : 0u);
    return ((unsigned long long)mh << 32) | ml;
}
#endif  // __CUDACC__

}  // namespace bvhb200
