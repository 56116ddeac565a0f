// bvh_b200/csrc/csr.cuh -- the two-pass CSR walk that every batched walk except the 3-D ray traversal produces its hit lists with:
// the traversal records of D = 3 and D = 4 and their fetch, the record walk generic in D, the count / fill kernel, the ordered
// traversal's kernel, the self-overlap and two-tree overlap kernels, the host driver of count -> scan -> fill, and the device
// drivers of the CSR families (queries, 4-D rays, nearest_candidates, ordered traversal, overlap, overlap between two trees), written
// once over the tree type and instantiated in traverse.cu (Tree<T>: D = 3, and D = 2 through the z = 0 lift) and dim4.cu (Tree4<T>).
// The triangle pairs (3-D only) reuse the overlap walk with a leaf policy and are instantiated in tripairs.cu; the point-in-polygon
// walk of 2-D trees (segments.cu) reuses its record loop, overlap_records.
// The 3-D ray kernels of traverse.cu use the same fetch.
//
// CSR: offsets[n + 1] (u32, saturated to 0xFFFFFFFF) and the hit list hits[total]; the fill pass stores hits[0 .. cap) only, so a
// short `cap` leaves a prefix of the full list.
#pragma once
#include "internal.h"
#include "queries.cuh"
#include <algorithm>

namespace bvhb200 {

// record, shape-box and ray types of the walk in D (3: TNodeF / TNodeD, the padded device boxes and bvh_ray3*; 4: TRec4F / TRec4D,
// the ABI boxes and bvh_ray4*)
template <int D, class T> struct CsrRecords;
template <class T> struct CsrRecords<3, T> { using Rec = typename Traits<T>::TNode; using Box = typename Traits<T>::DAabb; using Ray = typename Traits<T>::Ray; };
template <> struct CsrRecords<4, float> { using Rec = TRec4F; using Box = bvh_aabb4f; using Ray = bvh_ray4f; };
template <> struct CsrRecords<4, double> { using Rec = TRec4D; using Box = bvh_aabb4d; using Ray = bvh_ray4d; };

#ifdef __CUDACC__
// ---- record fetch: 128-bit non-coherent loads (LDG.E.128, the widest global load sm_90a has) ------------
// A divergent warp pays one L1 tag lookup ("wavefront") per distinct line per load instruction, and the ray
// kernels are L1-wavefront bound, so a record is fetched with as few load instructions as the ISA allows:
// two for a 32-byte f32 record, four for a 64-byte f64 record.
__device__ __forceinline__ void fetch(const TNodeF* __restrict__ p, float mn[3], float mx[3], uint32_t& skip, uint32_t& shape) {
    float sk, sh;
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(mn[0]), "=f"(mn[1]), "=f"(mn[2]), "=f"(sk) : "l"(p));
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(mx[0]), "=f"(mx[1]), "=f"(mx[2]), "=f"(sh) : "l"(reinterpret_cast<const char*>(p) + 16));
    skip = __float_as_uint(sk);
    shape = __float_as_uint(sh);
}
__device__ __forceinline__ void fetch(const TNodeD* __restrict__ p, double mn[3], double mx[3], uint32_t& skip, uint32_t& shape) {
    double links, pad;                         // {skip, shape} travel as the bits of the 7th double of the 64-byte record
    const char* c = reinterpret_cast<const char*>(p);
    asm volatile("ld.global.nc.v2.f64 {%0,%1}, [%2];" : "=d"(mn[0]), "=d"(mn[1]) : "l"(c));
    asm volatile("ld.global.nc.v2.f64 {%0,%1}, [%2];" : "=d"(mn[2]), "=d"(mx[0]) : "l"(c + 16));
    asm volatile("ld.global.nc.v2.f64 {%0,%1}, [%2];" : "=d"(mx[1]), "=d"(mx[2]) : "l"(c + 32));
    asm volatile("ld.global.nc.v2.f64 {%0,%1}, [%2];" : "=d"(links), "=d"(pad) : "l"(c + 48));
    const unsigned long long b = (unsigned long long)__double_as_longlong(links);
    skip = (uint32_t)b; shape = (uint32_t)(b >> 32);
}
__device__ __forceinline__ void fetch(const TRec4F* p, float mn[4], float mx[4], uint32_t& skip, uint32_t& shape) {
    uint32_t a, b, c, d;
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(mn[0]), "=f"(mn[1]), "=f"(mn[2]), "=f"(mn[3]) : "l"(p));
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(mx[0]), "=f"(mx[1]), "=f"(mx[2]), "=f"(mx[3]) : "l"(reinterpret_cast<const char*>(p) + 16));
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "l"(reinterpret_cast<const char*>(p) + 32));
    skip = a; shape = b;
}
__device__ __forceinline__ void fetch(const TRec4D* p, double mn[4], double mx[4], uint32_t& skip, uint32_t& shape) {
    const char* c = reinterpret_cast<const char*>(p);
    uint32_t a, b, x, y;
    asm volatile("ld.global.nc.v2.f64 {%0,%1}, [%2];" : "=d"(mn[0]), "=d"(mn[1]) : "l"(c));
    asm volatile("ld.global.nc.v2.f64 {%0,%1}, [%2];" : "=d"(mn[2]), "=d"(mn[3]) : "l"(c + 16));
    asm volatile("ld.global.nc.v2.f64 {%0,%1}, [%2];" : "=d"(mx[0]), "=d"(mx[1]) : "l"(c + 32));
    asm volatile("ld.global.nc.v2.f64 {%0,%1}, [%2];" : "=d"(mx[2]), "=d"(mx[3]) : "l"(c + 48));
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(a), "=r"(b), "=r"(x), "=r"(y) : "l"(c + 64));
    skip = a; shape = b;
}

// ---- shape boxes: the padded 3-D device layout and the 4-D ABI layout (already whole sectors) ----
__device__ __forceinline__ void load4(const bvh_aabb4f* p, float mn[4], float mx[4]) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
    mn[0] = a.x; mn[1] = a.y; mn[2] = a.z; mn[3] = a.w; mx[0] = b.x; mx[1] = b.y; mx[2] = b.z; mx[3] = b.w;
}
__device__ __forceinline__ void load4(const bvh_aabb4d* p, double mn[4], double mx[4]) {
    const double2* q = reinterpret_cast<const double2*>(p);
    const double2 a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + 2), d = __ldg(q + 3);
    mn[0] = a.x; mn[1] = a.y; mn[2] = b.x; mn[3] = b.y; mx[0] = c.x; mx[1] = c.y; mx[2] = d.x; mx[3] = d.y;
}
__device__ __forceinline__ void load_box(const DAabbF* p, float mn[3], float mx[3]) { load_aabb(p, mn, mx); }
__device__ __forceinline__ void load_box(const DAabbD* p, double mn[3], double mx[3]) { load_aabb(p, mn, mx); }
__device__ __forceinline__ void load_box(const bvh_aabb4f* p, float mn[4], float mx[4]) { load4(p, mn, mx); }
__device__ __forceinline__ void load_box(const bvh_aabb4d* p, double mn[4], double mx[4]) { load4(p, mn, mx); }

// ---- rays of the C ABI: origin and inv_direction (the direction is not needed by a slab test) ----
template <class T> __device__ __forceinline__ void load_ray3(const T* p, T o[3], T inv[3]) {
#pragma unroll
    for (int k = 0; k < 3; ++k) { o[k] = __ldg(p + k); inv[k] = __ldg(p + 6 + k); }
}
__device__ __forceinline__ void load_ray_full(const bvh_ray3f* p, float o[3], float inv[3]) { load_ray3(reinterpret_cast<const float*>(p), o, inv); }
__device__ __forceinline__ void load_ray_full(const bvh_ray3d* p, double o[3], double inv[3]) { load_ray3(reinterpret_cast<const double*>(p), o, inv); }
__device__ __forceinline__ void load_ray_full(const bvh_ray4f* p, float o[4], float inv[4]) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 2);
    o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; inv[0] = b.x; inv[1] = b.y; inv[2] = b.z; inv[3] = b.w;
}
__device__ __forceinline__ void load_ray_full(const bvh_ray4d* p, double o[4], double inv[4]) {
    const double2* q = reinterpret_cast<const double2*>(p);
    const double2 a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + 4), d = __ldg(q + 5);
    o[0] = a.x; o[1] = a.y; o[2] = b.x; o[3] = b.y; inv[0] = c.x; inv[1] = c.y; inv[2] = d.x; inv[3] = d.y;
}

// ---- the walk: stackless over the preorder records, hit -> next record, miss -> skip, so hits come out in the reference's
// left-first DFS order.  `probe.hit(mn, mx)` is the predicate; `emit(shape)` is called for every reported shape. ----
template <int D, class T, bool FLAT, class Rec, class Box, class Probe, class Emit>
__device__ __forceinline__ void walk_records(const Rec* __restrict__ trec, uint32_t n_rec, const Box* __restrict__ aabb, const Probe& probe, Emit emit) {
    uint32_t i = 0;
    while (i < n_rec) {
        T mn[D], mx[D];
        uint32_t skip, shape;
        fetch(trec + i, mn, mx, skip, shape);
        if (probe.hit(mn, mx)) {
            if (shape != BVH_INVALID) {
                bool report = true;
                if (FLAT) {                                    // flat_bvh.rs:412-416: a reached leaf re-tests the shape's AABB
                    T smn[D], smx[D];
                    load_box(aabb + shape, smn, smx);
                    report = probe.hit(smn, smx);
                }
                if (report) emit(shape);
            }
            ++i;
        } else {
            i = skip;
        }
    }
}

// Count pass (FILL = false) and fill pass (FILL = true) over n items, one per thread.  A probe has load(src, r), which reads item r
// of the batch, and hit(mn, mx).  The fill pass writes offsets[0 .. n] from the scan (saturated to 0xFFFFFFFF) and drops the hits
// at positions >= cap.
template <int D, class T, bool FLAT, bool FILL, class Probe>
__global__ void __launch_bounds__(256) csr_walk_kernel(const typename CsrRecords<D, T>::Rec* __restrict__ trec, uint32_t n_rec,
                                                       const typename CsrRecords<D, T>::Box* __restrict__ aabb,
                                                       const void* __restrict__ src, uint32_t n, uint32_t* __restrict__ counts,
                                                       const uint32_t* __restrict__ local, const unsigned long long* __restrict__ blocksum,
                                                       const unsigned long long* __restrict__ total, uint32_t* __restrict__ offsets, uint32_t* __restrict__ hits,
                                                       unsigned long long cap) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (FILL && r == 0) { const unsigned long long t = *total; offsets[n] = t > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)t; }
    if (r >= n) return;
    Probe probe;
    probe.load(src, r);
    if (!FILL) {
        uint32_t cnt = 0;
        walk_records<D, T, FLAT>(trec, n_rec, aabb, probe, [&](uint32_t) { ++cnt; });
        counts[r] = cnt;
    } else {
        unsigned long long w = blocksum[r / CSR_SCAN_TILE] + local[r];
        offsets[r] = w > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)w;
        if (hits) walk_records<D, T, FLAT>(trec, n_rec, aabb, probe, [&](uint32_t shape) { if (w < cap) hits[w] = shape; ++w; });
    }
}

// ---- ordered traversal (SURVEY 8f N3): hits of every ray sorted by AABB entry distance (nearest first) or by exit
// distance (farthest first), with the distance.  The reference's DistanceTraverseIterator (src/bvh/distance_traverse.rs) is
// a best-effort heap walk ("not necessarily perfectly sorted", ties in heap order); this returns the same SET, perfectly
// sorted, ties in the reference's DFS order.  Distances are slab_slice (Ray::intersection_slice_for_aabb) of the record's box:
// the child box the parent stores for the leaf, or the shape's own box at a root leaf.  D = 3 and D = 4 over their records;
// D = 2 runs the D = 3 instance on the tree embedded in z = 0 (dim2.cu).  Count pass (FILL = false) and fill pass as
// csr_walk_kernel, then a stable insertion sort of the ray's list (lists are short).
template <int D, class T, bool FILL>
__global__ void __launch_bounds__(256) ordered_kernel(const typename CsrRecords<D, T>::Rec* __restrict__ trec, uint32_t n_rec,
                                                      const typename CsrRecords<D, T>::Ray* __restrict__ rays, uint32_t nrays, int ascending,
                                                      uint32_t* __restrict__ counts, const uint32_t* __restrict__ local,
                                                      const unsigned long long* __restrict__ blocksum, const unsigned long long* __restrict__ total,
                                                      uint32_t* __restrict__ offsets, uint32_t* __restrict__ hits, T* __restrict__ dists, unsigned long long cap) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (FILL && r == 0) { const unsigned long long t = *total; offsets[nrays] = t > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)t; }
    if (r >= nrays) return;
    T o[D], inv[D];
    load_ray_full(rays + r, o, inv);
    unsigned long long base = 0, w = 0;
    if (FILL) { base = blocksum[r / CSR_SCAN_TILE] + local[r]; offsets[r] = base > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)base; w = base; }
    uint32_t cnt = 0, i = 0;
    while (i < n_rec) {
        T mn[D], mx[D], t0, t1;
        uint32_t skip, shape;
        fetch(trec + i, mn, mx, skip, shape);
        if (slab_slice<D, T>(o, inv, mn, mx, t0, t1)) {
            if (shape != BVH_INVALID) {
                if (FILL) { if (w < cap) { hits[w] = shape; dists[w] = ascending ? t0 : t1; } ++w; }
                ++cnt;
            }
            i = i + 1;
        } else i = skip;
    }
    if (!FILL) { counts[r] = cnt; return; }
    // stable insertion sort of this ray's list: ascending entry distance / descending exit distance
    const unsigned long long end = w < cap ? w : cap;
    for (unsigned long long a = base + 1; a < end; ++a) {
        const T d = dists[a];
        const uint32_t h = hits[a];
        unsigned long long b = a;
        while (b > base && (ascending ? dists[b - 1] > d : dists[b - 1] < d)) { dists[b] = dists[b - 1]; hits[b] = hits[b - 1]; --b; }
        dists[b] = d; hits[b] = h;
    }
}

// ---- self-overlap (bvhgpu_overlap_pairs_*): row s lists every shape t with leaf(t) > leaf(s) whose own box intersects s's own box
// (Aabb::intersects_aabb: for every axis !(a.max < b.min || b.max < a.min)), in DFS order.  Record r is node r + 1, so the walk of s
// starts at record leaf(s), the node right after s's leaf in preorder: every node it can reach lies after the leaf, and each pair is
// found once, by whichever leaf comes first.  A record is entered when its box intersects s's box or has min > max on some axis (the
// Aabb::empty() child box of a "no split wins" node); every other record box contains the boxes of the shapes below it, so a miss
// prunes no pair.  Thread k walks the shape of leaf rank k (order[k], neighbouring threads walk neighbouring leaves); its row is
// written at the shape's scanned offset.  Count pass (FILL = false) and fill pass as csr_walk_kernel.
template <int D, class T>
__device__ __forceinline__ bool overlap_enter(const T smn[D], const T smx[D], const T mn[D], const T mx[D]) {
    bool hit = true, empty = false;
#pragma unroll
    for (int k = 0; k < D; ++k) {
        hit = hit && !(smx[k] < mn[k] || mx[k] < smn[k]);
        empty = empty || mn[k] > mx[k];
    }
    return hit || empty;
}
template <int D, class T>
__device__ __forceinline__ bool overlap_boxes(const T smn[D], const T smx[D], const T mn[D], const T mx[D]) {
    bool hit = true;
#pragma unroll
    for (int k = 0; k < D; ++k) hit = hit && !(smx[k] < mn[k] || mx[k] < smn[k]);
    return hit;
}
// The record loop of the overlap walks, from record i to n_rec: a record is entered when overlap_enter(smn, smx, its box) holds, and
// visit(shape) is called for every entered leaf record, in DFS order.  The overlap kernels below and the point-in-polygon walk of
// segments.cu (a point's box [px, +inf] x [py, py]) run it.
template <int D, class T, class Rec, class Visit>
__device__ __forceinline__ void overlap_records(const Rec* __restrict__ trec, uint32_t i, uint32_t n_rec, const T smn[D], const T smx[D], Visit visit) {
    while (i < n_rec) {
        T mn[D], mx[D];
        uint32_t skip, shape;
        fetch(trec + i, mn, mx, skip, shape);
        if (overlap_enter<D, T>(smn, smx, mn, mx)) {
            if (shape != BVH_INVALID) visit(shape);
            ++i;
        } else {
            i = skip;
        }
    }
}
// The leaf policy of the overlap kernels: the boxes decide.  A policy has row(s), false when row s is empty whatever the boxes say,
// and keep(t), which filters a shape whose box passed (TriPairsLeaf, tritri.cuh: the triangle pairs).
struct BoxesDecide {
    __device__ __forceinline__ bool row(uint32_t) const { return true; }
    __device__ __forceinline__ bool keep(uint32_t) const { return true; }
};
// The body of the overlap and triangle-pair kernels.  Self (CROSS = false): rows and records of one tree, own = other = its boxes, the
// walk of s starts at record node_index[s].  Cross (CROSS = true, bvhgpu_overlap_trees_*): thread k takes shape order[k] of tree A (A's
// leaf order), loads its box from `own` (A's boxes), and walks all of B's records from record 0, testing each reached leaf's shape
// against `other` (B's boxes); node_index is unused.  The exactness argument is the same: it only needs B's records.  A reached shape
// whose box passes is reported when leaf.keep(shape) holds.
template <int D, class T, bool FILL, bool CROSS, class Leaf = BoxesDecide>
__device__ __forceinline__ void overlap_walk(const typename CsrRecords<D, T>::Rec* __restrict__ trec, uint32_t n_rec,
                                             const typename CsrRecords<D, T>::Box* __restrict__ own, const typename CsrRecords<D, T>::Box* __restrict__ other,
                                             const uint32_t* __restrict__ node_index, const uint32_t* __restrict__ order, uint32_t n,
                                             uint32_t* __restrict__ counts, const uint32_t* __restrict__ local,
                                             const unsigned long long* __restrict__ blocksum, const unsigned long long* __restrict__ total,
                                             uint32_t* __restrict__ offsets, uint32_t* __restrict__ hits, unsigned long long cap,
                                             Leaf leaf = Leaf()) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (FILL && k == 0) { const unsigned long long t = *total; offsets[n] = t > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)t; }
    if (k >= n) return;
    const uint32_t s = __ldg(order + k);
    T smn[D], smx[D];
    load_box(own + s, smn, smx);
    unsigned long long w = 0;
    if (FILL) {
        w = blocksum[s / CSR_SCAN_TILE] + local[s];
        offsets[s] = w > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)w;
        if (!hits) return;                                        // offsets only
    }
    uint32_t cnt = 0, i = CROSS ? 0u : __ldg(node_index + s);
    if (!leaf.row(s)) i = n_rec;
    overlap_records<D, T>(trec, i, n_rec, smn, smx, [&](uint32_t shape) {
        T tmn[D], tmx[D];
        load_box(other + shape, tmn, tmx);
        if (overlap_boxes<D, T>(smn, smx, tmn, tmx) && leaf.keep(shape)) {
            if (FILL) { if (w < cap) hits[w] = shape; ++w; }
            else ++cnt;
        }
    });
    if (!FILL) counts[s] = cnt;
}
template <int D, class T, bool FILL>
__global__ void __launch_bounds__(256) overlap_kernel(const typename CsrRecords<D, T>::Rec* __restrict__ trec, uint32_t n_rec,
                                                      const typename CsrRecords<D, T>::Box* __restrict__ aabb, const uint32_t* __restrict__ node_index,
                                                      const uint32_t* __restrict__ order, uint32_t n, uint32_t* __restrict__ counts,
                                                      const uint32_t* __restrict__ local, const unsigned long long* __restrict__ blocksum,
                                                      const unsigned long long* __restrict__ total, uint32_t* __restrict__ offsets,
                                                      uint32_t* __restrict__ hits, unsigned long long cap) {
    overlap_walk<D, T, FILL, false>(trec, n_rec, aabb, aabb, node_index, order, n, counts, local, blocksum, total, offsets, hits, cap);
}
// ---- overlap between two trees (bvhgpu_overlap_trees_*): row a of tree A lists every shape b of tree B whose own box intersects a's
// own box, in B's DFS order.  trec / n_rec: B's records; aabb_b: B's boxes; aabb_a, order_a, n_a: A's boxes and shapes in A's leaf
// order, so that neighbouring threads test neighbouring boxes.  Count pass and fill pass as overlap_kernel.
template <int D, class T, bool FILL>
__global__ void __launch_bounds__(256) overlap_trees_kernel(const typename CsrRecords<D, T>::Rec* __restrict__ trec, uint32_t n_rec,
                                                            const typename CsrRecords<D, T>::Box* __restrict__ aabb_b,
                                                            const typename CsrRecords<D, T>::Box* __restrict__ aabb_a,
                                                            const uint32_t* __restrict__ order_a, uint32_t n_a, uint32_t* __restrict__ counts,
                                                            const uint32_t* __restrict__ local, const unsigned long long* __restrict__ blocksum,
                                                            const unsigned long long* __restrict__ total, uint32_t* __restrict__ offsets,
                                                            uint32_t* __restrict__ hits, unsigned long long cap) {
    overlap_walk<D, T, FILL, true>(trec, n_rec, aabb_a, aabb_b, nullptr, order_a, n_a, counts, local, blocksum, total, offsets, hits, cap);
}
// ---- triangle pairs (bvhgpu_triangle_pairs_*, D = 3): the overlap walks with the leaf policy TriPairsLeaf (tritri.cuh, included by the
// translation unit that instantiates them), which keeps a box pair only when the two closed triangles meet.  Self (CROSS = false): the
// rows, records, boxes and triangles of one tree.  Cross: A's boxes, triangles and leaf order against B's records, boxes and triangles.
template <class T> struct TriPairsLeaf;
template <class T, bool FILL, bool CROSS>
__global__ void __launch_bounds__(256) triangle_pairs_kernel(const typename CsrRecords<3, T>::Rec* __restrict__ trec, uint32_t n_rec,
                                                             const typename CsrRecords<3, T>::Box* __restrict__ aabb_own,
                                                             const typename CsrRecords<3, T>::Box* __restrict__ aabb_other,
                                                             const DTri<T>* __restrict__ tris_own, const DTri<T>* __restrict__ tris_other,
                                                             int skip_shared, const uint32_t* __restrict__ node_index,
                                                             const uint32_t* __restrict__ order, uint32_t n, uint32_t* __restrict__ counts,
                                                             const uint32_t* __restrict__ local, const unsigned long long* __restrict__ blocksum,
                                                             const unsigned long long* __restrict__ total, uint32_t* __restrict__ offsets,
                                                             uint32_t* __restrict__ hits, unsigned long long cap) {
    TriPairsLeaf<T> leaf;
    leaf.own = tris_own; leaf.other = tris_other; leaf.skip_shared = skip_shared;
    overlap_walk<3, T, FILL, CROSS, TriPairsLeaf<T>&>(trec, n_rec, aabb_own, aabb_other, node_index, order, n, counts, local, blocksum,
                                                      total, offsets, hits, cap, leaf);
}

// ---- host: count -> scan -> fill ----
// A walk is what the driver launches: walk.count(stream, n, counts) enqueues the count pass, walk.fill(stream, n, local, sums, total,
// offsets, hits, cap) the fill pass.  CsrWalk is the one of csr_walk_kernel, OrderedWalk the one of ordered_kernel.
template <int D, class T, class Probe> struct CsrWalk {
    bool flat;
    const typename CsrRecords<D, T>::Rec* trec;
    uint32_t n_rec;
    const typename CsrRecords<D, T>::Box* aabb;       // the FLAT leaf re-test's shape boxes
    const void* src;                                  // the batch, read by Probe::load
    template <bool FILL> void launch(cudaStream_t st, uint32_t n, uint32_t* counts, const uint32_t* local, const unsigned long long* sums,
                                     const unsigned long long* total, uint32_t* offsets, uint32_t* hits, size_t cap) const {
        const unsigned grid = (n + 255) / 256;
        if (flat) csr_walk_kernel<D, T, true, FILL, Probe><<<grid, 256, 0, st>>>(trec, n_rec, aabb, src, n, counts, local, sums, total, offsets, hits, (unsigned long long)cap);
        else      csr_walk_kernel<D, T, false, FILL, Probe><<<grid, 256, 0, st>>>(trec, n_rec, aabb, src, n, counts, local, sums, total, offsets, hits, (unsigned long long)cap);
    }
    void count(cudaStream_t st, uint32_t n, uint32_t* counts) const { launch<false>(st, n, counts, nullptr, nullptr, nullptr, nullptr, nullptr, 0); }
    void fill(cudaStream_t st, uint32_t n, const uint32_t* local, const unsigned long long* sums, const unsigned long long* total,
              uint32_t* offsets, uint32_t* hits, size_t cap) const { launch<true>(st, n, nullptr, local, sums, total, offsets, hits, cap); }
};
template <int D, class T> struct OrderedWalk {
    const typename CsrRecords<D, T>::Rec* trec;
    uint32_t n_rec;
    const typename CsrRecords<D, T>::Ray* rays;
    int ascending;
    T* dists;                                         // written next to the hits, cap entries
    void count(cudaStream_t st, uint32_t n, uint32_t* counts) const {
        ordered_kernel<D, T, false><<<(n + 255) / 256, 256, 0, st>>>(trec, n_rec, rays, n, ascending, counts, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0);
    }
    void fill(cudaStream_t st, uint32_t n, const uint32_t* local, const unsigned long long* sums, const unsigned long long* total,
              uint32_t* offsets, uint32_t* hits, size_t cap) const {
        ordered_kernel<D, T, true><<<(n + 255) / 256, 256, 0, st>>>(trec, n_rec, rays, n, ascending, nullptr, local, sums, total, offsets, hits, dists, (unsigned long long)cap);
    }
};
// The walk of overlap_kernel over the tree's n shapes (n >= 2).  order: the shapes in leaf order (leaf_order_kernel).
template <int D, class T> struct OverlapWalk {
    const typename CsrRecords<D, T>::Rec* trec;
    uint32_t n_rec;
    const typename CsrRecords<D, T>::Box* aabb;       // the shapes' own boxes (D = 2: z = [0, 0])
    const uint32_t* node_index;
    const uint32_t* order;
    void count(cudaStream_t st, uint32_t n, uint32_t* counts) const {
        overlap_kernel<D, T, false><<<(n + 255) / 256, 256, 0, st>>>(trec, n_rec, aabb, node_index, order, n, counts, nullptr, nullptr, nullptr, nullptr, nullptr, 0);
    }
    void fill(cudaStream_t st, uint32_t n, const uint32_t* local, const unsigned long long* sums, const unsigned long long* total,
              uint32_t* offsets, uint32_t* hits, size_t cap) const {
        overlap_kernel<D, T, true><<<(n + 255) / 256, 256, 0, st>>>(trec, n_rec, aabb, node_index, order, n, nullptr, local, sums, total, offsets, hits, (unsigned long long)cap);
    }
};
// The walk of overlap_trees_kernel over tree A's n_a shapes (n_a >= 1) against tree B's records (n_b >= 1).  order_a: A's shapes in
// A's leaf order (leaf_order_kernel).
template <int D, class T> struct OverlapTreesWalk {
    const typename CsrRecords<D, T>::Rec* trec;       // B's records
    uint32_t n_rec;
    const typename CsrRecords<D, T>::Box* aabb_b;     // B's own boxes (D = 2: z = [0, 0])
    const typename CsrRecords<D, T>::Box* aabb_a;     // A's own boxes (D = 2: z = [0, 0])
    const uint32_t* order_a;
    void count(cudaStream_t st, uint32_t n, uint32_t* counts) const {
        overlap_trees_kernel<D, T, false><<<(n + 255) / 256, 256, 0, st>>>(trec, n_rec, aabb_b, aabb_a, order_a, n, counts, nullptr, nullptr, nullptr, nullptr, nullptr, 0);
    }
    void fill(cudaStream_t st, uint32_t n, const uint32_t* local, const unsigned long long* sums, const unsigned long long* total,
              uint32_t* offsets, uint32_t* hits, size_t cap) const {
        overlap_trees_kernel<D, T, true><<<(n + 255) / 256, 256, 0, st>>>(trec, n_rec, aabb_b, aabb_a, order_a, n, nullptr, local, sums, total, offsets, hits, (unsigned long long)cap);
    }
};
// The walk of triangle_pairs_kernel: self over one tree's n >= 2 shapes (CROSS = false; node_index of that tree) or tree A's n_a >= 1
// shapes against tree B (CROSS = true, n_b >= 1).  order: the row tree's shapes in its leaf order.
template <class T, bool CROSS> struct TrianglePairsWalk {
    const typename CsrRecords<3, T>::Rec* trec;       // the walked tree's records (B's in the cross form)
    uint32_t n_rec;
    const typename CsrRecords<3, T>::Box* aabb_own;   // the row tree's own boxes
    const typename CsrRecords<3, T>::Box* aabb_other; // the walked tree's own boxes
    const DTri<T>* tris_own;
    const DTri<T>* tris_other;
    int skip_shared;
    const uint32_t* node_index;
    const uint32_t* order;
    void count(cudaStream_t st, uint32_t n, uint32_t* counts) const {
        triangle_pairs_kernel<T, false, CROSS><<<(n + 255) / 256, 256, 0, st>>>(trec, n_rec, aabb_own, aabb_other, tris_own, tris_other, skip_shared,
                                                                                 node_index, order, n, counts, nullptr, nullptr, nullptr, nullptr, nullptr, 0);
    }
    void fill(cudaStream_t st, uint32_t n, const uint32_t* local, const unsigned long long* sums, const unsigned long long* total,
              uint32_t* offsets, uint32_t* hits, size_t cap) const {
        triangle_pairs_kernel<T, true, CROSS><<<(n + 255) / 256, 256, 0, st>>>(trec, n_rec, aabb_own, aabb_other, tris_own, tris_other, skip_shared,
                                                                                node_index, order, n, nullptr, local, sums, total, offsets, hits,
                                                                                (unsigned long long)cap);
    }
};

// One CSR over n items (0 < n <= 2^31 - 1) on the context's stream, in two steps so that a caller can read the total between them.
// count_and_scan: the count pass, then the shared scan (scan_local_kernel / scan_blocks_kernel) into local offsets, 64-bit block
// offsets sums[0 .. nblk) and the total sums[nblk].  With read_total it also copies the total into the pinned word CSR_TOTAL_WORD
// and records ctx->ev_total, so that total() waits for that copy only, not for a fill enqueued after it.  The scratch lives as long
// as the object (released stream-ordered, after the fill).
struct CsrPasses {
    bvhgpu_ctx* ctx;
    uint32_t n, nblk;
    Scratch scratch;
    uint32_t *counts = nullptr, *local = nullptr;
    unsigned long long* sums = nullptr;

    CsrPasses(bvhgpu_ctx* c, uint32_t items) : ctx(c), n(items), nblk((items + CSR_SCAN_TILE - 1) / CSR_SCAN_TILE), scratch(c) {}
    unsigned long long* pinned_total() const { return reinterpret_cast<unsigned long long*>(ctx->h_pinned + CSR_TOTAL_WORD); }

    template <class Walk> int count_and_scan(const Walk& walk, bool read_total) {
        cudaStream_t st = ctx->stream;
        BVH_TRY(scratch.get(&counts, n));
        BVH_TRY(scratch.get(&local, n));
        BVH_TRY(scratch.get(&sums, (size_t)nblk + 1));
        BVH_CUDA_TRY(cudaMemsetAsync(sums + nblk, 0, sizeof(unsigned long long), st));
        walk.count(st, n, counts);
        scan_local_kernel<<<nblk, CSR_SCAN_THREADS, 0, st>>>(counts, n, local, sums, nullptr);
        scan_blocks_kernel<<<1, 1024, 0, st>>>(sums, nblk, sums + nblk);
        ctx->launches += 3;
        BVH_CUDA_TRY(cudaGetLastError());
        if (read_total) {
            BVH_CUDA_TRY(cudaMemcpyAsync(pinned_total(), sums + nblk, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
            BVH_CUDA_TRY(cudaEventRecord(ctx->ev_total, st));
        }
        return BVHGPU_OK;
    }
    template <class Walk> int fill(const Walk& walk, uint32_t* offsets, uint32_t* hits, size_t cap) {
        walk.fill(ctx->stream, n, local, sums, sums + nblk, offsets, hits, cap);
        ctx->launches++;
        BVH_CUDA_TRY(cudaGetLastError());
        return BVHGPU_OK;
    }
    // Waits for the total (count_and_scan with read_total) and stores it in *out.  BVHGPU_ERR_CAPACITY when it overflows the u32
    // offsets, or when hits != nullptr and it exceeds cap.  `what` names the entry point in the message.
    int total(const char* what, const uint32_t* hits, size_t cap, size_t* out) const {
        BVH_CUDA_TRY(cudaEventSynchronize(ctx->ev_total));
        const unsigned long long t = *pinned_total();
        *out = (size_t)t;
        if (t > 0xFFFFFFFFull) { set_error("%s: %llu hits overflow the u32 CSR offsets", what, t); return BVHGPU_ERR_CAPACITY; }
        if (hits && t > cap) { set_error("%s: %llu hits do not fit capacity %zu", what, t, cap); return BVHGPU_ERR_CAPACITY; }
        return BVHGPU_OK;
    }
};

// The whole CSR of a device-pointer call.  Without `total` nothing synchronises.  With it, the call waits for the total only (the
// fill pass may still run when it returns) and returns CsrPasses::total's verdict.
template <class Walk> int csr_two_pass(bvhgpu_ctx* ctx, const Walk& walk, uint32_t n, const char* what, uint32_t* offsets, uint32_t* hits,
                                       size_t cap, size_t* total) {
    CsrPasses passes(ctx, n);
    BVH_TRY(passes.count_and_scan(walk, total != nullptr));
    BVH_TRY(passes.fill(walk, offsets, hits, cap));
    return total ? passes.total(what, hits, cap, total) : BVHGPU_OK;
}

// ---- the device drivers of the CSR families (declared in internal.h) ----
// Where a tree type differs they call an overload of internal.h: ensure_records, walk_aabbs, nearest_bound, keep_total.

// The status step: a call with nothing to walk does not wait for a build that may still run on the device.
template <class TreeT> int csr_status(TreeT* tree, size_t n) {
    return n || tree->failed_status != BVHGPU_OK ? resolve_status(tree) : BVHGPU_OK;
}
// The CSR of a call with nothing to walk: all-zero offsets; the host form does no device work.
template <class TreeT> int csr_zero(TreeT* tree, size_t n, const CsrOut& out) {
    if (out.host) {
        std::fill(out.offsets, out.offsets + n + 1, 0u);
        keep_total(tree, 0);
    } else {
        BVH_CUDA_TRY(cudaMemsetAsync(out.offsets, 0, sizeof(uint32_t) * (n + 1), tree->ctx->stream));
    }
    if (out.total) *out.total = 0;
    return BVHGPU_OK;
}
// The CSR of a walk over n > 0 items.  Device form: csr_two_pass.  Host form: count and scan once, fill into the tree's retained
// buffers, read the total; when it did not fit and fits the u32 offsets, grow the hit buffer to it and fill again from the same
// scan, if the list is wanted: the caller's cap holds it, or a 3-D tree keeps it for bvhgpu_traverse_fetch_*.  (2-D and 4-D have no
// fetch: a short cap needs the offsets only, which the first fill completed.)  Then copy_retained.
template <class TreeT, class Walk> int csr_run(TreeT* tree, const Walk& walk, size_t n, const CsrOut& out, const char* what) {
    if (!out.host) return csr_two_pass(tree->ctx, walk, (uint32_t)n, what, out.offsets, out.hits, out.cap, out.total);
    BVH_TRY(ensure_result_buffers(tree, n, std::max<size_t>(std::max<size_t>(tree->hits_cap, out.per_item * n), 1024)));
    CsrPasses passes(tree->ctx, (uint32_t)n);
    BVH_TRY(passes.count_and_scan(walk, true));
    BVH_TRY(passes.fill(walk, tree->d_offsets, tree->d_hits, tree->hits_cap));
    size_t tot = 0;
    const int rc = passes.total(what, nullptr, 0, &tot);
    if (out.total) *out.total = tot;
    if (rc == BVHGPU_OK || rc == BVHGPU_ERR_CAPACITY) keep_total(tree, tot);
    if (rc != BVHGPU_OK) return rc;
    if (tot > tree->hits_cap && (tree->dims == 3 || (out.hits && tot <= out.cap))) {
        BVH_TRY(ensure_result_buffers(tree, n, tot));
        BVH_TRY(passes.fill(walk, tree->d_offsets, tree->d_hits, tree->hits_cap));
    }
    return copy_retained(tree, what, n, tot, out.offsets, out.hits, out.cap);
}

// One probe over the records: status, empty input, then the walk (FLAT: leaves re-test the shape's own box).
template <class Probe, class TreeT> int probe_csr(TreeT* tree, bool flat, const void* src, size_t n, const CsrOut& out, const char* what) {
    BVH_TRY(csr_status(tree, n));
    if (n == 0 || tree->n == 0) return csr_zero(tree, n, out);     // nothing to walk / empty Bvh: no hits (bvh_impl.rs:109-112)
    BVH_TRY(ensure_records(tree));
    const CsrWalk<TreeT::D, typename TreeT::Scalar, Probe> walk{flat, tree->d_tnodes, tree->n_trec, walk_aabbs(tree), src};
    return csr_run(tree, walk, n, out, what);
}
inline int check_walk(const char* what, size_t n, int mode) {
    BVH_TRY(check_n(what, n));
    if (mode != BVHGPU_TRAVERSE_BVH && mode != BVHGPU_TRAVERSE_FLAT) { set_error("%s: bad mode %d", what, mode); return BVHGPU_ERR_INVALID; }
    return BVHGPU_OK;
}
template <class TreeT> int query_csr(TreeT* tree, int mode, int kind, const void* src, size_t n, const CsrOut& out, const char* what) {
    using T = typename TreeT::Scalar;
    constexpr int D = TreeT::D;
    BVH_TRY(check_walk(what, n, mode));
    const bool flat = mode == BVHGPU_TRAVERSE_FLAT;
    switch (kind) {
    case BVHGPU_QUERY_AABB: return probe_csr<Query<T, BVHGPU_QUERY_AABB, D>>(tree, flat, src, n, out, what);
    case BVHGPU_QUERY_POINT: return probe_csr<Query<T, BVHGPU_QUERY_POINT, D>>(tree, flat, src, n, out, what);
    case BVHGPU_QUERY_BALL: return probe_csr<Query<T, BVHGPU_QUERY_BALL, D>>(tree, flat, src, n, out, what);
    case QUERY_WITHIN: return probe_csr<Query<T, QUERY_WITHIN, D>>(tree, flat, src, n, out, what);
    default: set_error("%s: bad kind %d", what, kind); return BVHGPU_ERR_INVALID;
    }
}

template <class TreeT> int nearest_candidates_csr(TreeT* tree, const typename TreeT::Scalar* points, size_t n, const CsrOut& out) {
    using T = typename TreeT::Scalar;
    const char* what = "nearest_candidates";
    BVH_TRY(check_n(what, n));
    BVH_TRY(csr_status(tree, n));
    if (n == 0 || tree->n == 0) return csr_zero(tree, n, out);
    Scratch scratch(tree->ctx);
    T* rec = nullptr;
    BVH_TRY(scratch.get(&rec, (TreeT::D + 1) * n));
    BVH_TRY(nearest_bound(tree, points, (uint32_t)n, rec));
    return probe_csr<Query<T, QUERY_WITHIN, TreeT::D>>(tree, true, rec, n, out, what);
}

// Ordered traversal: ordered_kernel over the records (a 2-D tree walks the lifted rays of dim2_expand_rays in its embedding).
template <class TreeT> int ordered_csr(TreeT* tree, const void* rays, size_t n, int ascending, uint32_t* d_offsets, uint32_t* d_hits,
                                       typename TreeT::Scalar* d_dists, size_t cap, size_t* total) {
    using T = typename TreeT::Scalar;
    const char* what = "traverse_ordered";
    BVH_TRY(check_n(what, n));
    BVH_TRY(csr_status(tree, n));
    if (n == 0 || tree->n == 0) return csr_zero(tree, n, CsrOut::device(d_offsets, d_hits, cap, total));
    BVH_TRY(ensure_records(tree));
    const OrderedWalk<TreeT::D, T> walk{tree->d_tnodes, tree->n_trec, reinterpret_cast<const typename CsrRecords<TreeT::D, T>::Ray*>(rays), ascending, d_dists};
    return csr_two_pass(tree->ctx, walk, (uint32_t)n, what, d_offsets, d_hits, cap, total);
}

// The shapes of a tree in leaf (DFS) order, as long as `scratch` lives (released stream-ordered after the fill).
template <class TreeT> int leaf_order(TreeT* tree, Scratch& scratch, uint32_t** order) {
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_TRY(scratch.get(order, tree->n));
    leaf_order_kernel<<<(tree->n + 255) / 256, 256, 0, ctx->stream>>>(tree->d_node_index, tree->d_node_start, tree->n, *order);
    ctx->launches++;
    BVH_CUDA_TRY(cudaGetLastError());
    return BVHGPU_OK;
}
// Self-overlap: overlap_kernel over the records and the shapes' own boxes.  A 2-D tree tests d_aabb (z = [0, 0]) and walks the records
// of its embedding, whose z = [-1, +1] contains that slab.
template <class TreeT> int overlap_csr(TreeT* tree, const CsrOut& out, const char* what) {
    BVH_TRY(resolve_status(tree));
    if (tree->n < 2) return csr_zero(tree, tree->n, out);
    BVH_TRY(ensure_records(tree));
    Scratch scratch(tree->ctx);
    uint32_t* order = nullptr;
    BVH_TRY(leaf_order(tree, scratch, &order));
    const OverlapWalk<TreeT::D, typename TreeT::Scalar> walk{tree->d_tnodes, tree->n_trec, tree->d_aabb, tree->d_node_index, order};
    return csr_run(tree, walk, tree->n, out, what);
}
// Overlap between two trees: overlap_trees_kernel, A's shapes in A's leaf order against B's records and B's own boxes (2-D trees as
// above: both d_aabb have z = [0, 0], B's records z = [-1, +1]).
template <class TreeT> int overlap_trees_csr(TreeT* a, TreeT* b, const CsrOut& out, const char* what) {
    BVH_TRY(resolve_status(a));
    BVH_TRY(resolve_status(b));
    if (a->n == 0 || b->n == 0) return csr_zero(a, a->n, out);
    BVH_TRY(ensure_records(b));
    Scratch scratch(a->ctx);
    uint32_t* order = nullptr;
    BVH_TRY(leaf_order(a, scratch, &order));
    const OverlapTreesWalk<TreeT::D, typename TreeT::Scalar> walk{b->d_tnodes, b->n_trec, b->d_aabb, a->d_aabb, order};
    return csr_run(a, walk, a->n, out, what);
}
// Triangle pairs (D = 3): the overlap rows filtered by the triangles' predicate.  The checks run in this order: the sticky failure
// (A's before B's), then the triangles of every non-empty tree.
template <class T> int triangle_pairs_check(Tree<T>* tree, const char* what) {
    if (tree->n && !tree->d_tris) { set_error("%s: needs bvhgpu_tree_set_triangles_* first", what); return BVHGPU_ERR_INVALID; }
    return BVHGPU_OK;
}
template <class T> int triangle_pairs_csr(Tree<T>* tree, int skip_shared, const CsrOut& out, const char* what) {
    BVH_TRY(resolve_status(tree));
    BVH_TRY(triangle_pairs_check(tree, what));
    if (tree->n < 2) return csr_zero(tree, tree->n, out);
    BVH_TRY(ensure_records(tree));
    Scratch scratch(tree->ctx);
    uint32_t* order = nullptr;
    BVH_TRY(leaf_order(tree, scratch, &order));
    const DTri<T>* tris = reinterpret_cast<const DTri<T>*>(tree->d_tris);
    const TrianglePairsWalk<T, false> walk{tree->d_tnodes, tree->n_trec, tree->d_aabb, tree->d_aabb, tris, tris, skip_shared != 0,
                                           tree->d_node_index, order};
    return csr_run(tree, walk, tree->n, out, what);
}
template <class T> int triangle_pairs_trees_csr(Tree<T>* a, Tree<T>* b, const CsrOut& out, const char* what) {
    BVH_TRY(resolve_status(a));
    BVH_TRY(resolve_status(b));
    BVH_TRY(triangle_pairs_check(a, what));
    BVH_TRY(triangle_pairs_check(b, what));
    if (a->n == 0 || b->n == 0) return csr_zero(a, a->n, out);
    BVH_TRY(ensure_records(b));
    Scratch scratch(a->ctx);
    uint32_t* order = nullptr;
    BVH_TRY(leaf_order(a, scratch, &order));
    const TrianglePairsWalk<T, true> walk{b->d_tnodes, b->n_trec, a->d_aabb, b->d_aabb, reinterpret_cast<const DTri<T>*>(a->d_tris),
                                          reinterpret_cast<const DTri<T>*>(b->d_tris), 0, nullptr, order};
    return csr_run(a, walk, a->n, out, what);
}

// Explicit instantiations of the drivers of one tree type (traverse.cu: Tree<T>, dim4.cu: Tree4<T>).
#define BVH_INSTANTIATE_CSR(TR, T)                                                                                                  \
    template int query_csr<TR>(TR*, int, int, const void*, size_t, const CsrOut&, const char*);                                    \
    template int nearest_candidates_csr<TR>(TR*, const T*, size_t, const CsrOut&);                                                  \
    template int ordered_csr<TR>(TR*, const void*, size_t, int, uint32_t*, uint32_t*, T*, size_t, size_t*);                         \
    template int overlap_csr<TR>(TR*, const CsrOut&, const char*);                                                                  \
    template int overlap_trees_csr<TR>(TR*, TR*, const CsrOut&, const char*);
#endif  // __CUDACC__

}  // namespace bvhb200
