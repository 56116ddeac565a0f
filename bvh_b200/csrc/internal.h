// bvh_b200/csrc/internal.h -- host-side structures shared by the translation units of libbvh_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <string>
#include <cstdio>
#include "common.cuh"

namespace bvhb200 {

void set_error(const char* fmt, ...);

#define BVH_CUDA_TRY(expr)                                                                          \
    do {                                                                                            \
        cudaError_t _e = (expr);                                                                    \
        if (_e != cudaSuccess) {                                                                    \
            ::bvhb200::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return BVHGPU_ERR_CUDA;                                                                 \
        }                                                                                           \
    } while (0)

#define BVH_TRY(expr)                  \
    do {                               \
        int _s = (expr);               \
        if (_s != BVHGPU_OK) return _s; \
    } while (0)

}  // namespace bvhb200

// Device status block a build writes (read back lazily).
struct BuildStatus {
    uint32_t error;        // bvhgpu_status raised on the device (timeout / internal)
    uint32_t nan_found;    // prep kernel saw a NaN coordinate
    uint32_t tickets;      // queue tickets handed out (diagnostics)
    uint32_t leaves_done;  // must equal n at the end
    uint32_t rebuilt;      // optimize: shapes in the subtrees that were rebuilt
    uint32_t pad[3];
};

struct bvhgpu_ctx {
    int device = 0;
    int sm_count = 0;
    cudaStream_t own_stream = nullptr;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev_switch = nullptr; // set_stream / reset_stream: recorded on the outgoing stream, waited on by the incoming one
    uint64_t launches = 0;
    int64_t traverse_slots = -1;   // per-ray hit slots of the single-pass traversal (0 = two-pass, -1 = auto by batch size)
    int64_t traverse_persistent = 2;   // 0: one ray per thread, 1: persistent refill kernel, 2: coherence probe decides on the device
    int walk_grid = 0;             // persistent grid size: one full wave (computed once), or the value of option "walk_grid"
    bool walk_grid_forced = false;
    bool top_attr_set = false;     // walk_top_kernel's dynamic shared memory limit has been raised on this device
    int64_t build_gang = -1;       // exact builder: co-resident warp gangs for the top levels (-1 / 1 on, 0 off = queue tiles only)
    int64_t build_subtree = -1;    // exact builder: in-register subtrees for ranges <= 32 shapes (-1 auto, 0 never, 1 always)
    int64_t build_small = -1;      // exact builder: defer ranges <= 16 shapes to the thread-per-range kernel (-1 auto by size, 0 never, 1 always)
    // small pinned read-back area (256 words): 0-25 the ray traversal's scan tail, 64-79 the streamed path's per-chunk values,
    // 128-129 the stream probe, 200-217 the entry points' checks (200 staged boxes, 204 synchronize, 208-209 changed boxes, 212 added
    // boxes, 216-217 removal lists), 220 the group count of an add, 224-225 the 4-D group seeds, 232-235 the 4-D build, CSR_TOTAL_WORD
    // (236-237) the total of the two-pass CSR walks (csr.cuh), 244-248 the 4-D rebuild seeds
    uint32_t* h_pinned = nullptr;
    int64_t profile = 0;           // bracket dominant kernels with events
    cudaEvent_t ev_walk[2] = {nullptr, nullptr};
    cudaEvent_t ev_build[2] = {nullptr, nullptr};
    bool have_walk = false, have_build = false;
    // host-pointer traversal: H2D chunks on a second stream, overlapped with the walks
    cudaStream_t copy_stream = nullptr, d2h_stream = nullptr;
    cudaEvent_t ev_order = nullptr, ev_total = nullptr;
    cudaEvent_t ev_chunk[16] = {}, ev_emit[16] = {};
    cudaEvent_t ev_e2e[5] = {};    // profile: start, walk end, last H2D done, last emit, last D2H
    bool have_e2e = false;
    // host-pointer traversal, streaming form (rays consumed by a running kernel while they arrive): only when a kernel launch
    // does not block the host and no tool serialises / replays launches.  -1 = not probed yet, 0 = never stream, 1 = ok.
    int stream_ok = -1;
    double host_us[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // profile: host-side time stamps of the last host-pointer traversal (us since entry)
    uint64_t slot_budget_words = 0; // traversal slot scratch budget (a quarter of the memory that was free at first use, in 4-byte words / 4)
    int last_streamed = -1;        // did the last host-pointer traversal stream (1) or copy-then-walk (0)
    int64_t traverse_stream = -1;  // option "traverse_stream": -1 auto (probe), 0 never, 1 force
    int64_t traverse_top = -1;     // option "traverse_top": shared-memory top-of-tree walk: -1 auto, 0 off, 1 on
    uint32_t* d_ready = nullptr;       // cudaMalloc'ed word the streamed host path bumps with cuStreamWriteValue32 (refused on pool memory)
    int wv_ok = -1;                    // did the last streamed call use stream write-value flags (1) or 4-byte copies (0)
    uint32_t* d_async_err = nullptr;   // sticky device-side error word of asynchronous calls (sharded exchange): surfaced by bvhgpu_synchronize
    int numa_node = -1;            // NUMA node of the device (sysfs), -1 unknown
};
#define BVH_MAX_CHUNKS 16u

namespace bvhb200 {

// The device layout of a triangle of bvhgpu_tree_set_triangles_* (Tree::d_tris).
template <class T> struct DTri { T a[3], pa, b[3], pb, c[3], pc; };       // 48 B / 96 B: three vector loads per triangle
// The device layout of a segment of bvhgpu_tree_set_segments_* (Tree::d_segs, 2-D trees): the ABI's 4 T as they are.
template <class T> struct DSeg { T a[2], b[2]; };                         // 16 B / 32 B: one / two vector loads per segment

template <class T> struct Tree {
    using Tr = Traits<T>;
    // what the dynamic drivers of dynamic.cu see: a 2-D tree runs the D = 3 kernels in the plane z = 0
    static constexpr int D = 3;
    using Scalar = T; using Node = typename Tr::Node; using Aabb = typename Tr::Aabb; using Box = typename Tr::DAabb;
    bvhgpu_ctx* ctx = nullptr;
    uint32_t n = 0;          // shapes
    uint32_t n_nodes = 0;    // 2n-1
    int dims = 3;            // 2: a Bvh<T,2> embedded in the plane z = 0 (dim2.cu)
    typename Tr::DAabb* d_aabb = nullptr;     // [n]      shape AABBs (padded device layout)
    typename Tr::DAabb* d_aabb_trav = nullptr; // [n]     dims == 2 only: the same with z = [-1, +1] for the FLAT leaf re-test
    typename Tr::Node* d_nodes = nullptr;     // [2n-1]   Bvh.nodes, reference preorder layout
    uint32_t* d_node_index = nullptr;         // [n]      leaf node of every shape
    uint32_t* d_node_start = nullptr;         // [2n-1]   first position of the node's shape range (== #leaves before it)
    typename Tr::TNode* d_tnodes = nullptr;   // [n_trec] traversal records
    uint32_t n_trec = 0;
    void* d_top = nullptr;                    // f32: top-of-tree records for walk_top_kernel (32-B header {n_top, C}, lo[n_top], hi[n_top] float4), built lazily
    uint32_t top_cap = 0, top_budget = 0;
    bool top_valid = false;
    uint32_t* d_arrive = nullptr;             // [2n-1] arrival counters of the incremental update (all zero between calls)
    uint8_t* d_bad = nullptr;                 // [2n-1] growth flags of the incremental update (all zero between calls)
    T* d_sa_base = nullptr;                   // [2n-1] surface area of every inner node when it was last (re)built: baseline of bvhgpu_optimize / update
    void* d_tris = nullptr;                   // [n] triangle vertices (padded), optional: bvhgpu_tree_set_triangles_*
    void* d_segs = nullptr;                   // [n] dims == 2 only: segment end points (DSeg<T>), optional: bvhgpu_tree_set_segments_*
    typename Tr::Flat* d_flat = nullptr;      // [n_flat] reference-layout FlatBvh (built on demand)
    size_t n_flat = 0;
    bool have_flat = false;
    // deferred build status
    BuildStatus* d_status = nullptr;
    BuildStatus* h_status = nullptr;          // pinned
    bool status_pending = false;
    int failed_status = 0;                    // sticky: first failure of build / refit / optimize (BVHGPU_OK = healthy)
    std::string failed_message;
    // retained result of the last traversal
    uint32_t* d_offsets = nullptr; size_t offsets_cap = 0;
    uint32_t* d_hits = nullptr;    size_t hits_cap = 0;
    size_t last_total = 0, last_nrays = 0;
    uint64_t last_visits = 0;
};

// Resolve the deferred device status of a build / refit (synchronises the stream once).
template <class T> int resolve_status(Tree<T>* tree);

// The message of the last failed call on this thread (bvhgpu_last_error).
const char* last_error();
// A failure that leaves a tree's arrays inconsistent (a build, refit, rebuild or relocation that failed half-way) is STICKY: every
// later entry point on that tree reports the same status again, and only bvhgpu_tree_free_* is meaningful afterwards.  `msg` is the
// message as it is; without one it reads "<who> failed after the tree was modified (<last error>)".  A tree that has failed already
// keeps its first failure.  Serves Tree<T> and Tree4<T> (dim4.cu).
template <class TreeT> int mark_failed(TreeT* tree, int rc, const char* who, const char* msg = nullptr) {
    if (tree->failed_status != BVHGPU_OK) return tree->failed_status;
    char buf[1200];
    if (!msg) { snprintf(buf, sizeof buf, "%s failed after the tree was modified (%s); the tree is unusable", who, last_error()); msg = buf; }
    tree->failed_status = rc; tree->failed_message = msg;
    set_error("%s", msg);
    return rc;
}

// ---- memory (stream-ordered pool) ----
int dalloc(bvhgpu_ctx* ctx, void** p, size_t bytes);
void dfree(bvhgpu_ctx* ctx, void* p);
template <class P> inline int dalloc_t(bvhgpu_ctx* ctx, P** p, size_t count) { return dalloc(ctx, (void**)p, count * sizeof(P)); }
// The result buffers a tree retains for its host-pointer CSR calls (d_offsets / d_hits), grown to at least n + 1 offsets and hits_cap
// hits; they are never shrunk.  Serves Tree<T> and Tree4<T>.
template <class TreeT> int ensure_result_buffers(TreeT* tree, size_t n, size_t hits_cap) {
    bvhgpu_ctx* ctx = tree->ctx;
    if (tree->offsets_cap < n + 1) {
        dfree(ctx, tree->d_offsets); tree->d_offsets = nullptr; tree->offsets_cap = 0;
        const int rc = dalloc_t(ctx, &tree->d_offsets, n + 1);
        if (rc != BVHGPU_OK) return rc;
        tree->offsets_cap = n + 1;
    }
    if (tree->hits_cap < hits_cap) {
        dfree(ctx, tree->d_hits); tree->d_hits = nullptr; tree->hits_cap = 0;
        const int rc = dalloc_t(ctx, &tree->d_hits, hits_cap);
        if (rc != BVHGPU_OK) return rc;
        tree->hits_cap = hits_cap;
    }
    return BVHGPU_OK;
}
// The CSR a host-pointer call left in the tree's retained buffers, copied back: the offsets always, the hits when they fit `cap`;
// otherwise BVHGPU_ERR_CAPACITY, with a hint that depends on whether the tree type has bvhgpu_traverse_fetch_* (D = 3 only).
// Synchronises.
template <class TreeT> int copy_retained(TreeT* tree, const char* what, size_t n, size_t tot, uint32_t* offsets, uint32_t* hits, size_t cap) {
    cudaStream_t st = tree->ctx->stream;
    BVH_CUDA_TRY(cudaMemcpyAsync(offsets, tree->d_offsets, sizeof(uint32_t) * (n + 1), cudaMemcpyDeviceToHost, st));
    int ret = BVHGPU_OK;
    if (hits && tot <= cap) { if (tot) BVH_CUDA_TRY(cudaMemcpyAsync(hits, tree->d_hits, sizeof(uint32_t) * tot, cudaMemcpyDeviceToHost, st)); }
    else if (tot > cap) {
        set_error("%s: %zu hits do not fit the caller's capacity %zu (%s)", what, tot, cap,
                  tree->dims == 3 ? "use bvhgpu_traverse_fetch_*" : "call again with cap = *total");
        ret = BVHGPU_ERR_CAPACITY;
    }
    BVH_CUDA_TRY(cudaStreamSynchronize(st));
    return ret;
}
// The size guard of the batched calls: n must fit the kernels' u32 item indices.
inline int check_n(const char* what, size_t n) {
    if (n > 0x7FFFFFFFull) { set_error("%s: n = %zu exceeds 2^31-1", what, n); return BVHGPU_ERR_INVALID; }
    return BVHGPU_OK;
}
// Scratch that is released (stream-ordered) when the scope ends, on every return path.
struct Scratch {
    bvhgpu_ctx* ctx;
    void* ptrs[16];
    int n = 0;
    explicit Scratch(bvhgpu_ctx* c) : ctx(c) {}
    Scratch(const Scratch&) = delete;
    Scratch& operator=(const Scratch&) = delete;
    ~Scratch() { for (int i = 0; i < n; ++i) dfree(ctx, ptrs[i]); }
    template <class P> int get(P** p, size_t count) {
        *p = nullptr;
        if (n >= 16) { set_error("internal: scratch table full"); return BVHGPU_ERR_INTERNAL; }
        const int rc = dalloc(ctx, (void**)p, count * sizeof(P));
        if (rc == BVHGPU_OK) ptrs[n++] = (void*)*p;
        return rc;
    }
};

// ---- build_sah.cu ----
// in_aabbs: device pointer to n AABBs in the C-ABI layout (24 B / 48 B).  Fills tree->d_aabb, d_nodes,
// d_node_index, d_node_start (allocated here).  Asynchronous; errors are reported via tree->d_status.
template <class T> int build_exact_sah(bvhgpu_ctx* ctx, const typename Traits<T>::Aabb* in_aabbs, uint32_t n, Tree<T>* tree);
// Converts ABI-layout AABBs to the device layout only (used by tree_from_nodes and refit).
template <class T> int convert_aabbs(bvhgpu_ctx* ctx, const typename Traits<T>::Aabb* in_aabbs, uint32_t n,
                                     typename Traits<T>::DAabb* out, uint32_t* d_nan_flag);

// ---- treelet session (build_sah.cu), used by lbvh.cu for BVHGPU_BUILD_LBVH_TREELET ----
struct BuildCtl;
template <class T> struct QSlot;
template <class T> struct TreeletSession { void* params = nullptr; QSlot<T>* q = nullptr; uint32_t* qseq = nullptr; uint32_t qmask = 0; BuildCtl* ctl = nullptr; };
template <class T> int treelet_begin(bvhgpu_ctx* ctx, Tree<T>* tree, uint32_t* sorted_ids, TreeletSession<T>* S);
template <class T> int treelet_finish(bvhgpu_ctx* ctx, Tree<T>* tree, TreeletSession<T>* S);

// ---- rebuild session (build_sah.cu), used by optimize(): the exact builder restarted from inner nodes.  d_roots[0 .. *d_n_roots)
// are node indices of disjoint subtrees, cb[node][6] the bounds of the shape centres below every node, idx0 the shapes in
// leaf order.  Rewrites d_nodes / d_node_index / d_node_start of those subtrees in place.
// cb_by_root: cb holds 6 values per ROOT (in d_roots order) instead of per node
template <class T> int rebuild_subtrees(bvhgpu_ctx* ctx, Tree<T>* tree, const uint32_t* d_roots, const uint32_t* d_n_roots, const T* cb, uint32_t* idx0, bool cb_by_root);

// ---- lbvh.cu ----
template <class T> int build_lbvh(bvhgpu_ctx* ctx, const typename Traits<T>::Aabb* in_aabbs, uint32_t n, Tree<T>* tree, bool treelets);

// ---- flatten.cu ----
template <class T> int build_traversal_records(Tree<T>* tree);   // d_tnodes
template <class T> int build_flat(Tree<T>* tree);                // d_flat (reference FlatNode layout)
int build_top_records(Tree<float>* tree, uint32_t budget);        // d_top
template <class T> int sah_cost(Tree<T>* tree, double* out2);
template <class T> int optimize(Tree<T>* tree, double max_growth);   // refit + exact rebuild of the degraded subtrees
// idx[node_start[node_index[s]]] = s for s < n: the shapes in leaf (DFS) order, of a 3-D or a 4-D tree
__global__ void __launch_bounds__(256) leaf_order_kernel(const uint32_t* __restrict__ node_index, const uint32_t* __restrict__ node_start,
                                                         uint32_t n, uint32_t* __restrict__ idx);
// Caches after the boxes changed in place (node count unchanged, dynamic.cu): the FLAT leaf boxes of a 2-D tree first (the records
// read them), then the traversal records, then the flat array if it was built.
template <class T> int refresh_caches(Tree<T>* tree);
// After a relocation (new node count or shape numbering, dynamic.cu): update buffers dropped, records and flat array rebuilt at the
// new size.
template <class T> int finish_relayout(Tree<T>* tree);
// dirty[0 .. cnts[0]) = the nodes whose box changed, tree->d_bad = their growth flags.  Rebuilds in place the outermost degraded subtrees
// (cnts[1], zero on entry, counts them), gives them fresh baselines and clears the flags.  The shapes rebuilt are counted in
// tree->d_status (`rebuilt` and `who` serve the 4-D overload).
template <class T> int rebuild_degraded(Tree<T>* tree, const uint32_t* d_dirty, uint32_t* d_cnts, size_t* rebuilt, const char* who);

// ---- dynamic.cu: refit, update_shapes, add_shape / remove_shape (batched) of Tree<T> and Tree4<T> ----
// The shapes of the tree type's ABI box, checked on the device (flags read back, synchronises): a NaN coordinate, an index >= n when
// d_changed is given (otherwise box i belongs to shape i).  A failure leaves the tree untouched.
template <class TreeT> int check_boxes(TreeT* tree, const uint32_t* d_changed, const typename TreeT::Aabb* d_fresh, uint32_t m, Scratch& scratch,
                                       const char* who);
template <class TreeT> int scatter_boxes(TreeT* tree, const uint32_t* d_changed, const typename TreeT::Aabb* d_fresh, uint32_t m);   // into d_aabb
template <class TreeT> int ensure_sa_base(TreeT* tree);   // the growth baseline: the tree as it is now, unless one exists already
template <class TreeT> int refit(TreeT* tree);            // child boxes bottom-up from d_aabb, then the caches
// The shapes d_changed[0 .. m) already carry their new boxes in d_aabb.  max_growth <= 0: boxes only.  *rebuilt: shapes in the rebuilt
// subtrees (4-D; a 3-D tree counts them in its status).
template <class TreeT> int update_incremental(TreeT* tree, const uint32_t* d_changed, uint32_t m, double max_growth, size_t* rebuilt);
// aabb_all: [n + k] device boxes (the tree's n followed by the k new ones, checked for NaN); becomes tree->d_aabb.  A failure with
// tree->d_aabb != aabb_all left the tree untouched; after that point the caller marks it failed.  *rebuilt as update_incremental.
template <class TreeT> int add_shapes(TreeT* tree, typename TreeT::Box* aabb_all, uint32_t k, double max_growth, size_t* rebuilt);
// d_rm: [n + 1] removed flag of every shape (0 / 1, the last word 0), k = number of removed shapes, 1 <= k <= n.  A failure with
// tree->d_nodes unchanged left the tree untouched.
template <class TreeT> int remove_shapes(TreeT* tree, const uint32_t* d_rm, uint32_t k);
// validation of a removal list: d_rm[n + 1] zeroed by the caller; d_flags[0] = index >= n, d_flags[1] = duplicate index
int remove_check(bvhgpu_ctx* ctx, const uint32_t* d_idx, uint32_t k, uint32_t n, uint32_t* d_rm, uint32_t* d_flags);

// ---- traverse.cu ----
// d_rays: rays on the device; fmt: BVHGPU_RAYS_FULL (9 scalars: the C-ABI Ray) or BVHGPU_RAYS_OD (6 scalars: origin, direction).
// shard != nullptr: multi-GPU step, results go to every rank's peer-mapped global CSR (d_offsets / d_hits unused).
template <class T> int traverse_device(Tree<T>* tree, int mode, const void* d_rays, uint32_t fmt,
                                       size_t nrays, uint32_t* d_offsets, uint32_t* d_hits, size_t cap, size_t* total,
                                       const bvhgpu_shard* shard = nullptr);
// Every argument check of a sharded step (rank / world, seq >= 1, ray layout, non-null peer buffers, shard sizes): BVHGPU_OK or the
// status the entry point returns before it enqueues anything.
int check_shard(const bvhgpu_shard* shard, size_t nrays);
// Loads the sharded step's kernels (scan_post_kernel<true>, emit_goffsets_kernel) on the current device before any step runs.
int preload_shard_kernels();
// Host rays in, host CSR out; H2D / walk+scan+emit / D2H overlapped.  Needs tree->d_offsets / d_hits sized by the caller.
template <class T> int traverse_host_pipelined(Tree<T>* tree, int mode, const void* h_rays, uint32_t fmt, size_t nrays,
                                               uint32_t* h_offsets, uint32_t* h_hits, size_t h_cap, size_t* total);
// nearest_to for a batch of points (device pointers): exact reference walk for AABB-distance shapes; candidate lists for any shape
template <class T> int nearest_device(Tree<T>* tree, int mode, const T* d_points, size_t nq, uint32_t* d_shape, T* d_dist, int use_triangles = 0);
// k nearest shapes of every point (device pointers: 3 T per point, nq limits or nullptr, nq * k outputs), on the context's stream.
// Checks nq, k and the tree's status; the pointers are checked by the caller.
template <class T> int knn_device(Tree<T>* tree, const T* d_points, size_t nq, uint32_t k, const T* d_max_dist, uint32_t* d_shape, T* d_dist);
// k nearest triangles (bvhgpu_tree_set_triangles_*), as knn_device with Triangle::distance_squared keys; d_closest (nq * k * 3 T) may be
// nullptr.  Also refuses a non-empty tree without triangles.
template <class T> int knn_tri_device(Tree<T>* tree, const T* d_points, size_t nq, uint32_t k, const T* d_max_dist, uint32_t* d_shape, T* d_dist,
                                      T* d_closest);
// CSR scan of per-item counts (traverse.cu), launched by the count -> scan -> fill driver of csr.cuh (CsrPasses) for every two-pass
// walk: scan_local_kernel runs CSR_SCAN_THREADS threads per block over CSR_SCAN_TILE counts and leaves local exclusive offsets
// (saturated at 0xFFFFFFFF) and 64-bit block totals; scan_blocks_kernel (one block of 1024 threads) turns the block totals into exclusive 64-bit block offsets and adds the
// grand total to *total (zeroed by the caller).
constexpr int CSR_SCAN_THREADS = 256;
constexpr int CSR_SCAN_TILE = 2048;
constexpr int CSR_TOTAL_WORD = 236;        // h_pinned word (8-byte aligned) of the two-pass total
__global__ void __launch_bounds__(256) scan_local_kernel(const uint32_t* __restrict__ counts, uint32_t n, uint32_t* __restrict__ local,
                                                         unsigned long long* __restrict__ blocksum, uint32_t* __restrict__ maxcount);
__global__ void __launch_bounds__(1024) scan_blocks_kernel(unsigned long long* __restrict__ blocksum, uint32_t nblocks, unsigned long long* __restrict__ total);
// ---- dim2.cu ----
template <class T> int dim2_expand_aabbs(bvhgpu_ctx* ctx, const T* d_in4, uint32_t n, T* d_out6);
template <class T> int dim2_expand_rays(bvhgpu_ctx* ctx, const T* d_in6, uint32_t n, T* d_out9);
// n records of nvec 2-vectors and nscal scalars -> the same with every vector lifted to z = 0 (query records, nearest_to points)
template <class T> int dim2_lift(bvhgpu_ctx* ctx, const T* d_in, uint32_t n, int nvec, int nscal, T* d_out);
template <class T> int dim2_finish_build(Tree<T>* tree);
template <class T, class N2> int dim2_nodes_out(Tree<T>* tree, N2* d_out);
template <class T, class F2> int dim2_flat_out(Tree<T>* tree, F2* d_out);
// ---- closest.cu ----
template <class T> int set_triangles(Tree<T>* tree, const T* tris9, size_t n, bool dev_input);
template <class T> int closest_hit_device(Tree<T>* tree, const void* d_rays, uint32_t fmt, size_t nrays, int use_triangles, uint32_t* d_shape, T* d_dist, T* d_uv);
// AABB-mode closest hit of a 2-D tree (D = 2: the 3-D nodes and boxes it is embedded in, x and y tested, 2-D rays of 6 T) or a 4-D
// tree (D = 4: its bvh_node4* and ABI boxes, rays of 12 T); device pointers, on the context's stream, nothing synchronises.  Arguments
// and the tree's status are checked by the caller.
template <int D, class T> struct ClosestLayout { using Node = typename Traits<T>::Node; using Box = typename Traits<T>::DAabb; };   // D = 2, 3
template <> struct ClosestLayout<4, float> { using Node = bvh_node4f; using Box = bvh_aabb4f; };
template <> struct ClosestLayout<4, double> { using Node = bvh_node4d; using Box = bvh_aabb4d; };
template <int D, class T> int closest_aabb_device(bvhgpu_ctx* ctx, const typename ClosestLayout<D, T>::Node* nodes, uint32_t n_shapes,
                                                  const typename ClosestLayout<D, T>::Box* aabb, const T* d_rays, size_t nrays, uint32_t* d_shape, T* d_dist);
// Any hit (closest.cu): per ray the first leaf the closest walk accepts with distance < tmax (d_tmax: nrays limits, or nullptr for
// +inf), BVH_INVALID without one; device pointers, on the context's stream.  any_hit_device checks its arguments and the tree's
// status as closest_hit_device does; any_hit_aabb_device (D = 2, 4) leaves both to the caller, as closest_aabb_device.
template <class T> int any_hit_device(Tree<T>* tree, const void* d_rays, uint32_t fmt, size_t nrays, const T* d_tmax, int use_triangles, uint32_t* d_shape);
template <int D, class T> int any_hit_aabb_device(bvhgpu_ctx* ctx, const typename ClosestLayout<D, T>::Node* nodes, uint32_t n_shapes,
                                                  const typename ClosestLayout<D, T>::Box* aabb, const T* d_rays, size_t nrays, const T* d_tmax, uint32_t* d_shape);
// Multi hit (closest.cu): per ray the first k hits of the closest walk's keys with distance < tmax (d_tmax: nrays limits or nullptr
// for no limit), rows of k slots (nrays * k outputs, d_uv: 2 T per slot or nullptr), padded with (BVH_INVALID, +inf, 0, 0); device
// pointers, on the context's stream.  1 <= k <= BVHGPU_KNN_MAX_K is checked by the caller.  multi_hit_device checks the other
// arguments and the tree's status as any_hit_device does; multi_hit_aabb_device (D = 2, 4) leaves them to the caller.
template <class T> int multi_hit_device(Tree<T>* tree, const void* d_rays, uint32_t fmt, size_t nrays, uint32_t k, const T* d_tmax, int use_triangles,
                                        uint32_t* d_shape, T* d_dist, T* d_uv);
template <int D, class T> int multi_hit_aabb_device(bvhgpu_ctx* ctx, const typename ClosestLayout<D, T>::Node* nodes, uint32_t n_shapes,
                                                    const typename ClosestLayout<D, T>::Box* aabb, const T* d_rays, size_t nrays, uint32_t k,
                                                    const T* d_tmax, uint32_t* d_shape, T* d_dist);
// Crossing counts, point-in-mesh and signed distance (closest.cu, crossings_kernel): device pointers, on the context's stream, nothing
// synchronises.  Each checks n (<= 2^31-1), its layout / rule, then (n > 0) the tree's status and the triangles; the pointers are
// checked by the caller.  An empty tree gives zeros (counts, inside); signed_distance_device is knn_tri_device (k = 1, no limit), the
// containment walk into scratch and the sign.
template <class T> int count_hits_device(Tree<T>* tree, const void* d_rays, uint32_t fmt, size_t nrays, const T* d_tmax, uint32_t* d_front,
                                         uint32_t* d_back);
template <class T> int contains_points_device(Tree<T>* tree, const T* d_points, size_t n, int rule, uint8_t* d_inside);
template <class T> int signed_distance_device(Tree<T>* tree, const T* d_points, size_t n, int rule, uint32_t* d_shape, T* d_dist, T* d_closest);
template <class T> int rays_new_device(bvhgpu_ctx* ctx, const T* d_origins, const T* d_dirs, size_t n,
                                       typename Traits<T>::Ray* d_rays);
// ---- segments.cu: polygons of 2-D trees (DESIGN.md §4.23) ----
// The segments of every shape, host pointer: 4 T per segment (ax, ay, bx, by), n == tree->n.  Synchronises.
template <class T> int set_segments(Tree<T>* tree, const T* segs4, size_t n);
// Point-in-polygon, k nearest segments and signed distance, device pointers (2 T per point), on the context's stream, nothing
// synchronises.  Each checks n (<= 2^31-1), its rule / k, the tree's status, then the segments; the pointers are checked by the caller.
// d_winding and d_closest (2 T per slot) may be nullptr.
template <class T> int polygon_contains_device(Tree<T>* tree, const T* d_points, size_t n, int rule, uint8_t* d_class, int32_t* d_winding);
template <class T> int knn_seg_device(Tree<T>* tree, const T* d_points, size_t n, uint32_t k, const T* d_max_dist, uint32_t* d_shape, T* d_dist,
                                      T* d_closest);
template <class T> int polygon_distance_device(Tree<T>* tree, const T* d_points, size_t n, int rule, uint32_t* d_shape, T* d_dist, T* d_closest);

// ---- dim4.cu: D = 4 ----
// Traversal record: the AABB the node has in its parent, `skip` (first record behind the subtree) and the shape index of a leaf.
// Sized in whole 16-byte granules so that a record is fetched with 128-bit non-coherent loads only: 3 for f32, 5 for f64.
struct __align__(16) TRec4F { float min[4]; float max[4]; uint32_t skip, shape, pad[2]; };    // 48 B
struct __align__(16) TRec4D { double min[4]; double max[4]; uint32_t skip, shape, pad[2]; };  // 80 B
static_assert(sizeof(TRec4F) == 48 && sizeof(TRec4D) == 80, "4-D record size");
static_assert(sizeof(bvh_aabb4f) == 32 && sizeof(bvh_aabb4d) == 64 && sizeof(bvh_ray4f) == 48 && sizeof(bvh_ray4d) == 96, "4-D POD size");
static_assert(sizeof(bvh_node4f) == 80 && sizeof(bvh_node4d) == 144 && sizeof(bvh_flat4f) == 44 && sizeof(bvh_flat4d) == 80, "4-D POD size");

template <class T> struct D4;
template <> struct D4<float> { using Aabb = bvh_aabb4f; using Ray = bvh_ray4f; using Node = bvh_node4f; using Flat = bvh_flat4f; using Rec = TRec4F; };
template <> struct D4<double> { using Aabb = bvh_aabb4d; using Ray = bvh_ray4d; using Node = bvh_node4d; using Flat = bvh_flat4d; using Rec = TRec4D; };

// Bvh<T,4>: its own node types and pipeline (a fourth axis cannot hide in the 3-D kernels the way D = 2 hides in z = 0).
template <class T> struct Tree4 {
    using Aabb = typename D4<T>::Aabb; using Node = typename D4<T>::Node; using Flat = typename D4<T>::Flat; using Rec = typename D4<T>::Rec;
    static constexpr int D = 4, dims = 4;
    using Scalar = T; using Box = Aabb;   // the shape boxes keep the ABI layout on the device
    bvhgpu_ctx* ctx = nullptr;
    uint32_t n = 0, n_nodes = 0;
    Aabb* d_aabb = nullptr;            // [n]      shape AABBs (ABI layout: already whole sectors)
    Node* d_nodes = nullptr;           // [2n-1]   Bvh.nodes, reference preorder layout
    uint32_t* d_node_index = nullptr;  // [n]      leaf node of every shape
    uint32_t* d_node_start = nullptr;  // [2n-1]   first position of the node's shape range (== leaves before it)
    Rec* d_tnodes = nullptr;           // [n_trec] traversal records (built on first use)
    uint32_t n_trec = 0;
    Flat* d_flat = nullptr;            // [n_flat] FlatBvh (built on demand)
    size_t n_flat = 0;
    int failed_status = 0;             // sticky (mark_failed)
    std::string failed_message;
    uint32_t* d_offsets = nullptr; size_t offsets_cap = 0;   // result buffers of the host-pointer traversal
    uint32_t* d_hits = nullptr;    size_t hits_cap = 0;
    T* d_sa_base = nullptr;            // [2n-1] surface area of every inner node when it was last (re)built: baseline of update (first update)
    uint32_t* d_arrive = nullptr;      // [2n-1] arrival counters of the incremental update (all zero between calls)
    uint8_t* d_bad = nullptr;          // [2n-1] growth flags of the incremental update (all zero between calls)
};
// The status check of a 4-D tree: its build is synchronous, so only a sticky failure (mark_failed) is left to report.
template <class T> inline int resolve_status(const Tree4<T>* t) {
    if (t->failed_status != BVHGPU_OK) set_error("%s", t->failed_message.c_str());
    return t->failed_status;
}
// The device-side drivers of dim4.cu (the CSR walks are the shared drivers declared below).  Arguments and the tree's status are
// checked by the caller unless said otherwise; everything runs on the context's stream.
// Exact SAH build of tree->n shapes (tree->n, n_nodes set, n >= 1) from `aabbs` (kind: the direction of that copy).  Synchronous.
template <class T> int build4(Tree4<T>* tree, const typename D4<T>::Aabb* aabbs, cudaMemcpyKind kind);
template <class T> int build_flat4(Tree4<T>* tree);                 // tree->n_flat; d_flat built once
// nearest_to (4 T per point); an empty tree gives BVH_INVALID and 0 for every point.
template <class T> int nearest4_device(Tree4<T>* tree, int mode, const T* d_points, size_t n, uint32_t* d_shape, T* d_dist);
// k nearest shapes: checks n, k and the tree's status, as knn_device does.
template <class T> int knn4_device(Tree4<T>* tree, const T* d_points, size_t n, uint32_t k, const T* d_max_dist, uint32_t* d_shape, T* d_dist);
// The 4-D overloads of the steps the dynamic drivers of dynamic.cu leave to the tree type (the 3-D ones are declared above):
// records and flat array, if built, rewritten in place from the new boxes
template <class T> int refresh_caches(Tree4<T>* tree);
// after a relocation: records and flat array dropped (rebuilt at the new size on first use), update buffers dropped
template <class T> int finish_relayout(Tree4<T>* tree);
// the growth rebuild of the level loop and small4_kernel of the build; *rebuilt = shapes in the rebuilt subtrees
template <class T> int rebuild_degraded(Tree4<T>* tree, const uint32_t* d_dirty, uint32_t* d_cnts, size_t* rebuilt, const char* who);
// Exact-SAH subtrees built in place under the roots d_roots[0 .. *d_n_roots) (at most max_roots): their shapes in leaf order in
// idx[0 .. n) (idx holds the builder's two index buffers, 2 n), their centre bounds as keys in cb[8 slot ..].  Synchronous.
template <class T> int build_subtrees(Tree4<T>* tree, const uint32_t* d_roots, const uint32_t* d_n_roots, uint32_t max_roots,
                                      const typename Traits<T>::Key* cb, uint32_t* idx, const char* who);

// ---- the CSR walks of every D (csr.cuh): one device driver per family over the tree type, instantiated for Tree<T> in traverse.cu
// and for Tree4<T> in dim4.cu.  Each checks, in this order, the size of the batch, the mode, the query kind, the tree's status and
// the empty input; the pointers are checked by the caller.  A call with nothing to walk (n = 0) does not wait for a build still
// running on the device: it reports only a failure that is already known.
// Where a driver leaves its CSR: device pointers (CsrOut::device), enqueued on the context's stream and synchronising only to return
// *total; or host pointers (CsrOut::to_host) through the tree's retained buffers (csr_run): the offsets always, the hits when they fit
// `cap`, otherwise BVHGPU_ERR_CAPACITY.  per_item sizes the first retained hit buffer: max(hits_cap, per_item * n, 1024).
struct CsrOut {
    uint32_t* offsets;
    uint32_t* hits;
    size_t cap;
    size_t* total;
    bool host;
    size_t per_item;
    static CsrOut device(uint32_t* d_offsets, uint32_t* d_hits, size_t cap, size_t* total) { return {d_offsets, d_hits, cap, total, false, 0}; }
    static CsrOut to_host(uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total, size_t per_item) {
        return {offsets, hits, cap, total, true, per_item};
    }
};
// Aabb / Point / Ball queries and the internal QUERY_WITHIN (queries.cuh) over `src`: records of 2D / D / D + 1 / D + 1 T.
template <class TreeT> int query_csr(TreeT* tree, int mode, int kind, const void* src, size_t n, const CsrOut& out, const char* what);
// Ray traversal of a 4-D tree (rays of 12 T): the query walk with the 4-wide slab test.  D = 2, 3 have traverse_device.
template <class T> int traverse_csr(Tree4<T>* tree, int mode, const void* rays, size_t n, const CsrOut& out, const char* what);
// Candidate lists that contain the nearest shape of every point (D T per point): the candidate bound, then QUERY_WITHIN, FLAT.
template <class TreeT> int nearest_candidates_csr(TreeT* tree, const typename TreeT::Scalar* points, size_t n, const CsrOut& out);
// Hits sorted by entry (ascending) / exit (descending) distance, with the distances (device pointers, cap entries each).
template <class TreeT> int ordered_csr(TreeT* tree, const void* rays, size_t n, int ascending, uint32_t* d_offsets, uint32_t* d_hits,
                                       typename TreeT::Scalar* d_dists, size_t cap, size_t* total);
// Every pair of shapes whose own boxes intersect, once, in the row of the earlier leaf; n < 2 gives all-zero offsets.
template <class TreeT> int overlap_csr(TreeT* tree, const CsrOut& out, const char* what);
// Every pair (a, b) of a shape of tree A and a shape of tree B whose own boxes intersect, in A's row, B's DFS order (A and B share a
// context).  A's status is checked before B's; n_a = 0 or n_b = 0 give all-zero offsets.  A host CSR uses A's retained buffers.
template <class TreeT> int overlap_trees_csr(TreeT* a, TreeT* b, const CsrOut& out, const char* what);
// The overlap rows of overlap_csr / overlap_trees_csr (D = 3) keeping only the pairs whose triangles (bvhgpu_tree_set_triangles_*)
// meet (tritri.cuh); skip_shared: the self form drops pairs that share a vertex.  A non-empty tree without triangles: BVHGPU_ERR_INVALID,
// checked after the sticky failures.  Instantiated in tripairs.cu.
template <class T> int triangle_pairs_csr(Tree<T>* tree, int skip_shared, const CsrOut& out, const char* what);
template <class T> int triangle_pairs_trees_csr(Tree<T>* a, Tree<T>* b, const CsrOut& out, const char* what);

// The steps in which the CSR drivers tell the tree types apart.
// The traversal records (d_tnodes, n_trec), built on first use.
template <class T> inline int ensure_records(Tree<T>* t) { return t->d_tnodes ? BVHGPU_OK : build_traversal_records(t); }
template <class T> int ensure_records(Tree4<T>* t);
// The shape boxes of the FLAT leaf re-test: a 2-D tree re-tests the boxes with z = [-1, +1] (dim2.cu).
template <class T> inline const typename Traits<T>::DAabb* walk_aabbs(const Tree<T>* t) { return t->dims == 2 && t->d_aabb_trav ? t->d_aabb_trav : t->d_aabb; }
template <class T> inline const typename D4<T>::Aabb* walk_aabbs(const Tree4<T>* t) { return t->d_aabb; }
// nearest_candidates' first pass: records {p, U} of D + 1 T per point, U the farthest-corner bound (nearest_bound_kernel of
// traverse.cu, nearest_bound4_kernel of dim4.cu).
template <class T> int nearest_bound(Tree<T>* t, const T* d_points, uint32_t n, T* d_records);
template <class T> int nearest_bound(Tree4<T>* t, const T* d_points, uint32_t n, T* d_records);
// The total of the last host CSR call, which bvhgpu_traverse_fetch_* and bvhgpu_traverse_stats_* of a 3-D tree read.
template <class T> inline void keep_total(Tree<T>* t, size_t total) { t->last_total = total; }
template <class T> inline void keep_total(Tree4<T>*, size_t) {}

}  // namespace bvhb200

struct bvhgpu_tree3f : bvhb200::Tree<float> {};
struct bvhgpu_tree3d : bvhb200::Tree<double> {};
struct bvhgpu_tree2f : bvhb200::Tree<float> {};
struct bvhgpu_tree2d : bvhb200::Tree<double> {};
struct bvhgpu_tree4f : bvhb200::Tree4<float> {};
struct bvhgpu_tree4d : bvhb200::Tree4<double> {};
