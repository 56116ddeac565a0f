/* ============================================================================
 * include/bvh_b200.h -- C ABI of libbvh_b200.so
 *
 * H100-native (sm_90a) replacement for the ONE data-parallel hot path of the
 * Rust crate svenstaro/bvh 0.12.0:
 *
 *     Bvh::build  ->  Bvh::flatten  ->  batched Ray traversal
 *
 * This header is the drop-in boundary: plain pointers and sizes only, so a Rust
 * shim (`impl BoundingHierarchy<T,3> for GpuBvh<T>`, see INTEGRATION.md) can bind
 * it with `extern "C"`.  Every entry point cites the reference interface it
 * replaces (file:line relative to the reference checkout).
 *
 * There is NO CPU fallback behind any of these calls: without a CUDA device
 * `bvhgpu_create` fails with BVHGPU_ERR_CUDA.
 *
 * Conventions
 *   - all functions return a bvhgpu_status (0 = ok); `bvhgpu_last_error()` gives
 *     the message for the calling thread.  The reference panics on the same
 *     conditions (NaN centroid: src/bvh/bvh_node.rs:214-217); the shim turns a
 *     non-zero status into `panic!`.
 *   - `*_dev_*` variants take DEVICE pointers, enqueue on the context's stream
 *     and do not synchronise unless they must return a host value.
 *   - n == 0 and n == 1 behave as the reference does (empty tree / root leaf,
 *     src/bvh/bvh_impl.rs:57-59, src/bvh/bvh_node.rs:95-104, 314).
 * ========================================================================== */
#ifndef BVH_B200_H
#define BVH_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BVHGPU_INVALID_INDEX 0xFFFFFFFFu /* u32::MAX sentinel, src/flat_bvh.rs:36-45 */

/* ---- POD mirrors (Rust's Aabb / Ray / BvhNode / FlatNode are not repr(C)) ---- */

/* Aabb<f32,3> / Aabb<f64,3>: src/aabb/aabb_impl.rs:10-16 */
typedef struct { float min[3]; float max[3]; } bvh_aabb3f;    /* 24 B */
typedef struct { double min[3]; double max[3]; } bvh_aabb3d;  /* 48 B */

/* Ray<T,3>: src/ray/ray_impl.rs:17-29 (direction already normalised, inv = 1/direction) */
typedef struct { float origin[3]; float direction[3]; float inv_direction[3]; } bvh_ray3f;     /* 36 B */
typedef struct { double origin[3]; double direction[3]; double inv_direction[3]; } bvh_ray3d;  /* 72 B */

/* BvhNode<T,3> (enum, src/bvh/bvh_node.rs:21-47) flattened:
 *   Leaf: child_l == child_r == BVHGPU_INVALID_INDEX, shape = shape_index, AABBs = Aabb::empty()
 *   Node: child_l / child_r = child node indices, shape = number of shapes under the node
 *         (extra information the reference does not store), l_aabb / r_aabb = child AABBs.
 * Indices are u32 (the reference uses usize; FlatNode already limits trees to u32). */
typedef struct { uint32_t parent, child_l, child_r, shape; bvh_aabb3f l_aabb, r_aabb; } bvh_node3f;  /*  64 B */
typedef struct { uint32_t parent, child_l, child_r, shape; bvh_aabb3d l_aabb, r_aabb; } bvh_node3d;  /* 112 B */

/* FlatNode<T,3>: src/flat_bvh.rs:17-46 */
typedef struct { bvh_aabb3f aabb; uint32_t entry_index, exit_index, shape_index; } bvh_flat3f;             /* 36 B */
typedef struct { bvh_aabb3d aabb; uint32_t entry_index, exit_index, shape_index, _pad; } bvh_flat3d;      /* 64 B */

/* D = 2 twins (the reference is generic in D; 2-D slab tests: src/ray/intersect_simd.rs:99-133, 181-191) */
typedef struct { float min[2]; float max[2]; } bvh_aabb2f;                                                   /* 16 B */
typedef struct { double min[2]; double max[2]; } bvh_aabb2d;                                                 /* 32 B */
typedef struct { float origin[2]; float direction[2]; float inv_direction[2]; } bvh_ray2f;                   /* 24 B */
typedef struct { double origin[2]; double direction[2]; double inv_direction[2]; } bvh_ray2d;                /* 48 B */
typedef struct { uint32_t parent, child_l, child_r, shape; bvh_aabb2f l_aabb, r_aabb; } bvh_node2f;          /* 48 B */
typedef struct { uint32_t parent, child_l, child_r, shape; bvh_aabb2d l_aabb, r_aabb; } bvh_node2d;          /* 80 B */
typedef struct { bvh_aabb2f aabb; uint32_t entry_index, exit_index, shape_index; } bvh_flat2f;               /* 28 B */
typedef struct { bvh_aabb2d aabb; uint32_t entry_index, exit_index, shape_index, _pad; } bvh_flat2d;         /* 48 B */

/* D = 4 twins (4-wide slab tests: src/ray/intersect_simd.rs:38-45, 123-133 (f32), 202-209, 226-246, 260-270 (f64)) */
typedef struct { float min[4]; float max[4]; } bvh_aabb4f;                                                   /* 32 B */
typedef struct { double min[4]; double max[4]; } bvh_aabb4d;                                                 /* 64 B */
typedef struct { float origin[4]; float direction[4]; float inv_direction[4]; } bvh_ray4f;                   /* 48 B */
typedef struct { double origin[4]; double direction[4]; double inv_direction[4]; } bvh_ray4d;                /* 96 B */
typedef struct { uint32_t parent, child_l, child_r, shape; bvh_aabb4f l_aabb, r_aabb; } bvh_node4f;          /* 80 B */
typedef struct { uint32_t parent, child_l, child_r, shape; bvh_aabb4d l_aabb, r_aabb; } bvh_node4d;          /* 144 B */
typedef struct { bvh_aabb4f aabb; uint32_t entry_index, exit_index, shape_index; } bvh_flat4f;               /* 44 B */
typedef struct { bvh_aabb4d aabb; uint32_t entry_index, exit_index, shape_index, _pad; } bvh_flat4d;         /* 80 B */

typedef enum {
    BVHGPU_OK = 0,
    BVHGPU_ERR_INVALID = 1,     /* bad argument */
    BVHGPU_ERR_CUDA = 2,        /* CUDA runtime error / no device */
    BVHGPU_ERR_NAN = 3,         /* NaN in an input AABB (reference: panic, bvh_node.rs:214-217) */
    BVHGPU_ERR_CAPACITY = 4,    /* caller buffer too small; *total / *len holds the needed size */
    BVHGPU_ERR_TIMEOUT = 5,     /* device watchdog fired */
    BVHGPU_ERR_UNSUPPORTED = 6,
    BVHGPU_ERR_INTERNAL = 7
} bvhgpu_status;

typedef enum {
    BVHGPU_BUILD_EXACT_SAH = 0, /* bit-identical to Bvh::build (6-bucket SAH, src/bvh/bvh_node.rs:81-279) */
    BVHGPU_BUILD_LBVH = 1,      /* Morton/Karras LBVH: same hit sets, different topology */
    BVHGPU_BUILD_LBVH_TREELET = 2 /* LBVH top + every subtree of <= 512 shapes rebuilt with the reference's 6-bucket SAH (shared memory) */
} bvhgpu_build_mode;

typedef enum {
    BVHGPU_TRAVERSE_BVH = 0,    /* Bvh::traverse semantics     (src/bvh/bvh_node.rs:288-319): leaves are not re-tested */
    BVHGPU_TRAVERSE_FLAT = 1    /* FlatBvh::traverse semantics (src/flat_bvh.rs:396-431): reached leaves re-test the shape AABB */
} bvhgpu_traverse_mode;

/* Ray batch layouts at the boundary.  FULL is the crate's Ray (bvh_ray3f / bvh_ray3d).  OD carries only what Ray::new keeps
 * besides the reciprocal: 6 scalars per ray {origin[3], direction[3]} with `direction` exactly as Ray stores it (normalised);
 * the device recomputes inv_direction = 1/direction with the same IEEE division Ray::new performs (src/ray/ray_impl.rs:76-78),
 * so both layouts give bit-identical results -- OD moves 24 instead of 36 bytes per f32 ray across PCIe. */
typedef enum { BVHGPU_RAYS_FULL = 0, BVHGPU_RAYS_OD = 1 } bvhgpu_ray_layout;

typedef struct bvhgpu_ctx bvhgpu_ctx;       /* one per device: stream, scratch pool           */
typedef struct bvhgpu_tree3f bvhgpu_tree3f; /* device-resident Bvh<f32,3> (+ FlatBvh, shape AABBs) */
typedef struct bvhgpu_tree3d bvhgpu_tree3d; /* device-resident Bvh<f64,3>                      */
typedef struct bvhgpu_tree2f bvhgpu_tree2f; /* device-resident Bvh<f32,2>                      */
typedef struct bvhgpu_tree2d bvhgpu_tree2d; /* device-resident Bvh<f64,2>                      */
typedef struct bvhgpu_tree4f bvhgpu_tree4f; /* device-resident Bvh<f32,4>                      */
typedef struct bvhgpu_tree4d bvhgpu_tree4d; /* device-resident Bvh<f64,4>                      */

/* ---- context ------------------------------------------------------------------ */
int bvhgpu_create(int device, bvhgpu_ctx** out);
void bvhgpu_destroy(bvhgpu_ctx* ctx);
const char* bvhgpu_last_error(void);
const char* bvhgpu_version(void);
/* Enqueue on an externally owned cudaStream_t (e.g. torch's current stream; 0 is CUDA's legacy default
 * stream and is honoured as such, on either side of a switch).  bvhgpu_reset_stream returns to the context's own stream.
 * Ordering: when the stream changes, the context records an event on the outgoing stream and makes the incoming stream
 * wait for it (no host synchronisation).  So every call on a context is ordered after every earlier call on that context,
 * on whatever stream each one ran -- builds, refits, updates, tree frees and the stream-ordered pool allocations and frees
 * inside them included.  Setting the stream the context already uses is a no-op.  If a CUDA call fails the function
 * returns BVHGPU_ERR_CUDA and the context stays on its previous stream.
 * What stays the caller's job: ordering the production of its input buffers (device rays, boxes, triangles, ...) before
 * the call, and the consumption of its output buffers after it, against the stream it installs.
 * Out of scope: switching streams while a CUDA graph is being captured, and calls on one context from several host
 * threads at once. */
int bvhgpu_set_stream(bvhgpu_ctx* ctx, void* cuda_stream);
int bvhgpu_reset_stream(bvhgpu_ctx* ctx);
/* Waits for the context's stream, and so (see bvhgpu_set_stream) for every earlier call on the context, including work
 * enqueued on streams it used before.  Also the point where errors of asynchronous multi-GPU steps surface: a peer that
 * never answered (BVHGPU_ERR_TIMEOUT) is reported here, once, and the step's result must not be used. */
int bvhgpu_synchronize(bvhgpu_ctx* ctx);
/* Pinned host memory for ray / result staging, placed on the NUMA node the device hangs off (sysfs numa_node of the
 * PCI function) -- on a two-socket host a buffer pinned on the far socket moves at a fraction of the PCIe rate. */
int bvhgpu_host_alloc(bvhgpu_ctx* ctx, size_t bytes, void** out);
int bvhgpu_host_free(bvhgpu_ctx* ctx, void* p);
/* Number of kernels this context has launched so far (bench.py's gpu_launches). */
uint64_t bvhgpu_launch_count(const bvhgpu_ctx* ctx);
/* Tunables: "traverse_slots" (per-ray hit slots of the single-pass path, 0 = two-pass count/fill, -1 = auto),
 * "traverse_persistent" (0 = one ray per thread, 1 = persistent refill kernel, 2 = decided per batch by a coherence probe),
 * "build_small" (exact builder: finish ranges of <= 16 shapes with one thread each in a second kernel; -1 auto by type and size, 0 never, 1 always),
 * "build_subtree" (exact builder: build ranges of <= 32 shapes in registers, one warp per subtree; -1 auto, 0 never, 1 always),
 * "build_gang" (exact builder: co-resident warp gangs walk the top levels behind device-wide barriers; -1 auto by size, 0 never, 1 always),
 * -- every combination produces the same bits; the switches exist for measurement (tools/build_sweep.py) --
 * "traverse_stream" (host-pointer traversal: consume the rays in a running kernel while the copy is still in flight;
 *   -1 auto = only when launches are asynchronous and no profiler / debugger / sanitizer is attached, 0 never, 1 force),
 * "traverse_top" (f32 persistent walk with the top of the tree in shared memory: -1 auto = trees with >= 5 MB of traversal records,
 *   0 never, 1 always, > 1 = always with at most that many top entries; the results are the same bits either way),
 * "walk_grid" (CTAs of the plain persistent walk; 0 = automatic: 4..8 per SM by batch size),
 * "profile" (1: bracket the dominant kernels with CUDA events, read back with bvhgpu_get_metric). */
int bvhgpu_set_option(bvhgpu_ctx* ctx, const char* name, int64_t value);
/* Measurements of the last profiled call on this context: "walk_ms" (traversal walk kernel),
 * "build_ms" (persistent SAH build kernel).  Synchronises on the recorded events. */
int bvhgpu_get_metric(bvhgpu_ctx* ctx, const char* name, double* out);

/* ---- build: replaces BoundingHierarchy::build / build_par for Bvh ----------------
 * (src/bounding_hierarchy.rs:158-177, src/bvh/bvh_impl.rs:40-96, src/bvh/bvh_node.rs:81-279).
 * `aabbs[i]` is `shapes[i].aabb()` (Bounded::aabb, src/aabb/aabb_impl.rs:55) gathered by the shim.
 * The tree stays on the device; fetch Bvh.nodes / the per-shape node indices with
 * bvhgpu_tree_nodes_*.  build_par == build (rayon is off the hot path). */
int bvhgpu_build_f32x3(bvhgpu_ctx* ctx, const bvh_aabb3f* aabbs, size_t n, int mode, bvhgpu_tree3f** out);
int bvhgpu_build_f64x3(bvhgpu_ctx* ctx, const bvh_aabb3d* aabbs, size_t n, int mode, bvhgpu_tree3d** out);
int bvhgpu_build_dev_f32x3(bvhgpu_ctx* ctx, const void* dev_aabbs, size_t n, int mode, bvhgpu_tree3f** out);
int bvhgpu_build_dev_f64x3(bvhgpu_ctx* ctx, const void* dev_aabbs, size_t n, int mode, bvhgpu_tree3d** out);

/* Upload an existing reference-layout Bvh (`Bvh.nodes` in the preorder layout Bvh::build emits:
 * child_l == i+1, src/bvh/bvh_node.rs:138-142) together with the shapes' AABBs. */
int bvhgpu_tree_from_nodes_f32x3(bvhgpu_ctx* ctx, const bvh_node3f* nodes, size_t n_nodes,
                                 const bvh_aabb3f* aabbs, size_t n, bvhgpu_tree3f** out);
int bvhgpu_tree_from_nodes_f64x3(bvhgpu_ctx* ctx, const bvh_node3d* nodes, size_t n_nodes,
                                 const bvh_aabb3d* aabbs, size_t n, bvhgpu_tree3d** out);

void bvhgpu_tree_free_f32x3(bvhgpu_tree3f* tree);
void bvhgpu_tree_free_f64x3(bvhgpu_tree3d* tree);
size_t bvhgpu_tree_num_shapes_f32x3(const bvhgpu_tree3f* tree);
size_t bvhgpu_tree_num_shapes_f64x3(const bvhgpu_tree3d* tree);
size_t bvhgpu_tree_num_nodes_f32x3(const bvhgpu_tree3f* tree);   /* 2n-1 (0 for n == 0) */
size_t bvhgpu_tree_num_nodes_f64x3(const bvhgpu_tree3d* tree);

/* Materialise `Bvh.nodes` (pub field, src/bvh/bvh_impl.rs:27-33) and the leaf node index of every
 * shape (BHShape::set_bh_node_index, src/bounding_hierarchy.rs:58; written at src/bvh/bvh_node.rs:103).
 * Either pointer may be NULL. */
int bvhgpu_tree_nodes_f32x3(bvhgpu_tree3f* tree, bvh_node3f* out_nodes, uint32_t* out_node_index);
int bvhgpu_tree_nodes_f64x3(bvhgpu_tree3d* tree, bvh_node3d* out_nodes, uint32_t* out_node_index);

/* ---- D = 2: Bvh<T,2>::build / nodes / flatten / traverse (SURVEY.md 8f N4).  Host pointers; semantics, modes, error codes and
 * the CSR output exactly as the 3-D entry points above.  The scene is embedded in the plane z = 0 of the 3-D kernels in a way that
 * reproduces the 2-D arithmetic bit for bit (dim2.cu). */
int bvhgpu_build_f32x2(bvhgpu_ctx* ctx, const bvh_aabb2f* aabbs, size_t n, int mode, bvhgpu_tree2f** out);
int bvhgpu_build_f64x2(bvhgpu_ctx* ctx, const bvh_aabb2d* aabbs, size_t n, int mode, bvhgpu_tree2d** out);
void bvhgpu_tree_free_f32x2(bvhgpu_tree2f* tree);
void bvhgpu_tree_free_f64x2(bvhgpu_tree2d* tree);
size_t bvhgpu_tree_num_shapes_f32x2(const bvhgpu_tree2f* tree);
size_t bvhgpu_tree_num_shapes_f64x2(const bvhgpu_tree2d* tree);
int bvhgpu_tree_nodes_f32x2(bvhgpu_tree2f* tree, bvh_node2f* out_nodes, uint32_t* out_node_index);
int bvhgpu_tree_nodes_f64x2(bvhgpu_tree2d* tree, bvh_node2d* out_nodes, uint32_t* out_node_index);
int bvhgpu_flatten_f32x2(bvhgpu_tree2f* tree, bvh_flat2f* out, size_t cap, size_t* len);
int bvhgpu_flatten_f64x2(bvhgpu_tree2d* tree, bvh_flat2d* out, size_t cap, size_t* len);
int bvhgpu_traverse_f32x2(bvhgpu_tree2f* tree, int mode, const bvh_ray2f* rays, size_t nrays,
                          uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_traverse_f64x2(bvhgpu_tree2d* tree, int mode, const bvh_ray2d* rays, size_t nrays,
                          uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
/* D = 2 queries and nearest_to: the semantics of bvhgpu_query_f32x3 / bvhgpu_nearest_f32x3 / bvhgpu_nearest_candidates_f32x3 below
 * (section "the other IntersectsAabb implementors" and section "nearest_to") with 2 components, host pointers.  Query records:
 * Aabb {min, max} = 4 T, Point = 2 T, Ball {center, radius} = 3 T; nearest points: 2 T.  The records are lifted to z = 0 and run
 * through the 3-D kernels on the embedded tree; every z term is exactly neutral, so the results are the 2-D ones bit for bit (dim2.cu).
 * `kind` outside 1..3, a bad mode, a null argument or n > 2^31-1: BVHGPU_ERR_INVALID, nothing is read or written.  There is no fetch
 * call: when the hits (candidates) do not fit `cap`, offsets and *total are valid and the call returns BVHGPU_ERR_CAPACITY; call
 * again with cap = *total. */
int bvhgpu_query_f32x2(bvhgpu_tree2f* tree, int mode, int kind, const float* queries, size_t n,
                       uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_query_f64x2(bvhgpu_tree2d* tree, int mode, int kind, const double* queries, size_t n,
                       uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_nearest_f32x2(bvhgpu_tree2f* tree, int mode, const float* points, size_t n, uint32_t* out_shape, float* out_dist);
int bvhgpu_nearest_f64x2(bvhgpu_tree2d* tree, int mode, const double* points, size_t n, uint32_t* out_shape, double* out_dist);
int bvhgpu_nearest_candidates_f32x2(bvhgpu_tree2f* tree, const float* points, size_t n, uint32_t* offsets, uint32_t* cand,
                                    size_t cap, size_t* total);
int bvhgpu_nearest_candidates_f64x2(bvhgpu_tree2d* tree, const double* points, size_t n, uint32_t* offsets, uint32_t* cand,
                                    size_t cap, size_t* total);

/* ---- D = 4: Bvh<T,4>::build / nodes / flatten / traverse (the reference is generic in D, src/bvh/bvh_node.rs:81-279,
 * src/flat_bvh.rs:60-143, 396-431; 4-wide slab tests src/ray/intersect_simd.rs; generic slab test src/ray/intersect_default.rs:16-37).
 * Its own device pipeline (dim4.cu): a fourth axis cannot be embedded in the 3-D kernels.  Semantics, error codes and the CSR output as
 * the 3-D entry points, except:
 *   - build: only BVHGPU_BUILD_EXACT_SAH exists (bit-identical to Bvh<T,4>::build); the LBVH modes return BVHGPU_ERR_UNSUPPORTED.
 *     NaN in any coordinate: BVHGPU_ERR_NAN; n > 2^30 or a null argument: BVHGPU_ERR_INVALID.  The build is synchronous and a build
 *     that fails hands out no tree.  Node layout, leaves and inner-node `shape` (= shapes below the node) as bvh_node3f.
 *   - traverse: there is no fetch call.  When the hits do not fit `cap`, offsets and *total are valid and the call returns
 *     BVHGPU_ERR_CAPACITY; call again with cap = *total.  BVHGPU_TRAVERSE_BVH re-tests the shape AABB only at a root leaf
 *     (src/bvh/bvh_node.rs:314), BVHGPU_TRAVERSE_FLAT at every reached leaf.
 *   - traverse_dev: device pointers, enqueued on the context's stream; `total` may be NULL (no host synchronisation); hits beyond
 *     `cap` are dropped, as bvhgpu_traverse_dev_f32x3. */
int bvhgpu_build_f32x4(bvhgpu_ctx* ctx, const bvh_aabb4f* aabbs, size_t n, int mode, bvhgpu_tree4f** out);
int bvhgpu_build_f64x4(bvhgpu_ctx* ctx, const bvh_aabb4d* aabbs, size_t n, int mode, bvhgpu_tree4d** out);
void bvhgpu_tree_free_f32x4(bvhgpu_tree4f* tree);
void bvhgpu_tree_free_f64x4(bvhgpu_tree4d* tree);
size_t bvhgpu_tree_num_shapes_f32x4(const bvhgpu_tree4f* tree);
size_t bvhgpu_tree_num_shapes_f64x4(const bvhgpu_tree4d* tree);
int bvhgpu_tree_nodes_f32x4(bvhgpu_tree4f* tree, bvh_node4f* out_nodes, uint32_t* out_node_index);
int bvhgpu_tree_nodes_f64x4(bvhgpu_tree4d* tree, bvh_node4d* out_nodes, uint32_t* out_node_index);
int bvhgpu_flatten_f32x4(bvhgpu_tree4f* tree, bvh_flat4f* out, size_t cap, size_t* len);
int bvhgpu_flatten_f64x4(bvhgpu_tree4d* tree, bvh_flat4d* out, size_t cap, size_t* len);
int bvhgpu_traverse_f32x4(bvhgpu_tree4f* tree, int mode, const bvh_ray4f* rays, size_t nrays,
                          uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_traverse_f64x4(bvhgpu_tree4d* tree, int mode, const bvh_ray4d* rays, size_t nrays,
                          uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_traverse_dev_f32x4(bvhgpu_tree4f* tree, int mode, const void* dev_rays, size_t nrays,
                              void* dev_offsets, void* dev_hits, size_t cap, size_t* total);
int bvhgpu_traverse_dev_f64x4(bvhgpu_tree4d* tree, int mode, const void* dev_rays, size_t nrays,
                              void* dev_offsets, void* dev_hits, size_t cap, size_t* total);
/* D = 4 queries and nearest_to: the semantics of the 3-D functions (section "the other IntersectsAabb implementors" and section
 * "nearest_to") with 4 components, run by dim4.cu's own kernels.  Query records: Aabb {min, max} = 8 T, Point = 4 T,
 * Ball {center, radius} = 5 T; nearest points: 4 T.  `kind` outside 1..3, a bad mode, a null argument or n > 2^31-1:
 * BVHGPU_ERR_INVALID, nothing is read or written.  An empty tree gives all-zero offsets; nearest gives BVHGPU_INVALID_INDEX and
 * distance 0.  Host forms: no fetch call; when the hits (candidates) do not fit `cap`, offsets and *total are valid and the call
 * returns BVHGPU_ERR_CAPACITY; call again with cap = *total.  query_dev: device pointers, enqueued on the context's stream, the
 * contract of bvhgpu_query_dev_f32x3 (offsets always complete, hits[0 .. cap) a prefix of the full list, `total` may be NULL: then
 * there is no host synchronisation). */
int bvhgpu_query_f32x4(bvhgpu_tree4f* tree, int mode, int kind, const float* queries, size_t n,
                       uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_query_f64x4(bvhgpu_tree4d* tree, int mode, int kind, const double* queries, size_t n,
                       uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_query_dev_f32x4(bvhgpu_tree4f* tree, int mode, int kind, const void* dev_queries, size_t n,
                           void* dev_offsets, void* dev_hits, size_t cap, size_t* total);
int bvhgpu_query_dev_f64x4(bvhgpu_tree4d* tree, int mode, int kind, const void* dev_queries, size_t n,
                           void* dev_offsets, void* dev_hits, size_t cap, size_t* total);
int bvhgpu_nearest_f32x4(bvhgpu_tree4f* tree, int mode, const float* points, size_t n, uint32_t* out_shape, float* out_dist);
int bvhgpu_nearest_f64x4(bvhgpu_tree4d* tree, int mode, const double* points, size_t n, uint32_t* out_shape, double* out_dist);
int bvhgpu_nearest_candidates_f32x4(bvhgpu_tree4f* tree, const float* points, size_t n, uint32_t* offsets, uint32_t* cand,
                                    size_t cap, size_t* total);
int bvhgpu_nearest_candidates_f64x4(bvhgpu_tree4d* tree, const double* points, size_t n, uint32_t* offsets, uint32_t* cand,
                                    size_t cap, size_t* total);

/* ---- D = 2 and D = 4 refit and update_shapes (Bvh::update_shapes and its refit fix_aabbs_ascending, src/bvh/optimization.rs:17,
 * 304-351, generic in D).  The contract of bvhgpu_refit_f32x3 / bvhgpu_update_f32x3 below, with D components:
 *   - refit: `aabbs` are the new boxes of all n shapes; every node's child boxes are recomputed bottom-up.  Topology, node indices and
 *     node_start are kept; leaves keep their Aabb::empty() child boxes.  n != the tree's shape count: BVHGPU_ERR_INVALID.
 *   - update: `changed[i]` is a shape index, `changed_aabbs[i]` its new box; only the root paths of the changed leaves are refitted.
 *     max_growth >= 1: then the outermost subtrees that hold a node whose surface area grew by more than max_growth are rebuilt in
 *     place with the exact builder (the node array stays in Bvh::build's preorder layout; node indices of the shapes in them change).
 *     Growth is judged against the surface area every node had when it was last (re)built; the baseline is taken at the first update,
 *     so slow drift over many calls adds up.  max_growth <= 0: boxes only.  0 < max_growth < 1: BVHGPU_ERR_INVALID.  *rebuilt (may
 *     be NULL) = number of shapes in the rebuilt subtrees.  m = 0 is a no-op.
 *   - every changed index (< n) and every new box (no NaN) is checked on the device, and the verdict read back, before anything is
 *     written: a refused call (BVHGPU_ERR_INVALID / BVHGPU_ERR_NAN) leaves the tree byte for byte as it was.
 *   - traversal records and the flat array built by earlier traverse / query / flatten / nearest_to calls are rewritten in place, so
 *     every later call sees the new boxes.
 *   - a failure after the tree was modified is sticky, as a failed build's.
 * D = 2 runs the 3-D refit and update on the tree embedded in z = [0, 0] (exact, dim2.cu); host pointers only.  D = 4 has its own
 * kernels (dim4.cu) and rebuilds with the 4-D exact builder; the calls are synchronous (the builder reads one word per level).
 * update_dev / refit_dev: device pointers (C-ABI layout), enqueued on the context's stream. */
int bvhgpu_refit_f32x2(bvhgpu_tree2f* tree, const bvh_aabb2f* aabbs, size_t n);
int bvhgpu_refit_f64x2(bvhgpu_tree2d* tree, const bvh_aabb2d* aabbs, size_t n);
int bvhgpu_update_f32x2(bvhgpu_tree2f* tree, const uint32_t* changed, const bvh_aabb2f* changed_aabbs, size_t m, double max_growth, size_t* rebuilt);
int bvhgpu_update_f64x2(bvhgpu_tree2d* tree, const uint32_t* changed, const bvh_aabb2d* changed_aabbs, size_t m, double max_growth, size_t* rebuilt);
int bvhgpu_refit_f32x4(bvhgpu_tree4f* tree, const bvh_aabb4f* aabbs, size_t n);
int bvhgpu_refit_f64x4(bvhgpu_tree4d* tree, const bvh_aabb4d* aabbs, size_t n);
int bvhgpu_refit_dev_f32x4(bvhgpu_tree4f* tree, const void* dev_aabbs, size_t n);
int bvhgpu_refit_dev_f64x4(bvhgpu_tree4d* tree, const void* dev_aabbs, size_t n);
int bvhgpu_update_f32x4(bvhgpu_tree4f* tree, const uint32_t* changed, const bvh_aabb4f* changed_aabbs, size_t m, double max_growth, size_t* rebuilt);
int bvhgpu_update_f64x4(bvhgpu_tree4d* tree, const uint32_t* changed, const bvh_aabb4d* changed_aabbs, size_t m, double max_growth, size_t* rebuilt);
int bvhgpu_update_dev_f32x4(bvhgpu_tree4f* tree, const void* dev_changed, const void* dev_changed_aabbs, size_t m, double max_growth, size_t* rebuilt);
int bvhgpu_update_dev_f64x4(bvhgpu_tree4d* tree, const void* dev_changed, const void* dev_changed_aabbs, size_t m, double max_growth, size_t* rebuilt);

/* ---- D = 2 and D = 4 add / remove shapes (Bvh::add_shape / Bvh::remove_shape, src/bvh/optimization.rs:67-301, generic in D).  The
 * contract of bvhgpu_add_shapes_f32x3 / bvhgpu_remove_shapes_f32x3 below, with D components: the descent, the grafts (exact-SAH
 * subtrees over the shapes that chose one insertion point), the growth test and rebuild with max_growth >= 1, the contraction and the
 * swap renumbering of remove, the checks before the tree is touched (NaN, indices >= n, duplicates, k > n, n + k > 2^30,
 * 0 < max_growth < 1), *rebuilt = shapes in the subtrees rebuilt by the growth test, k = 0 is a no-op, add to an empty tree is
 * bvhgpu_build_*, removing every shape leaves the tree of an n = 0 build, a failure after the tree was modified is sticky.  Traversal
 * records and flat arrays built earlier follow the new tree.  The node index of every shape may change: re-read them with
 * bvhgpu_tree_nodes_* after every call.
 * D = 2 runs the 3-D add / remove on the tree embedded in z = [0, 0] (exact, dim2.cu); host pointers only.  D = 4 has its own drivers
 * (dim4.cu) and builds the group subtrees and the growth rebuilds with the 4-D exact builder; the calls are synchronous (the builder
 * reads one word per level).  _dev_: inputs on the device (C-ABI layout). */
int bvhgpu_add_shapes_f32x2(bvhgpu_tree2f* tree, const bvh_aabb2f* aabbs, size_t k, double max_growth, size_t* rebuilt);
int bvhgpu_add_shapes_f64x2(bvhgpu_tree2d* tree, const bvh_aabb2d* aabbs, size_t k, double max_growth, size_t* rebuilt);
int bvhgpu_remove_shapes_f32x2(bvhgpu_tree2f* tree, const uint32_t* indices, size_t k);
int bvhgpu_remove_shapes_f64x2(bvhgpu_tree2d* tree, const uint32_t* indices, size_t k);
int bvhgpu_add_shapes_f32x4(bvhgpu_tree4f* tree, const bvh_aabb4f* aabbs, size_t k, double max_growth, size_t* rebuilt);
int bvhgpu_add_shapes_f64x4(bvhgpu_tree4d* tree, const bvh_aabb4d* aabbs, size_t k, double max_growth, size_t* rebuilt);
int bvhgpu_add_shapes_dev_f32x4(bvhgpu_tree4f* tree, const void* dev_aabbs, size_t k, double max_growth, size_t* rebuilt);
int bvhgpu_add_shapes_dev_f64x4(bvhgpu_tree4d* tree, const void* dev_aabbs, size_t k, double max_growth, size_t* rebuilt);
int bvhgpu_remove_shapes_f32x4(bvhgpu_tree4f* tree, const uint32_t* indices, size_t k);
int bvhgpu_remove_shapes_f64x4(bvhgpu_tree4d* tree, const uint32_t* indices, size_t k);
int bvhgpu_remove_shapes_dev_f32x4(bvhgpu_tree4f* tree, const void* dev_indices, size_t k);
int bvhgpu_remove_shapes_dev_f64x4(bvhgpu_tree4d* tree, const void* dev_indices, size_t k);

/* ---- D = 2 and D = 4 distance-ordered traversal and closest hit (Bvh::nearest_traverse_iterator / farthest_traverse_iterator and
 * the child variants, src/bvh/bvh_impl.rs:145-220, src/bvh/distance_traverse.rs, child_distance_traverse.rs, over
 * Ray::intersection_slice_for_aabb, src/ray/ray_impl.rs:118-145, all generic in D).  The contract of bvhgpu_traverse_ordered_f32x3
 * and of bvhgpu_closest_hit_f32x3 with use_triangles == 0 below, with D components: the set of bvhgpu_traverse_* in BVH semantics
 * with its offsets, sorted by entry distance ascending (`ascending` != 0) or exit distance descending of the child box the tree stores
 * for each leaf (empty boxes of "no split wins" nodes: entry 0 / exit +inf), ties in DFS order, that distance in `dists`; closest =
 * the shape whose own AABB the ray enters first, key (entry distance, DFS order), exact, BVHGPU_INVALID_INDEX / +inf without a hit.
 * Differences:
 *   - there is no triangle mode: Ray::intersects_triangle needs a 3-D cross product.  (The primitives of a 2-D tree are the segments
 *     of bvhgpu_tree_set_segments_*x2, which serve point-in-polygon, k nearest segments and signed distance: see "polygons" below.)
 *   - a null argument or nrays > 2^31-1: BVHGPU_ERR_INVALID, nothing is read or written.  An empty tree gives all-zero offsets or
 *     no-hit results; a root leaf (n = 1) is decided by the shape's own box, as in the reference.
 *   - ordered, host pointers, `cap` entries in hits and dists: there is no fetch call.  When the hits do not fit `cap`, offsets and
 *     *total are valid and the call returns BVHGPU_ERR_CAPACITY; call again with cap = *total.
 *   - D = 2: ordered runs the 3-D kernel on the tree embedded in z = 0 (exact, dim2.cu); closest tests x and y of the embedded tree
 *     and reads the 2-D rays as they are.  Host pointers only.
 *   - closest_hit_dev (D = 4 only): device pointers, full 4-D rays (12 T), enqueued on the context's stream, no synchronisation.
 *     A sticky failure of the tree is reported as by the other 4-D calls. */
int bvhgpu_traverse_ordered_f32x2(bvhgpu_tree2f* tree, const bvh_ray2f* rays, size_t nrays, int ascending,
                                  uint32_t* offsets, uint32_t* hits, float* dists, size_t cap, size_t* total);
int bvhgpu_traverse_ordered_f64x2(bvhgpu_tree2d* tree, const bvh_ray2d* rays, size_t nrays, int ascending,
                                  uint32_t* offsets, uint32_t* hits, double* dists, size_t cap, size_t* total);
int bvhgpu_traverse_ordered_f32x4(bvhgpu_tree4f* tree, const bvh_ray4f* rays, size_t nrays, int ascending,
                                  uint32_t* offsets, uint32_t* hits, float* dists, size_t cap, size_t* total);
int bvhgpu_traverse_ordered_f64x4(bvhgpu_tree4d* tree, const bvh_ray4d* rays, size_t nrays, int ascending,
                                  uint32_t* offsets, uint32_t* hits, double* dists, size_t cap, size_t* total);
int bvhgpu_closest_hit_f32x2(bvhgpu_tree2f* tree, const bvh_ray2f* rays, size_t nrays, uint32_t* out_shape, float* out_dist);
int bvhgpu_closest_hit_f64x2(bvhgpu_tree2d* tree, const bvh_ray2d* rays, size_t nrays, uint32_t* out_shape, double* out_dist);
int bvhgpu_closest_hit_f32x4(bvhgpu_tree4f* tree, const bvh_ray4f* rays, size_t nrays, uint32_t* out_shape, float* out_dist);
int bvhgpu_closest_hit_f64x4(bvhgpu_tree4d* tree, const bvh_ray4d* rays, size_t nrays, uint32_t* out_shape, double* out_dist);
int bvhgpu_closest_hit_dev_f32x4(bvhgpu_tree4f* tree, const void* dev_rays, size_t nrays, void* dev_shape, void* dev_dist);
int bvhgpu_closest_hit_dev_f64x4(bvhgpu_tree4d* tree, const void* dev_rays, size_t nrays, void* dev_shape, void* dev_dist);

/* ---- flatten: replaces Bvh::flatten (src/flat_bvh.rs:60-143, 240-251, 312-319) -----
 * Writes the FlatBvh (3n-2 FlatNodes for n >= 2, 1 for n == 1, 0 for n == 0) into `out`
 * (may be NULL to only build the device copy) and its length into *len. */
int bvhgpu_flatten_f32x3(bvhgpu_tree3f* tree, bvh_flat3f* out, size_t cap, size_t* len);
int bvhgpu_flatten_f64x3(bvhgpu_tree3d* tree, bvh_flat3d* out, size_t cap, size_t* len);

/* ---- traverse: batched Bvh::traverse / FlatBvh::traverse for Ray queries -----------
 * (src/bvh/bvh_impl.rs:104-119, src/bvh/bvh_node.rs:288-319, src/flat_bvh.rs:396-431,
 *  slab test src/ray/intersect_default.rs:16-37).
 * Output is CSR: hits of ray r are hits[offsets[r] .. offsets[r+1]) = shape indices in the
 * reference's DFS (left-first) order.  If the hit list does not fit `cap`, offsets and *total
 * are still valid, the call returns BVHGPU_ERR_CAPACITY and bvhgpu_traverse_fetch_* can copy the
 * retained result without traversing again.  Shape AABBs are the ones given at build time. */
int bvhgpu_traverse_f32x3(bvhgpu_tree3f* tree, int mode, const bvh_ray3f* rays, size_t nrays,
                          uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_traverse_f64x3(bvhgpu_tree3d* tree, int mode, const bvh_ray3d* rays, size_t nrays,
                          uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_traverse_fetch_f32x3(bvhgpu_tree3f* tree, uint32_t* hits, size_t cap);
int bvhgpu_traverse_fetch_f64x3(bvhgpu_tree3d* tree, uint32_t* hits, size_t cap);
/* The same with the compact ray layout BVHGPU_RAYS_OD: `origin_dir` holds 6 scalars per ray. */
int bvhgpu_traverse_od_f32x3(bvhgpu_tree3f* tree, int mode, const float* origin_dir, size_t nrays,
                             uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_traverse_od_f64x3(bvhgpu_tree3d* tree, int mode, const double* origin_dir, size_t nrays,
                             uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
/* Device-resident variant: rays / offsets / hits are device pointers.  `total` may be NULL
 * (no host synchronisation); hits beyond `cap` are dropped and reported through *total. */
int bvhgpu_traverse_dev_f32x3(bvhgpu_tree3f* tree, int mode, const void* dev_rays, size_t nrays,
                              void* dev_offsets, void* dev_hits, size_t cap, size_t* total);
int bvhgpu_traverse_dev_f64x3(bvhgpu_tree3d* tree, int mode, const void* dev_rays, size_t nrays,
                              void* dev_offsets, void* dev_hits, size_t cap, size_t* total);
int bvhgpu_traverse_od_dev_f32x3(bvhgpu_tree3f* tree, int mode, const void* dev_origin_dir, size_t nrays,
                                 void* dev_offsets, void* dev_hits, size_t cap, size_t* total);
int bvhgpu_traverse_od_dev_f64x3(bvhgpu_tree3d* tree, int mode, const void* dev_origin_dir, size_t nrays,
                                 void* dev_offsets, void* dev_hits, size_t cap, size_t* total);
/* ---- multi-GPU ray sharding with the exchange fused into the traversal (no NCCL on the data path) -------------
 * Every rank owns a contiguous shard of the ray batch and a replica of the tree.  Every rank ends the step with its own
 * copy of the GLOBAL CSR in original ray order -- the all-gather of hit lists north_star asks for -- built over peer
 * memory (buffers allocated with bvhgpu_peer_alloc and opened on the other ranks through CUDA IPC):
 *   1. the scan kernel behind the local walk stores every 2048-ray tile's hit COUNTS, narrowed to 1 / 2 / 4 bytes by the
 *      tile's largest count, into every rank's staging (8/16-byte P2P stores over NVLink); its last block adds the table of
 *      tile offsets and publishes the rank's hit total in all mailboxes;
 *   2. the emit kernel waits for the peers' posts (which fixes its hit base), writes its hit lists into its own copy of
 *      the global hit buffer, and every block ships its contiguous piece to all peers with whole 16-byte P2P stores
 *      (4-byte stores scattered straight from the emit loop reach only a small fraction of the NVLink rate); the last
 *      block raises the done flags;
 *   3. extra blocks of the same launch rebuild the global u32 offsets on every rank from the staged counts (1 byte per ray
 *      crossed NVLink instead of 4) and end the step by waiting for the peers' done flags: when the stream reaches the end of
 *      the step, this rank's copy of the global CSR is complete.  Same number of launches as a single-GPU step.
 * `seq` must increase by one per call on all ranks, starting at 1: seq 0 is refused with BVHGPU_ERR_INVALID (the mailbox
 * starts zeroed, so a wait for 0 would pass before any peer posted).  Every argument check (rank / world, seq, ray_layout, a
 * null peer buffer or offsets, an empty shard, shard_rays[rank] != nrays) fails before the call enqueues anything.  No host
 * synchronisation; failures (a peer that never answers) are reported by bvhgpu_synchronize.  A global hit total past 2^32
 * leaves every offset at or past 2^32 as 0xFFFFFFFF (the closing entry included).  Mailbox layout (trace words for diagnostics
 * included): traverse.cu. */
#define BVHGPU_MAX_PEERS 8
#define BVHGPU_MAILBOX_BYTES 65536
#define BVHGPU_IPC_HANDLE_BYTES 64
#define BVHGPU_SHARD_STAGE_BYTES(nrays_global) ((8200 * ((size_t)(nrays_global) / 2048 + 2 * BVHGPU_MAX_PEERS) + 255) & ~(size_t)255)
typedef struct {
    int rank, world;
    void* peer_counts[BVHGPU_MAX_PEERS];    /* 2 * BVHGPU_SHARD_STAGE_BYTES(nrays_global) on every rank (index = rank): two halves, alternating per step */
    void* peer_hits[BVHGPU_MAX_PEERS];      /* u32[cap] on every rank: the global hit lists                          */
    void* peer_mailbox[BVHGPU_MAX_PEERS];   /* BVHGPU_MAILBOX_BYTES on every rank, zero-initialised                  */
    void* offsets;                          /* LOCAL device memory, u32[nrays_global + 1]: the global CSR offsets     */
    uint64_t seq;                           /* 1, 2, 3, ... identical on all ranks for the same step (0: refused)    */
    size_t shard_rays[BVHGPU_MAX_PEERS];    /* rays of every rank's shard (shard_rays[rank] == nrays of the call)     */
    size_t cap;                             /* capacity of the global hit buffers                                    */
    int ray_layout;                         /* bvhgpu_ray_layout of dev_rays                                         */
} bvhgpu_shard;
int bvhgpu_traverse_sharded_dev_f32x3(bvhgpu_tree3f* tree, int mode, const void* dev_rays, size_t nrays, const bvhgpu_shard* shard);
int bvhgpu_traverse_sharded_dev_f64x3(bvhgpu_tree3d* tree, int mode, const void* dev_rays, size_t nrays, const bvhgpu_shard* shard);
/* Peer-mappable device memory (plain cudaMalloc + cudaIpcGetMemHandle / cudaIpcOpenMemHandle). */
int bvhgpu_peer_alloc(bvhgpu_ctx* ctx, size_t bytes, void** dev_ptr, void* handle64);
int bvhgpu_peer_open(bvhgpu_ctx* ctx, const void* handle64, void** dev_ptr);
int bvhgpu_peer_close(bvhgpu_ctx* ctx, void* dev_ptr);
int bvhgpu_peer_free(bvhgpu_ctx* ctx, void* dev_ptr);
/* Synchronous device -> host copy on the context's stream (lets a binding read peer-allocated buffers). */
int bvhgpu_memcpy_d2h(bvhgpu_ctx* ctx, void* host_dst, const void* dev_src, size_t bytes);
/* Asynchronous host -> device copy on the context's stream (host memory should be pinned: bvhgpu_host_alloc). */
int bvhgpu_memcpy_h2d_async(bvhgpu_ctx* ctx, void* dev_dst, const void* host_src, size_t bytes);

/* Counters of the last traversal on this tree: [0] node records visited, [1] hits. */
int bvhgpu_traverse_stats_f32x3(bvhgpu_tree3f* tree, uint64_t* out2);
int bvhgpu_traverse_stats_f64x3(bvhgpu_tree3d* tree, uint64_t* out2);

/* ---- the other IntersectsAabb implementors as batched queries (SURVEY.md 8f N2) ------------------------------
 * Bvh::traverse / FlatBvh::traverse with an Aabb (src/aabb/aabb_impl.rs:240-248, src/aabb/intersection.rs:35-39),
 * a Point (Aabb::contains, src/aabb/aabb_impl.rs:175-177, intersection.rs:41-45) or a Ball (src/ball.rs:85-106) as the
 * query.  `queries` holds n records of 6 T {min,max}, 3 T {point} or 4 T {center, radius}.  Output: CSR as for rays.
 * `kind` other than the three below: BVHGPU_ERR_INVALID, nothing is read or written.
 * query_dev: device pointers, enqueued on the context's stream.  `total` may be NULL (no host synchronisation, no capacity
 * check).  The offsets are always complete; hits[0 .. cap) receives the first `cap` entries of the full CSR hit list (a prefix:
 * the hits at positions >= cap are dropped).  With `total` given and more than `cap` hits, *total holds the full count and the
 * call returns BVHGPU_ERR_CAPACITY. */
typedef enum { BVHGPU_QUERY_AABB = 1, BVHGPU_QUERY_POINT = 2, BVHGPU_QUERY_BALL = 3 } bvhgpu_query_kind;
int bvhgpu_query_f32x3(bvhgpu_tree3f* tree, int mode, int kind, const float* queries, size_t n,
                       uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_query_f64x3(bvhgpu_tree3d* tree, int mode, int kind, const double* queries, size_t n,
                       uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_query_dev_f32x3(bvhgpu_tree3f* tree, int mode, int kind, const void* dev_queries, size_t n,
                           void* dev_offsets, void* dev_hits, size_t cap, size_t* total);
int bvhgpu_query_dev_f64x3(bvhgpu_tree3d* tree, int mode, int kind, const void* dev_queries, size_t n,
                           void* dev_offsets, void* dev_hits, size_t cap, size_t* total);

/* ---- distance-ordered traversal (SURVEY.md 8f N3): batched counterpart of Bvh::nearest_traverse_iterator /
 * farthest_traverse_iterator (src/bvh/distance_traverse.rs, src/bvh/bvh_impl.rs).  Per ray: the same set as
 * bvhgpu_traverse_* in BVH semantics, sorted by the entry distance ascending
 * (`ascending` != 0) or the exit distance descending of the child box the tree stores for each leaf, with that distance in
 * `dists` (Ray::intersection_slice_for_aabb, src/ray/ray_impl.rs:118-145; distance_traverse.rs:100-116 slices the same box).
 * On tight trees that box is the shape's AABB.  Where surface areas overflow, "no split wins" nodes store Aabb::empty()
 * children, which every ray passes at entry 0 / exit inf: those leaves are listed whether or not the ray hits the shape itself.
 * The reference iterator is best-effort ("not necessarily perfectly sorted"); this result is perfectly sorted, ties in the
 * reference's DFS order.  Host pointers; `cap` entries in hits and dists. */
int bvhgpu_traverse_ordered_f32x3(bvhgpu_tree3f* tree, const bvh_ray3f* rays, size_t nrays, int ascending,
                                  uint32_t* offsets, uint32_t* hits, float* dists, size_t cap, size_t* total);
int bvhgpu_traverse_ordered_f64x3(bvhgpu_tree3d* tree, const bvh_ray3d* rays, size_t nrays, int ascending,
                                  uint32_t* offsets, uint32_t* hits, double* dists, size_t cap, size_t* total);

/* ---- closest hit with distance pruning (SURVEY.md 8f N3): what callers of the reference build from Bvh::traverse (or the distance
 * iterators, src/bvh/distance_traverse.rs, child_distance_traverse.rs) + Ray::intersects_triangle (src/ray/ray_impl.rs:154-213; the
 * loop itself: src/bvh/iter.rs:330-365) -- per ray, front to back, subtrees entered behind the best hit are never opened.
 *   use_triangles == 0: out_shape = the shape whose AABB the ray enters first, key (entry distance as
 *       Ray::intersection_slice_for_aabb, src/ray/ray_impl.rs:118-145, then DFS order) = the first element of a perfectly sorted
 *       nearest_traverse_iterator; out_dist = that entry distance.  Exact (ties are never pruned).
 *   use_triangles != 0: the triangles given with bvhgpu_tree_set_triangles_* (9 scalars per shape: a, b, c; shape i's AABB must
 *       contain triangle i); out_shape = the triangle with the smallest Moeller-Trumbore distance (backface culled, the reference's
 *       operation order, no FMA), ties to the lower index; out_dist = that distance, out_uv (may be NULL) = its u, v.  A subtree is
 *       skipped when its entry distance exceeds best * (1 + 2^-16).  The result G differs from the unpruned minimum W (the loop over
 *       Bvh::traverse) only where W's Moeller-Trumbore distance lies more than 2^-16 in front of the slab entry of W's own AABB
 *       (grazing hits); then d_W <= d_G, that entry exceeds fl(d_G * (1 + 2^-16)), and W's exact intersection lies behind d_G.
 * No hit: out_shape = BVHGPU_INVALID_INDEX, out_dist = +inf. */
int bvhgpu_tree_set_triangles_f32x3(bvhgpu_tree3f* tree, const float* triangles, size_t n);
int bvhgpu_tree_set_triangles_f64x3(bvhgpu_tree3d* tree, const double* triangles, size_t n);
int bvhgpu_tree_set_triangles_dev_f32x3(bvhgpu_tree3f* tree, const void* dev_triangles, size_t n);
int bvhgpu_tree_set_triangles_dev_f64x3(bvhgpu_tree3d* tree, const void* dev_triangles, size_t n);
int bvhgpu_closest_hit_f32x3(bvhgpu_tree3f* tree, const bvh_ray3f* rays, size_t nrays, int use_triangles,
                             uint32_t* out_shape, float* out_dist, float* out_uv);
int bvhgpu_closest_hit_f64x3(bvhgpu_tree3d* tree, const bvh_ray3d* rays, size_t nrays, int use_triangles,
                             uint32_t* out_shape, double* out_dist, double* out_uv);
int bvhgpu_closest_hit_dev_f32x3(bvhgpu_tree3f* tree, const void* dev_rays, int ray_layout, size_t nrays, int use_triangles,
                                 void* dev_shape, void* dev_dist, void* dev_uv);
int bvhgpu_closest_hit_dev_f64x3(bvhgpu_tree3d* tree, const void* dev_rays, int ray_layout, size_t nrays, int use_triangles,
                                 void* dev_shape, void* dev_dist, void* dev_uv);

/* ---- any hit (occlusion) with a per-ray distance limit: the other loop callers of the reference write over Bvh::traverse +
 * Ray::intersects_triangle -- traverse(..).iter().any(|s| ray.intersects_triangle(..).distance < tmax), a shadow ray, a line of sight,
 * a segment against the scene.  Per ray r, with the limit tmax[r] (`tmax` == NULL: +inf for every ray):
 *   use_triangles == 0 (D = 2, 3, 4): out_shape[r] = a shape s of Bvh::traverse's set (reached through the stored child boxes, the NaN
 *       rule applied at every ancestor) whose own AABB the ray enters at e_s < tmax[r], e_s the entry of
 *       Ray::intersection_slice_for_aabb bit for bit as bvhgpu_closest_hit_* uses it; BVHGPU_INVALID_INDEX exactly when there is none.
 *       Exact: a hit exists iff the AABB-mode closest_hit distance is < tmax[r].  Slab entries are monotone under box containment and
 *       every stored child box contains the boxes below it ("no split wins" empty boxes pass at entry 0), so subtrees entered at or
 *       beyond tmax[r] are never opened without losing a shape.
 *   use_triangles != 0 (D = 3, triangles from bvhgpu_tree_set_triangles_*): a reported shape always has a Moeller-Trumbore distance
 *       (the reference's operation order, no FMA) < tmax[r].  A child is entered when its entry <= fl(tmax[r] * (1 + 2^-16)), the
 *       margin of closest_hit, for the same reason; so "no hit" where the unpruned loop has one happens only in the grazing case:
 *       every qualifying triangle's Moeller-Trumbore distance lies more than 2^-16 in front of the slab entry of its own AABB (its
 *       entry then exceeds fl(tmax[r] * (1 + 2^-16)) > its distance).
 *   Which shape: the first leaf the walk accepts, the closest_hit walk (stackless, near child first by entry, left on ties) with the
 *       per-ray bound above; deterministic, the same across calls, host and device forms and both 3-D ray layouts.
 *   tmax[r] <= 0 (-0 included) or NaN: no hit (the comparison is a strict <).  An empty tree: no hit for every ray; n = 1: the shape's
 *   own box decides, as in the reference.  nrays > 2^31-1, an unknown ray_layout, a null argument, or use_triangles without triangles
 *   (also after bvhgpu_add_shapes_* dropped them): BVHGPU_ERR_INVALID.  A failed build is reported sticky.  The _dev forms take device
 *   pointers (dev_tmax may be NULL) and enqueue on the context's stream without synchronising; D = 2 has host pointers only. */
int bvhgpu_any_hit_f32x3(bvhgpu_tree3f* tree, const bvh_ray3f* rays, size_t nrays, const float* tmax, int use_triangles, uint32_t* out_shape);
int bvhgpu_any_hit_f64x3(bvhgpu_tree3d* tree, const bvh_ray3d* rays, size_t nrays, const double* tmax, int use_triangles, uint32_t* out_shape);
int bvhgpu_any_hit_dev_f32x3(bvhgpu_tree3f* tree, const void* dev_rays, int ray_layout, size_t nrays, const void* dev_tmax,
                             int use_triangles, void* dev_shape);      /* FULL or OD rays, as bvhgpu_closest_hit_dev_* */
int bvhgpu_any_hit_dev_f64x3(bvhgpu_tree3d* tree, const void* dev_rays, int ray_layout, size_t nrays, const void* dev_tmax,
                             int use_triangles, void* dev_shape);
int bvhgpu_any_hit_f32x2(bvhgpu_tree2f* tree, const bvh_ray2f* rays, size_t nrays, const float* tmax, uint32_t* out_shape);
int bvhgpu_any_hit_f64x2(bvhgpu_tree2d* tree, const bvh_ray2d* rays, size_t nrays, const double* tmax, uint32_t* out_shape);
int bvhgpu_any_hit_f32x4(bvhgpu_tree4f* tree, const bvh_ray4f* rays, size_t nrays, const float* tmax, uint32_t* out_shape);
int bvhgpu_any_hit_f64x4(bvhgpu_tree4d* tree, const bvh_ray4d* rays, size_t nrays, const double* tmax, uint32_t* out_shape);
int bvhgpu_any_hit_dev_f32x4(bvhgpu_tree4f* tree, const void* dev_rays, size_t nrays, const void* dev_tmax, void* dev_shape);
int bvhgpu_any_hit_dev_f64x4(bvhgpu_tree4d* tree, const void* dev_rays, size_t nrays, const void* dev_tmax, void* dev_shape);

/* ---- k nearest shapes with an optional per-point radius: the query of point-cloud, neighbour-search and collision code that the
 * reference leaves to a loop over Bvh::traverse with a guessed Ball and a sort.  `points`: D T per point (D = 2, 3, 4).  For point i
 * the key of shape s is d2_s = Aabb::min_distance_squared(p_i) of the shape's OWN CURRENT AABB (after refit, update, add and remove;
 * src/aabb/aabb_impl.rs:618-629, the reference's operation order, no FMA; the clamp maps NaN to 0, so no key is NaN).
 * Shape s qualifies when `max_dist` is NULL, or when max_dist[i] >= 0 (-0 included) and d2_s <= fl(max_dist[i] * max_dist[i]), the
 * comparison of Ball::intersects_aabb.  max_dist[i] < 0 or NaN: nothing qualifies; +inf: everything does.
 * Output, row-major, k slots per point: out_shape[i*k + j] is the j-th qualifying shape in ascending (d2_s, s) order and
 * out_dist[i*k + j] = fl(sqrt(d2_s)), the distance bvhgpu_nearest_* returns; slots past the qualifying shapes hold
 * BVHGPU_INVALID_INDEX and +inf.  Exact: every row is the first min(k, #qualifying) entries of a stable brute-force sort, for every
 * input (points with NaN or infinite coordinates included).  Pruning uses a lower bound of the distance (rounding slack per axis,
 * monotone under box containment) with ties entered, and empty child boxes ("no split wins" nodes) are always entered.
 *   k = 1 is NOT bvhgpu_nearest_*: Bvh::nearest_to prunes with the rounded reference distance, which is not monotone, and on large
 *   coordinates can return a shape that brute force does not pick.  k = 1 is the brute-force minimum of min_distance_squared, ties
 *   to the lower index.
 *   Distances are the AABB's (the UnitBox PointDistance of bvhgpu_nearest_*); bvhgpu_knn_triangles_* below is the triangle form.
 * 1 <= k <= BVHGPU_KNN_MAX_K.  k out of range, a null argument or n > 2^31-1: BVHGPU_ERR_INVALID, nothing written.  n = 0: no-op.
 * An empty tree: rows of padding.  A failed build is reported sticky.  The _dev forms take device pointers (dev_max_dist may be
 * NULL), check k and the pointers on the host and enqueue on the context's stream without synchronising; D = 2 has host pointers only. */
#define BVHGPU_KNN_MAX_K 64
int bvhgpu_knn_f32x3(bvhgpu_tree3f* tree, const float* points, size_t n, uint32_t k, const float* max_dist, uint32_t* out_shape, float* out_dist);
int bvhgpu_knn_f64x3(bvhgpu_tree3d* tree, const double* points, size_t n, uint32_t k, const double* max_dist, uint32_t* out_shape, double* out_dist);
int bvhgpu_knn_dev_f32x3(bvhgpu_tree3f* tree, const void* dev_points, size_t n, uint32_t k, const void* dev_max_dist, void* dev_shape, void* dev_dist);
int bvhgpu_knn_dev_f64x3(bvhgpu_tree3d* tree, const void* dev_points, size_t n, uint32_t k, const void* dev_max_dist, void* dev_shape, void* dev_dist);
int bvhgpu_knn_f32x2(bvhgpu_tree2f* tree, const float* points, size_t n, uint32_t k, const float* max_dist, uint32_t* out_shape, float* out_dist);
int bvhgpu_knn_f64x2(bvhgpu_tree2d* tree, const double* points, size_t n, uint32_t k, const double* max_dist, uint32_t* out_shape, double* out_dist);
int bvhgpu_knn_f32x4(bvhgpu_tree4f* tree, const float* points, size_t n, uint32_t k, const float* max_dist, uint32_t* out_shape, float* out_dist);
int bvhgpu_knn_f64x4(bvhgpu_tree4d* tree, const double* points, size_t n, uint32_t k, const double* max_dist, uint32_t* out_shape, double* out_dist);
int bvhgpu_knn_dev_f32x4(bvhgpu_tree4f* tree, const void* dev_points, size_t n, uint32_t k, const void* dev_max_dist, void* dev_shape, void* dev_dist);
int bvhgpu_knn_dev_f64x4(bvhgpu_tree4d* tree, const void* dev_points, size_t n, uint32_t k, const void* dev_max_dist, void* dev_shape, void* dev_dist);

/* ---- k nearest triangles with an optional per-point radius (D = 3): point-to-mesh distance, signed-distance fields, ICP, contact
 * generation.  The triangles are those of bvhgpu_tree_set_triangles_*; a non-empty tree without them (never set, or dropped by
 * bvhgpu_add_shapes_*) gives BVHGPU_ERR_INVALID.  After bvhgpu_remove_shapes_* the triangles follow their shapes.
 *   Key: key_s = Triangle::distance_squared(p_i, tri_s) (closest_point_triangle, src/testbase.rs:353-443, the reference's operation
 *   order, no FMA), bit for bit the distance bvhgpu_nearest_triangles_* evaluates.  Shape s qualifies when key_s is not NaN and either
 *   `max_dist` is NULL or max_dist[i] >= 0 (-0 included) and key_s <= fl(max_dist[i] * max_dist[i]).  A NaN key (overflow-scale
 *   coordinates, a 0 * inf in the interior branch, a point with a NaN coordinate) never qualifies.
 *   Row i, k slots (arguments and refusals as bvhgpu_knn_*x3): the first min(k, #qualifying) triangles of a stable sort by (key_s, s),
 *   out_dist = fl(sqrt(key_s)) and out_closest (may be NULL; 3 T per slot, row-major n * k * 3) = the point q that
 *   closest_point_triangle computed for that key.  Padding slots: BVHGPU_INVALID_INDEX, +inf, NaN x 3.
 *   Guarantee: the walk prunes with the lower bound of bvhgpu_knn_* on the stored child boxes, so a triangle can be lost only where its
 *   rounded key lies below box_lower_d2(p, AABB_s) of its own current box; call it bounded at p when it does not.  Where every
 *   qualifying triangle is bounded, the row is the brute-force row exactly (shapes, distances and closest points bit for bit).
 *   Elsewhere every entry is a real (s, key_s) in ascending order, every bounded qualifying triangle that sorts before the row's last
 *   entry is in it, and a row that is not full holds every bounded qualifying triangle.  A triangle inside its box is proven bounded
 *   in every branch of closest_point_triangle except the interior branch of a near-degenerate triangle, where no counterexample is
 *   known (DESIGN.md section 4.17); a triangle outside its box (a stale triangle after a refit) need not be bounded.
 *   A refused call (k outside 1 .. BVHGPU_KNN_MAX_K, a null argument, n > 2^31-1, missing triangles) writes nothing; n = 0 is a no-op
 *   and an empty tree gives rows of padding.  A failed build is reported sticky, before missing triangles.
 *   k = 1 is the brute-force minimum of key_s over the bounded triangles, not bvhgpu_nearest_triangles_*, which replays
 *   Bvh::nearest_to's pruning with the reference's rounded, non-monotone box distance.
 * The _dev forms take device pointers (dev_max_dist and dev_closest may be NULL) and enqueue on the context's stream without
 * synchronising. */
int bvhgpu_knn_triangles_f32x3(bvhgpu_tree3f* tree, const float* points, size_t n, uint32_t k, const float* max_dist, uint32_t* out_shape,
                               float* out_dist, float* out_closest);
int bvhgpu_knn_triangles_f64x3(bvhgpu_tree3d* tree, const double* points, size_t n, uint32_t k, const double* max_dist, uint32_t* out_shape,
                               double* out_dist, double* out_closest);
int bvhgpu_knn_triangles_dev_f32x3(bvhgpu_tree3f* tree, const void* dev_points, size_t n, uint32_t k, const void* dev_max_dist,
                                   void* dev_shape, void* dev_dist, void* dev_closest);
int bvhgpu_knn_triangles_dev_f64x3(bvhgpu_tree3d* tree, const void* dev_points, size_t n, uint32_t k, const void* dev_max_dist,
                                   void* dev_shape, void* dev_dist, void* dev_closest);

/* ---- multi hit: the first k hits along each ray, with an optional per-ray distance limit (transparency and layered surfaces, LiDAR
 * with several returns, entry plus exit for wall thickness, inside / outside counting).  The closest_hit walk keeping a sorted list of
 * k keys instead of one.  Output, row-major, k slots per ray: row r is the first min(k, #qualifying) entries of a stable sort of the
 * qualifying set by key; slots past them hold BVHGPU_INVALID_INDEX, +inf and uv (0, 0) (what closest_hit writes for no hit).
 * Limit: `tmax` NULL: none (no comparison, as closest_hit).  Otherwise an entry qualifies only if its distance is < tmax[r], the strict
 * comparison of any_hit, so tmax[r] <= 0 (-0 included) or NaN gives an empty row.
 *   use_triangles == 0 (D = 2, 3, 4): the candidates are the shapes of Bvh::traverse's set (BVH semantics); s qualifies when the slab
 *       test of its own AABB passes.  Key (e_s, the leaf's node index): e_s the entry of Ray::intersection_slice_for_aabb bit for bit as
 *       closest_hit computes it, ties in DFS order (closest_hit's rule).  out_dist = e_s; out_uv, if given, zeros.  EXACT for every
 *       input: a child is pruned only when its slab test fails, its entry exceeds the current k-th key or (with a limit) its entry is
 *       >= tmax[r]; slab entries are monotone under box containment ("no split wins" empty boxes pass at entry 0).  On a built tree
 *       without "no split wins" nodes and with tmax NULL, a row is the head of bvhgpu_traverse_ordered_* (ascending).
 *   use_triangles != 0 (D = 3, triangles from bvhgpu_tree_set_triangles_*): key (d_s, s), d_s = Ray::intersects_triangle
 *       (Moeller-Trumbore with backface culling, the reference's operation order, no FMA; the function of closest_hit); s qualifies
 *       when d_s is finite.  out_uv (may be NULL) = the u, v of that evaluation.  Leaves are reached through their stored boxes only; a
 *       child is entered when its slab test passes and entry <= min(fl(kth * (1 + 2^-16)), fl(tmax[r] * (1 + 2^-16))), kth = +inf
 *       until the list is full: the margins of closest_hit / any_hit.  Call s bounded on ray r when the box its parent stores for it
 *       passes the slab test with entry <= fl(d_s * (1 + 2^-16)).  Where every triangle of the unpruned row (the stable sort of the loop
 *       over Bvh::traverse with intersects_triangle) is bounded, the row equals it bit for bit: shapes, distances and uv.  Elsewhere (the
 *       grazing hits closest_hit documents) every entry is still a real qualifying (s, d_s), in ascending order.
 *   Identities: k = 1 with tmax NULL is closest_hit (shape, distance, uv) in both modes and every D; with tmax given, a row is empty
 *   exactly where any_hit with the same tmax reports no hit.
 *   1 <= k <= BVHGPU_KNN_MAX_K.  k out of range, a null argument, nrays > 2^31-1, an unknown ray_layout, or use_triangles without
 *   triangles (never set, or dropped by bvhgpu_add_shapes_*): BVHGPU_ERR_INVALID, nothing written.  nrays = 0: no-op.  An empty tree:
 *   rows of padding; n = 1: the shape's own box decides.  A failed build is reported sticky, before missing triangles.  After
 *   bvhgpu_remove_shapes_* the triangles follow their shapes.  The _dev forms take device pointers (dev_tmax and dev_uv may be NULL),
 *   check k and the pointers on the host and enqueue on the context's stream without synchronising; D = 2 has host pointers only. */
int bvhgpu_multi_hit_f32x3(bvhgpu_tree3f* tree, const bvh_ray3f* rays, size_t nrays, uint32_t k, const float* tmax, int use_triangles,
                           uint32_t* out_shape, float* out_dist, float* out_uv);
int bvhgpu_multi_hit_f64x3(bvhgpu_tree3d* tree, const bvh_ray3d* rays, size_t nrays, uint32_t k, const double* tmax, int use_triangles,
                           uint32_t* out_shape, double* out_dist, double* out_uv);
int bvhgpu_multi_hit_dev_f32x3(bvhgpu_tree3f* tree, const void* dev_rays, int ray_layout, size_t nrays, uint32_t k, const void* dev_tmax,
                               int use_triangles, void* dev_shape, void* dev_dist, void* dev_uv);   /* FULL or OD rays */
int bvhgpu_multi_hit_dev_f64x3(bvhgpu_tree3d* tree, const void* dev_rays, int ray_layout, size_t nrays, uint32_t k, const void* dev_tmax,
                               int use_triangles, void* dev_shape, void* dev_dist, void* dev_uv);
int bvhgpu_multi_hit_f32x2(bvhgpu_tree2f* tree, const bvh_ray2f* rays, size_t nrays, uint32_t k, const float* tmax, uint32_t* out_shape,
                           float* out_dist);
int bvhgpu_multi_hit_f64x2(bvhgpu_tree2d* tree, const bvh_ray2d* rays, size_t nrays, uint32_t k, const double* tmax, uint32_t* out_shape,
                           double* out_dist);
int bvhgpu_multi_hit_f32x4(bvhgpu_tree4f* tree, const bvh_ray4f* rays, size_t nrays, uint32_t k, const float* tmax, uint32_t* out_shape,
                           float* out_dist);
int bvhgpu_multi_hit_f64x4(bvhgpu_tree4d* tree, const bvh_ray4d* rays, size_t nrays, uint32_t k, const double* tmax, uint32_t* out_shape,
                           double* out_dist);
int bvhgpu_multi_hit_dev_f32x4(bvhgpu_tree4f* tree, const void* dev_rays, size_t nrays, uint32_t k, const void* dev_tmax, void* dev_shape,
                               void* dev_dist);
int bvhgpu_multi_hit_dev_f64x4(bvhgpu_tree4d* tree, const void* dev_rays, size_t nrays, uint32_t k, const void* dev_tmax, void* dev_shape,
                               void* dev_dist);

/* ---- crossing counts per ray (D = 3): how many triangles a ray crosses, front and back faces apart.  The triangles are those of
 * bvhgpu_tree_set_triangles_* (shape s carries triangle (a, b, c)).  mt(o, d, a, b, c) = Ray::intersects_triangle (Moeller-Trumbore
 * with back-face culling, the reference's operation order, no FMA; the function of closest_hit), evaluated twice per triangle:
 *   out_front[r] = #{ s : mt(o, d, a, b, c) is finite and < tmax[r] }
 *   out_back[r]  = #{ s : mt(o, d, a, c, b) is finite and < tmax[r] }   (b and c exchanged: the back-face test, the same function)
 * A triangle whose two evaluations are both finite counts in both columns.  `tmax` NULL: no limit and no comparison; tmax[r] <= 0 (-0
 * included) or NaN gives 0 / 0 (the comparison is strict).
 *   Candidates: Bvh::traverse's set (BVH semantics: leaves reached through the child boxes their ancestors store, a NaN slab value
 *   rejects; n = 1: the shape's own box).  No distance pruning.  With a limit, a child is entered when its slab test passes and its
 *   entry <= fl(tmax[r] * (1 + 2^-16)), the margin of any_hit.
 *   tmax NULL: the counts are EXACTLY the loop over Bvh::traverse(ray) with both windings, for every input.
 *   With a limit: the same wherever every counted triangle is bounded: the box its parent stores for it passes the slab test with
 *   entry <= fl(d_s * (1 + 2^-16)), d_s the distance it is counted with.  A triangle that is not bounded (a grazing hit whose rounded
 *   distance lies more than 2^-16 in front of its box's entry, or a stale triangle outside its box) may be missed; then its exact
 *   intersection lies beyond tmax.  Every count is at most the unpruned one.
 *   A null argument, nrays > 2^31-1, an unknown ray_layout, or a non-empty tree without triangles (never set, or dropped by
 *   bvhgpu_add_shapes_*): BVHGPU_ERR_INVALID, nothing written.  nrays = 0: no-op.  An empty tree gives zeros.  A failed build is
 *   reported sticky, before missing triangles.  After bvhgpu_remove_shapes_* the triangles follow their shapes.  The _dev forms take
 *   device pointers (FULL or OD rays, dev_tmax may be NULL) and enqueue on the context's stream without synchronising. */
int bvhgpu_count_hits_f32x3(bvhgpu_tree3f* tree, const bvh_ray3f* rays, size_t nrays, const float* tmax, uint32_t* out_front,
                            uint32_t* out_back);
int bvhgpu_count_hits_f64x3(bvhgpu_tree3d* tree, const bvh_ray3d* rays, size_t nrays, const double* tmax, uint32_t* out_front,
                            uint32_t* out_back);
int bvhgpu_count_hits_dev_f32x3(bvhgpu_tree3f* tree, const void* dev_rays, int ray_layout, size_t nrays, const void* dev_tmax,
                                void* dev_front, void* dev_back);   /* FULL or OD rays, as closest_hit_dev */
int bvhgpu_count_hits_dev_f64x3(bvhgpu_tree3d* tree, const void* dev_rays, int ray_layout, size_t nrays, const void* dev_tmax,
                                void* dev_front, void* dev_back);

/* ---- point-in-mesh (D = 3): is each point inside the closed triangle mesh of bvhgpu_tree_set_triangles_*?  (voxelisation, occupancy
 * grids, particle-in-body tests.)  From every point p three rays r_j = Ray::new(p, D_j) are cast, j = 0, 1, 2, with the fixed directions
 * BVHGPU_CONTAINS_DIRECTIONS (normalised as bvhgpu_rays_new_dev_* normalises, bit for bit; in f32 each literal is first rounded to
 * float).  They are not axis-aligned, not parallel to a face diagonal of an axis-aligned cube, and not parallel to each other.  Each
 * ray counts (front_j, back_j) as bvhgpu_count_hits_* with no limit and votes inside:
 *   BVHGPU_FILL_EVEN_ODD   front_j + back_j odd.  Ignores orientation (flipped triangles do not matter); overlapping closed parts cancel.
 *   BVHGPU_FILL_NONZERO    back_j != front_j.  Needs consistently oriented (outward) shells; gives the union of overlapping parts.
 * out_inside[i] = 1 when at least two of the three rays vote inside, else 0.  The vote is there because Moeller-Trumbore is not
 * watertight: a ray through a shared edge or vertex can count twice or not at all; three directions make one such ray harmless.
 * Limits:
 *   - the result is meaningful for closed meshes only (an open mesh, such as a scene without its floor, gives whatever the rays count);
 *   - a point on the surface is undefined;
 *   - a triangle with |det| < eps (f32::EPSILON / f64::EPSILON, the reference's test) is invisible to every ray.  det scales with the
 *     square of the edge lengths (the directions are normalised), so in f32 triangles with edges below about 3e-4 never count: a mesh
 *     whose triangles are all that small (a tiny mesh in absolute units) contains no point; scale it up first.
 * A point with a NaN coordinate gives 0.  An unknown `rule`: BVHGPU_ERR_INVALID; the other refusals, the sticky failure and the empty
 * tree (all 0) as bvhgpu_count_hits_*.  The _dev form takes device pointers and enqueues on the context's stream without synchronising. */
typedef enum { BVHGPU_FILL_EVEN_ODD = 0, BVHGPU_FILL_NONZERO = 1 } bvhgpu_fill_rule;
#define BVHGPU_CONTAINS_DIRECTIONS \
    { { 0.7548776662466927, 0.5698402909980532, 0.3247179572447460 },  \
      { -0.5698402909980532, 0.3247179572447460, 0.7548776662466927 }, \
      { 0.3247179572447460, -0.7548776662466927, 0.5698402909980532 } }
int bvhgpu_contains_points_f32x3(bvhgpu_tree3f* tree, const float* points, size_t n, int rule, uint8_t* out_inside);
int bvhgpu_contains_points_f64x3(bvhgpu_tree3d* tree, const double* points, size_t n, int rule, uint8_t* out_inside);
int bvhgpu_contains_points_dev_f32x3(bvhgpu_tree3f* tree, const void* dev_points, size_t n, int rule, void* dev_inside);
int bvhgpu_contains_points_dev_f64x3(bvhgpu_tree3d* tree, const void* dev_points, size_t n, int rule, void* dev_inside);

/* ---- signed distance to a closed triangle mesh (D = 3): SDF generation, penetration depth, contact.  out_shape, |out_dist| and
 * out_closest (may be NULL) are bit for bit bvhgpu_knn_triangles_* with k = 1 and no radius, with its guarantee (the brute-force
 * nearest triangle wherever the qualifying triangles are bounded).  out_dist is negated exactly where bvhgpu_contains_points_* with the
 * same rule says inside (inside at distance 0 gives -0).  A point without a qualifying triangle keeps +inf, BVHGPU_INVALID_INDEX and a
 * NaN closest point, whatever its vote.  The limits of bvhgpu_contains_points_* apply to the sign.  Refusals as
 * bvhgpu_contains_points_*, nothing written.  The _dev form enqueues the k = 1 query, the containment walk and the sign on the
 * context's stream without synchronising. */
int bvhgpu_signed_distance_f32x3(bvhgpu_tree3f* tree, const float* points, size_t n, int rule, uint32_t* out_shape, float* out_dist,
                                 float* out_closest);
int bvhgpu_signed_distance_f64x3(bvhgpu_tree3d* tree, const double* points, size_t n, int rule, uint32_t* out_shape, double* out_dist,
                                 double* out_closest);
int bvhgpu_signed_distance_dev_f32x3(bvhgpu_tree3f* tree, const void* dev_points, size_t n, int rule, void* dev_shape, void* dev_dist,
                                     void* dev_closest);
int bvhgpu_signed_distance_dev_f64x3(bvhgpu_tree3d* tree, const void* dev_points, size_t n, int rule, void* dev_shape, void* dev_dist,
                                     void* dev_closest);

/* ---- polygons (D = 2): exact point-in-polygon with winding numbers, k nearest segments and signed distance over line segments (GIS
 * point-in-outline tests, 2-D physics and games, occupancy maps, font and vector SDFs).  bvhgpu_tree_set_segments_* gives shape s the
 * segment (ax, ay, bx, by): 4 T per shape, n must equal the tree's shape count (else BVHGPU_ERR_INVALID).  The caller guarantees that
 * shape s's current AABB contains segment s; it is not checked.  The segments follow their shapes through bvhgpu_remove_shapes_*,
 * bvhgpu_add_shapes_* drops them (every segment call refuses until they are set again), bvhgpu_refit_* and bvhgpu_update_* keep them
 * (they can go stale: a segment outside its box may then be missed).  Host pointers; set_segments synchronises.
 *
 * bvhgpu_contains_points_*x2: per point p (2 T), with every comparison exact and every sign decided in exact real arithmetic:
 *   excluded   a segment with a non-finite coordinate or a == b contributes nothing and is never boundary.
 *   relevant   a non-excluded s with min(ay, by) <= py <= max(ay, by) and max(ax, bx) >= px (its own end points, not its box).
 *   o          sign(orient2d(a, b, p)), orient2d(a, b, c) = (a - c) x (b - c): positive when p lies left of a -> b.
 *   contribution of a relevant s: +1 if ay <= py < by and o > 0; -1 if by <= py < ay and o < 0; else 0 (horizontal segments give 0).
 *   boundary   o == 0 and p in the closed box of a and b.
 *   out_winding[i] (may be NULL) = the sum of the contributions: the winding number of closed loops around a point not on them.
 *   out_class[i] = BVHGPU_POINT_BOUNDARY when p is boundary of some relevant segment (this wins); else BVHGPU_POINT_UNDECIDED (f64 only,
 *   below); else BVHGPU_POINT_INSIDE when the winding is odd (BVHGPU_FILL_EVEN_ODD) / nonzero (BVHGPU_FILL_NONZERO); else
 *   BVHGPU_POINT_OUTSIDE.  A point with a non-finite coordinate: class 0, winding 0.
 *   f64 range: the signs are exact for coordinates that are zero or of magnitude in [2^-300, 2^300] (f32: every finite value).  A point
 *   with a nonzero coordinate outside it gets class 3 and winding 0 and is not walked; a relevant segment with such a coordinate
 *   contributes nothing and makes the point class 3 unless it is boundary.
 *   EXACT for every tree the library builds or maintains (the walk enters "no split wins" empty boxes), as long as every segment lies
 *   in its shape's box.
 * bvhgpu_knn_segments_*x2: as bvhgpu_knn_triangles_*x3 (radius rule, stable sort by (key_s, s), padding BVHGPU_INVALID_INDEX / +inf /
 *   NaN x 2, out_dist = fl(sqrt(key_s)), refusals), out_closest 2 T per slot.  key_s in T, in this order, without FMA:
 *     ex = bx - ax; ey = by - ay; wx = px - ax; wy = py - ay; num = wx*ex + wy*ey; den = ex*ex + ey*ey;
 *     q = a if num <= 0; q = b if num >= den; otherwise t = num / den, q = (ax + t*ex, ay + t*ey) (a NaN num lands here);
 *     key = (px - qx)*(px - qx) + (py - qy)*(py - qy).
 *   A NaN key never qualifies; nothing else is excluded (a zero-length segment is a point).  Guarantee, with the wording of
 *   bvhgpu_knn_triangles_*: a segment is bounded at p when its key is not below box_lower_d2(p, AABB_s); where every qualifying
 *   segment is bounded the row is the brute-force row bit for bit.  Every finite segment inside its box is bounded at every finite
 *   point, at every scale (DESIGN.md section 4.23); a stale segment outside its box need not be.
 * bvhgpu_signed_distance_*x2: out_shape, |out_dist| and out_closest (may be NULL) are bvhgpu_knn_segments_* with k = 1 and no radius,
 *   bit for bit; out_dist is negated exactly where bvhgpu_contains_points_*x2 with the same rule gives class 1 (inside at distance 0
 *   gives -0).  Boundary and undecided points keep a non-negative distance; a point without a qualifying segment keeps +inf.
 * Refusals (nothing written): a null argument, n > 2^31-1, an unknown rule, k outside 1 .. BVHGPU_KNN_MAX_K, or a non-empty tree
 * without segments: BVHGPU_ERR_INVALID.  A failed build is reported sticky, before missing segments.  n = 0: no-op.  An empty tree:
 * class 0 / winding 0, rows of padding. */
#define BVHGPU_POINT_OUTSIDE 0
#define BVHGPU_POINT_INSIDE 1
#define BVHGPU_POINT_BOUNDARY 2
#define BVHGPU_POINT_UNDECIDED 3
int bvhgpu_tree_set_segments_f32x2(bvhgpu_tree2f* tree, const float* segments, size_t n);
int bvhgpu_tree_set_segments_f64x2(bvhgpu_tree2d* tree, const double* segments, size_t n);
int bvhgpu_contains_points_f32x2(bvhgpu_tree2f* tree, const float* points, size_t n, int rule, uint8_t* out_class, int32_t* out_winding);
int bvhgpu_contains_points_f64x2(bvhgpu_tree2d* tree, const double* points, size_t n, int rule, uint8_t* out_class, int32_t* out_winding);
int bvhgpu_knn_segments_f32x2(bvhgpu_tree2f* tree, const float* points, size_t n, uint32_t k, const float* max_dist, uint32_t* out_shape,
                              float* out_dist, float* out_closest);
int bvhgpu_knn_segments_f64x2(bvhgpu_tree2d* tree, const double* points, size_t n, uint32_t k, const double* max_dist, uint32_t* out_shape,
                              double* out_dist, double* out_closest);
int bvhgpu_signed_distance_f32x2(bvhgpu_tree2f* tree, const float* points, size_t n, int rule, uint32_t* out_shape, float* out_dist,
                                 float* out_closest);
int bvhgpu_signed_distance_f64x2(bvhgpu_tree2d* tree, const double* points, size_t n, int rule, uint32_t* out_shape, double* out_dist,
                                 double* out_closest);

/* ---- self-overlap pairs: every pair of shapes of the tree whose AABBs intersect, each once (the broad phase of physics, mesh
 * self-intersection, duplicate and contact detection in point and particle sets).  leaf(s) = the preorder node index of shape s's leaf
 * (out_node_index of bvhgpu_tree_nodes_*).  Output: a CSR indexed by shape, offsets[n + 1]; row s lists every shape t with
 * leaf(t) > leaf(s) and intersects(box_s, box_t), in ascending leaf(t) order (DFS order).
 *   intersects = Aabb::intersects_aabb (src/aabb/aabb_impl.rs:240-248): for every axis !(a.max < b.min || b.max < a.min).  Touching
 *   faces overlap; an empty box (min > max) overlaps no finite box; an inverted finite box follows the formula literally.  The boxes are
 *   the shapes' own current boxes: from the build or the latest refit, update_shapes or add_shapes, in the numbering after
 *   remove_shapes.  Each unordered pair {s, t}, s != t, appears exactly once, in the row of whichever leaf comes first; no shape is
 *   paired with itself.
 *   EXACT (equal to the brute force over all pairs) for every tree the library builds or maintains, every build mode, after refit /
 *   update_shapes / add_shapes / remove_shapes, on overflow-scale, infinite, coincident and subnormal boxes: a record is entered when
 *   its box intersects box_s or has min > max on some axis (the Aabb::empty() child box of a "no split wins" node); every other stored
 *   child box contains the boxes of the shapes below it, and containment makes the test monotone.  For a tree from
 *   bvhgpu_tree_from_nodes_* the result is exact only when the caller's node boxes contain their shapes (or are empty); otherwise it
 *   is a subset of the true pairs, still each pair at most once.
 *   Capacity as bvhgpu_query_*: the offsets are always complete; the hits are copied when they fit `cap`, else BVHGPU_ERR_CAPACITY
 *   with *total (in 3-D bvhgpu_traverse_fetch_* then fetches the retained list; in 2-D and 4-D call again with cap = *total).  The
 *   _dev forms (D = 3, 4) take device pointers and enqueue on the context's stream; `total` may be NULL (nothing synchronises), and
 *   dev_hits receives a prefix of length cap.  Offsets saturate at 0xFFFFFFFF; a total above 2^32-1 returns BVHGPU_ERR_CAPACITY
 *   (with the saturated offsets in the _dev forms, with *total only in the host forms).
 *   n = 0 and n = 1: all-zero offsets.  A null tree or offsets pointer: BVHGPU_ERR_INVALID, nothing written.  A failed build is
 *   reported sticky first. */
int bvhgpu_overlap_pairs_f32x2(bvhgpu_tree2f* tree, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_overlap_pairs_f64x2(bvhgpu_tree2d* tree, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_overlap_pairs_f32x3(bvhgpu_tree3f* tree, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_overlap_pairs_f64x3(bvhgpu_tree3d* tree, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_overlap_pairs_f32x4(bvhgpu_tree4f* tree, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_overlap_pairs_f64x4(bvhgpu_tree4d* tree, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_overlap_pairs_dev_f32x3(bvhgpu_tree3f* tree, void* dev_offsets, void* dev_hits, size_t cap, size_t* total);
int bvhgpu_overlap_pairs_dev_f64x3(bvhgpu_tree3d* tree, void* dev_offsets, void* dev_hits, size_t cap, size_t* total);
int bvhgpu_overlap_pairs_dev_f32x4(bvhgpu_tree4f* tree, void* dev_offsets, void* dev_hits, size_t cap, size_t* total);
int bvhgpu_overlap_pairs_dev_f64x4(bvhgpu_tree4d* tree, void* dev_offsets, void* dev_hits, size_t cap, size_t* total);

/* ---- overlap pairs between two trees: every pair of a shape of tree A and a shape of tree B whose AABBs intersect (a moving body
 * against static scenery, one mesh against another, particles against obstacles).  leaf_B(b) = the preorder node index of shape b's
 * leaf in B.  Output: a CSR indexed by A's shapes, offsets[n_a + 1]; row a lists every shape b of B with intersects(box_a, box_b), in
 * ascending leaf_B(b) order (B's DFS order, the order of bvhgpu_query_* hits).
 *   intersects = Aabb::intersects_aabb taken literally, as for bvhgpu_overlap_pairs_*; touching faces overlap.  The boxes are each
 *   tree's own current shape boxes: from the build or the latest refit, update_shapes or add_shapes, in the numbering after
 *   remove_shapes.
 *   EXACT (equal to the brute force over all n_a x n_b pairs) for every tree the library builds or maintains, every build mode, after
 *   every dynamic call, on overflow-scale, infinite, coincident and subnormal boxes: a record of B is entered when its box intersects
 *   box_a or has min > max on some axis (the Aabb::empty() child box of a "no split wins" node), the argument of the self-overlap
 *   pairs applied to B.  For a B from bvhgpu_tree_from_nodes_* the result is exact only when the caller's node boxes contain their
 *   shapes (or are empty); otherwise it is a subset of the true pairs.
 *   A and B must belong to the same context (its one stream orders the walk after every call pending on either tree); otherwise
 *   BVHGPU_ERR_INVALID, nothing written.  a == b is allowed and gives the full symmetric relation, (s, s) included for every box that
 *   intersects itself.
 *   Capacity, saturation and the _dev forms as bvhgpu_overlap_pairs_*: the host forms of D = 2 and 3 keep the retained list on tree A
 *   (in 3-D bvhgpu_traverse_fetch_*(a, ...) fetches it after BVHGPU_ERR_CAPACITY; in 2-D and 4-D call again with cap = *total).
 *   n_a = 0: offsets[0] = 0.  n_b = 0: all-zero offsets, no device work.  A null a, b or offsets pointer: BVHGPU_ERR_INVALID, nothing
 *   written.  A failed build is reported sticky, A's before B's.  The _dev forms exist for D = 3 and 4. */
int bvhgpu_overlap_trees_f32x2(bvhgpu_tree2f* a, bvhgpu_tree2f* b, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_overlap_trees_f64x2(bvhgpu_tree2d* a, bvhgpu_tree2d* b, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_overlap_trees_f32x3(bvhgpu_tree3f* a, bvhgpu_tree3f* b, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_overlap_trees_f64x3(bvhgpu_tree3d* a, bvhgpu_tree3d* b, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_overlap_trees_f32x4(bvhgpu_tree4f* a, bvhgpu_tree4f* b, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_overlap_trees_f64x4(bvhgpu_tree4d* a, bvhgpu_tree4d* b, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_overlap_trees_dev_f32x3(bvhgpu_tree3f* a, bvhgpu_tree3f* b, void* dev_offsets, void* dev_hits, size_t cap, size_t* total);
int bvhgpu_overlap_trees_dev_f64x3(bvhgpu_tree3d* a, bvhgpu_tree3d* b, void* dev_offsets, void* dev_hits, size_t cap, size_t* total);
int bvhgpu_overlap_trees_dev_f32x4(bvhgpu_tree4f* a, bvhgpu_tree4f* b, void* dev_offsets, void* dev_hits, size_t cap, size_t* total);
int bvhgpu_overlap_trees_dev_f64x4(bvhgpu_tree4d* a, bvhgpu_tree4d* b, void* dev_offsets, void* dev_hits, size_t cap, size_t* total);

/* ---- triangle pairs (D = 3): which triangles of a mesh cut each other (self-intersection, mesh repair), where one mesh touches another
 * (contact, boolean operations, clearance checks).  The narrow phase of the overlap pairs, decided exactly.  The triangles are those of
 * bvhgpu_tree_set_triangles_* (shape s carries triangle (a, b, c)).  The CSR is a filter of the overlap CSR:
 *   self:   row s of bvhgpu_triangle_pairs_* is row s of bvhgpu_overlap_pairs_*, in the same order (ascending leaf(t)), keeping only the
 *           shapes t with meets(tri_s, tri_t).  Every pair appears once.
 *   trees:  row a of bvhgpu_triangle_pairs_trees_*(a, b) is row a of bvhgpu_overlap_trees_*(a, b), filtered the same way, A's triangle
 *           against B's.
 * So the result equals the brute force over all pairs exactly where the overlap pairs do, provided every triangle lies inside its
 * shape's own box (the condition bvhgpu_tree_set_triangles_* asks for).  With stale triangles (a refit or update without a new
 * set_triangles) it is still precisely the filtered overlap row.
 * meets(P, Q), in this order:
 *   1. Excluded triangles meet nothing: a coordinate that is not finite, or degenerate: (b - a) x (c - a) exactly zero (collinear
 *      points, a repeated vertex, a single point).
 *   2. f64 only: a triangle with a nonzero coordinate of magnitude outside [2^-300, 2^300] is unchecked: it is never excluded as
 *      degenerate, and a pair with it (the other triangle not excluded) is KEPT as its boxes decided it.  A stated superset: no contact
 *      is dropped, and overflow-scale and subnormal scenes get a defined result.
 *   3. Shared vertex: some vertex of P equals some vertex of Q (all three coordinates compare ==, so -0 equals +0).  With
 *      skip_shared != 0 (self form only) the pair is NOT reported: the usual "non-adjacent self-intersections" of mesh repair tools;
 *      the cost is that a fold-over between two triangles that share a vertex is not reported either.  Otherwise (skip_shared = 0, and
 *      always between trees) it IS reported: the closed triangles share that point.  No predicate runs.
 *   4. Otherwise: true exactly when the closed triangles, as sets of real points with the input coordinates as exact real numbers,
 *      have a point in common.  Touching counts: a vertex on a face, an edge on an edge, coplanar triangles that only touch; coplanar
 *      overlap counts too.
 * Exactness of 4: every sign comes from orient3d / orient2d evaluated in double with a static error bound and, where that cannot
 * decide, in exact double-precision expansion arithmetic (DESIGN.md §4.22).  f32: exact for every finite input (f32 values are
 * multiples of 2^-149 below 2^128; nothing underflows or overflows).  f64: exact on [2^-300, 2^300] and zero, the range of step 2.
 * Refusals: a null tree, a or b, or offsets pointer; a non-empty tree without triangles (never set, or dropped by
 * bvhgpu_add_shapes_*); two trees of different contexts: BVHGPU_ERR_INVALID, nothing written.  A failed build is reported sticky
 * first, A's before B's, before missing triangles.  Self with n < 2: all-zero offsets.  Trees: n_a = 0 gives offsets[0] = 0, n_b = 0
 * all-zero offsets.  a == b is allowed and gives the full symmetric relation, (s, s) included for every non-excluded triangle.
 * After bvhgpu_remove_shapes_* the triangles follow their shapes.
 * Capacity, u32 saturation, BVHGPU_ERR_CAPACITY with *total, and the retained list for bvhgpu_traverse_fetch_* (kept on tree A) as
 * bvhgpu_overlap_pairs_* / bvhgpu_overlap_trees_*.  The _dev forms take device pointers and enqueue on the context's stream; with
 * `total` NULL they never synchronise the host, and dev_hits receives a prefix of length cap. */
int bvhgpu_triangle_pairs_f32x3(bvhgpu_tree3f* tree, int skip_shared, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_triangle_pairs_f64x3(bvhgpu_tree3d* tree, int skip_shared, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_triangle_pairs_dev_f32x3(bvhgpu_tree3f* tree, int skip_shared, void* dev_offsets, void* dev_hits, size_t cap, size_t* total);
int bvhgpu_triangle_pairs_dev_f64x3(bvhgpu_tree3d* tree, int skip_shared, void* dev_offsets, void* dev_hits, size_t cap, size_t* total);
int bvhgpu_triangle_pairs_trees_f32x3(bvhgpu_tree3f* a, bvhgpu_tree3f* b, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_triangle_pairs_trees_f64x3(bvhgpu_tree3d* a, bvhgpu_tree3d* b, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total);
int bvhgpu_triangle_pairs_trees_dev_f32x3(bvhgpu_tree3f* a, bvhgpu_tree3f* b, void* dev_offsets, void* dev_hits, size_t cap, size_t* total);
int bvhgpu_triangle_pairs_trees_dev_f64x3(bvhgpu_tree3d* a, bvhgpu_tree3d* b, void* dev_offsets, void* dev_hits, size_t cap, size_t* total);

/* ---- nearest_to (SURVEY.md 8f N4): batched Bvh::nearest_to (src/bvh/bvh_impl.rs:221-238, src/bvh/bvh_node.rs:327-372) and
 * FlatBvh::nearest_to (src/flat_bvh.rs:513-562).  The reference calls the shape's own PointDistance::distance_squared at the
 * leaves (user code), so there are two forms.  `points`: 3 T per query point, host pointers.
 *   bvhgpu_nearest_*            for shapes whose distance IS their AABB's (as the reference's UnitBox, src/testbase.rs:101-105):
 *                               the reference's walk replayed exactly (children ordered by Aabb::min_distance_squared,
 *                               src/aabb/aabb_impl.rs:618-629; strict `<`; first minimum kept).  out_shape[i] = shape index
 *                               (BVHGPU_INVALID_INDEX for an empty tree), out_dist[i] = distance (sqrt, as the reference returns).
 *                               `mode` selects Bvh (BVHGPU_TRAVERSE_BVH) or FlatBvh (BVHGPU_TRAVERSE_FLAT) visiting order.
 *   bvhgpu_nearest_candidates_* for ANY shape contained in its AABB: CSR lists of the shapes whose AABB is at most as far as
 *                               the smallest farthest-corner distance of any shape's AABB, both sides widened per axis by a
 *                               rounding slack of 16 eps max(|p|, -min, max, max - min).  Every list contains every shape at the
 *                               minimal exact distance, the shape bvhgpu_nearest_* (Bvh::nearest_to) returns, and the shape of
 *                               smallest Aabb::min_distance_squared over all shapes.  A shape's own distance is guaranteed only
 *                               in exact arithmetic; its rounded form is user code.  The shim evaluates distance_squared on the
 *                               short list and keeps the minimum.  Below an empty child box ("no split wins" nodes, where surface areas
 *                               overflow) the box bounds nothing, so every shape under it is listed. */
int bvhgpu_nearest_f32x3(bvhgpu_tree3f* tree, int mode, const float* points, size_t n, uint32_t* out_shape, float* out_dist);
int bvhgpu_nearest_f64x3(bvhgpu_tree3d* tree, int mode, const double* points, size_t n, uint32_t* out_shape, double* out_dist);
/* The same walk with the TRIANGLE's own distance at the leaves -- Triangle::distance_squared of the reference's test shape
 * (closest_point_triangle, src/testbase.rs:353-443), operation for operation; triangles from bvhgpu_tree_set_triangles_*.  This is
 * the PointDistance of every benchmark scene of the reference, evaluated on the device: same shape, bit-identical distance. */
int bvhgpu_nearest_triangles_f32x3(bvhgpu_tree3f* tree, int mode, const float* points, size_t n, uint32_t* out_shape, float* out_dist);
int bvhgpu_nearest_triangles_f64x3(bvhgpu_tree3d* tree, int mode, const double* points, size_t n, uint32_t* out_shape, double* out_dist);
int bvhgpu_nearest_candidates_f32x3(bvhgpu_tree3f* tree, const float* points, size_t n, uint32_t* offsets, uint32_t* cand,
                                    size_t cap, size_t* total);
int bvhgpu_nearest_candidates_f64x3(bvhgpu_tree3d* tree, const double* points, size_t n, uint32_t* offsets, uint32_t* cand,
                                    size_t cap, size_t* total);

/* Ray::new for a batch (src/ray/ray_impl.rs:70-80): normalise, inv = 1/direction. Device pointers. */
int bvhgpu_rays_new_dev_f32x3(bvhgpu_ctx* ctx, const void* dev_origins, const void* dev_directions, size_t n, void* dev_rays);
int bvhgpu_rays_new_dev_f64x3(bvhgpu_ctx* ctx, const void* dev_origins, const void* dev_directions, size_t n, void* dev_rays);

/* ---- whole-tree SAH cost (definition: DESIGN.md; the reference only has the per-split cost,
 * src/bvh/bvh_node.rs:236-238).  out2[0]: with the reference's surface_area (2*|size|^2,
 * src/aabb/aabb_impl.rs:551-554), out2[1]: geometric area. */
int bvhgpu_sah_cost_f32x3(bvhgpu_tree3f* tree, double* out2);
int bvhgpu_sah_cost_f64x3(bvhgpu_tree3d* tree, double* out2);

/* ---- refit: bottom-up AABB update after shapes moved (the data-parallel part of
 * Bvh::update_shapes, src/bvh/optimization.rs:304-351 fix_aabbs_ascending).  Topology is kept. */
int bvhgpu_refit_f32x3(bvhgpu_tree3f* tree, const bvh_aabb3f* aabbs, size_t n);
int bvhgpu_refit_f64x3(bvhgpu_tree3d* tree, const bvh_aabb3d* aabbs, size_t n);
/* The AABBs are already on the device (C-ABI layout): nothing is uploaded.  A NaN in the new AABBs is rejected
 * (BVHGPU_ERR_NAN) before the tree is touched, in every refit / optimize / update variant. */
int bvhgpu_refit_dev_f32x3(bvhgpu_tree3f* tree, const void* dev_aabbs, size_t n);
int bvhgpu_refit_dev_f64x3(bvhgpu_tree3d* tree, const void* dev_aabbs, size_t n);

/* ---- optimize: replaces Bvh::update_shapes after shapes moved (src/bvh/optimization.rs:290-302) ----
 * The reference removes and re-inserts every changed shape sequentially (remove_shape :208-288, add_shape :70-206).
 * The data-parallel counterpart: refit, then rebuild -- in place, with the exact 6-bucket SAH builder -- the
 * outermost subtrees that contain a node whose surface area grew by more than `max_growth` (>= 1; e.g. 1.5).
 * `aabbs` are the CURRENT AABBs of all n shapes (no list of changed indices is needed: unchanged subtrees are
 * found by the growth test).  The node array stays in Bvh::build's preorder layout (the reference's does not,
 * it appends and swap-removes nodes), node indices of shapes in rebuilt subtrees change: fetch them with
 * bvhgpu_tree_nodes_* and pass them to BHShape::set_bh_node_index.  *rebuilt (may be NULL) = number of shapes in
 * the rebuilt subtrees (0: the call was a pure refit).  Not the reference's tree: parity is on the invariants
 * (assert_consistent, assert_tight), on hit sets, and on SAH cost against the oracle's update_shapes. */
int bvhgpu_optimize_f32x3(bvhgpu_tree3f* tree, const bvh_aabb3f* aabbs, size_t n, double max_growth, size_t* rebuilt);
int bvhgpu_optimize_f64x3(bvhgpu_tree3d* tree, const bvh_aabb3d* aabbs, size_t n, double max_growth, size_t* rebuilt);
int bvhgpu_optimize_dev_f32x3(bvhgpu_tree3f* tree, const void* dev_aabbs, size_t n, double max_growth, size_t* rebuilt);
int bvhgpu_optimize_dev_f64x3(bvhgpu_tree3d* tree, const void* dev_aabbs, size_t n, double max_growth, size_t* rebuilt);
/* The same with Bvh::update_shapes' own signature (src/bvh/optimization.rs:304-315: the indices of the changed shapes + the shapes):
 * `changed[i]` is a shape index, `changed_aabbs[i]` its new AABB -- only the m changed shapes cross the boundary (10 M f64 shapes,
 * 1 % moved: 5 MB instead of 480 MB).  max_growth >= 1: refit + rebuild of the degraded subtrees as bvhgpu_optimize_*;
 * max_growth <= 0: refit only.  Indices >= n or NaN AABBs are rejected before the tree is touched.  Growth is judged against the
 * surface area every node had when it was last (re)built, so slow drift over many calls adds up and is rebuilt eventually. */
int bvhgpu_update_f32x3(bvhgpu_tree3f* tree, const uint32_t* changed, const bvh_aabb3f* changed_aabbs, size_t m, double max_growth, size_t* rebuilt);
int bvhgpu_update_f64x3(bvhgpu_tree3d* tree, const uint32_t* changed, const bvh_aabb3d* changed_aabbs, size_t m, double max_growth, size_t* rebuilt);
int bvhgpu_update_dev_f32x3(bvhgpu_tree3f* tree, const void* dev_changed, const void* dev_changed_aabbs, size_t m, double max_growth, size_t* rebuilt);
int bvhgpu_update_dev_f64x3(bvhgpu_tree3d* tree, const void* dev_changed, const void* dev_changed_aabbs, size_t m, double max_growth, size_t* rebuilt);

/* ---- add / remove shapes: Bvh::add_shape / Bvh::remove_shape (src/bvh/optimization.rs:67-301), batched ----
 * add: the k new shapes get indices n .. n+k-1 in the order given (the reference's shapes.push(s); add_shape(len-1)).  Every new
 * shape picks its insertion point by the reference's descent, evaluated against the tree as it was before the call (all k descents
 * are independent).  At each insertion point p a new inner node takes p's place: its left child is the exact-SAH subtree over the
 * shapes that chose p (ascending index order; a leaf for one shape), its right child p's old subtree; the ancestors' boxes are
 * refitted.  For k = 1 this is the reference's own topology, and its own tree whenever the boxes are tight (every built tree except
 * trees whose surface areas overflow -- coordinates from about 1e19 in f32, 1e154 in f64 -- where the builder stores empty child
 * boxes: there the device refits the affected paths up to the root, the reference stops at the first box that does not change, so
 * boxes on those paths can differ; traversal then follows the device's boxes).  max_growth >= 1: then the growth test of bvhgpu_update_* runs on the
 * changed ancestors and the degraded subtrees are rebuilt in place; *rebuilt (may be NULL) = shapes in those subtrees.
 * max_growth <= 0: no rebuild, *rebuilt = 0.  n == 0: the call is bvhgpu_build_* over the k AABBs.  Triangles set with
 * bvhgpu_tree_set_triangles_* are discarded (the triangle forms of closest_hit / nearest return BVHGPU_ERR_INVALID until set again).
 * remove: `indices` are distinct shape indices (numbering before the call).  Removed leaves go; an inner node left with one child
 * is replaced by that child (the reference's connect_nodes); boxes on the affected paths are refitted (same caveat for non-tight trees
 * as for add: the topology and node indices are the reference's, the boxes are on tight trees); nothing is rebuilt.
 * Renumbering (remove_shape with swap_shape = true): the survivors with index >= n-k move into the vacated indices < n-k, in
 * ascending order on both sides (smallest hole <- smallest surviving tail index).  For k = 1 that is remove_shape(i, true) + pop();
 * for k > 1 it is NOT k sequential swap-removes (removing {0,1,2} of 5 shapes sequentially gives [4,3], here [3,4]).  Triangles
 * follow their shapes.  swap_shape == false is not representable: device trees number their shapes densely.
 * Both: NaN AABBs (BVHGPU_ERR_NAN), indices >= n, duplicates, k > n on remove and n + k > 2^30 (BVHGPU_ERR_INVALID) are rejected
 * before the tree is touched.  The node index of EVERY shape may change (preorder positions shift): re-read them with
 * bvhgpu_tree_nodes_* after every call.  The tree stays in Bvh::build's preorder layout: it is the same tree that
 * bvhgpu_tree_from_nodes_* makes from its node array and AABBs.  _dev_: inputs on the device; validated synchronously, the rest
 * is asynchronous (as bvhgpu_update_dev_*). */
int bvhgpu_add_shapes_f32x3(bvhgpu_tree3f* tree, const bvh_aabb3f* aabbs, size_t k, double max_growth, size_t* rebuilt);
int bvhgpu_add_shapes_f64x3(bvhgpu_tree3d* tree, const bvh_aabb3d* aabbs, size_t k, double max_growth, size_t* rebuilt);
int bvhgpu_add_shapes_dev_f32x3(bvhgpu_tree3f* tree, const void* dev_aabbs, size_t k, double max_growth, size_t* rebuilt);
int bvhgpu_add_shapes_dev_f64x3(bvhgpu_tree3d* tree, const void* dev_aabbs, size_t k, double max_growth, size_t* rebuilt);
int bvhgpu_remove_shapes_f32x3(bvhgpu_tree3f* tree, const uint32_t* indices, size_t k);
int bvhgpu_remove_shapes_f64x3(bvhgpu_tree3d* tree, const uint32_t* indices, size_t k);
int bvhgpu_remove_shapes_dev_f32x3(bvhgpu_tree3f* tree, const void* dev_indices, size_t k);
int bvhgpu_remove_shapes_dev_f64x3(bvhgpu_tree3d* tree, const void* dev_indices, size_t k);

#ifdef __cplusplus
}
#endif
#endif /* BVH_B200_H */
