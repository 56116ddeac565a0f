// bvh_b200/csrc/capi.cu -- the extern "C" surface declared in include/bvh_b200.h.
#include "internal.h"
#include <cstdarg>
#include <cstring>
#include <vector>
#include <new>
#include <algorithm>
#include <cctype>
#include <sched.h>
#include <type_traits>

namespace bvhb200 {

static thread_local std::string g_last_error;
const char* last_error() { return g_last_error.c_str(); }

void set_error(const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_last_error = buf;
}

int dalloc(bvhgpu_ctx* ctx, void** p, size_t bytes) {
    *p = nullptr;
    if (bytes == 0) bytes = 16;
    BVH_CUDA_TRY(cudaMallocAsync(p, bytes, ctx->stream));
    return BVHGPU_OK;
}
void dfree(bvhgpu_ctx* ctx, void* p) {
    if (p) cudaFreeAsync(p, ctx->stream);
}

// Resolve the deferred device status of a build (synchronises the stream once).
// A failure is STICKY (mark_failed): the node arrays of a tree whose build / refit / optimize failed are uninitialised or half
// rewritten (the reference panicked at this point and the Bvh never existed).
template <class T> int resolve_status(Tree<T>* tree) {
    if (tree->failed_status != BVHGPU_OK) { set_error("%s", tree->failed_message.c_str()); return tree->failed_status; }
    if (!tree->status_pending) return BVHGPU_OK;
    bvhgpu_ctx* ctx = tree->ctx;
    BuildStatus h;
    BVH_CUDA_TRY(cudaMemcpyAsync(&h, tree->d_status, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    tree->status_pending = false;
    char msg[512];
    int rc = BVHGPU_OK;
    if (h.nan_found) { snprintf(msg, sizeof msg, "build: NaN coordinate in an input AABB (the reference panics here, src/bvh/bvh_node.rs:214-217); the tree is unusable"); rc = BVHGPU_ERR_NAN; }
    else if (h.error == BVHGPU_ERR_TIMEOUT) { snprintf(msg, sizeof msg, "build: device watchdog fired (tickets=%u leaves=%u/%u); the tree is unusable", h.tickets, h.leaves_done, tree->n); rc = BVHGPU_ERR_TIMEOUT; }
    else if (h.error) { snprintf(msg, sizeof msg, "build: device reported status %u (tickets=%u leaves=%u/%u); the tree is unusable", h.error, h.tickets, h.leaves_done, tree->n); rc = (int)h.error; }
    return rc == BVHGPU_OK ? rc : mark_failed(tree, rc, nullptr, msg);
}

template int resolve_status<float>(Tree<float>*);
template int resolve_status<double>(Tree<double>*);

template <class T> static void tree_release(Tree<T>* t) {
    if (!t) return;
    bvhgpu_ctx* ctx = t->ctx;
    if (ctx) {
        dfree(ctx, t->d_aabb); dfree(ctx, t->d_aabb_trav); dfree(ctx, t->d_nodes); dfree(ctx, t->d_node_index); dfree(ctx, t->d_node_start);
        dfree(ctx, t->d_tris); dfree(ctx, t->d_segs); dfree(ctx, t->d_sa_base); dfree(ctx, t->d_arrive); dfree(ctx, t->d_bad); dfree(ctx, t->d_tnodes); dfree(ctx, t->d_top); dfree(ctx, t->d_flat); dfree(ctx, t->d_status); dfree(ctx, t->d_offsets); dfree(ctx, t->d_hits);
    }
}

template <class T> static void tree_release(Tree4<T>* t) {
    if (!t || !t->ctx) return;
    bvhgpu_ctx* ctx = t->ctx;
    dfree(ctx, t->d_aabb); dfree(ctx, t->d_nodes); dfree(ctx, t->d_node_index); dfree(ctx, t->d_node_start);
    dfree(ctx, t->d_tnodes); dfree(ctx, t->d_flat); dfree(ctx, t->d_offsets); dfree(ctx, t->d_hits);
    dfree(ctx, t->d_sa_base); dfree(ctx, t->d_arrive); dfree(ctx, t->d_bad);
}

template <class T, class TreeT>
static int build_impl(bvhgpu_ctx* ctx, const typename Traits<T>::Aabb* aabbs, size_t n, int mode, bool host_input, TreeT** out) {
    if (!ctx || !out || (n && !aabbs)) { set_error("build: null argument"); return BVHGPU_ERR_INVALID; }
    *out = nullptr;
    if (n > (1ull << 30)) { set_error("build: n = %zu exceeds 2^30 shapes (u32 node indices)", n); return BVHGPU_ERR_INVALID; }
    if (mode != BVHGPU_BUILD_EXACT_SAH && mode != BVHGPU_BUILD_LBVH && mode != BVHGPU_BUILD_LBVH_TREELET) { set_error("build: unknown mode %d", mode); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    TreeT* tree = new (std::nothrow) TreeT();
    if (!tree) { set_error("build: out of host memory"); return BVHGPU_ERR_INTERNAL; }
    tree->ctx = ctx;
    const typename Traits<T>::Aabb* d_in = aabbs;
    typename Traits<T>::Aabb* staged = nullptr;
    int rc = BVHGPU_OK;
    if (host_input && n) {
        rc = dalloc_t(ctx, &staged, n);
        if (rc == BVHGPU_OK) {
            cudaError_t e = cudaMemcpyAsync(staged, aabbs, n * sizeof(*aabbs), cudaMemcpyHostToDevice, ctx->stream);
            if (e != cudaSuccess) { set_error("build: H2D copy failed: %s", cudaGetErrorString(e)); rc = BVHGPU_ERR_CUDA; }
        }
        d_in = staged;
    }
    if (rc == BVHGPU_OK) rc = mode == BVHGPU_BUILD_EXACT_SAH ? build_exact_sah<T>(ctx, d_in, (uint32_t)n, tree) : build_lbvh<T>(ctx, d_in, (uint32_t)n, tree, mode == BVHGPU_BUILD_LBVH_TREELET);
    if (staged) dfree(ctx, staged);
    if (rc == BVHGPU_OK && host_input) rc = resolve_status(tree);     // host entry point reports errors eagerly
    if (rc != BVHGPU_OK) { tree_release(tree); delete tree; return rc; }
    *out = tree;
    return BVHGPU_OK;
}

// Upload of an existing reference-layout Bvh: validate the preorder invariant on the host, derive the
// per-node shape counts / range starts the device kernels rely on.
template <class T, class TreeT>
static int from_nodes_impl(bvhgpu_ctx* ctx, const typename Traits<T>::Node* nodes, size_t n_nodes,
                           const typename Traits<T>::Aabb* aabbs, size_t n, TreeT** out) {
    using Node = typename Traits<T>::Node;
    if (!ctx || !out) { set_error("tree_from_nodes: null argument"); return BVHGPU_ERR_INVALID; }
    *out = nullptr;
    if ((n == 0) != (n_nodes == 0) || (n && n_nodes != 2 * n - 1)) { set_error("tree_from_nodes: n_nodes must be 2n-1"); return BVHGPU_ERR_INVALID; }
    if (n > (1ull << 30)) { set_error("tree_from_nodes: too many shapes"); return BVHGPU_ERR_INVALID; }
    if (n && (!nodes || !aabbs)) { set_error("tree_from_nodes: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    std::vector<Node> fixed(nodes, nodes + n_nodes);
    std::vector<uint32_t> count(n_nodes), start(n_nodes), node_index(n, BVH_INVALID);
    for (size_t ii = n_nodes; ii-- > 0;) {                       // children have larger indices in preorder
        Node& nd = fixed[ii];
        if (nd.child_l == BVH_INVALID) {
            if (nd.shape >= n) { set_error("tree_from_nodes: leaf %zu has shape %u out of range", ii, nd.shape); return BVHGPU_ERR_INVALID; }
            count[ii] = 1;
        } else {
            if (nd.child_l != ii + 1 || nd.child_l >= n_nodes || nd.child_r >= n_nodes || nd.child_r <= nd.child_l) {
                set_error("tree_from_nodes: node %zu is not in the preorder layout Bvh::build emits (child_l must be i+1)", ii);
                return BVHGPU_ERR_UNSUPPORTED;
            }
            if (nd.child_r != ii + 2 * (size_t)count[nd.child_l]) {
                set_error("tree_from_nodes: node %zu: child_r != i + 2*n_l", ii);
                return BVHGPU_ERR_UNSUPPORTED;
            }
            count[ii] = count[nd.child_l] + count[nd.child_r];
            nd.shape = count[ii];
        }
    }
    if (n_nodes && count[0] != n) { set_error("tree_from_nodes: tree does not cover all shapes"); return BVHGPU_ERR_INVALID; }
    if (n_nodes) start[0] = 0;
    for (size_t ii = 0; ii < n_nodes; ++ii) {
        const Node& nd = fixed[ii];
        if (nd.child_l == BVH_INVALID) { node_index[nd.shape] = (uint32_t)ii; continue; }
        start[nd.child_l] = start[ii];
        start[nd.child_r] = start[ii] + count[nd.child_l];
        if (fixed[nd.child_l].parent != ii || fixed[nd.child_r].parent != ii) { set_error("tree_from_nodes: bad parent link under node %zu", ii); return BVHGPU_ERR_INVALID; }
    }
    for (size_t s = 0; s < n; ++s) if (node_index[s] == BVH_INVALID) { set_error("tree_from_nodes: shape %zu is in no leaf", s); return BVHGPU_ERR_INVALID; }

    TreeT* tree = new (std::nothrow) TreeT();
    if (!tree) { set_error("out of host memory"); return BVHGPU_ERR_INTERNAL; }
    tree->ctx = ctx; tree->n = (uint32_t)n; tree->n_nodes = (uint32_t)n_nodes;
    int rc = BVHGPU_OK;
    typename Traits<T>::Aabb* staged = nullptr;
    auto fail = [&](int code) { if (staged) dfree(ctx, staged); tree_release(tree); delete tree; return code; };
    if ((rc = dalloc_t(ctx, &tree->d_status, 1)) != BVHGPU_OK) return fail(rc);
    cudaMemsetAsync(tree->d_status, 0, sizeof(BuildStatus), ctx->stream);
    if (n) {
        if ((rc = dalloc_t(ctx, &tree->d_aabb, n)) != BVHGPU_OK) return fail(rc);
        if ((rc = dalloc_t(ctx, &tree->d_nodes, n_nodes)) != BVHGPU_OK) return fail(rc);
        if ((rc = dalloc_t(ctx, &tree->d_node_index, n)) != BVHGPU_OK) return fail(rc);
        if ((rc = dalloc_t(ctx, &tree->d_node_start, n_nodes)) != BVHGPU_OK) return fail(rc);
        if ((rc = dalloc_t(ctx, &staged, n)) != BVHGPU_OK) return fail(rc);
        cudaMemcpyAsync(staged, aabbs, n * sizeof(*aabbs), cudaMemcpyHostToDevice, ctx->stream);
        cudaMemcpyAsync(tree->d_nodes, fixed.data(), n_nodes * sizeof(Node), cudaMemcpyHostToDevice, ctx->stream);
        cudaMemcpyAsync(tree->d_node_index, node_index.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream);
        cudaMemcpyAsync(tree->d_node_start, start.data(), n_nodes * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream);
        if ((rc = convert_aabbs<T>(ctx, staged, (uint32_t)n, tree->d_aabb, &tree->d_status->nan_found)) != BVHGPU_OK) return fail(rc);
        cudaError_t e = cudaStreamSynchronize(ctx->stream);       // the host vectors go out of scope
        if (e != cudaSuccess) { set_error("tree_from_nodes: %s", cudaGetErrorString(e)); return fail(BVHGPU_ERR_CUDA); }
        dfree(ctx, staged);
        staged = nullptr;
        tree->status_pending = true;                              // the NaN flag of convert_aabbs
        if ((rc = resolve_status(tree)) != BVHGPU_OK) return fail(rc);
    }
    *out = tree;
    return BVHGPU_OK;
}

template <class T> static int tree_nodes_impl(Tree<T>* tree, typename Traits<T>::Node* out_nodes, uint32_t* out_node_index) {
    if (!tree) { set_error("tree_nodes: null tree"); return BVHGPU_ERR_INVALID; }
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(resolve_status(tree));
    if (tree->n == 0) return BVHGPU_OK;
    if (out_nodes) BVH_CUDA_TRY(cudaMemcpyAsync(out_nodes, tree->d_nodes, sizeof(*out_nodes) * tree->n_nodes, cudaMemcpyDeviceToHost, ctx->stream));
    if (out_node_index) BVH_CUDA_TRY(cudaMemcpyAsync(out_node_index, tree->d_node_index, sizeof(uint32_t) * tree->n, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return BVHGPU_OK;
}

template <class T> static int flatten_impl(Tree<T>* tree, typename Traits<T>::Flat* out, size_t cap, size_t* len) {
    if (!tree) { set_error("flatten: null tree"); return BVHGPU_ERR_INVALID; }
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    if (out || tree->failed_status != BVHGPU_OK) BVH_TRY(resolve_status(tree));   // never map a node array whose build failed
    BVH_TRY(build_flat(tree));
    if (len) *len = tree->n_flat;
    if (out) {
        if (cap < tree->n_flat) { set_error("flatten: capacity %zu < %zu flat nodes", cap, tree->n_flat); return BVHGPU_ERR_CAPACITY; }
        if (tree->n_flat) {
            BVH_CUDA_TRY(cudaMemcpyAsync(out, tree->d_flat, sizeof(*out) * tree->n_flat, cudaMemcpyDeviceToHost, ctx->stream));
            BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
        }
    }
    return BVHGPU_OK;
}

// ---- D = 4 (dim4.cu): exact SAH build only, synchronous; node and flat arrays in the ABI layout already ----
template <class T, class TreeT> static int build4_impl(bvhgpu_ctx* ctx, const typename D4<T>::Aabb* aabbs, size_t n, int mode, TreeT** out) {
    if (!ctx || !out || (n && !aabbs)) { set_error("build: null argument"); return BVHGPU_ERR_INVALID; }
    *out = nullptr;
    if (n > (1ull << 30)) { set_error("build: n = %zu exceeds 2^30 shapes", n); return BVHGPU_ERR_INVALID; }
    if (mode == BVHGPU_BUILD_LBVH || mode == BVHGPU_BUILD_LBVH_TREELET) {
        set_error("build: D = 4 has the exact SAH build only (BVHGPU_BUILD_EXACT_SAH); the LBVH modes are not implemented for D = 4");
        return BVHGPU_ERR_UNSUPPORTED;
    }
    if (mode != BVHGPU_BUILD_EXACT_SAH) { set_error("build: unknown mode %d", mode); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    TreeT* tree = new (std::nothrow) TreeT();
    if (!tree) { set_error("build: out of host memory"); return BVHGPU_ERR_INTERNAL; }
    tree->ctx = ctx;
    tree->n = (uint32_t)n;
    tree->n_nodes = n ? 2 * (uint32_t)n - 1 : 0;
    const int rc = n ? build4<T>(tree, aabbs, cudaMemcpyHostToDevice) : (int)BVHGPU_OK;
    if (rc != BVHGPU_OK) { tree_release<T>(tree); delete tree; return rc; }
    *out = tree;
    return BVHGPU_OK;
}
template <class T> static int tree_nodes_impl(Tree4<T>* tree, typename D4<T>::Node* out_nodes, uint32_t* out_node_index) {
    if (!tree) { set_error("tree_nodes: null tree"); return BVHGPU_ERR_INVALID; }
    BVH_TRY(resolve_status(tree));
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    if (tree->n == 0) return BVHGPU_OK;
    if (out_nodes) BVH_CUDA_TRY(cudaMemcpyAsync(out_nodes, tree->d_nodes, sizeof(*out_nodes) * tree->n_nodes, cudaMemcpyDeviceToHost, ctx->stream));
    if (out_node_index) BVH_CUDA_TRY(cudaMemcpyAsync(out_node_index, tree->d_node_index, sizeof(uint32_t) * tree->n, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return BVHGPU_OK;
}
template <class T> static int flatten_impl(Tree4<T>* tree, typename D4<T>::Flat* out, size_t cap, size_t* len) {
    if (!tree) { set_error("flatten: null tree"); return BVHGPU_ERR_INVALID; }
    BVH_TRY(resolve_status(tree));
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(build_flat4(tree));
    if (len) *len = tree->n_flat;
    if (out) {
        if (cap < tree->n_flat) { set_error("flatten: capacity %zu < %zu flat nodes", cap, tree->n_flat); return BVHGPU_ERR_CAPACITY; }
        if (tree->n_flat) BVH_CUDA_TRY(cudaMemcpyAsync(out, tree->d_flat, sizeof(*out) * tree->n_flat, cudaMemcpyDeviceToHost, ctx->stream));
        BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    }
    return BVHGPU_OK;
}

// The tree type of dimension D: Bvh<T,2> lives embedded in the 3-D tree (dim2.cu), Bvh<T,4> has its own (dim4.cu).
template <int D, class T> using TreeOf = typename std::conditional<D == 4, Tree4<T>, Tree<T>>::type;

// A host batch staged on the device.  D = 3, 4: the C-ABI records as they are.  D = 2: records of 2-vectors (a Bvh<T,2> embedded in
// z = 0), lifted on the device before they reach the 3-D kernels: nvec 2-vectors and nscal scalars per record (dim2_lift), or
// RAY_RECORD: rays of 6 T (dim2_expand_rays, 9 T), or AABB_RECORD: boxes of 4 T (dim2_expand_aabbs, 6 T).  There is no fetch
// call for D = 2, so a short `cap` is answered with "call again with cap = *total" and the retained buffers are re-used by that call.
constexpr int RAY_RECORD = -1, AABB_RECORD = -2;
template <int D, class T> static int upload_records(bvhgpu_ctx* ctx, Scratch& scratch, const void* h, size_t n, int nvec, int nscal, T** d_out) {
    const size_t in_w = nvec == RAY_RECORD ? 3 * D : nvec == AABB_RECORD ? 2 * D : (size_t)D * nvec + nscal;
    T* d_in = nullptr;
    BVH_TRY(scratch.get(&d_in, n * in_w));
    BVH_CUDA_TRY(cudaMemcpyAsync(d_in, h, sizeof(T) * n * in_w, cudaMemcpyHostToDevice, ctx->stream));
    if (D != 2) { *d_out = d_in; return BVHGPU_OK; }
    T* d_lift = nullptr;
    BVH_TRY(scratch.get(&d_lift, n * (nvec == RAY_RECORD ? 9 : nvec == AABB_RECORD ? 6 : 3 * (size_t)nvec + nscal)));
    if (nvec == RAY_RECORD) BVH_TRY(dim2_expand_rays<T>(ctx, d_in, (uint32_t)n, d_lift));
    else if (nvec == AABB_RECORD) BVH_TRY(dim2_expand_aabbs<T>(ctx, d_in, (uint32_t)n, d_lift));
    else BVH_TRY(dim2_lift<T>(ctx, d_in, (uint32_t)n, nvec, nscal, d_lift));
    *d_out = d_lift;
    return BVHGPU_OK;
}
// The host-pointer ray traversal of a 2-D or 3-D tree runs into the tree's retained buffers, which bvhgpu_traverse_fetch_* reads
// later.  The hit buffer starts at max(hits_cap, 4 n, 1024).  traverse_device has a scan of its own and cannot fill again from it:
// when run(d_offsets, d_hits, cap, &tot) reports BVHGPU_ERR_CAPACITY with a total the u32 offsets can hold, the buffer grows to that
// total and the call runs once more.  (The other CSR walks grow their buffer between the passes, csr_run of csr.cuh.)
template <class T, class Run> static int run_retained(Tree<T>* tree, size_t n, size_t* tot, Run run) {
    size_t want = std::max<size_t>(std::max<size_t>(tree->hits_cap, 4 * n), 1024);
    int rc = BVHGPU_OK;
    for (int attempt = 0; attempt < 2; ++attempt) {
        rc = ensure_result_buffers(tree, n, want);
        if (rc != BVHGPU_OK) break;
        rc = run(tree->d_offsets, tree->d_hits, tree->hits_cap, tot);
        if (rc == BVHGPU_ERR_CAPACITY && *tot <= 0xFFFFFFFFull && *tot > tree->hits_cap && attempt == 0) { want = *tot; continue; }   // grow once and redo
        break;
    }
    return rc;
}

static bool bad_mode(int mode) { return mode != BVHGPU_TRAVERSE_BVH && mode != BVHGPU_TRAVERSE_FLAT; }

// Ray traversal, host pointers.  D = 3: the streamed host traversal.  D = 2: rays of 6 T lifted on the device (dim2_expand_rays)
// and walked by traverse_device.  D = 4: rays of 12 T through traverse_csr.
template <int D, class T>
static int traverse_host_impl(TreeOf<D, T>* tree, int mode, const void* rays, uint32_t fmt, size_t nrays,
                              uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total) {
    if (!tree || (nrays && !rays) || !offsets) { set_error("traverse: null argument"); return BVHGPU_ERR_INVALID; }
    if (D != 2) BVH_TRY(check_n("traverse", nrays));
    if (D == 4 && bad_mode(mode)) { set_error("traverse: bad mode %d", mode); return BVHGPU_ERR_INVALID; }
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(resolve_status(tree));
    if (D == 2) BVH_TRY(check_n("traverse", nrays));            // a 2-D tree reports a sticky failure first
    Scratch scratch(ctx);
    T* d_rays = nullptr;
    if constexpr (D == 4) {
        if (nrays && tree->n) BVH_TRY(upload_records<D>(ctx, scratch, rays, nrays, RAY_RECORD, 0, &d_rays));
        return traverse_csr<T>(tree, mode, d_rays, nrays, CsrOut::to_host(offsets, hits, cap, total, 4), "traverse");
    } else if constexpr (D == 2) {
        if (nrays) BVH_TRY(upload_records<D>(ctx, scratch, rays, nrays, RAY_RECORD, 0, &d_rays));
        size_t tot = 0;
        const int rc = run_retained(tree, nrays, &tot, [&](uint32_t* d_off, uint32_t* d_hits, size_t hcap, size_t* t) {
            return traverse_device<T>(tree, mode, d_rays, BVHGPU_RAYS_FULL, nrays, d_off, d_hits, hcap, t);
        });
        if (total) *total = tot;
        if (rc != BVHGPU_OK) return rc;
        return copy_retained(tree, "traverse", nrays, tot, offsets, hits, cap);
    } else {
        if (nrays == 0 || tree->n == 0) {                            // nothing to pipeline
            size_t tot0 = 0;
            BVH_TRY(ensure_result_buffers(tree, nrays, 1024));
            BVH_TRY(traverse_device<T>(tree, mode, nullptr, fmt, nrays, tree->d_offsets, tree->d_hits, tree->hits_cap, &tot0));
            BVH_CUDA_TRY(cudaMemcpyAsync(offsets, tree->d_offsets, sizeof(uint32_t) * (nrays + 1), cudaMemcpyDeviceToHost, ctx->stream));
            BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
            if (total) *total = 0;
            return BVHGPU_OK;
        }
        size_t tot = 0;
        const int rc = run_retained(tree, nrays, &tot, [&](uint32_t*, uint32_t*, size_t, size_t* t) {   // copies back for itself
            return traverse_host_pipelined<T>(tree, mode, rays, fmt, nrays, offsets, hits, cap, t);
        });
        if (total) *total = tot;
        if (rc != BVHGPU_OK) return rc;
        if (tot > cap) {
            set_error("traverse: %zu hits do not fit the caller's capacity %zu (use bvhgpu_traverse_fetch_*)", tot, cap);
            return BVHGPU_ERR_CAPACITY;
        }
        return BVHGPU_OK;
    }
}
// Ray traversal, device pointers (D = 3, 4): enqueued on the context's stream; synchronises only to return *total.
template <int D, class T>
static int traverse_dev_impl(TreeOf<D, T>* tree, int mode, const void* d_rays, uint32_t fmt, size_t nrays, uint32_t* d_offsets, uint32_t* d_hits,
                             size_t cap, size_t* total, const char* what) {
    if (!tree || !d_offsets || (nrays && !d_rays)) { set_error("%s: null argument", what); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(tree->ctx->device));
    if constexpr (D == 4) return traverse_csr<T>(tree, mode, d_rays, nrays, CsrOut::device(d_offsets, d_hits, cap, total), "traverse");
    else return traverse_device<T>(tree, mode, d_rays, fmt, nrays, d_offsets, d_hits, cap, total);
}

// Aabb / Point / Ball queries, host pointers: records of 2D / D / D + 1 T.  query_csr also serves the library's internal kinds
// (nearest_candidates): only the public ones get through here.
template <int D, class T>
static int query_host_impl(TreeOf<D, T>* tree, int mode, int kind, const T* queries, size_t n, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total) {
    if (!tree || (n && !queries) || !offsets) { set_error("query: null argument"); return BVHGPU_ERR_INVALID; }
    if (kind < BVHGPU_QUERY_AABB || kind > BVHGPU_QUERY_BALL) { set_error("query: bad kind %d", kind); return BVHGPU_ERR_INVALID; }
    BVH_TRY(check_n("query", n));
    if (bad_mode(mode)) { set_error("query: bad mode %d", mode); return BVHGPU_ERR_INVALID; }
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(resolve_status(tree));
    const int nvec = kind == BVHGPU_QUERY_AABB ? 2 : 1, nscal = kind == BVHGPU_QUERY_BALL ? 1 : 0;
    T* d_q = nullptr;
    Scratch scratch(ctx);                                           // released on every return path
    if (n) BVH_TRY(upload_records<D>(ctx, scratch, queries, n, nvec, nscal, &d_q));
    return query_csr(tree, mode, kind, d_q, n, CsrOut::to_host(offsets, hits, cap, total, 16), "query");
}
// Queries, device pointers (D = 3, 4).  With `total` given the call synchronises, and the CSR is complete when it returns.
template <int D, class T>
static int query_dev_impl(TreeOf<D, T>* tree, int mode, int kind, const void* d_queries, size_t n, uint32_t* d_offsets, uint32_t* d_hits, size_t cap, size_t* total) {
    if (!tree || !d_offsets || (n && !d_queries)) { set_error("query_dev: null argument"); return BVHGPU_ERR_INVALID; }
    if (kind < BVHGPU_QUERY_AABB || kind > BVHGPU_QUERY_BALL) { set_error("query_dev: bad kind %d", kind); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(tree->ctx->device));
    const int rc = query_csr(tree, mode, kind, d_queries, n, CsrOut::device(d_offsets, d_hits, cap, total), "query_dev");
    if (total && (rc == BVHGPU_OK || rc == BVHGPU_ERR_CAPACITY)) BVH_CUDA_TRY(cudaStreamSynchronize(tree->ctx->stream));
    return rc;
}

// Self-overlap pairs, host pointers: through the retained buffers (bvhgpu_traverse_fetch_* reads them in 3-D).  n < 2: all-zero
// offsets, no device work.
template <int D, class T>
static int overlap_host_impl(TreeOf<D, T>* tree, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total) {
    if (!tree || !offsets) { set_error("overlap_pairs: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(tree->ctx->device));
    return overlap_csr(tree, CsrOut::to_host(offsets, hits, cap, total, 4), "overlap_pairs");
}
// Self-overlap pairs, device pointers (D = 3, 4), on the context's stream.  With `total` the call returns once the total is known
// and the CSR is complete.
template <int D, class T>
static int overlap_dev_impl(TreeOf<D, T>* tree, void* d_offsets, void* d_hits, size_t cap, size_t* total) {
    if (!tree || !d_offsets) { set_error("overlap_pairs_dev: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(tree->ctx->device));
    const int rc = overlap_csr(tree, CsrOut::device((uint32_t*)d_offsets, (uint32_t*)d_hits, cap, total), "overlap_pairs_dev");
    if (total && (rc == BVHGPU_OK || rc == BVHGPU_ERR_CAPACITY)) BVH_CUDA_TRY(cudaStreamSynchronize(tree->ctx->stream));
    return rc;
}

// Overlap between two trees: the arguments of both forms.  The trees must share a context, whose one stream then orders the walk
// after every call pending on either tree.
template <class Tr> static int overlap_trees_args(const char* what, const Tr* a, const Tr* b, const void* offsets) {
    if (!a || !b || !offsets) { set_error("%s: null argument", what); return BVHGPU_ERR_INVALID; }
    if (a->ctx != b->ctx) { set_error("%s: the two trees belong to different contexts", what); return BVHGPU_ERR_INVALID; }
    return BVHGPU_OK;
}
// Overlap between two trees, host pointers: through A's retained buffers (bvhgpu_traverse_fetch_* on A reads them in 3-D).
// n_a = 0 or n_b = 0: all-zero offsets, no device work.
template <int D, class T>
static int overlap_trees_host_impl(TreeOf<D, T>* a, TreeOf<D, T>* b, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total) {
    BVH_TRY(overlap_trees_args("overlap_trees", a, b, offsets));
    BVH_CUDA_TRY(cudaSetDevice(a->ctx->device));
    return overlap_trees_csr(a, b, CsrOut::to_host(offsets, hits, cap, total, 4), "overlap_trees");
}
// Overlap between two trees, device pointers (D = 3, 4), on the context's stream.  With `total` the call returns once the total is
// known and the CSR is complete.
template <int D, class T>
static int overlap_trees_dev_impl(TreeOf<D, T>* a, TreeOf<D, T>* b, void* d_offsets, void* d_hits, size_t cap, size_t* total) {
    BVH_TRY(overlap_trees_args("overlap_trees_dev", a, b, d_offsets));
    BVH_CUDA_TRY(cudaSetDevice(a->ctx->device));
    const int rc = overlap_trees_csr(a, b, CsrOut::device((uint32_t*)d_offsets, (uint32_t*)d_hits, cap, total), "overlap_trees_dev");
    if (total && (rc == BVHGPU_OK || rc == BVHGPU_ERR_CAPACITY)) BVH_CUDA_TRY(cudaStreamSynchronize(a->ctx->stream));
    return rc;
}

// Triangle pairs (D = 3): the overlap forms above with the triangles' predicate.  Self: host pointers through the retained buffers,
// device pointers on the context's stream.
template <class T>
static int triangle_pairs_host_impl(Tree<T>* tree, int skip_shared, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total) {
    if (!tree || !offsets) { set_error("triangle_pairs: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(tree->ctx->device));
    return triangle_pairs_csr(tree, skip_shared, CsrOut::to_host(offsets, hits, cap, total, 4), "triangle_pairs");
}
template <class T>
static int triangle_pairs_dev_impl(Tree<T>* tree, int skip_shared, void* d_offsets, void* d_hits, size_t cap, size_t* total) {
    if (!tree || !d_offsets) { set_error("triangle_pairs_dev: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(tree->ctx->device));
    const int rc = triangle_pairs_csr(tree, skip_shared, CsrOut::device((uint32_t*)d_offsets, (uint32_t*)d_hits, cap, total), "triangle_pairs_dev");
    if (total && (rc == BVHGPU_OK || rc == BVHGPU_ERR_CAPACITY)) BVH_CUDA_TRY(cudaStreamSynchronize(tree->ctx->stream));
    return rc;
}
template <class T>
static int triangle_pairs_trees_host_impl(Tree<T>* a, Tree<T>* b, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total) {
    BVH_TRY(overlap_trees_args("triangle_pairs_trees", a, b, offsets));
    BVH_CUDA_TRY(cudaSetDevice(a->ctx->device));
    return triangle_pairs_trees_csr(a, b, CsrOut::to_host(offsets, hits, cap, total, 4), "triangle_pairs_trees");
}
template <class T>
static int triangle_pairs_trees_dev_impl(Tree<T>* a, Tree<T>* b, void* d_offsets, void* d_hits, size_t cap, size_t* total) {
    BVH_TRY(overlap_trees_args("triangle_pairs_trees_dev", a, b, d_offsets));
    BVH_CUDA_TRY(cudaSetDevice(a->ctx->device));
    const int rc = triangle_pairs_trees_csr(a, b, CsrOut::device((uint32_t*)d_offsets, (uint32_t*)d_hits, cap, total), "triangle_pairs_trees_dev");
    if (total && (rc == BVHGPU_OK || rc == BVHGPU_ERR_CAPACITY)) BVH_CUDA_TRY(cudaStreamSynchronize(a->ctx->stream));
    return rc;
}

// nearest_to, host pointers: D T per point.  The mode of a 3-D call is checked by nearest_device.
template <int D, class T>
static int nearest_host_impl(TreeOf<D, T>* tree, int mode, const T* points, size_t n, uint32_t* out_shape, T* out_dist, int use_triangles = 0) {
    if (!tree || (n && (!points || !out_shape || !out_dist))) { set_error("nearest: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_TRY(check_n("nearest", n));
    if (D != 3 && bad_mode(mode)) { set_error("nearest: bad mode %d", mode); return BVHGPU_ERR_INVALID; }
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(resolve_status(tree));
    if (n == 0) return BVHGPU_OK;
    T *d_p = nullptr, *d_d = nullptr;
    uint32_t* d_s = nullptr;
    Scratch scratch(ctx);
    BVH_TRY(upload_records<D>(ctx, scratch, points, n, 1, 0, &d_p));
    BVH_TRY(scratch.get(&d_d, n));
    BVH_TRY(scratch.get(&d_s, n));
    int rc;
    if constexpr (D == 4) rc = nearest4_device<T>(tree, mode, d_p, n, d_s, d_d);
    else rc = nearest_device<T>(tree, mode, d_p, n, d_s, d_d, use_triangles);
    if (rc == BVHGPU_OK) {
        BVH_CUDA_TRY(cudaMemcpyAsync(out_shape, d_s, sizeof(uint32_t) * n, cudaMemcpyDeviceToHost, ctx->stream));
        BVH_CUDA_TRY(cudaMemcpyAsync(out_dist, d_d, sizeof(T) * n, cudaMemcpyDeviceToHost, ctx->stream));
        BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    }
    return rc;
}

// k nearest shapes, host pointers: D T per point (D = 2 lifted to z = 0, dim2.cu), n optional limits; n * k results copied back.
template <int D, class T>
static int knn_host_impl(TreeOf<D, T>* tree, const T* points, size_t n, uint32_t k, const T* max_dist, uint32_t* out_shape, T* out_dist) {
    if (!tree || (n && (!points || !out_shape || !out_dist))) { set_error("knn: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_TRY(check_n("knn", n));
    if (k < 1 || k > BVHGPU_KNN_MAX_K) { set_error("knn: k = %u outside 1 .. %d", k, BVHGPU_KNN_MAX_K); return BVHGPU_ERR_INVALID; }
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(resolve_status(tree));
    if (n == 0) return BVHGPU_OK;
    T *d_p = nullptr, *d_r = nullptr, *d_d = nullptr;
    uint32_t* d_s = nullptr;
    Scratch scratch(ctx);
    BVH_TRY(upload_records<D>(ctx, scratch, points, n, 1, 0, &d_p));
    if (max_dist) {
        BVH_TRY(scratch.get(&d_r, n));
        BVH_CUDA_TRY(cudaMemcpyAsync(d_r, max_dist, sizeof(T) * n, cudaMemcpyHostToDevice, ctx->stream));
    }
    BVH_TRY(scratch.get(&d_s, n * k));
    BVH_TRY(scratch.get(&d_d, n * k));
    if constexpr (D == 4) BVH_TRY(knn4_device<T>(tree, d_p, n, k, d_r, d_s, d_d));
    else BVH_TRY(knn_device<T>(tree, d_p, n, k, d_r, d_s, d_d));
    BVH_CUDA_TRY(cudaMemcpyAsync(out_shape, d_s, sizeof(uint32_t) * n * k, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaMemcpyAsync(out_dist, d_d, sizeof(T) * n * k, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return BVHGPU_OK;
}
// k nearest shapes, device pointers (D = 3, 4): the device driver checks n, k and the tree's status.
template <int D, class T>
static int knn_dev_impl(TreeOf<D, T>* tree, const void* d_points, size_t n, uint32_t k, const void* d_max_dist, void* d_shape, void* d_dist) {
    if (!tree || (n && (!d_points || !d_shape || !d_dist))) { set_error("knn_dev: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(tree->ctx->device));
    if constexpr (D == 4) return knn4_device<T>(tree, (const T*)d_points, n, k, (const T*)d_max_dist, (uint32_t*)d_shape, (T*)d_dist);
    else return knn_device<T>(tree, (const T*)d_points, n, k, (const T*)d_max_dist, (uint32_t*)d_shape, (T*)d_dist);
}
// k nearest triangles (D = 3), host pointers: as knn_host_impl, plus n * k * 3 closest-point coordinates when out_closest is given.
// Every check (pointers, n, k, triangles, status) runs in knn_tri_device or before it, so a refused call writes nothing.
template <class T>
static int knn_tri_host_impl(Tree<T>* tree, const T* points, size_t n, uint32_t k, const T* max_dist, uint32_t* out_shape, T* out_dist, T* out_closest) {
    if (!tree || (n && (!points || !out_shape || !out_dist))) { set_error("knn_triangles: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_TRY(check_n("knn_triangles", n));
    if (k < 1 || k > BVHGPU_KNN_MAX_K) { set_error("knn_triangles: k = %u outside 1 .. %d", k, BVHGPU_KNN_MAX_K); return BVHGPU_ERR_INVALID; }
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    if (n == 0) return knn_tri_device<T>(tree, nullptr, 0, k, nullptr, nullptr, nullptr, nullptr);      // the triangle and status checks
    T *d_p = nullptr, *d_r = nullptr, *d_d = nullptr, *d_q = nullptr;
    uint32_t* d_s = nullptr;
    Scratch scratch(ctx);
    BVH_TRY(upload_records<3>(ctx, scratch, points, n, 1, 0, &d_p));
    if (max_dist) {
        BVH_TRY(scratch.get(&d_r, n));
        BVH_CUDA_TRY(cudaMemcpyAsync(d_r, max_dist, sizeof(T) * n, cudaMemcpyHostToDevice, ctx->stream));
    }
    const size_t nk = n * k;
    BVH_TRY(scratch.get(&d_s, nk));
    BVH_TRY(scratch.get(&d_d, nk));
    if (out_closest) BVH_TRY(scratch.get(&d_q, 3 * nk));
    BVH_TRY(knn_tri_device<T>(tree, d_p, n, k, d_r, d_s, d_d, d_q));
    BVH_CUDA_TRY(cudaMemcpyAsync(out_shape, d_s, sizeof(uint32_t) * nk, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaMemcpyAsync(out_dist, d_d, sizeof(T) * nk, cudaMemcpyDeviceToHost, ctx->stream));
    if (out_closest) BVH_CUDA_TRY(cudaMemcpyAsync(out_closest, d_q, sizeof(T) * 3 * nk, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return BVHGPU_OK;
}
// k nearest triangles, device pointers: knn_tri_device checks n, k, the triangles and the tree's status.
template <class T>
static int knn_tri_dev_impl(Tree<T>* tree, const void* d_points, size_t n, uint32_t k, const void* d_max_dist, void* d_shape, void* d_dist, void* d_closest) {
    if (!tree || (n && (!d_points || !d_shape || !d_dist))) { set_error("knn_triangles_dev: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(tree->ctx->device));
    return knn_tri_device<T>(tree, (const T*)d_points, n, k, (const T*)d_max_dist, (uint32_t*)d_shape, (T*)d_dist, (T*)d_closest);
}

template <int D, class T>
static int nearest_candidates_host_impl(TreeOf<D, T>* tree, const T* points, size_t n, uint32_t* offsets, uint32_t* cand, size_t cap, size_t* total) {
    if (!tree || (n && !points) || !offsets) { set_error("nearest_candidates: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_TRY(check_n("nearest_candidates", n));
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(resolve_status(tree));
    T* d_p = nullptr;
    Scratch scratch(ctx);
    if (n) BVH_TRY(upload_records<D>(ctx, scratch, points, n, 1, 0, &d_p));
    return nearest_candidates_csr(tree, d_p, n, CsrOut::to_host(offsets, cand, cap, total, 16));
}

// Distance-ordered traversal, host pointers.  D = 3, 4: the C-ABI rays as they are.  D = 2: rays of 6 T lifted on the device
// (dim2_expand_rays: origin.z = 0, inv_direction.z = +inf) and walked by the 3-D ordered kernel on the embedded tree, whose records
// span z = [-1, +1]: the z slab is (-inf, +inf) and leaves both the set and the distances of the 2-D slice unchanged (dim2.cu).
template <int D, class T>
static int ordered_host_impl(TreeOf<D, T>* tree, const void* rays, size_t nrays, int ascending,
                             uint32_t* offsets, uint32_t* hits, T* dists, size_t cap, size_t* total) {
    if (!tree || (nrays && !rays) || !offsets || (cap && (!hits || !dists))) { set_error("traverse_ordered: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_TRY(check_n("traverse_ordered", nrays));
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(resolve_status(tree));
    T* d_rays = nullptr;
    uint32_t *d_off = nullptr, *d_hits = nullptr;
    T* d_dists = nullptr;
    Scratch scratch(ctx);
    if (nrays) BVH_TRY(upload_records<D>(ctx, scratch, rays, nrays, RAY_RECORD, 0, &d_rays));
    BVH_TRY(scratch.get(&d_off, nrays + 1));
    BVH_TRY(scratch.get(&d_hits, cap));
    BVH_TRY(scratch.get(&d_dists, cap));
    size_t tot = 0;
    int rc = ordered_csr(tree, d_rays, nrays, ascending, d_off, d_hits, d_dists, cap, &tot);
    if (total) *total = tot;
    if (rc == BVHGPU_OK || rc == BVHGPU_ERR_CAPACITY) {
        cudaMemcpyAsync(offsets, d_off, sizeof(uint32_t) * (nrays + 1), cudaMemcpyDeviceToHost, ctx->stream);
        const size_t m = std::min(tot, cap);
        if (m) { cudaMemcpyAsync(hits, d_hits, sizeof(uint32_t) * m, cudaMemcpyDeviceToHost, ctx->stream); cudaMemcpyAsync(dists, d_dists, sizeof(T) * m, cudaMemcpyDeviceToHost, ctx->stream); }
        cudaError_t e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) { set_error("traverse_ordered: %s", cudaGetErrorString(e)); rc = BVHGPU_ERR_CUDA; }
    }
    return rc;
}

// Closest hit / any hit on the device.  D = 3: closest_hit_device / any_hit_device (rays of 9 or 6 T, AABB or triangle mode; they
// check n, the layout and the tree's status).  D = 2, 4: AABB mode, rays of 3D T straight to closest_aabb_device<D, T> /
// any_hit_aabb_device<D, T> (D = 2 tests x and y of the embedded tree), which leave the checks to the caller.
template <int D, class T>
static int closest_driver(TreeOf<D, T>* tree, const void* d_rays, uint32_t fmt, size_t nrays, int use_triangles, uint32_t* d_shape, T* d_dist, T* d_uv) {
    if constexpr (D == 3) return closest_hit_device<T>(tree, d_rays, fmt, nrays, use_triangles, d_shape, d_dist, d_uv);
    else return closest_aabb_device<D, T>(tree->ctx, tree->d_nodes, tree->n, tree->d_aabb, (const T*)d_rays, nrays, d_shape, d_dist);
}
template <int D, class T>
static int any_hit_driver(TreeOf<D, T>* tree, const void* d_rays, uint32_t fmt, size_t nrays, const T* d_tmax, int use_triangles, uint32_t* d_shape) {
    if constexpr (D == 3) return any_hit_device<T>(tree, d_rays, fmt, nrays, d_tmax, use_triangles, d_shape);
    else return any_hit_aabb_device<D, T>(tree->ctx, tree->d_nodes, tree->n, tree->d_aabb, (const T*)d_rays, nrays, d_tmax, d_shape);
}

template <int D, class T>
static int closest_host_impl(TreeOf<D, T>* tree, const void* rays, uint32_t fmt, size_t nrays, int use_triangles, uint32_t* out_shape, T* out_dist, T* out_uv) {
    if (!tree || (nrays && (!rays || !out_shape || !out_dist))) { set_error("closest_hit: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_TRY(check_n("closest_hit", nrays));
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(resolve_status(tree));
    if (nrays == 0) return BVHGPU_OK;
    Scratch scratch(ctx);
    const size_t ray_bytes = (D != 3 ? 3 * D : fmt == BVHGPU_RAYS_FULL ? 9 : 6) * sizeof(T);
    unsigned char* d_rays = nullptr;
    uint32_t* d_s = nullptr;
    T *d_d = nullptr, *d_uv = nullptr;
    BVH_TRY(scratch.get(&d_rays, ray_bytes * nrays));
    BVH_TRY(scratch.get(&d_s, nrays));
    BVH_TRY(scratch.get(&d_d, nrays));
    if (out_uv) BVH_TRY(scratch.get(&d_uv, 2 * nrays));
    BVH_CUDA_TRY(cudaMemcpyAsync(d_rays, rays, ray_bytes * nrays, cudaMemcpyHostToDevice, ctx->stream));
    BVH_TRY((closest_driver<D, T>(tree, d_rays, fmt, nrays, use_triangles, d_s, d_d, d_uv)));
    BVH_CUDA_TRY(cudaMemcpyAsync(out_shape, d_s, sizeof(uint32_t) * nrays, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaMemcpyAsync(out_dist, d_d, sizeof(T) * nrays, cudaMemcpyDeviceToHost, ctx->stream));
    if (out_uv) BVH_CUDA_TRY(cudaMemcpyAsync(out_uv, d_uv, sizeof(T) * 2 * nrays, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return BVHGPU_OK;
}
template <int D, class T>
static int closest_dev_impl(TreeOf<D, T>* tree, const void* d_rays, uint32_t fmt, size_t nrays, int use_triangles, void* d_shape, void* d_dist, void* d_uv) {
    if (!tree || (nrays && (!d_rays || !d_shape || !d_dist))) { set_error("closest_hit_dev: null argument"); return BVHGPU_ERR_INVALID; }
    if (D == 4) BVH_TRY(check_n("closest_hit_dev", nrays));
    if (D == 4) BVH_TRY(resolve_status(tree));
    BVH_CUDA_TRY(cudaSetDevice(tree->ctx->device));
    return closest_driver<D, T>(tree, d_rays, fmt, nrays, use_triangles, (uint32_t*)d_shape, (T*)d_dist, (T*)d_uv);
}

// Any hit, host pointers: rays and the optional limits (nullptr: +inf) staged as closest_host_impl stages the rays.
template <int D, class T>
static int any_hit_host_impl(TreeOf<D, T>* tree, const void* rays, size_t nrays, const T* tmax, int use_triangles, uint32_t* out_shape) {
    if (!tree || (nrays && (!rays || !out_shape))) { set_error("any_hit: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_TRY(check_n("any_hit", nrays));
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(resolve_status(tree));
    if (nrays == 0) return BVHGPU_OK;
    Scratch scratch(ctx);
    const size_t ray_w = 3 * D;
    T *d_rays = nullptr, *d_tmax = nullptr;
    uint32_t* d_s = nullptr;
    BVH_TRY(scratch.get(&d_rays, ray_w * nrays));
    BVH_TRY(scratch.get(&d_s, nrays));
    BVH_CUDA_TRY(cudaMemcpyAsync(d_rays, rays, sizeof(T) * ray_w * nrays, cudaMemcpyHostToDevice, ctx->stream));
    if (tmax) {
        BVH_TRY(scratch.get(&d_tmax, nrays));
        BVH_CUDA_TRY(cudaMemcpyAsync(d_tmax, tmax, sizeof(T) * nrays, cudaMemcpyHostToDevice, ctx->stream));
    }
    BVH_TRY((any_hit_driver<D, T>(tree, d_rays, BVHGPU_RAYS_FULL, nrays, d_tmax, use_triangles, d_s)));
    BVH_CUDA_TRY(cudaMemcpyAsync(out_shape, d_s, sizeof(uint32_t) * nrays, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return BVHGPU_OK;
}
template <int D, class T>
static int any_hit_dev_impl(TreeOf<D, T>* tree, const void* d_rays, uint32_t fmt, size_t nrays, const void* d_tmax, int use_triangles, void* d_shape) {
    if (!tree || (nrays && (!d_rays || !d_shape))) { set_error("any_hit_dev: null argument"); return BVHGPU_ERR_INVALID; }
    if (D == 4) BVH_TRY(check_n("any_hit_dev", nrays));
    if (D == 4) BVH_TRY(resolve_status(tree));
    BVH_CUDA_TRY(cudaSetDevice(tree->ctx->device));
    return any_hit_driver<D, T>(tree, d_rays, fmt, nrays, (const T*)d_tmax, use_triangles, (uint32_t*)d_shape);
}

// Multi hit: the first k hits per ray, rows of k slots.  D = 3: multi_hit_device (checks n, the layout, the status and the triangles);
// D = 2, 4: multi_hit_aabb_device, as any_hit_driver.
template <int D, class T>
static int multi_hit_driver(TreeOf<D, T>* tree, const void* d_rays, uint32_t fmt, size_t nrays, uint32_t k, const T* d_tmax, int use_triangles,
                            uint32_t* d_shape, T* d_dist, T* d_uv) {
    if constexpr (D == 3) return multi_hit_device<T>(tree, d_rays, fmt, nrays, k, d_tmax, use_triangles, d_shape, d_dist, d_uv);
    else return multi_hit_aabb_device<D, T>(tree->ctx, tree->d_nodes, tree->n, tree->d_aabb, (const T*)d_rays, nrays, k, d_tmax, d_shape, d_dist);
}
static int check_k(const char* what, uint32_t k) {
    if (k < 1 || k > BVHGPU_KNN_MAX_K) { set_error("%s: k = %u outside 1 .. %d", what, k, BVHGPU_KNN_MAX_K); return BVHGPU_ERR_INVALID; }
    return BVHGPU_OK;
}
// Multi hit, host pointers: rays and the optional limits staged as any_hit_host_impl stages them, nrays * k slots copied back.  Every
// refusal happens before the first copy to the caller's buffers.
template <int D, class T>
static int multi_hit_host_impl(TreeOf<D, T>* tree, const void* rays, size_t nrays, uint32_t k, const T* tmax, int use_triangles, uint32_t* out_shape,
                               T* out_dist, T* out_uv) {
    if (!tree || (nrays && (!rays || !out_shape || !out_dist))) { set_error("multi_hit: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_TRY(check_n("multi_hit", nrays));
    BVH_TRY(check_k("multi_hit", k));
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(resolve_status(tree));
    if (nrays == 0) return BVHGPU_OK;
    Scratch scratch(ctx);
    const size_t ray_w = 3 * D, slots = nrays * k;
    T *d_rays = nullptr, *d_tmax = nullptr, *d_d = nullptr, *d_uv = nullptr;
    uint32_t* d_s = nullptr;
    BVH_TRY(scratch.get(&d_rays, ray_w * nrays));
    BVH_TRY(scratch.get(&d_s, slots));
    BVH_TRY(scratch.get(&d_d, slots));
    if (out_uv) BVH_TRY(scratch.get(&d_uv, 2 * slots));
    BVH_CUDA_TRY(cudaMemcpyAsync(d_rays, rays, sizeof(T) * ray_w * nrays, cudaMemcpyHostToDevice, ctx->stream));
    if (tmax) {
        BVH_TRY(scratch.get(&d_tmax, nrays));
        BVH_CUDA_TRY(cudaMemcpyAsync(d_tmax, tmax, sizeof(T) * nrays, cudaMemcpyHostToDevice, ctx->stream));
    }
    BVH_TRY((multi_hit_driver<D, T>(tree, d_rays, BVHGPU_RAYS_FULL, nrays, k, d_tmax, use_triangles, d_s, d_d, d_uv)));
    BVH_CUDA_TRY(cudaMemcpyAsync(out_shape, d_s, sizeof(uint32_t) * slots, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaMemcpyAsync(out_dist, d_d, sizeof(T) * slots, cudaMemcpyDeviceToHost, ctx->stream));
    if (out_uv) BVH_CUDA_TRY(cudaMemcpyAsync(out_uv, d_uv, sizeof(T) * 2 * slots, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return BVHGPU_OK;
}
template <int D, class T>
static int multi_hit_dev_impl(TreeOf<D, T>* tree, const void* d_rays, uint32_t fmt, size_t nrays, uint32_t k, const void* d_tmax, int use_triangles,
                              void* d_shape, void* d_dist, void* d_uv) {
    if (!tree || (nrays && (!d_rays || !d_shape || !d_dist))) { set_error("multi_hit_dev: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_TRY(check_k("multi_hit_dev", k));
    if (D == 4) BVH_TRY(check_n("multi_hit_dev", nrays));
    if (D == 4) BVH_TRY(resolve_status(tree));
    BVH_CUDA_TRY(cudaSetDevice(tree->ctx->device));
    return multi_hit_driver<D, T>(tree, d_rays, fmt, nrays, k, (const T*)d_tmax, use_triangles, (uint32_t*)d_shape, (T*)d_dist, (T*)d_uv);
}

// Crossing counts, point-in-mesh and signed distance (D = 3).  Host forms: the null checks, n, the rule, the tree's status and n = 0 are
// settled before anything is staged; the device drivers (closest.cu) check the layout, the status and the triangles before they launch,
// and the caller's buffers are written only after they returned OK.
template <class T>
static int count_hits_host_impl(Tree<T>* tree, const void* rays, size_t nrays, const T* tmax, uint32_t* out_front, uint32_t* out_back) {
    if (!tree || (nrays && (!rays || !out_front || !out_back))) { set_error("count_hits: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_TRY(check_n("count_hits", nrays));
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(resolve_status(tree));
    if (nrays == 0) return BVHGPU_OK;
    Scratch scratch(ctx);
    T *d_rays = nullptr, *d_tmax = nullptr;
    uint32_t *d_f = nullptr, *d_b = nullptr;
    BVH_TRY(scratch.get(&d_rays, 9 * nrays));
    BVH_TRY(scratch.get(&d_f, nrays));
    BVH_TRY(scratch.get(&d_b, nrays));
    BVH_CUDA_TRY(cudaMemcpyAsync(d_rays, rays, sizeof(T) * 9 * nrays, cudaMemcpyHostToDevice, ctx->stream));
    if (tmax) {
        BVH_TRY(scratch.get(&d_tmax, nrays));
        BVH_CUDA_TRY(cudaMemcpyAsync(d_tmax, tmax, sizeof(T) * nrays, cudaMemcpyHostToDevice, ctx->stream));
    }
    BVH_TRY(count_hits_device<T>(tree, d_rays, BVHGPU_RAYS_FULL, nrays, d_tmax, d_f, d_b));
    BVH_CUDA_TRY(cudaMemcpyAsync(out_front, d_f, sizeof(uint32_t) * nrays, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaMemcpyAsync(out_back, d_b, sizeof(uint32_t) * nrays, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return BVHGPU_OK;
}
template <class T>
static int count_hits_dev_impl(Tree<T>* tree, const void* d_rays, uint32_t fmt, size_t nrays, const void* d_tmax, void* d_front, void* d_back) {
    if (!tree || (nrays && (!d_rays || !d_front || !d_back))) { set_error("count_hits_dev: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(tree->ctx->device));
    return count_hits_device<T>(tree, d_rays, fmt, nrays, (const T*)d_tmax, (uint32_t*)d_front, (uint32_t*)d_back);
}
static int check_fill_rule(const char* what, int rule) {
    if (rule != BVHGPU_FILL_EVEN_ODD && rule != BVHGPU_FILL_NONZERO) { set_error("%s: unknown fill rule %d", what, rule); return BVHGPU_ERR_INVALID; }
    return BVHGPU_OK;
}
template <class T>
static int contains_host_impl(Tree<T>* tree, const T* points, size_t n, int rule, uint8_t* out_inside) {
    if (!tree || (n && (!points || !out_inside))) { set_error("contains_points: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_TRY(check_n("contains_points", n));
    BVH_TRY(check_fill_rule("contains_points", rule));
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(resolve_status(tree));
    if (n == 0) return BVHGPU_OK;
    Scratch scratch(ctx);
    T* d_p = nullptr;
    uint8_t* d_in = nullptr;
    BVH_TRY(upload_records<3>(ctx, scratch, points, n, 1, 0, &d_p));
    BVH_TRY(scratch.get(&d_in, n));
    BVH_TRY(contains_points_device<T>(tree, d_p, n, rule, d_in));
    BVH_CUDA_TRY(cudaMemcpyAsync(out_inside, d_in, n, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return BVHGPU_OK;
}
template <class T>
static int contains_dev_impl(Tree<T>* tree, const void* d_points, size_t n, int rule, void* d_inside) {
    if (!tree || (n && (!d_points || !d_inside))) { set_error("contains_points_dev: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(tree->ctx->device));
    return contains_points_device<T>(tree, (const T*)d_points, n, rule, (uint8_t*)d_inside);
}
template <class T>
static int signed_distance_host_impl(Tree<T>* tree, const T* points, size_t n, int rule, uint32_t* out_shape, T* out_dist, T* out_closest) {
    if (!tree || (n && (!points || !out_shape || !out_dist))) { set_error("signed_distance: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_TRY(check_n("signed_distance", n));
    BVH_TRY(check_fill_rule("signed_distance", rule));
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(resolve_status(tree));
    if (n == 0) return BVHGPU_OK;
    Scratch scratch(ctx);
    T *d_p = nullptr, *d_d = nullptr, *d_q = nullptr;
    uint32_t* d_s = nullptr;
    BVH_TRY(upload_records<3>(ctx, scratch, points, n, 1, 0, &d_p));
    BVH_TRY(scratch.get(&d_s, n));
    BVH_TRY(scratch.get(&d_d, n));
    if (out_closest) BVH_TRY(scratch.get(&d_q, 3 * n));
    BVH_TRY(signed_distance_device<T>(tree, d_p, n, rule, d_s, d_d, d_q));
    BVH_CUDA_TRY(cudaMemcpyAsync(out_shape, d_s, sizeof(uint32_t) * n, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaMemcpyAsync(out_dist, d_d, sizeof(T) * n, cudaMemcpyDeviceToHost, ctx->stream));
    if (out_closest) BVH_CUDA_TRY(cudaMemcpyAsync(out_closest, d_q, sizeof(T) * 3 * n, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return BVHGPU_OK;
}
template <class T>
static int signed_distance_dev_impl(Tree<T>* tree, const void* d_points, size_t n, int rule, void* d_shape, void* d_dist, void* d_closest) {
    if (!tree || (n && (!d_points || !d_shape || !d_dist))) { set_error("signed_distance_dev: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(tree->ctx->device));
    return signed_distance_device<T>(tree, (const T*)d_points, n, rule, (uint32_t*)d_shape, (T*)d_dist, (T*)d_closest);
}

// Polygons of a 2-D tree (segments.cu), host pointers: 2 T per point, copied back after the device driver, whose checks (n, rule / k,
// status, segments) all run before anything is written.
template <class T>
static int polygon_contains_host_impl(Tree<T>* tree, const T* points, size_t n, int rule, uint8_t* out_class, int32_t* out_winding) {
    if (!tree || (n && (!points || !out_class))) { set_error("contains_points: null argument"); return BVHGPU_ERR_INVALID; }
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    if (n == 0) return polygon_contains_device<T>(tree, nullptr, 0, rule, nullptr, nullptr);
    BVH_TRY(check_n("contains_points", n));
    Scratch scratch(ctx);
    T* d_p = nullptr;
    uint8_t* d_c = nullptr;
    int32_t* d_w = nullptr;
    BVH_TRY(scratch.get(&d_p, 2 * n));
    BVH_TRY(scratch.get(&d_c, n));
    if (out_winding) BVH_TRY(scratch.get(&d_w, n));
    BVH_CUDA_TRY(cudaMemcpyAsync(d_p, points, sizeof(T) * 2 * n, cudaMemcpyHostToDevice, ctx->stream));
    BVH_TRY(polygon_contains_device<T>(tree, d_p, n, rule, d_c, d_w));
    BVH_CUDA_TRY(cudaMemcpyAsync(out_class, d_c, n, cudaMemcpyDeviceToHost, ctx->stream));
    if (out_winding) BVH_CUDA_TRY(cudaMemcpyAsync(out_winding, d_w, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return BVHGPU_OK;
}
template <class T>
static int knn_seg_host_impl(Tree<T>* tree, const T* points, size_t n, uint32_t k, const T* max_dist, uint32_t* out_shape, T* out_dist, T* out_closest) {
    if (!tree || (n && (!points || !out_shape || !out_dist))) { set_error("knn_segments: null argument"); return BVHGPU_ERR_INVALID; }
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    if (n == 0) return knn_seg_device<T>(tree, nullptr, 0, k, nullptr, nullptr, nullptr, nullptr);
    BVH_TRY(check_n("knn_segments", n));
    if (k < 1 || k > BVHGPU_KNN_MAX_K) { set_error("knn_segments: k = %u outside 1 .. %d", k, BVHGPU_KNN_MAX_K); return BVHGPU_ERR_INVALID; }
    Scratch scratch(ctx);
    T *d_p = nullptr, *d_r = nullptr, *d_d = nullptr, *d_q = nullptr;
    uint32_t* d_s = nullptr;
    const size_t nk = n * k;
    BVH_TRY(scratch.get(&d_p, 2 * n));
    if (max_dist) BVH_TRY(scratch.get(&d_r, n));
    BVH_TRY(scratch.get(&d_s, nk));
    BVH_TRY(scratch.get(&d_d, nk));
    if (out_closest) BVH_TRY(scratch.get(&d_q, 2 * nk));
    BVH_CUDA_TRY(cudaMemcpyAsync(d_p, points, sizeof(T) * 2 * n, cudaMemcpyHostToDevice, ctx->stream));
    if (max_dist) BVH_CUDA_TRY(cudaMemcpyAsync(d_r, max_dist, sizeof(T) * n, cudaMemcpyHostToDevice, ctx->stream));
    BVH_TRY(knn_seg_device<T>(tree, d_p, n, k, d_r, d_s, d_d, d_q));
    BVH_CUDA_TRY(cudaMemcpyAsync(out_shape, d_s, sizeof(uint32_t) * nk, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaMemcpyAsync(out_dist, d_d, sizeof(T) * nk, cudaMemcpyDeviceToHost, ctx->stream));
    if (out_closest) BVH_CUDA_TRY(cudaMemcpyAsync(out_closest, d_q, sizeof(T) * 2 * nk, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return BVHGPU_OK;
}
template <class T>
static int polygon_distance_host_impl(Tree<T>* tree, const T* points, size_t n, int rule, uint32_t* out_shape, T* out_dist, T* out_closest) {
    if (!tree || (n && (!points || !out_shape || !out_dist))) { set_error("signed_distance: null argument"); return BVHGPU_ERR_INVALID; }
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    if (n == 0) return polygon_distance_device<T>(tree, nullptr, 0, rule, nullptr, nullptr, nullptr);
    BVH_TRY(check_n("signed_distance", n));
    Scratch scratch(ctx);
    T *d_p = nullptr, *d_d = nullptr, *d_q = nullptr;
    uint32_t* d_s = nullptr;
    BVH_TRY(scratch.get(&d_p, 2 * n));
    BVH_TRY(scratch.get(&d_s, n));
    BVH_TRY(scratch.get(&d_d, n));
    if (out_closest) BVH_TRY(scratch.get(&d_q, 2 * n));
    BVH_CUDA_TRY(cudaMemcpyAsync(d_p, points, sizeof(T) * 2 * n, cudaMemcpyHostToDevice, ctx->stream));
    BVH_TRY(polygon_distance_device<T>(tree, d_p, n, rule, d_s, d_d, d_q));
    BVH_CUDA_TRY(cudaMemcpyAsync(out_shape, d_s, sizeof(uint32_t) * n, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaMemcpyAsync(out_dist, d_d, sizeof(T) * n, cudaMemcpyDeviceToHost, ctx->stream));
    if (out_closest) BVH_CUDA_TRY(cudaMemcpyAsync(out_closest, d_q, sizeof(T) * 2 * n, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return BVHGPU_OK;
}

template <class T> static int fetch_impl(Tree<T>* tree, uint32_t* hits, size_t cap) {
    if (!tree || !hits) { set_error("traverse_fetch: null argument"); return BVHGPU_ERR_INVALID; }
    if (cap < tree->last_total) { set_error("traverse_fetch: capacity %zu < %zu hits", cap, tree->last_total); return BVHGPU_ERR_CAPACITY; }
    if (tree->last_total == 0) return BVHGPU_OK;
    if (!tree->d_hits || tree->hits_cap < tree->last_total) { set_error("traverse_fetch: no retained result"); return BVHGPU_ERR_INVALID; }
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_CUDA_TRY(cudaMemcpyAsync(hits, tree->d_hits, sizeof(uint32_t) * tree->last_total, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return BVHGPU_OK;
}

// New shape AABBs for refit / optimize: converted into a TEMPORARY device array and checked for NaN before the tree is touched,
// so a rejected update (BVHGPU_ERR_NAN) leaves the tree exactly as it was.  dev_input: `aabbs` is a device pointer.
template <class T>
static int stage_new_aabbs(Tree<T>* tree, const typename Traits<T>::Aabb* aabbs, size_t n, bool dev_input, const char* who) {
    bvhgpu_ctx* ctx = tree->ctx;
    Scratch scratch(ctx);
    typename Traits<T>::Aabb* staged = nullptr;
    const typename Traits<T>::Aabb* d_in = aabbs;
    if (!dev_input) {
        BVH_TRY(scratch.get(&staged, n));
        BVH_CUDA_TRY(cudaMemcpyAsync(staged, aabbs, n * sizeof(*aabbs), cudaMemcpyHostToDevice, ctx->stream));
        d_in = staged;
    }
    typename Traits<T>::DAabb* fresh = nullptr;
    uint32_t* flag = nullptr;
    BVH_TRY(dalloc_t(ctx, &fresh, n));
    int rc = scratch.get(&flag, 1);
    if (rc == BVHGPU_OK && cudaMemsetAsync(flag, 0, sizeof(uint32_t), ctx->stream) != cudaSuccess) rc = BVHGPU_ERR_CUDA;
    if (rc == BVHGPU_OK) rc = convert_aabbs<T>(ctx, d_in, (uint32_t)n, fresh, flag);
    uint32_t* h = ctx->h_pinned + 200;
    if (rc == BVHGPU_OK && (cudaMemcpyAsync(h, flag, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
                            cudaStreamSynchronize(ctx->stream) != cudaSuccess)) { set_error("%s: CUDA error while staging the AABBs", who); rc = BVHGPU_ERR_CUDA; }
    if (rc == BVHGPU_OK && *h) { set_error("%s: NaN coordinate in an input AABB; the tree was left unchanged", who); rc = BVHGPU_ERR_NAN; }
    if (rc != BVHGPU_OK) { dfree(ctx, fresh); return rc; }
    dfree(ctx, tree->d_aabb);
    tree->d_aabb = fresh;
    return BVHGPU_OK;
}

// 4-D: the boxes are checked (the tree is left untouched if that fails), then copied into the tree: the ABI box is the device layout.
template <class T>
static int stage_new_aabbs(Tree4<T>* tree, const typename D4<T>::Aabb* d_in, size_t n, bool, const char* who) {
    Scratch scratch(tree->ctx);
    BVH_TRY(check_boxes(tree, nullptr, d_in, (uint32_t)n, scratch, who));
    if (cudaMemcpyAsync(tree->d_aabb, d_in, sizeof(*d_in) * n, cudaMemcpyDeviceToDevice, tree->ctx->stream) != cudaSuccess)
        return mark_failed(tree, BVHGPU_ERR_CUDA, who);
    return BVHGPU_OK;
}

// A 3-D tree's deferred build status is cleared before a call enqueues builder work; a 4-D tree reports its errors synchronously.
template <class T> static int reset_status(Tree<T>* tree) {
    BVH_CUDA_TRY(cudaMemsetAsync(tree->d_status, 0, sizeof(BuildStatus), tree->ctx->stream));
    return BVHGPU_OK;
}
template <class T> static int reset_status(Tree4<T>*) { return BVHGPU_OK; }

// The end of a call that changed the tree.  Tree<T>: the status stays pending for device pointers unless the caller asked for the
// rebuilt count, and is resolved otherwise; the status counts the rebuilt shapes.  Tree4<T>: host pointers synchronise, and the
// count is the driver's `shapes`.
template <class T> static int complete(Tree<T>* tree, bool dev_input, size_t* rebuilt, size_t, const char*) {
    tree->status_pending = true;
    if (!rebuilt) return dev_input ? (int)BVHGPU_OK : resolve_status(tree);
    BuildStatus hs;
    BVH_CUDA_TRY(cudaMemcpyAsync(&hs, tree->d_status, sizeof(hs), cudaMemcpyDeviceToHost, tree->ctx->stream));
    BVH_TRY(resolve_status(tree));                                      // synchronises
    *rebuilt = hs.rebuilt;
    return BVHGPU_OK;
}
template <class T> static int complete(Tree4<T>* tree, bool dev_input, size_t* rebuilt, size_t shapes, const char* who) {
    if (!dev_input && cudaStreamSynchronize(tree->ctx->stream) != cudaSuccess) { set_error("%s: CUDA error", who); return mark_failed(tree, BVHGPU_ERR_CUDA, who); }
    if (rebuilt) *rebuilt = shapes;
    return BVHGPU_OK;
}

// Refit from n new shape boxes (ABI layout of D).  D = 2 (host pointers): the 2-D boxes are lifted to z = [0, 0] on the device.
// Surface areas with z = [0, 0] are exact and largest_axis never picks z (dim2.cu), so the 3-D refit, growth test and rebuild are the
// 2-D ones.  The boxes are checked before the tree is touched; a refit that fails after that leaves the tree failed.
template <int D, class T>
static int refit_impl(TreeOf<D, T>* tree, const void* aabbs, size_t n, bool dev_input) {
    if (!tree || (n && !aabbs)) { set_error("refit: null argument"); return BVHGPU_ERR_INVALID; }
    if (D == 4) BVH_TRY(resolve_status(tree));                     // a 4-D tree reports a sticky failure before the size
    if (n != tree->n) { set_error("refit: %zu AABBs for a tree over %u shapes", n, tree->n); return BVHGPU_ERR_INVALID; }
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    if (D != 4) BVH_TRY(resolve_status(tree));
    if (n == 0) return BVHGPU_OK;
    Scratch scratch(ctx);
    if (D != 3 && !dev_input) {
        T* staged = nullptr;
        BVH_TRY(upload_records<D>(ctx, scratch, aabbs, n, AABB_RECORD, 0, &staged));
        aabbs = staged;
    }
    BVH_TRY(stage_new_aabbs<T>(tree, static_cast<const typename TreeOf<D, T>::Aabb*>(aabbs), n, dev_input || D != 3, "refit"));
    int rc = reset_status(tree);
    if (rc == BVHGPU_OK) rc = refit(tree);
    if (rc != BVHGPU_OK) return mark_failed(tree, rc, "refit");
    return complete(tree, dev_input, nullptr, 0, "refit");
}

template <class T>
static int optimize_impl(Tree<T>* tree, const typename Traits<T>::Aabb* aabbs, size_t n, double max_growth, size_t* rebuilt, bool dev_input) {
    if (!tree || (n && !aabbs)) { set_error("optimize: null argument"); return BVHGPU_ERR_INVALID; }
    if (n != tree->n) { set_error("optimize: %zu AABBs for a tree over %u shapes", n, tree->n); return BVHGPU_ERR_INVALID; }
    if (!(max_growth >= 1.0)) { set_error("optimize: max_growth = %g, must be >= 1", max_growth); return BVHGPU_ERR_INVALID; }
    if (rebuilt) *rebuilt = 0;
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(resolve_status(tree));
    if (n == 0) return BVHGPU_OK;
    BVH_TRY(stage_new_aabbs<T>(tree, aabbs, n, dev_input, "optimize"));
    BVH_CUDA_TRY(cudaMemsetAsync(tree->d_status, 0, sizeof(BuildStatus), ctx->stream));
    BVH_TRY(optimize(tree, max_growth));
    tree->status_pending = true;
    if (dev_input && !rebuilt) return BVHGPU_OK;                        // asynchronous: errors surface at the next call on the tree
    BuildStatus h;
    BVH_CUDA_TRY(cudaMemcpyAsync(&h, tree->d_status, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
    BVH_TRY(resolve_status(tree));                                      // synchronises
    if (rebuilt) *rebuilt = h.rebuilt;
    return BVHGPU_OK;
}

// ---- D = 2 (dim2.cu): host PODs in, converted on the device, run through the 3-D path --------------------------------------
template <class T, class TREE2, class AABB2>
static int build2_impl(bvhgpu_ctx* ctx, const AABB2* aabbs, size_t n, int mode, TREE2** out) {
    if (!ctx || !out || (n && !aabbs)) { set_error("build: null argument"); return BVHGPU_ERR_INVALID; }
    *out = nullptr;
    if (n > (1ull << 30)) { set_error("build: n = %zu exceeds 2^30 shapes", n); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    Scratch scratch(ctx);
    T* in6 = nullptr;
    if (n) BVH_TRY(upload_records<2>(ctx, scratch, aabbs, n, AABB_RECORD, 0, &in6));
    TREE2* tree = nullptr;
    BVH_TRY((build_impl<T, TREE2>(ctx, reinterpret_cast<const typename Traits<T>::Aabb*>(in6), n, mode, false, &tree)));
    int rc = dim2_finish_build<T>(tree);
    if (rc == BVHGPU_OK) rc = resolve_status(tree);
    if (rc != BVHGPU_OK) { tree_release<T>(tree); delete tree; return rc; }
    *out = tree;
    return BVHGPU_OK;
}
template <class T, class N2>
static int tree_nodes2_impl(Tree<T>* tree, N2* out_nodes, uint32_t* out_node_index) {
    if (!tree) { set_error("tree_nodes: null tree"); return BVHGPU_ERR_INVALID; }
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(resolve_status(tree));
    if (tree->n == 0) return BVHGPU_OK;
    Scratch scratch(ctx);
    if (out_nodes) {
        N2* d = nullptr;
        BVH_TRY(scratch.get(&d, tree->n_nodes));
        BVH_TRY((dim2_nodes_out<T, N2>(tree, d)));
        BVH_CUDA_TRY(cudaMemcpyAsync(out_nodes, d, sizeof(N2) * tree->n_nodes, cudaMemcpyDeviceToHost, ctx->stream));
    }
    if (out_node_index) BVH_CUDA_TRY(cudaMemcpyAsync(out_node_index, tree->d_node_index, sizeof(uint32_t) * tree->n, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return BVHGPU_OK;
}
template <class T, class F2>
static int flatten2_impl(Tree<T>* tree, F2* out, size_t cap, size_t* len) {
    if (!tree) { set_error("flatten: null tree"); return BVHGPU_ERR_INVALID; }
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(resolve_status(tree));
    BVH_TRY(build_flat(tree));
    if (len) *len = tree->n_flat;
    if (out) {
        if (cap < tree->n_flat) { set_error("flatten: capacity %zu < %zu flat nodes", cap, tree->n_flat); return BVHGPU_ERR_CAPACITY; }
        if (tree->n_flat) {
            Scratch scratch(ctx);
            F2* d = nullptr;
            BVH_TRY(scratch.get(&d, tree->n_flat));
            BVH_TRY((dim2_flat_out<T, F2>(tree, d)));
            BVH_CUDA_TRY(cudaMemcpyAsync(out, d, sizeof(F2) * tree->n_flat, cudaMemcpyDeviceToHost, ctx->stream));
            BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
        }
    }
    return BVHGPU_OK;
}
// Bvh::update_shapes(changed_shape_indices, shapes): only the m changed shapes cross the boundary.  The tree is touched only after
// the new AABBs passed the NaN / index check.  max_growth <= 0: refit only (topology kept).
template <int D, class T>
static int update_impl(TreeOf<D, T>* tree, const uint32_t* changed, const void* fresh, size_t m, double max_growth, size_t* rebuilt, bool dev_input) {
    if (!tree || (m && (!changed || !fresh))) { set_error("update: null argument"); return BVHGPU_ERR_INVALID; }
    if (max_growth > 0.0 && !(max_growth >= 1.0)) { set_error("update: max_growth = %g, must be >= 1 (or <= 0 for a pure refit)", max_growth); return BVHGPU_ERR_INVALID; }
    if (m > 0xFFFFFFFFull) { set_error("update: too many changed shapes"); return BVHGPU_ERR_INVALID; }
    if (rebuilt) *rebuilt = 0;
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(resolve_status(tree));
    if (m == 0 || tree->n == 0) return BVHGPU_OK;
    Scratch scratch(ctx);
    const uint32_t* d_changed = changed;
    if (!dev_input) {
        uint32_t* c = nullptr;
        T* f = nullptr;
        BVH_TRY(scratch.get(&c, m));
        BVH_CUDA_TRY(cudaMemcpyAsync(c, changed, sizeof(uint32_t) * m, cudaMemcpyHostToDevice, ctx->stream));
        BVH_TRY(upload_records<D>(ctx, scratch, fresh, m, AABB_RECORD, 0, &f));
        d_changed = c; fresh = f;
    }
    const auto* d_fresh = static_cast<const typename TreeOf<D, T>::Aabb*>(fresh);
    BVH_TRY(check_boxes(tree, d_changed, d_fresh, (uint32_t)m, scratch, "update"));
    BVH_TRY(reset_status(tree));
    size_t shapes = 0;
    int rc = scatter_boxes(tree, d_changed, d_fresh, (uint32_t)m);
    if (rc == BVHGPU_OK) rc = update_incremental(tree, d_changed, (uint32_t)m, max_growth, &shapes);   // touches the root paths of the changed leaves only
    if (rc != BVHGPU_OK) return mark_failed(tree, rc, "update");
    return complete(tree, dev_input, rebuilt, shapes, "update");
}

// Adding to an empty tree is exactly bvhgpu_build_* over the k boxes (device pointers), which replaces the tree's arrays.
template <class T> static int build_into_empty(Tree<T>* tree, const typename Traits<T>::Aabb* d_in, uint32_t k, bool dev_input) {
    bvhgpu_ctx* ctx = tree->ctx;
    Tree<T> fresh;
    int rc = build_exact_sah<T>(ctx, d_in, k, &fresh);
    if (rc == BVHGPU_OK) rc = resolve_status(&fresh);
    if (rc != BVHGPU_OK) { tree_release(&fresh); return rc; }
    dfree(ctx, tree->d_status); dfree(ctx, tree->d_sa_base); dfree(ctx, tree->d_tris); dfree(ctx, tree->d_segs);
    tree->d_sa_base = nullptr; tree->d_tris = nullptr; tree->d_segs = nullptr;
    tree->n = fresh.n; tree->n_nodes = fresh.n_nodes; tree->d_status = fresh.d_status;
    tree->d_aabb = fresh.d_aabb; tree->d_nodes = fresh.d_nodes; tree->d_node_index = fresh.d_node_index; tree->d_node_start = fresh.d_node_start;
    if (tree->dims == 2) {                                              // the FLAT leaf boxes, read by the records, at the new n
        dfree(ctx, tree->d_aabb_trav); tree->d_aabb_trav = nullptr;
        BVH_TRY(dim2_finish_build<T>(tree));
    }
    BVH_TRY(build_traversal_records(tree));
    if (tree->have_flat) BVH_TRY(build_flat(tree));
    tree->status_pending = true;
    return dev_input ? (int)BVHGPU_OK : resolve_status(tree);
}
template <class T> static int build_into_empty(Tree4<T>* tree, const typename D4<T>::Aabb* d_in, uint32_t k, bool) {
    bvhgpu_ctx* ctx = tree->ctx;
    {
        Scratch scratch(ctx);
        BVH_TRY(check_boxes(tree, nullptr, d_in, k, scratch, "add_shapes"));
    }
    Tree4<T> fresh;
    fresh.ctx = ctx; fresh.n = k; fresh.n_nodes = 2 * k - 1;
    const int rc = build4<T>(&fresh, d_in, cudaMemcpyDeviceToDevice);  // synchronous
    if (rc != BVHGPU_OK) { tree_release(&fresh); return rc; }
    dfree(ctx, tree->d_sa_base); tree->d_sa_base = nullptr;
    tree->d_aabb = fresh.d_aabb; tree->d_nodes = fresh.d_nodes; tree->d_node_index = fresh.d_node_index; tree->d_node_start = fresh.d_node_start;
    tree->n = fresh.n; tree->n_nodes = fresh.n_nodes;
    return finish_relayout(tree);
}

// The tree's n boxes followed by the k new ones, in a new device array, checked for NaN before the tree is touched.  3-D: the new
// boxes are converted to the padded device layout; 4-D: checked, then copied as they are.
template <class T> static int stage_added(Tree<T>* tree, const typename Traits<T>::Aabb* d_in, uint32_t k, typename Traits<T>::DAabb** out) {
    bvhgpu_ctx* ctx = tree->ctx;
    const uint32_t n = tree->n;
    Scratch scratch(ctx);
    typename Traits<T>::DAabb* all = nullptr;
    uint32_t* flag = nullptr;
    BVH_TRY(scratch.get(&flag, 1));
    BVH_TRY(dalloc_t(ctx, &all, (size_t)n + k));
    int rc = cudaMemsetAsync(flag, 0, sizeof(uint32_t), ctx->stream) == cudaSuccess ? BVHGPU_OK : BVHGPU_ERR_CUDA;
    if (rc == BVHGPU_OK && cudaMemcpyAsync(all, tree->d_aabb, sizeof(*all) * n, cudaMemcpyDeviceToDevice, ctx->stream) != cudaSuccess) rc = BVHGPU_ERR_CUDA;
    if (rc == BVHGPU_OK) rc = convert_aabbs<T>(ctx, d_in, k, all + n, flag);
    uint32_t* h = ctx->h_pinned + 212;
    if (rc == BVHGPU_OK && (cudaMemcpyAsync(h, flag, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
                            cudaStreamSynchronize(ctx->stream) != cudaSuccess)) { set_error("add_shapes: CUDA error while staging the AABBs"); rc = BVHGPU_ERR_CUDA; }
    if (rc == BVHGPU_OK && *h) { set_error("add_shapes: NaN coordinate in a new AABB; the tree was left unchanged"); rc = BVHGPU_ERR_NAN; }
    if (rc != BVHGPU_OK) { dfree(ctx, all); return rc; }
    *out = all;
    return BVHGPU_OK;
}
template <class T> static int stage_added(Tree4<T>* tree, const typename D4<T>::Aabb* d_in, uint32_t k, typename D4<T>::Aabb** out) {
    using Aabb = typename D4<T>::Aabb;
    bvhgpu_ctx* ctx = tree->ctx;
    const uint32_t n = tree->n;
    {
        Scratch scratch(ctx);
        BVH_TRY(check_boxes(tree, nullptr, d_in, k, scratch, "add_shapes"));
    }
    Aabb* all = nullptr;
    BVH_TRY(dalloc_t(ctx, &all, (size_t)n + k));
    if (cudaMemcpyAsync(all, tree->d_aabb, sizeof(Aabb) * n, cudaMemcpyDeviceToDevice, ctx->stream) != cudaSuccess ||
        cudaMemcpyAsync(all + n, d_in, sizeof(Aabb) * k, cudaMemcpyDeviceToDevice, ctx->stream) != cudaSuccess) {
        dfree(ctx, all);
        set_error("add_shapes: CUDA error while staging the AABBs");
        return BVHGPU_ERR_CUDA;
    }
    *out = all;
    return BVHGPU_OK;
}

// Bvh::add_shape, batched: the k new shapes get indices n .. n+k-1.  The AABBs are staged next to the tree's own and checked for NaN
// before the tree is touched.  n == 0: the call is bvhgpu_build_* over the k AABBs.
template <int D, class T>
static int add_impl(TreeOf<D, T>* tree, const void* aabbs, size_t k, double max_growth, size_t* rebuilt, bool dev_input) {
    if (!tree || (k && !aabbs)) { set_error("add_shapes: null argument"); return BVHGPU_ERR_INVALID; }
    if (max_growth > 0.0 && !(max_growth >= 1.0)) { set_error("add_shapes: max_growth = %g, must be >= 1 (or <= 0 for no rebuild)", max_growth); return BVHGPU_ERR_INVALID; }
    if (rebuilt) *rebuilt = 0;
    if ((uint64_t)tree->n + k > (1ull << 30)) { set_error("add_shapes: %u + %zu shapes exceed 2^30 (u32 node indices); the tree was left unchanged", tree->n, k); return BVHGPU_ERR_INVALID; }
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(resolve_status(tree));
    if (k == 0) return BVHGPU_OK;
    Scratch scratch(ctx);
    if (!dev_input) {
        T* staged = nullptr;
        BVH_TRY(upload_records<D>(ctx, scratch, aabbs, k, AABB_RECORD, 0, &staged));
        aabbs = staged;
    }
    const auto* d_in = static_cast<const typename TreeOf<D, T>::Aabb*>(aabbs);
    if (tree->n == 0) return build_into_empty(tree, d_in, (uint32_t)k, dev_input);
    typename TreeOf<D, T>::Box* all = nullptr;
    BVH_TRY(stage_added(tree, d_in, (uint32_t)k, &all));
    size_t shapes = 0;
    int rc = reset_status(tree);
    if (rc == BVHGPU_OK) rc = add_shapes(tree, all, (uint32_t)k, max_growth, &shapes);
    if (rc != BVHGPU_OK) {
        if (tree->d_aabb != all) { dfree(ctx, all); return rc; }            // failed before the tree was touched
        return mark_failed(tree, rc, "add_shapes");
    }
    return complete(tree, dev_input, rebuilt, shapes, "add_shapes");
}

// Bvh::remove_shape(i, swap_shape = true), batched: `indices` are distinct shape indices before the call; survivors >= n-k take the
// vacated indices < n-k, smallest hole first.  Checked (range, duplicates) before the tree is touched.
template <int D, class T>
static int remove_impl(TreeOf<D, T>* tree, const uint32_t* indices, size_t k, bool dev_input) {
    if (!tree || (k && !indices)) { set_error("remove_shapes: null argument"); return BVHGPU_ERR_INVALID; }
    if (k > tree->n) { set_error("remove_shapes: %zu indices for a tree over %u shapes; the tree was left unchanged", k, tree->n); return BVHGPU_ERR_INVALID; }
    bvhgpu_ctx* ctx = tree->ctx;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(resolve_status(tree));
    if (k == 0) return BVHGPU_OK;
    const uint32_t n = tree->n;
    Scratch scratch(ctx);
    const uint32_t* d_idx = indices;
    if (!dev_input) {
        uint32_t* c = nullptr;
        BVH_TRY(scratch.get(&c, k));
        BVH_CUDA_TRY(cudaMemcpyAsync(c, indices, sizeof(uint32_t) * k, cudaMemcpyHostToDevice, ctx->stream));
        d_idx = c;
    }
    uint32_t *rm = nullptr, *flags = nullptr;
    BVH_TRY(scratch.get(&rm, (size_t)n + 1));
    BVH_TRY(scratch.get(&flags, 2));
    BVH_CUDA_TRY(cudaMemsetAsync(rm, 0, sizeof(uint32_t) * ((size_t)n + 1), ctx->stream));
    BVH_CUDA_TRY(cudaMemsetAsync(flags, 0, 2 * sizeof(uint32_t), ctx->stream));
    BVH_TRY(remove_check(ctx, d_idx, (uint32_t)k, n, rm, flags));
    uint32_t* h = ctx->h_pinned + 216;
    BVH_CUDA_TRY(cudaMemcpyAsync(h, flags, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (h[0]) { set_error("remove_shapes: a shape index is >= %u; the tree was left unchanged", n); return BVHGPU_ERR_INVALID; }
    if (h[1]) { set_error("remove_shapes: a shape index is listed twice; the tree was left unchanged"); return BVHGPU_ERR_INVALID; }
    const void* nodes_before = tree->d_nodes;
    BVH_TRY(reset_status(tree));
    const int rc = remove_shapes(tree, rm, (uint32_t)k);
    if (rc != BVHGPU_OK) return tree->d_nodes == nodes_before ? rc : mark_failed(tree, rc, "remove_shapes");
    return complete(tree, dev_input, nullptr, 0, "remove_shapes");
}

}  // namespace bvhb200

using namespace bvhb200;

#define BVH_EXPORT extern "C" __attribute__((visibility("default")))

BVH_EXPORT const char* bvhgpu_last_error(void) { return g_last_error.c_str(); }
BVH_EXPORT const char* bvhgpu_version(void) { return "bvh_b200 0.1.0 (sm_90a)"; }

BVH_EXPORT int bvhgpu_create(int device, bvhgpu_ctx** out) {
    if (!out) { set_error("create: null out"); return BVHGPU_ERR_INVALID; }
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        set_error("create: no CUDA device (%s); libbvh_b200 has no CPU fallback", e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
        return BVHGPU_ERR_CUDA;
    }
    if (device < 0 || device >= count) { set_error("create: device %d out of range (0..%d)", device, count - 1); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(device));
    cudaDeviceProp prop;
    BVH_CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) { set_error("create: device %d is sm_%d%d; this library contains sm_90a code only", device, prop.major, prop.minor); return BVHGPU_ERR_UNSUPPORTED; }
    bvhgpu_ctx* ctx = new (std::nothrow) bvhgpu_ctx();
    if (!ctx) { set_error("create: out of host memory"); return BVHGPU_ERR_INTERNAL; }
    ctx->device = device;
    ctx->sm_count = prop.multiProcessorCount;
    BVH_CUDA_TRY(cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking));
    ctx->stream = ctx->own_stream;
    BVH_CUDA_TRY(cudaMallocHost((void**)&ctx->h_pinned, 256 * sizeof(uint32_t)));
    for (int i = 0; i < 2; ++i) { BVH_CUDA_TRY(cudaEventCreate(&ctx->ev_walk[i])); BVH_CUDA_TRY(cudaEventCreate(&ctx->ev_build[i])); }
    BVH_CUDA_TRY(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
    BVH_CUDA_TRY(cudaStreamCreateWithFlags(&ctx->d2h_stream, cudaStreamNonBlocking));
    for (unsigned i = 0; i < BVH_MAX_CHUNKS; ++i) BVH_CUDA_TRY(cudaEventCreateWithFlags(&ctx->ev_emit[i], cudaEventDisableTiming));
    for (int i = 0; i < 5; ++i) BVH_CUDA_TRY(cudaEventCreate(&ctx->ev_e2e[i]));
    BVH_CUDA_TRY(cudaEventCreateWithFlags(&ctx->ev_order, cudaEventDisableTiming));
    BVH_CUDA_TRY(cudaEventCreateWithFlags(&ctx->ev_total, cudaEventDisableTiming));
    BVH_CUDA_TRY(cudaEventCreateWithFlags(&ctx->ev_switch, cudaEventDisableTiming));
    for (unsigned i = 0; i < BVH_MAX_CHUNKS; ++i) BVH_CUDA_TRY(cudaEventCreateWithFlags(&ctx->ev_chunk[i], cudaEventDisableTiming));
    BVH_CUDA_TRY(cudaMalloc((void**)&ctx->d_async_err, 256));
    BVH_CUDA_TRY(cudaMemset(ctx->d_async_err, 0, 256));
    ctx->d_ready = ctx->d_async_err + 32;                         // its own 128-byte line of the same small allocation
    {   // NUMA node of the device (bvhgpu_host_alloc): /sys/bus/pci/devices/<domain:bus:dev.fn>/numa_node
        char bus[32] = {0}, path[128];
        if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) == cudaSuccess) {
            for (char* c = bus; *c; ++c) *c = (char)tolower(*c);
            snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
            if (FILE* f = fopen(path, "r")) { int nn = -1; if (fscanf(f, "%d", &nn) == 1) ctx->numa_node = nn; fclose(f); }
        }
    }
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
        unsigned long long thr = ~0ull;                       // keep freed blocks cached: alloc/free pairs stay cheap
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
    *out = ctx;
    return BVHGPU_OK;
}
BVH_EXPORT void bvhgpu_destroy(bvhgpu_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    if (ctx->d2h_stream) cudaStreamDestroy(ctx->d2h_stream);
    for (unsigned i = 0; i < BVH_MAX_CHUNKS; ++i) if (ctx->ev_emit[i]) cudaEventDestroy(ctx->ev_emit[i]);
    if (ctx->ev_order) cudaEventDestroy(ctx->ev_order);
    if (ctx->ev_total) cudaEventDestroy(ctx->ev_total);
    if (ctx->ev_switch) cudaEventDestroy(ctx->ev_switch);
    for (unsigned i = 0; i < BVH_MAX_CHUNKS; ++i) if (ctx->ev_chunk[i]) cudaEventDestroy(ctx->ev_chunk[i]);
    if (ctx->h_pinned) cudaFreeHost(ctx->h_pinned);
    if (ctx->d_async_err) cudaFree(ctx->d_async_err);
    for (int i = 0; i < 5; ++i) if (ctx->ev_e2e[i]) cudaEventDestroy(ctx->ev_e2e[i]);
    for (int i = 0; i < 2; ++i) { if (ctx->ev_walk[i]) cudaEventDestroy(ctx->ev_walk[i]); if (ctx->ev_build[i]) cudaEventDestroy(ctx->ev_build[i]); }
    delete ctx;
}
// Move the context to another stream without breaking the order of its calls: the incoming stream waits for everything
// enqueued on the outgoing one (kernels, copies and the pool frees / allocations inside them). No host synchronisation.
static int switch_stream(bvhgpu_ctx* ctx, cudaStream_t incoming) {
    if (incoming == ctx->stream) return BVHGPU_OK;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_CUDA_TRY(cudaEventRecord(ctx->ev_switch, ctx->stream));
    BVH_CUDA_TRY(cudaStreamWaitEvent(incoming, ctx->ev_switch, 0));
    ctx->stream = incoming;
    return BVHGPU_OK;
}
BVH_EXPORT int bvhgpu_set_stream(bvhgpu_ctx* ctx, void* cuda_stream) {
    if (!ctx) { set_error("set_stream: null ctx"); return BVHGPU_ERR_INVALID; }
    return switch_stream(ctx, (cudaStream_t)cuda_stream);
}
BVH_EXPORT int bvhgpu_reset_stream(bvhgpu_ctx* ctx) {
    if (!ctx) { set_error("reset_stream: null ctx"); return BVHGPU_ERR_INVALID; }
    return switch_stream(ctx, ctx->own_stream);
}
BVH_EXPORT int bvhgpu_synchronize(bvhgpu_ctx* ctx) {
    if (!ctx) { set_error("synchronize: null ctx"); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    uint32_t* h = ctx->h_pinned + 204;
    BVH_CUDA_TRY(cudaMemcpyAsync(h, ctx->d_async_err, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (*h) {                                                     // raised by an asynchronous multi-GPU step; reported once
        const int rc = (int)*h;
        cudaMemsetAsync(ctx->d_async_err, 0, sizeof(uint32_t), ctx->stream);
        set_error("sharded traversal: a peer did not answer within the exchange time-out (status %d); the step's result is invalid", rc);
        return rc;
    }
    return BVHGPU_OK;
}
BVH_EXPORT uint64_t bvhgpu_launch_count(const bvhgpu_ctx* ctx) { return ctx ? ctx->launches : 0; }
BVH_EXPORT int bvhgpu_set_option(bvhgpu_ctx* ctx, const char* name, int64_t value) {
    if (!ctx || !name) { set_error("set_option: null argument"); return BVHGPU_ERR_INVALID; }
    if (!strcmp(name, "traverse_slots")) { ctx->traverse_slots = value; return BVHGPU_OK; }
    if (!strcmp(name, "profile")) { ctx->profile = value; return BVHGPU_OK; }
    if (!strcmp(name, "build_small")) { ctx->build_small = value; return BVHGPU_OK; }
    if (!strcmp(name, "build_gang")) { ctx->build_gang = value; return BVHGPU_OK; }
    if (!strcmp(name, "build_subtree")) { ctx->build_subtree = value; return BVHGPU_OK; }
    if (!strcmp(name, "traverse_persistent")) { ctx->traverse_persistent = value; return BVHGPU_OK; }
    if (!strcmp(name, "traverse_stream")) { ctx->traverse_stream = value; return BVHGPU_OK; }
    if (!strcmp(name, "traverse_top")) { ctx->traverse_top = value; return BVHGPU_OK; }
    if (!strcmp(name, "walk_grid")) { ctx->walk_grid = value <= 0 ? 0 : (int)value; ctx->walk_grid_forced = value > 0; return BVHGPU_OK; }   // CTAs of the persistent walk (0 = one full wave)
    set_error("set_option: unknown option '%s'", name);
    return BVHGPU_ERR_INVALID;
}

BVH_EXPORT int bvhgpu_get_metric(bvhgpu_ctx* ctx, const char* name, double* out) {
    if (!ctx || !name || !out) { set_error("get_metric: null argument"); return BVHGPU_ERR_INVALID; }
    cudaEvent_t* ev = nullptr;
    if (!strncmp(name, "e2e_host_us_", 12) && name[12] >= '0' && name[12] <= '7' && !name[13]) { *out = ctx->host_us[name[12] - '0']; return BVHGPU_OK; }
    if (!strcmp(name, "stream_write_value")) { *out = (double)ctx->wv_ok; return BVHGPU_OK; }
    if (!strcmp(name, "host_streamed")) { *out = (double)ctx->last_streamed; return BVHGPU_OK; }
    if (!strcmp(name, "numa_node")) { *out = (double)ctx->numa_node; return BVHGPU_OK; }
    if (!strcmp(name, "walk_ms") && ctx->have_walk) ev = ctx->ev_walk;
    else if (!strcmp(name, "build_ms") && ctx->have_build) ev = ctx->ev_build;
    if (!ev && ctx->have_e2e && !strncmp(name, "e2e_", 4)) {      // e2e_walk_ms / e2e_h2d_ms / e2e_emit_ms / e2e_d2h_ms: since call start
        int k = !strcmp(name, "e2e_walk_ms") ? 1 : !strcmp(name, "e2e_h2d_ms") ? 2 : !strcmp(name, "e2e_emit_ms") ? 3 : !strcmp(name, "e2e_d2h_ms") ? 4 : 0;
        if (k) {
            BVH_CUDA_TRY(cudaEventSynchronize(ctx->ev_e2e[k]));
            float ms = 0.f;
            BVH_CUDA_TRY(cudaEventElapsedTime(&ms, ctx->ev_e2e[0], ctx->ev_e2e[k]));
            *out = (double)ms;
            return BVHGPU_OK;
        }
    }
    if (!ev) { set_error("get_metric: '%s' not recorded (set option profile=1 and run the call first)", name); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_CUDA_TRY(cudaEventSynchronize(ev[1]));
    float ms = 0.f;
    BVH_CUDA_TRY(cudaEventElapsedTime(&ms, ev[0], ev[1]));
    *out = (double)ms;
    return BVHGPU_OK;
}

BVH_EXPORT int bvhgpu_peer_alloc(bvhgpu_ctx* ctx, size_t bytes, void** dev_ptr, void* handle64) {
    if (!ctx || !dev_ptr || !handle64) { set_error("peer_alloc: null argument"); return BVHGPU_ERR_INVALID; }
    static_assert(sizeof(cudaIpcMemHandle_t) == BVHGPU_IPC_HANDLE_BYTES, "ipc handle size");
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    BVH_TRY(preload_shard_kernels());                            // every rank allocates before its first step
    BVH_CUDA_TRY(cudaMalloc(dev_ptr, bytes ? bytes : 16));
    BVH_CUDA_TRY(cudaMemset(*dev_ptr, 0, bytes ? bytes : 16));
    BVH_CUDA_TRY(cudaIpcGetMemHandle((cudaIpcMemHandle_t*)handle64, *dev_ptr));
    return BVHGPU_OK;
}
BVH_EXPORT int bvhgpu_peer_open(bvhgpu_ctx* ctx, const void* handle64, void** dev_ptr) {
    if (!ctx || !dev_ptr || !handle64) { set_error("peer_open: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, sizeof(h));
    BVH_CUDA_TRY(cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return BVHGPU_OK;
}
BVH_EXPORT int bvhgpu_peer_close(bvhgpu_ctx* ctx, void* dev_ptr) {
    if (!ctx) { set_error("peer_close: null ctx"); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    if (dev_ptr) BVH_CUDA_TRY(cudaIpcCloseMemHandle(dev_ptr));
    return BVHGPU_OK;
}
BVH_EXPORT int bvhgpu_peer_free(bvhgpu_ctx* ctx, void* dev_ptr) {
    if (!ctx) { set_error("peer_free: null ctx"); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    if (dev_ptr) BVH_CUDA_TRY(cudaFree(dev_ptr));
    return BVHGPU_OK;
}

BVH_EXPORT int bvhgpu_memcpy_d2h(bvhgpu_ctx* ctx, void* host_dst, const void* dev_src, size_t bytes) {
    if (!ctx || (bytes && (!host_dst || !dev_src))) { set_error("memcpy_d2h: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    if (bytes) BVH_CUDA_TRY(cudaMemcpyAsync(host_dst, dev_src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    BVH_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return BVHGPU_OK;
}

BVH_EXPORT int bvhgpu_memcpy_h2d_async(bvhgpu_ctx* ctx, void* dev_dst, const void* host_src, size_t bytes) {
    if (!ctx || (bytes && (!host_src || !dev_dst))) { set_error("memcpy_h2d_async: null argument"); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    if (bytes) BVH_CUDA_TRY(cudaMemcpyAsync(dev_dst, host_src, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return BVHGPU_OK;
}

// Pinned host memory on the device's NUMA node: the calling thread is moved onto that node's CPUs while the pages are
// allocated and first touched (first-touch placement; needs no privilege, unlike mbind), then moved back.
BVH_EXPORT int bvhgpu_host_alloc(bvhgpu_ctx* ctx, size_t bytes, void** out) {
    if (!ctx || !out) { set_error("host_alloc: null argument"); return BVHGPU_ERR_INVALID; }
    *out = nullptr;
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    cpu_set_t old_set, node_set;
    bool moved = false;
    if (ctx->numa_node >= 0 && sched_getaffinity(0, sizeof old_set, &old_set) == 0) {
        char path[128];
        snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", ctx->numa_node);
        CPU_ZERO(&node_set);
        int ncpu = 0;
        if (FILE* f = fopen(path, "r")) {                         // "0-31,64-95"
            int a, b;
            char sep;
            while (fscanf(f, "%d", &a) == 1) {
                b = a;
                int c = fgetc(f);
                if (c == '-') { if (fscanf(f, "%d", &b) != 1) break; c = fgetc(f); }
                for (int k = a; k <= b && k < CPU_SETSIZE; ++k) if (CPU_ISSET(k, &old_set)) { CPU_SET(k, &node_set); ++ncpu; }
                if (c != ',') break;
                (void)sep;
            }
            fclose(f);
        }
        if (ncpu > 0 && sched_setaffinity(0, sizeof node_set, &node_set) == 0) moved = true;
    }
    void* p = nullptr;
    cudaError_t e = cudaHostAlloc(&p, bytes ? bytes : 16, cudaHostAllocPortable);
    if (e == cudaSuccess) memset(p, 0, bytes ? bytes : 16);
    if (moved) sched_setaffinity(0, sizeof old_set, &old_set);
    if (e != cudaSuccess) { set_error("host_alloc: cudaHostAlloc(%zu) failed: %s", bytes, cudaGetErrorString(e)); return BVHGPU_ERR_CUDA; }
    *out = p;
    return BVHGPU_OK;
}
BVH_EXPORT int bvhgpu_host_free(bvhgpu_ctx* ctx, void* p) {
    if (!ctx) { set_error("host_free: null ctx"); return BVHGPU_ERR_INVALID; }
    BVH_CUDA_TRY(cudaSetDevice(ctx->device));
    if (p) BVH_CUDA_TRY(cudaFreeHost(p));
    return BVHGPU_OK;
}

#define DEFINE_API(T, SUF, TREE, AABB, RAY, NODE, FLAT)                                                                   \
    BVH_EXPORT int bvhgpu_build_##SUF(bvhgpu_ctx* ctx, const AABB* aabbs, size_t n, int mode, TREE** out) {              \
        return build_impl<T, TREE>(ctx, aabbs, n, mode, true, out);                                                       \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_build_dev_##SUF(bvhgpu_ctx* ctx, const void* dev_aabbs, size_t n, int mode, TREE** out) {      \
        return build_impl<T, TREE>(ctx, (const AABB*)dev_aabbs, n, mode, false, out);                                     \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_tree_from_nodes_##SUF(bvhgpu_ctx* ctx, const NODE* nodes, size_t n_nodes, const AABB* aabbs,   \
                                                size_t n, TREE** out) {                                                   \
        return from_nodes_impl<T, TREE>(ctx, nodes, n_nodes, aabbs, n, out);                                              \
    }                                                                                                                     \
    BVH_EXPORT void bvhgpu_tree_free_##SUF(TREE* tree) {                                                                  \
        if (!tree) return;                                                                                                \
        if (tree->ctx) cudaSetDevice(tree->ctx->device);                                                                  \
        tree_release<T>(tree);                                                                                            \
        delete tree;                                                                                                      \
    }                                                                                                                     \
    BVH_EXPORT size_t bvhgpu_tree_num_shapes_##SUF(const TREE* tree) { return tree ? tree->n : 0; }                       \
    BVH_EXPORT size_t bvhgpu_tree_num_nodes_##SUF(const TREE* tree) { return tree ? tree->n_nodes : 0; }                  \
    BVH_EXPORT int bvhgpu_tree_nodes_##SUF(TREE* tree, NODE* out_nodes, uint32_t* out_node_index) {                       \
        return tree_nodes_impl<T>(tree, out_nodes, out_node_index);                                                       \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_flatten_##SUF(TREE* tree, FLAT* out, size_t cap, size_t* len) {                                 \
        return flatten_impl<T>(tree, out, cap, len);                                                                      \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_traverse_##SUF(TREE* tree, int mode, const RAY* rays, size_t nrays, uint32_t* offsets,          \
                                         uint32_t* hits, size_t cap, size_t* total) {                                     \
        return traverse_host_impl<3, T>(tree, mode, rays, BVHGPU_RAYS_FULL, nrays, offsets, hits, cap, total);               \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_traverse_od_##SUF(TREE* tree, int mode, const T* origin_dir, size_t nrays, uint32_t* offsets,   \
                                            uint32_t* hits, size_t cap, size_t* total) {                                  \
        return traverse_host_impl<3, T>(tree, mode, origin_dir, BVHGPU_RAYS_OD, nrays, offsets, hits, cap, total);           \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_traverse_fetch_##SUF(TREE* tree, uint32_t* hits, size_t cap) { return fetch_impl<T>(tree, hits, cap); } \
    BVH_EXPORT int bvhgpu_traverse_dev_##SUF(TREE* tree, int mode, const void* dev_rays, size_t nrays, void* dev_offsets, \
                                             void* dev_hits, size_t cap, size_t* total) {                                 \
        return traverse_dev_impl<3, T>(tree, mode, dev_rays, BVHGPU_RAYS_FULL, nrays, (uint32_t*)dev_offsets, (uint32_t*)dev_hits, cap, total, "traverse_dev"); \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_traverse_od_dev_##SUF(TREE* tree, int mode, const void* dev_origin_dir, size_t nrays, void* dev_offsets, \
                                                void* dev_hits, size_t cap, size_t* total) {                              \
        return traverse_dev_impl<3, T>(tree, mode, dev_origin_dir, BVHGPU_RAYS_OD, nrays, (uint32_t*)dev_offsets, (uint32_t*)dev_hits, cap, total, "traverse_od_dev"); \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_traverse_sharded_dev_##SUF(TREE* tree, int mode, const void* dev_rays, size_t nrays, const bvhgpu_shard* shard) { \
        if (!tree || !shard || (nrays && !dev_rays)) { set_error("traverse_sharded: null argument"); return BVHGPU_ERR_INVALID; } \
        if (nrays == 0 || tree->n == 0) { set_error("traverse_sharded: every rank needs a non-empty shard and tree"); return BVHGPU_ERR_UNSUPPORTED; } \
        BVH_TRY(check_shard(shard, nrays));                                                                               \
        BVH_CUDA_TRY(cudaSetDevice(tree->ctx->device));                                                                   \
        return traverse_device<T>(tree, mode, dev_rays, (uint32_t)shard->ray_layout, nrays, nullptr, nullptr, shard->cap, nullptr, shard); \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_query_##SUF(TREE* tree, int mode, int kind, const T* queries, size_t n, uint32_t* offsets, uint32_t* hits, \
                                      size_t cap, size_t* total) {                                                       \
        return query_host_impl<3, T>(tree, mode, kind, queries, n, offsets, hits, cap, total);                           \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_query_dev_##SUF(TREE* tree, int mode, int kind, const void* dev_queries, size_t n, void* dev_offsets, \
                                          void* dev_hits, size_t cap, size_t* total) {                                    \
        return query_dev_impl<3, T>(tree, mode, kind, dev_queries, n, (uint32_t*)dev_offsets, (uint32_t*)dev_hits, cap, total); \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_overlap_pairs_##SUF(TREE* tree, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total) { \
        return overlap_host_impl<3, T>(tree, offsets, hits, cap, total);                                                  \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_overlap_pairs_dev_##SUF(TREE* tree, void* dev_offsets, void* dev_hits, size_t cap, size_t* total) { \
        return overlap_dev_impl<3, T>(tree, dev_offsets, dev_hits, cap, total);                                           \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_overlap_trees_##SUF(TREE* a, TREE* b, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total) { \
        return overlap_trees_host_impl<3, T>(a, b, offsets, hits, cap, total);                                            \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_overlap_trees_dev_##SUF(TREE* a, TREE* b, void* dev_offsets, void* dev_hits, size_t cap, size_t* total) { \
        return overlap_trees_dev_impl<3, T>(a, b, dev_offsets, dev_hits, cap, total);                                     \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_triangle_pairs_##SUF(TREE* tree, int skip_shared, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total) { \
        return triangle_pairs_host_impl<T>(tree, skip_shared, offsets, hits, cap, total);                                 \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_triangle_pairs_dev_##SUF(TREE* tree, int skip_shared, void* dev_offsets, void* dev_hits, size_t cap, size_t* total) { \
        return triangle_pairs_dev_impl<T>(tree, skip_shared, dev_offsets, dev_hits, cap, total);                          \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_triangle_pairs_trees_##SUF(TREE* a, TREE* b, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total) { \
        return triangle_pairs_trees_host_impl<T>(a, b, offsets, hits, cap, total);                                        \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_triangle_pairs_trees_dev_##SUF(TREE* a, TREE* b, void* dev_offsets, void* dev_hits, size_t cap, size_t* total) { \
        return triangle_pairs_trees_dev_impl<T>(a, b, dev_offsets, dev_hits, cap, total);                                 \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_nearest_##SUF(TREE* tree, int mode, const T* points, size_t n, uint32_t* out_shape, T* out_dist) { \
        return nearest_host_impl<3, T>(tree, mode, points, n, out_shape, out_dist);                                         \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_nearest_triangles_##SUF(TREE* tree, int mode, const T* points, size_t n, uint32_t* out_shape, T* out_dist) { \
        return nearest_host_impl<3, T>(tree, mode, points, n, out_shape, out_dist, 1);                                      \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_nearest_candidates_##SUF(TREE* tree, const T* points, size_t n, uint32_t* offsets, uint32_t* cand, \
                                                   size_t cap, size_t* total) {                                           \
        return nearest_candidates_host_impl<3, T>(tree, points, n, offsets, cand, cap, total);                               \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_traverse_ordered_##SUF(TREE* tree, const RAY* rays, size_t nrays, int ascending, uint32_t* offsets,      \
                                                 uint32_t* hits, T* dists, size_t cap, size_t* total) {                  \
        return ordered_host_impl<3, T>(tree, rays, nrays, ascending, offsets, hits, dists, cap, total);                      \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_knn_##SUF(TREE* tree, const T* points, size_t n, uint32_t k, const T* max_dist, uint32_t* out_shape, T* out_dist) { \
        return knn_host_impl<3, T>(tree, points, n, k, max_dist, out_shape, out_dist);                                      \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_knn_dev_##SUF(TREE* tree, const void* dev_points, size_t n, uint32_t k, const void* dev_max_dist,  \
                                        void* dev_shape, void* dev_dist) {                                                \
        return knn_dev_impl<3, T>(tree, dev_points, n, k, dev_max_dist, dev_shape, dev_dist);                             \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_knn_triangles_##SUF(TREE* tree, const T* points, size_t n, uint32_t k, const T* max_dist, uint32_t* out_shape, \
                                              T* out_dist, T* out_closest) {                                              \
        return knn_tri_host_impl<T>(tree, points, n, k, max_dist, out_shape, out_dist, out_closest);                       \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_knn_triangles_dev_##SUF(TREE* tree, const void* dev_points, size_t n, uint32_t k, const void* dev_max_dist, \
                                                  void* dev_shape, void* dev_dist, void* dev_closest) {                   \
        return knn_tri_dev_impl<T>(tree, dev_points, n, k, dev_max_dist, dev_shape, dev_dist, dev_closest);                \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_tree_set_triangles_##SUF(TREE* tree, const T* triangles, size_t n) {                            \
        if (!tree || (n && !triangles)) { set_error("set_triangles: null argument"); return BVHGPU_ERR_INVALID; }         \
        BVH_CUDA_TRY(cudaSetDevice(tree->ctx->device));                                                                   \
        return set_triangles<T>(tree, triangles, n, false);                                                               \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_tree_set_triangles_dev_##SUF(TREE* tree, const void* dev_triangles, size_t n) {                 \
        if (!tree || (n && !dev_triangles)) { set_error("set_triangles_dev: null argument"); return BVHGPU_ERR_INVALID; } \
        BVH_CUDA_TRY(cudaSetDevice(tree->ctx->device));                                                                   \
        return set_triangles<T>(tree, (const T*)dev_triangles, n, true);                                                  \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_closest_hit_##SUF(TREE* tree, const RAY* rays, size_t nrays, int use_triangles, uint32_t* out_shape, \
                                            T* out_dist, T* out_uv) {                                                     \
        return closest_host_impl<3, T>(tree, rays, BVHGPU_RAYS_FULL, nrays, use_triangles, out_shape, out_dist, out_uv);     \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_closest_hit_dev_##SUF(TREE* tree, const void* dev_rays, int ray_layout, size_t nrays, int use_triangles, \
                                                void* dev_shape, void* dev_dist, void* dev_uv) {                          \
        return closest_dev_impl<3, T>(tree, dev_rays, (uint32_t)ray_layout, nrays, use_triangles, dev_shape, dev_dist, dev_uv); \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_any_hit_##SUF(TREE* tree, const RAY* rays, size_t nrays, const T* tmax, int use_triangles, uint32_t* out_shape) { \
        return any_hit_host_impl<3, T>(tree, rays, nrays, tmax, use_triangles, out_shape);                                   \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_any_hit_dev_##SUF(TREE* tree, const void* dev_rays, int ray_layout, size_t nrays, const void* dev_tmax, \
                                            int use_triangles, void* dev_shape) {                                         \
        return any_hit_dev_impl<3, T>(tree, dev_rays, (uint32_t)ray_layout, nrays, dev_tmax, use_triangles, dev_shape);    \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_multi_hit_##SUF(TREE* tree, const RAY* rays, size_t nrays, uint32_t k, const T* tmax, int use_triangles, \
                                          uint32_t* out_shape, T* out_dist, T* out_uv) {                                  \
        return multi_hit_host_impl<3, T>(tree, rays, nrays, k, tmax, use_triangles, out_shape, out_dist, out_uv);          \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_multi_hit_dev_##SUF(TREE* tree, const void* dev_rays, int ray_layout, size_t nrays, uint32_t k,  \
                                              const void* dev_tmax, int use_triangles, void* dev_shape, void* dev_dist,   \
                                              void* dev_uv) {                                                             \
        return multi_hit_dev_impl<3, T>(tree, dev_rays, (uint32_t)ray_layout, nrays, k, dev_tmax, use_triangles, dev_shape, \
                                        dev_dist, dev_uv);                                                                \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_count_hits_##SUF(TREE* tree, const RAY* rays, size_t nrays, const T* tmax, uint32_t* out_front, \
                                           uint32_t* out_back) {                                                          \
        return count_hits_host_impl<T>(tree, rays, nrays, tmax, out_front, out_back);                                     \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_count_hits_dev_##SUF(TREE* tree, const void* dev_rays, int ray_layout, size_t nrays, const void* dev_tmax, \
                                               void* dev_front, void* dev_back) {                                         \
        return count_hits_dev_impl<T>(tree, dev_rays, (uint32_t)ray_layout, nrays, dev_tmax, dev_front, dev_back);        \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_contains_points_##SUF(TREE* tree, const T* points, size_t n, int rule, uint8_t* out_inside) {  \
        return contains_host_impl<T>(tree, points, n, rule, out_inside);                                                  \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_contains_points_dev_##SUF(TREE* tree, const void* dev_points, size_t n, int rule, void* dev_inside) { \
        return contains_dev_impl<T>(tree, dev_points, n, rule, dev_inside);                                               \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_signed_distance_##SUF(TREE* tree, const T* points, size_t n, int rule, uint32_t* out_shape,    \
                                                T* out_dist, T* out_closest) {                                            \
        return signed_distance_host_impl<T>(tree, points, n, rule, out_shape, out_dist, out_closest);                     \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_signed_distance_dev_##SUF(TREE* tree, const void* dev_points, size_t n, int rule, void* dev_shape, \
                                                    void* dev_dist, void* dev_closest) {                                  \
        return signed_distance_dev_impl<T>(tree, dev_points, n, rule, dev_shape, dev_dist, dev_closest);                  \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_traverse_stats_##SUF(TREE* tree, uint64_t* out2) {                                              \
        if (!tree || !out2) { set_error("traverse_stats: null argument"); return BVHGPU_ERR_INVALID; }                    \
        out2[0] = tree->last_visits; out2[1] = tree->last_total;                                                          \
        return BVHGPU_OK;                                                                                                 \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_rays_new_dev_##SUF(bvhgpu_ctx* ctx, const void* dev_origins, const void* dev_directions, size_t n, void* dev_rays) { \
        if (!ctx || (n && (!dev_origins || !dev_directions || !dev_rays))) { set_error("rays_new: null argument"); return BVHGPU_ERR_INVALID; } \
        BVH_CUDA_TRY(cudaSetDevice(ctx->device));                                                                         \
        return rays_new_device<T>(ctx, (const T*)dev_origins, (const T*)dev_directions, n, (RAY*)dev_rays);               \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_sah_cost_##SUF(TREE* tree, double* out2) {                                                      \
        if (!tree || !out2) { set_error("sah_cost: null argument"); return BVHGPU_ERR_INVALID; }                          \
        BVH_CUDA_TRY(cudaSetDevice(tree->ctx->device));                                                                   \
        BVH_TRY(resolve_status<T>(tree));                                                                                 \
        return sah_cost<T>(tree, out2);                                                                                   \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_refit_##SUF(TREE* tree, const AABB* aabbs, size_t n) { return refit_impl<3, T>(tree, aabbs, n, false); } \
    BVH_EXPORT int bvhgpu_refit_dev_##SUF(TREE* tree, const void* dev_aabbs, size_t n) { return refit_impl<3, T>(tree, dev_aabbs, n, true); } \
    BVH_EXPORT int bvhgpu_optimize_##SUF(TREE* tree, const AABB* aabbs, size_t n, double max_growth, size_t* rebuilt) { \
        return optimize_impl<T>(tree, aabbs, n, max_growth, rebuilt, false);                                           \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_optimize_dev_##SUF(TREE* tree, const void* dev_aabbs, size_t n, double max_growth, size_t* rebuilt) { \
        return optimize_impl<T>(tree, (const AABB*)dev_aabbs, n, max_growth, rebuilt, true);                            \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_update_##SUF(TREE* tree, const uint32_t* changed, const AABB* changed_aabbs, size_t m, double max_growth, size_t* rebuilt) { \
        return update_impl<3, T>(tree, changed, changed_aabbs, m, max_growth, rebuilt, false);                              \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_update_dev_##SUF(TREE* tree, const void* dev_changed, const void* dev_changed_aabbs, size_t m, double max_growth, size_t* rebuilt) { \
        return update_impl<3, T>(tree, (const uint32_t*)dev_changed, dev_changed_aabbs, m, max_growth, rebuilt, true); \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_add_shapes_##SUF(TREE* tree, const AABB* aabbs, size_t k, double max_growth, size_t* rebuilt) { \
        return add_impl<3, T>(tree, aabbs, k, max_growth, rebuilt, false);                                                   \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_add_shapes_dev_##SUF(TREE* tree, const void* dev_aabbs, size_t k, double max_growth, size_t* rebuilt) { \
        return add_impl<3, T>(tree, dev_aabbs, k, max_growth, rebuilt, true);                                   \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_remove_shapes_##SUF(TREE* tree, const uint32_t* indices, size_t k) {                            \
        return remove_impl<3, T>(tree, indices, k, false);                                                                \
    }                                                                                                                     \
    BVH_EXPORT int bvhgpu_remove_shapes_dev_##SUF(TREE* tree, const void* dev_indices, size_t k) {                        \
        return remove_impl<3, T>(tree, (const uint32_t*)dev_indices, k, true);                                            \
    }

#define DEFINE_API2(T, SUF, TREE, AABB, RAY, NODE, FLAT)                                                                   \
    BVH_EXPORT int bvhgpu_build_##SUF(bvhgpu_ctx* ctx, const AABB* aabbs, size_t n, int mode, TREE** out) {               \
        return build2_impl<T, TREE, AABB>(ctx, aabbs, n, mode, out);                                                       \
    }                                                                                                                      \
    BVH_EXPORT void bvhgpu_tree_free_##SUF(TREE* tree) {                                                                   \
        if (!tree) return;                                                                                                 \
        if (tree->ctx) cudaSetDevice(tree->ctx->device);                                                                   \
        tree_release<T>(tree);                                                                                             \
        delete tree;                                                                                                       \
    }                                                                                                                      \
    BVH_EXPORT size_t bvhgpu_tree_num_shapes_##SUF(const TREE* tree) { return tree ? tree->n : 0; }                        \
    BVH_EXPORT int bvhgpu_tree_nodes_##SUF(TREE* tree, NODE* out_nodes, uint32_t* out_node_index) {                        \
        return tree_nodes2_impl<T, NODE>(tree, out_nodes, out_node_index);                                                 \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_flatten_##SUF(TREE* tree, FLAT* out, size_t cap, size_t* len) { return flatten2_impl<T, FLAT>(tree, out, cap, len); } \
    BVH_EXPORT int bvhgpu_traverse_##SUF(TREE* tree, int mode, const RAY* rays, size_t nrays, uint32_t* offsets, uint32_t* hits, \
                                         size_t cap, size_t* total) {                                                      \
        return traverse_host_impl<2, T>(tree, mode, rays, BVHGPU_RAYS_FULL, nrays, offsets, hits, cap, total);                                 \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_query_##SUF(TREE* tree, int mode, int kind, const T* queries, size_t n, uint32_t* offsets, uint32_t* hits, \
                                      size_t cap, size_t* total) {                                                        \
        return query_host_impl<2, T>(tree, mode, kind, queries, n, offsets, hits, cap, total);                             \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_overlap_pairs_##SUF(TREE* tree, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total) {  \
        return overlap_host_impl<2, T>(tree, offsets, hits, cap, total);                                                   \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_overlap_trees_##SUF(TREE* a, TREE* b, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total) { \
        return overlap_trees_host_impl<2, T>(a, b, offsets, hits, cap, total);                                             \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_nearest_##SUF(TREE* tree, int mode, const T* points, size_t n, uint32_t* out_shape, T* out_dist) { \
        return nearest_host_impl<2, T>(tree, mode, points, n, out_shape, out_dist);                                        \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_nearest_candidates_##SUF(TREE* tree, const T* points, size_t n, uint32_t* offsets, uint32_t* cand, \
                                                   size_t cap, size_t* total) {                                            \
        return nearest_candidates_host_impl<2, T>(tree, points, n, offsets, cand, cap, total);                             \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_knn_##SUF(TREE* tree, const T* points, size_t n, uint32_t k, const T* max_dist, uint32_t* out_shape, T* out_dist) { \
        return knn_host_impl<2, T>(tree, points, n, k, max_dist, out_shape, out_dist);                                     \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_traverse_ordered_##SUF(TREE* tree, const RAY* rays, size_t nrays, int ascending, uint32_t* offsets,     \
                                                 uint32_t* hits, T* dists, size_t cap, size_t* total) {                   \
        return ordered_host_impl<2, T>(tree, rays, nrays, ascending, offsets, hits, dists, cap, total);               \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_closest_hit_##SUF(TREE* tree, const RAY* rays, size_t nrays, uint32_t* out_shape, T* out_dist) {  \
        return closest_host_impl<2, T>(tree, rays, BVHGPU_RAYS_FULL, nrays, 0, out_shape, out_dist, nullptr);                                              \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_any_hit_##SUF(TREE* tree, const RAY* rays, size_t nrays, const T* tmax, uint32_t* out_shape) {   \
        return any_hit_host_impl<2, T>(tree, rays, nrays, tmax, 0, out_shape);                                                      \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_multi_hit_##SUF(TREE* tree, const RAY* rays, size_t nrays, uint32_t k, const T* tmax, uint32_t* out_shape, \
                                          T* out_dist) {                                                                   \
        return multi_hit_host_impl<2, T>(tree, rays, nrays, k, tmax, 0, out_shape, out_dist, nullptr);                     \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_refit_##SUF(TREE* tree, const AABB* aabbs, size_t n) { return refit_impl<2, T>(tree, aabbs, n, false); } \
    BVH_EXPORT int bvhgpu_update_##SUF(TREE* tree, const uint32_t* changed, const AABB* changed_aabbs, size_t m, double max_growth, \
                                       size_t* rebuilt) {                                                                  \
        return update_impl<2, T>(tree, changed, changed_aabbs, m, max_growth, rebuilt, false);                                \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_add_shapes_##SUF(TREE* tree, const AABB* aabbs, size_t k, double max_growth, size_t* rebuilt) {  \
        return add_impl<2, T>(tree, aabbs, k, max_growth, rebuilt, false);                                                    \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_remove_shapes_##SUF(TREE* tree, const uint32_t* indices, size_t k) {                             \
        return remove_impl<2, T>(tree, indices, k, false);                                                                 \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_tree_set_segments_##SUF(TREE* tree, const T* segments, size_t n) {                               \
        if (!tree || (n && !segments)) { set_error("set_segments: null argument"); return BVHGPU_ERR_INVALID; }            \
        BVH_CUDA_TRY(cudaSetDevice(tree->ctx->device));                                                                    \
        return set_segments<T>(tree, segments, n);                                                                         \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_contains_points_##SUF(TREE* tree, const T* points, size_t n, int rule, uint8_t* out_class,       \
                                                int32_t* out_winding) {                                                    \
        return polygon_contains_host_impl<T>(tree, points, n, rule, out_class, out_winding);                               \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_knn_segments_##SUF(TREE* tree, const T* points, size_t n, uint32_t k, const T* max_dist,         \
                                             uint32_t* out_shape, T* out_dist, T* out_closest) {                           \
        return knn_seg_host_impl<T>(tree, points, n, k, max_dist, out_shape, out_dist, out_closest);                       \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_signed_distance_##SUF(TREE* tree, const T* points, size_t n, int rule, uint32_t* out_shape,      \
                                                T* out_dist, T* out_closest) {                                             \
        return polygon_distance_host_impl<T>(tree, points, n, rule, out_shape, out_dist, out_closest);                     \
    }

#define DEFINE_API4(T, SUF, TREE, AABB, RAY, NODE, FLAT)                                                                   \
    BVH_EXPORT int bvhgpu_build_##SUF(bvhgpu_ctx* ctx, const AABB* aabbs, size_t n, int mode, TREE** out) {               \
        return build4_impl<T, TREE>(ctx, aabbs, n, mode, out);                                                             \
    }                                                                                                                      \
    BVH_EXPORT void bvhgpu_tree_free_##SUF(TREE* tree) {                                                                   \
        if (!tree) return;                                                                                                 \
        if (tree->ctx) cudaSetDevice(tree->ctx->device);                                                                   \
        tree_release<T>(tree);                                                                                             \
        delete tree;                                                                                                       \
    }                                                                                                                      \
    BVH_EXPORT size_t bvhgpu_tree_num_shapes_##SUF(const TREE* tree) { return tree ? tree->n : 0; }                        \
    BVH_EXPORT int bvhgpu_tree_nodes_##SUF(TREE* tree, NODE* out_nodes, uint32_t* out_node_index) {                        \
        return tree_nodes_impl<T>(tree, out_nodes, out_node_index);                                                        \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_flatten_##SUF(TREE* tree, FLAT* out, size_t cap, size_t* len) { return flatten_impl<T>(tree, out, cap, len); } \
    BVH_EXPORT int bvhgpu_traverse_##SUF(TREE* tree, int mode, const RAY* rays, size_t nrays, uint32_t* offsets, uint32_t* hits, \
                                         size_t cap, size_t* total) {                                                      \
        return traverse_host_impl<4, T>(tree, mode, rays, BVHGPU_RAYS_FULL, nrays, offsets, hits, cap, total);             \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_traverse_dev_##SUF(TREE* tree, int mode, const void* dev_rays, size_t nrays, void* dev_offsets,  \
                                             void* dev_hits, size_t cap, size_t* total) {                                  \
        return traverse_dev_impl<4, T>(tree, mode, dev_rays, BVHGPU_RAYS_FULL, nrays, (uint32_t*)dev_offsets, (uint32_t*)dev_hits, cap, total, "traverse_dev"); \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_query_##SUF(TREE* tree, int mode, int kind, const T* queries, size_t n, uint32_t* offsets,      \
                                      uint32_t* hits, size_t cap, size_t* total) {                                        \
        return query_host_impl<4, T>(tree, mode, kind, queries, n, offsets, hits, cap, total);                             \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_query_dev_##SUF(TREE* tree, int mode, int kind, const void* dev_queries, size_t n,              \
                                          void* dev_offsets, void* dev_hits, size_t cap, size_t* total) {                 \
        return query_dev_impl<4, T>(tree, mode, kind, dev_queries, n, (uint32_t*)dev_offsets, (uint32_t*)dev_hits, cap, total); \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_overlap_pairs_##SUF(TREE* tree, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total) {  \
        return overlap_host_impl<4, T>(tree, offsets, hits, cap, total);                                                   \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_overlap_pairs_dev_##SUF(TREE* tree, void* dev_offsets, void* dev_hits, size_t cap, size_t* total) { \
        return overlap_dev_impl<4, T>(tree, dev_offsets, dev_hits, cap, total);                                            \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_overlap_trees_##SUF(TREE* a, TREE* b, uint32_t* offsets, uint32_t* hits, size_t cap, size_t* total) { \
        return overlap_trees_host_impl<4, T>(a, b, offsets, hits, cap, total);                                             \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_overlap_trees_dev_##SUF(TREE* a, TREE* b, void* dev_offsets, void* dev_hits, size_t cap, size_t* total) { \
        return overlap_trees_dev_impl<4, T>(a, b, dev_offsets, dev_hits, cap, total);                                      \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_nearest_##SUF(TREE* tree, int mode, const T* points, size_t n, uint32_t* out_shape, T* out_dist) { \
        return nearest_host_impl<4, T>(tree, mode, points, n, out_shape, out_dist);                                        \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_nearest_candidates_##SUF(TREE* tree, const T* points, size_t n, uint32_t* offsets, uint32_t* cand, \
                                                   size_t cap, size_t* total) {                                            \
        return nearest_candidates_host_impl<4, T>(tree, points, n, offsets, cand, cap, total);                             \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_traverse_ordered_##SUF(TREE* tree, const RAY* rays, size_t nrays, int ascending, uint32_t* offsets,    \
                                                 uint32_t* hits, T* dists, size_t cap, size_t* total) {                   \
        return ordered_host_impl<4, T>(tree, rays, nrays, ascending, offsets, hits, dists, cap, total);                    \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_closest_hit_##SUF(TREE* tree, const RAY* rays, size_t nrays, uint32_t* out_shape, T* out_dist) {  \
        return closest_host_impl<4, T>(tree, rays, BVHGPU_RAYS_FULL, nrays, 0, out_shape, out_dist, nullptr);              \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_closest_hit_dev_##SUF(TREE* tree, const void* dev_rays, size_t nrays, void* dev_shape, void* dev_dist) { \
        return closest_dev_impl<4, T>(tree, dev_rays, BVHGPU_RAYS_FULL, nrays, 0, dev_shape, dev_dist, nullptr);           \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_any_hit_##SUF(TREE* tree, const RAY* rays, size_t nrays, const T* tmax, uint32_t* out_shape) {   \
        return any_hit_host_impl<4, T>(tree, rays, nrays, tmax, 0, out_shape);                                             \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_any_hit_dev_##SUF(TREE* tree, const void* dev_rays, size_t nrays, const void* dev_tmax, void* dev_shape) { \
        return any_hit_dev_impl<4, T>(tree, dev_rays, BVHGPU_RAYS_FULL, nrays, dev_tmax, 0, dev_shape);                    \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_multi_hit_##SUF(TREE* tree, const RAY* rays, size_t nrays, uint32_t k, const T* tmax, uint32_t* out_shape, \
                                          T* out_dist) {                                                                   \
        return multi_hit_host_impl<4, T>(tree, rays, nrays, k, tmax, 0, out_shape, out_dist, nullptr);                     \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_multi_hit_dev_##SUF(TREE* tree, const void* dev_rays, size_t nrays, uint32_t k, const void* dev_tmax, \
                                              void* dev_shape, void* dev_dist) {                                           \
        return multi_hit_dev_impl<4, T>(tree, dev_rays, BVHGPU_RAYS_FULL, nrays, k, dev_tmax, 0, dev_shape, dev_dist, nullptr); \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_knn_##SUF(TREE* tree, const T* points, size_t n, uint32_t k, const T* max_dist, uint32_t* out_shape, T* out_dist) { \
        return knn_host_impl<4, T>(tree, points, n, k, max_dist, out_shape, out_dist);                                     \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_knn_dev_##SUF(TREE* tree, const void* dev_points, size_t n, uint32_t k, const void* dev_max_dist, \
                                        void* dev_shape, void* dev_dist) {                                                 \
        return knn_dev_impl<4, T>(tree, dev_points, n, k, dev_max_dist, dev_shape, dev_dist);                              \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_refit_##SUF(TREE* tree, const AABB* aabbs, size_t n) { return refit_impl<4, T>(tree, aabbs, n, false); } \
    BVH_EXPORT int bvhgpu_refit_dev_##SUF(TREE* tree, const void* dev_aabbs, size_t n) { return refit_impl<4, T>(tree, dev_aabbs, n, true); } \
    BVH_EXPORT int bvhgpu_update_##SUF(TREE* tree, const uint32_t* changed, const AABB* changed_aabbs, size_t m,           \
                                       double max_growth, size_t* rebuilt) {                                               \
        return update_impl<4, T>(tree, changed, changed_aabbs, m, max_growth, rebuilt, false);                             \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_update_dev_##SUF(TREE* tree, const void* dev_changed, const void* dev_changed_aabbs, size_t m,   \
                                           double max_growth, size_t* rebuilt) {                                           \
        return update_impl<4, T>(tree, (const uint32_t*)dev_changed, dev_changed_aabbs, m, max_growth, rebuilt, true);     \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_add_shapes_##SUF(TREE* tree, const AABB* aabbs, size_t k, double max_growth, size_t* rebuilt) {  \
        return add_impl<4, T>(tree, aabbs, k, max_growth, rebuilt, false);                                                 \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_add_shapes_dev_##SUF(TREE* tree, const void* dev_aabbs, size_t k, double max_growth, size_t* rebuilt) { \
        return add_impl<4, T>(tree, dev_aabbs, k, max_growth, rebuilt, true);                                              \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_remove_shapes_##SUF(TREE* tree, const uint32_t* indices, size_t k) {                             \
        return remove_impl<4, T>(tree, indices, k, false);                                                                 \
    }                                                                                                                      \
    BVH_EXPORT int bvhgpu_remove_shapes_dev_##SUF(TREE* tree, const void* dev_indices, size_t k) {                         \
        return remove_impl<4, T>(tree, (const uint32_t*)dev_indices, k, true);                                             \
    }

DEFINE_API2(float, f32x2, bvhgpu_tree2f, bvh_aabb2f, bvh_ray2f, bvh_node2f, bvh_flat2f)
DEFINE_API2(double, f64x2, bvhgpu_tree2d, bvh_aabb2d, bvh_ray2d, bvh_node2d, bvh_flat2d)
DEFINE_API(float, f32x3, bvhgpu_tree3f, bvh_aabb3f, bvh_ray3f, bvh_node3f, bvh_flat3f)
DEFINE_API(double, f64x3, bvhgpu_tree3d, bvh_aabb3d, bvh_ray3d, bvh_node3d, bvh_flat3d)
DEFINE_API4(float, f32x4, bvhgpu_tree4f, bvh_aabb4f, bvh_ray4f, bvh_node4f, bvh_flat4f)
DEFINE_API4(double, f64x4, bvhgpu_tree4d, bvh_aabb4d, bvh_ray4d, bvh_node4d, bvh_flat4d)
