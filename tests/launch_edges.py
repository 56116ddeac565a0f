"""tests/launch_edges.py -- the batch sizes at which the batched calls' launch arithmetic changes, read from the CUDA sources so that a
retuned constant moves the sweep with it.  TEST INFRASTRUCTURE for tests/test_gpu_launch_edges.py; tests/test_launch_edges_cpu.py
checks that every constant is found.

    CONST            the constants, by name (KeyError-free: every name the sweep needs is present or the import fails)
    BLOCK            thread-block size of every per-item kernel, by kernel name
    edges(kind)      sorted batch sizes for one kind of kernel (see KINDS)
    chunk_bounds     the streamed host path's chunk bounds (traverse_host_pipelined's `bound` lambda), restated
    trec_bytes(n)    the bytes of an f32 tree's traversal records (which walk_top_kernel form runs depends on them)
    sm_count()       the device's SM count (torch), for the persistent grids
"""
import os
import re

_CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "bvh_b200", "csrc")


def _src(name):
    with open(os.path.join(_CSRC, name)) as f:
        return f.read()


def _one(pattern, text, what, flags=0):
    m = re.findall(pattern, text, flags)
    if len(m) != 1:
        raise LookupError(f"{what}: expected one match of {pattern!r}, found {len(m)}")
    return m[0]


def _read_constants():
    internal, trav, csr = _src("internal.h"), _src("traverse.cu"), _src("csr.cuh")
    c = {}
    c["BVH_MAX_CHUNKS"] = int(_one(r"#define\s+BVH_MAX_CHUNKS\s+(\d+)u?", internal, "BVH_MAX_CHUNKS"))
    c["CSR_SCAN_TILE"] = int(_one(r"constexpr\s+int\s+CSR_SCAN_TILE\s*=\s*(\d+)\s*;", internal, "CSR_SCAN_TILE"))
    c["CSR_SCAN_THREADS"] = int(_one(r"constexpr\s+int\s+CSR_SCAN_THREADS\s*=\s*(\d+)\s*;", internal, "CSR_SCAN_THREADS"))
    c["SCAN_ITEMS"] = int(_one(r"constexpr\s+int\s+SCAN_ITEMS\s*=\s*(\d+)\s*;", trav, "SCAN_ITEMS"))
    c["SCAN_THREADS"] = int(_one(r"constexpr\s+int\s+SCAN_THREADS\s*=\s*(\d+)\s*;", trav, "SCAN_THREADS"))
    _one(r"constexpr\s+int\s+SCAN_TILE\s*=\s*(SCAN_ITEMS\s*\*\s*SCAN_THREADS)\s*;", trav, "SCAN_TILE")
    c["SCAN_TILE"] = c["SCAN_ITEMS"] * c["SCAN_THREADS"]
    c["TOP_BUDGET"] = int(_one(r"constexpr\s+uint32_t\s+TOP_BUDGET\s*=\s*(\d+)\s*;", trav, "TOP_BUDGET"))
    # scan_blocks_kernel (the tile-sum scan of every two-pass CSR walk): its block and its loop step
    body = _one(r"scan_blocks_kernel\([^)]*\)\s*\{(.*?)\n\}", trav, "scan_blocks_kernel body", re.S)
    c["SCAN_BLOCKS_STEP"] = int(_one(r"b0\s*\+=\s*(\d+)\s*\)", body, "scan_blocks_kernel loop step"))
    c["SCAN_BLOCKS_THREADS"] = int(_one(r"scan_blocks_kernel<<<\s*1\s*,\s*(\d+)\s*,", csr, "scan_blocks_kernel launch"))
    # scan_post_kernel's last block scans the tile sums in steps of its own block
    post = _one(r"for \(uint32_t b0 = 0; b0 < gridDim\.x; b0 \+= (\w+)\)", trav, "scan_post_kernel tile-sum loop")
    c["SCAN_POST_STEP"] = c[post]
    # the host path: streamed from STREAM_MIN rays, min(BVH_MAX_CHUNKS, R / CHUNK_RAYS) chunks, emit in 4 slices from SLICE_MIN rays
    c["STREAM_MIN"] = int(_one(r"R < (\d+)u \? 1u", trav, "streaming threshold"))
    c["CHUNK_RAYS"] = int(_one(r"BVH_MAX_CHUNKS, R / (\d+)\)", trav, "rays per chunk"))
    c["SLICE_MIN"] = int(_one(r"const uint32_t nsl = R >= (\d+) \? \d+ : 1;", trav, "emit slices"))
    # the persistent grids: walk_top_kernel runs min(SMs, ceil(R / TOP_RAYS_PER_CTA)) CTAs; walk_persistent_kernel at most one CTA of
    # PERSISTENT_THREADS per PERSISTENT_THREADS rays, forced (option walk_grid) or sized from R / (6 * 256 * SMs)
    step, div = _one(r"\(uint64_t\)ctx->sm_count, \(\(uint64_t\)R \+ (\d+)\) / (\d+)\)", trav, "walk_top_kernel grid")
    assert int(step) + 1 == int(div)
    c["TOP_RAYS_PER_CTA"] = int(div)
    threads = int(_one(r"\(uint64_t\)R / \(\d+ull \* (\d+)ull \* sms\)", trav, "walk_persistent_kernel grid"))
    cap = _one(r"\* sms, \(\(uint64_t\)R \+ (\d+)\) / (\d+)\);", trav, "walk_persistent_kernel grid cap")
    assert int(cap[0]) + 1 == int(cap[1]) == threads
    c["PERSISTENT_THREADS"] = threads
    # walk_top_kernel makes 4 visits per vote on trees of at most TOP_UNROLL_MAX_BYTES of TNODE_F32_BYTES-byte records, 1 beyond
    c["TOP_UNROLL_MAX_BYTES"] = int(_one(r"TOP_UNROLL_MAX_BYTES = \(size_t\)(\d+) << 20;", trav, "TOP_UNROLL_MAX_BYTES")) << 20
    c["TNODE_F32_BYTES"] = int(_one(r"sizeof\(TNodeF\) == (\d+)", _src("common.cuh"), "sizeof(TNodeF)"))
    return c


def trec_bytes(n_shapes):
    """The traversal records of an f32 tree of n shapes (n - 1 inner nodes with two child records each, or one root leaf)."""
    return (1 if n_shapes == 1 else 2 * n_shapes - 2) * CONST["TNODE_F32_BYTES"]


def bound_source():
    """The body of traverse_host_pipelined's `bound` lambda and the unit count before it, whitespace collapsed: chunk_bounds restates
    exactly this text (tests/test_launch_edges_cpu.py compares them)."""
    trav = _src("traverse.cu")
    units = _one(r"const uint32_t nhalf = nchunks / 2, units = ([^;]*);", trav, "chunk units")
    body = _one(r"auto bound = \[&\]\(uint32_t c\) -> uint32_t \{(.*?)\};", trav, "bound lambda", re.S)
    return " ".join(units.split()), " ".join(body.split())


# kernel name -> set of block sizes over every launch of it (closest.cu, traverse.cu, dim4.cu, csr.cuh)
_LAUNCH = re.compile(r"(\w+_kernel)(?:<[^;<>]*(?:<[^;<>]*>[^;<>]*)*>)?<<<(?:[^;]*?),\s*(\d+)\s*,\s*\w+\s*,\s*[\w>.-]+>>>")


def _read_blocks():
    out = {}
    for name in ("closest.cu", "traverse.cu", "dim4.cu", "csr.cuh"):
        for k, b in _LAUNCH.findall(_src(name)):
            out.setdefault(k, set()).add(int(b))
    return out


CONST = _read_constants()
BLOCK = _read_blocks()

# the per-item kernels of the batched calls: a row past the end, or a missed last row, sits at the tail of one of their blocks
PER_ITEM_128 = ("closest_kernel", "multi_hit_kernel", "knn_kernel", "knn_tri_kernel", "nearest_kernel", "nearest4_kernel", "knn4_kernel")
PER_ITEM_256 = ("rays_new_kernel", "emit_kernel", "walk_count_kernel", "csr_walk_kernel", "ordered_kernel")
WARP = 32
KINDS = ("small", "scan_post", "scan_blocks", "host", "top")


def _around(x):
    return [x - 1, x, x + 1]


def block_sizes():
    """The block sizes of the per-item kernels (128 and 256 today)."""
    return sorted({b for k in PER_ITEM_128 + PER_ITEM_256 for b in BLOCK[k]})


def edges(kind, sms=None):
    """Sorted batch sizes where the launch arithmetic of one kind of kernel changes:
    small        1, one item either side of the warp, of every per-item block size, of walk_top_kernel's rays per CTA, of a scan tile,
                 and two tiles plus one (the second tile-sum step of the scans)
    scan_post    SCAN_TILE * SCAN_THREADS +- 1: the first size at which scan_post_kernel's last block loops over the tile sums
    scan_blocks  CSR_SCAN_TILE * the step of scan_blocks_kernel +- 1: the same for every two-pass CSR walk
    host         the streamed host path: one ray either side of streaming and of the sliced emit, and one batch that gets the largest
                 chunk count with a remainder
    top          walk_top_kernel at TOP_RAYS_PER_CTA * SMs +- 1 (needs `sms`)"""
    c = CONST
    if kind == "small":
        s = {1, 2 * c["SCAN_TILE"] + 1}
        for b in [WARP] + block_sizes() + [c["TOP_RAYS_PER_CTA"], c["SCAN_TILE"]]:
            s.update(_around(b))
        return sorted(s)
    if kind == "scan_post":
        return _around(c["SCAN_TILE"] * c["SCAN_POST_STEP"])
    if kind == "scan_blocks":
        return _around(c["CSR_SCAN_TILE"] * c["SCAN_BLOCKS_STEP"])
    if kind == "host":
        return sorted([c["STREAM_MIN"] - 1, c["STREAM_MIN"]] + _around(c["SLICE_MIN"]) + [c["CHUNK_RAYS"] * c["BVH_MAX_CHUNKS"] + 3])
    if kind == "top":
        if sms is None:
            raise ValueError("edges('top') needs the SM count")
        return _around(c["TOP_RAYS_PER_CTA"] * int(sms))
    raise ValueError(kind)


def chunks_for(R, forced=0):
    """The chunk count traverse_host_pipelined picks (forced > 0: BVHGPU_CHUNKS, clamped to BVH_MAX_CHUNKS)."""
    c = CONST
    if forced > 0:
        return min(c["BVH_MAX_CHUNKS"], forced)
    return 1 if R < c["STREAM_MIN"] else max(2, min(c["BVH_MAX_CHUNKS"], R // c["CHUNK_RAYS"]))


def chunk_bounds(R, nchunks, sched):
    """[bound(0), ..., bound(nchunks)]: schedule 1 gives the first half of the chunks two units each, schedule 0 one unit to every
    chunk; bound(c) = R * units_before(c) // units, in 64-bit integers."""
    nhalf = nchunks // 2
    units = nchunks + nhalf if sched == 1 else nchunks

    def bound(c):
        u = (2 * c if c <= nhalf else nhalf + c) if sched == 1 else c
        return R * u // units

    return [bound(c) for c in range(nchunks + 1)]


def sm_count(device=0):
    import torch

    return int(torch.cuda.get_device_properties(device).multi_processor_count)
