"""GPU tests added in round 2: compact ray layout, tool-safe host traversal, sticky build failures, NaN handling of the
update entry points, device-resident refit / optimize, the fused multi-GPU exchange on whatever GPUs the box has.
Run on an H100:  python -m pytest tests -m gpu"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle as O
from tests import prunedcheck as PC
from tests.scenes import rays_for, scene

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A

    return A


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("name", ["boxes21", "cubes1000", "random5000", "huge300"])
def test_compact_ray_layout_is_bit_identical(api, name, prec):
    """BVHGPU_RAYS_OD (origin + direction, inv_direction recomputed on the device) == the full Ray layout == the oracle,
    incl. axis-aligned rays (zero direction components: inv = +-inf, NaN rule of the slab test)."""
    from bvh_b200 import capi

    shapes = scene(name, prec)
    want = O.build(shapes, prec)
    bvh = api.Bvh.build(shapes, prec=prec)
    rays = rays_for(shapes, 3000, prec, seed=11, axis_aligned=400)
    for mode, omode in ((capi.TRAVERSE_BVH, O.MODE_RECURSIVE), (capi.TRAVERSE_FLAT, O.MODE_FLAT)):
        tree = want.nodes if omode == O.MODE_RECURSIVE else O.flatten(want.nodes, prec)
        r = O.traverse(tree, shapes, rays, omode, prec)
        for compact in (False, True):
            off, hits = bvh.traverse_batch(rays, mode=mode, compact=compact)
            assert np.array_equal(off.astype(np.uint64), r.offsets) and np.array_equal(hits, r.hits), (mode, compact)
    bvh.free()


def test_compact_layout_device_pointers_and_large_batch(api):
    """The device-pointer OD entry point and the streamed host path (>= 2 chunks) on 300 k rays."""
    import torch

    from bvh_b200 import capi

    shapes = O.create_n_cubes(2000)
    want = O.build(shapes)
    rays, _ = O.create_rays(300_000)
    r = O.traverse(want.nodes, shapes, rays, O.MODE_RECURSIVE, threads=O.hardware_threads())
    bvh = api.Bvh.build(shapes)
    for stream_opt in (-1, 0, 1):                       # auto / plain copy-then-walk / forced streaming
        bvh.ctx.set_option("traverse_stream", stream_opt)
        for compact in (False, True):
            off, hits = bvh.traverse_batch(rays, compact=compact)
            assert np.array_equal(off.astype(np.uint64), r.offsets) and np.array_equal(hits, r.hits), (stream_opt, compact)
    bvh.ctx.set_option("traverse_stream", -1)
    dev = torch.device("cuda", 0)
    od = np.empty((len(rays), 6), dtype=np.float32)
    od[:, :3], od[:, 3:] = rays["origin"], rays["direction"]
    d_od = torch.from_numpy(od.reshape(-1)).to(dev)
    d_off = torch.empty(len(rays) + 1, dtype=torch.int32, device=dev)
    d_hits = torch.empty(4 * len(rays), dtype=torch.int32, device=dev)
    tot = C.c_size_t(0)
    torch.cuda.synchronize(dev)
    capi.check(capi.lib().bvhgpu_traverse_od_dev_f32x3(bvh._h, 0, C.c_void_p(d_od.data_ptr()), len(rays), C.c_void_p(d_off.data_ptr()),
                                                       C.c_void_p(d_hits.data_ptr()), d_hits.numel(), C.byref(tot)))
    bvh.ctx.synchronize()
    assert tot.value == len(r.hits)
    assert np.array_equal(d_off.cpu().numpy().view(np.uint32).astype(np.uint64), r.offsets)
    assert np.array_equal(d_hits[: tot.value].cpu().numpy().view(np.uint32), r.hits)
    bvh.free()


_BLOCKING_SCRIPT = r"""
import sys, numpy as np
sys.path.insert(0, %r)
from oracle import oracle as O
from bvh_b200 import api
shapes = O.create_n_cubes(2000)
rays, _ = O.create_rays(300_000)
bvh = api.Bvh.build(shapes)
off, hits = bvh.traverse_batch(rays)
off2, hits2 = bvh.traverse_batch(rays, compact=True)
want = O.build(shapes)
r = O.traverse(want.nodes, shapes, rays, O.MODE_RECURSIVE, threads=8)
ok = np.array_equal(off.astype(np.uint64), r.offsets) and np.array_equal(hits, r.hits) and np.array_equal(off, off2) and np.array_equal(hits, hits2)
print("BLOCKING_OK" if ok else "BLOCKING_MISMATCH", len(hits))
"""


def test_host_traversal_survives_serialised_launches():
    """CUDA_LAUNCH_BLOCKING=1 makes every launch wait for the kernel: a walk kernel that waited for copies the host had yet to enqueue
    would never return (round 1: the driver's ncu pass hung for 900 s).  The host path must take the plain form here and finish."""
    env = dict(os.environ, CUDA_LAUNCH_BLOCKING="1")
    r = subprocess.run([sys.executable, "-c", _BLOCKING_SCRIPT % ROOT], capture_output=True, text=True, timeout=240, env=env)
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-1500:]
    assert "BLOCKING_OK" in r.stdout


_STREAMED_SCRIPT = _BLOCKING_SCRIPT + r"""
print("STREAMED", int(bvh.ctx.get_metric("host_streamed")))
"""


def test_host_traversal_falls_back_to_copy_then_walk_under_profiler_injection():
    """A profiler that replays kernels (Nsight Compute) would roll back the DMA-bumped arrival counter of the streamed host path, so
    the library must take the copy-then-walk form when a tool's injection marker is in the environment.  The marker used here is one
    only Nsight's own injection library reads; CUDA ignores it.  Control: the same 300 k-ray batch is streamed without it."""
    base = {k: v for k, v in os.environ.items() if k != "CUDA_LAUNCH_BLOCKING"}
    seen = {}
    for marked in (False, True):
        env = dict(base, NV_NSIGHT_INJECTION_TRANSPORT_TYPE="1") if marked else base
        r = subprocess.run([sys.executable, "-c", _STREAMED_SCRIPT % ROOT], capture_output=True, text=True, timeout=240, env=env)
        assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-1500:]
        assert "BLOCKING_OK" in r.stdout, r.stdout[-1500:]
        seen[marked] = r.stdout.split("STREAMED")[-1].split()[0]
    assert seen == {False: "1", True: "0"}, seen


def test_failed_build_is_sticky(api):
    """bvhgpu_build_dev_* defers the status: the first call on the tree reports the NaN, and so does EVERY later call (the node arrays
    were never written); nothing may walk them."""
    import torch

    from bvh_b200 import capi

    shapes = scene("random1000").copy()
    shapes["min"][77][0] = np.nan
    dev = torch.device("cuda", 0)
    d = torch.from_numpy(shapes.view(np.uint8).reshape(-1)).to(dev)
    torch.cuda.synchronize(dev)
    for mode in (capi.BUILD_EXACT_SAH, capi.BUILD_LBVH, capi.BUILD_LBVH_TREELET):
        bvh = api.Bvh.build_dev(d.data_ptr(), len(shapes), mode=mode)          # no error yet
        rays = rays_for(scene("random1000"), 100, seed=3)
        for attempt in range(3):
            with pytest.raises(capi.BvhGpuError) as e:
                bvh.traverse_batch(rays)
            assert e.value.status == capi.ERR_NAN, (mode, attempt)
        with pytest.raises(capi.BvhGpuError):
            bvh.flatten()
        with pytest.raises(capi.BvhGpuError):
            bvh.nodes
        bvh.free()


@pytest.mark.parametrize("mode", [0, 1, 2], ids=["exact", "lbvh", "lbvh_treelet"])
def test_nan_in_x_is_rejected_by_every_builder(api, mode):
    from bvh_b200 import capi

    shapes = scene("random3000").copy()
    shapes["max"][1234][0] = np.nan                      # the split axis of the root of this scene is x
    with pytest.raises(capi.BvhGpuError) as e:
        api.Bvh.build(shapes, mode=mode)
    assert e.value.status == capi.ERR_NAN


@pytest.mark.parametrize("what", ["refit", "optimize"])
def test_nan_update_leaves_the_tree_untouched(api, what):
    """A NaN in the new AABBs is refused BEFORE anything is overwritten: same nodes, still traversable (the reference would have
    panicked inside update_shapes with a half-modified Bvh)."""
    from bvh_b200 import capi

    shapes = scene("cubes1000").copy()
    bvh = api.Bvh.build(shapes)
    before = bvh.nodes.copy()
    bad = shapes.copy()
    bad["min"][5000][0] = np.nan
    with pytest.raises(capi.BvhGpuError) as e:
        bvh.refit(bad) if what == "refit" else bvh.optimize(bad)
    assert e.value.status == capi.ERR_NAN
    after = bvh.nodes
    assert np.array_equal(before.view(np.uint8), after.view(np.uint8))
    rays = rays_for(shapes, 500, seed=5)
    r = O.traverse(before, shapes, rays, O.MODE_RECURSIVE)
    off, hits = bvh.traverse_batch(rays)
    assert np.array_equal(off.astype(np.uint64), r.offsets) and np.array_equal(hits, r.hits)
    bvh.free()


def test_device_resident_refit_and_optimize(api):
    """bvhgpu_refit_dev_* / bvhgpu_optimize_dev_*: the new AABBs are already on the device (no upload) -- same result as the host forms."""
    import torch

    from bvh_b200 import capi

    shapes = scene("cubes1000").copy()
    rng = np.random.default_rng(21)
    moved = rng.choice(len(shapes), 600, replace=False)
    delta = rng.uniform(-3000, 3000, (600, 3)).astype(np.float32)
    new = shapes.copy()
    new["min"][moved] += delta
    new["max"][moved] += delta
    dev = torch.device("cuda", 0)
    d_new = torch.from_numpy(new.view(np.uint8).reshape(-1)).to(dev)
    torch.cuda.synchronize(dev)
    L = capi.lib()
    a, b = api.Bvh.build(shapes), api.Bvh.build(shapes)
    a.refit(new)
    capi.check(L.bvhgpu_refit_dev_f32x3(b._h, C.c_void_p(d_new.data_ptr()), len(new)))
    b._nodes = None
    assert np.array_equal(a.nodes.view(np.uint8), b.nodes.view(np.uint8))
    a2, b2 = api.Bvh.build(shapes), api.Bvh.build(shapes)
    ra = a2.optimize(new)
    rb = C.c_size_t(0)
    capi.check(L.bvhgpu_optimize_dev_f32x3(b2._h, C.c_void_p(d_new.data_ptr()), len(new), C.c_double(1.5), C.byref(rb)))
    b2._nodes = None
    assert ra == rb.value and ra > 0
    assert np.array_equal(a2.nodes.view(np.uint8), b2.nodes.view(np.uint8))
    assert O.is_consistent(b2.nodes, new) and O.is_tight(b2.nodes)
    for t in (a, b, a2, b2):
        t.free()


def test_pinned_numa_local_host_buffers(api):
    ctx = api.Context.default()
    arr = ctx.host_alloc(1 << 20, np.uint32)
    arr[:] = np.arange(len(arr), dtype=np.uint32)
    assert int(arr[12345]) == 12345
    ctx.host_free(arr)


@pytest.mark.parametrize("nproc", [1, 2])
def test_fused_multi_gpu_exchange(nproc):
    """tools/check_sharded.py under torchrun: the fused sharded traversal (counts pushed in 1 / 2 / 4-byte width, offsets rebuilt by
    the local scan, hit lists stored into every rank's buffer) == the NCCL all-gather path == the oracle, with uneven shards and with
    rays that have > 65 535 hits on one rank only.  nproc = 1 runs the whole exchange machinery on a single-GPU box."""
    import torch

    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs >= {nproc} GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1",
                        "--master-port", str(29533 + nproc), os.path.join(ROOT, "tools", "check_sharded.py")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count("fused==nccl True  fused==oracle True") == 2 * nproc


# ---- closest hit with distance pruning (SURVEY 8f N3) ----------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("name", ["cubes1", "boxes21", "cubes1000", "random5000", "points500", "huge300", "skew3000"])
def test_closest_hit_aabb_mode_is_exact(api, name, prec):
    """First AABB entered by the ray == the minimum (entry distance, DFS order) over Bvh::traverse's candidates, bit for bit -- although the
    device prunes subtrees behind the best entry so far and walks front to back (incl. the 3 000-deep skew tree: no stack)."""
    shapes = scene(name, prec)
    want = O.build(shapes, prec)
    bvh = api.Bvh.build(shapes, prec=prec)
    rays = rays_for(shapes, 3000, prec, seed=17, axis_aligned=300)
    ws, wd, _ = O.closest_hit(want.nodes, shapes, rays, prec=prec)
    gs, gd, _ = bvh.closest_hit(rays)
    assert np.array_equal(gs, ws)
    assert np.array_equal(gd, wd)
    if name.startswith("huge"):       # "no split wins" trees store EMPTY child boxes: the ordered traversal reports those (entry 0), this the shape's own AABB
        bvh.free()
        return
    # cross-check against the distance-ordered traversal: its first element per ray is the same shape
    off, hits, dists = bvh.traverse_ordered(rays, True)
    has = off[1:] > off[:-1]
    assert np.array_equal(has, gs != O.U32_MAX)
    assert np.array_equal(hits[off[:-1][has]], gs[has]) and np.array_equal(dists[off[:-1][has]], gd[has])
    bvh.free()


def _check_triangle_closest(api, shapes, tris, rays, prec="f32"):
    want = O.build(shapes, prec)
    bvh = api.Bvh.build(shapes, prec=prec)
    bvh.set_triangles(tris)
    ws, wd, wuv = O.closest_hit(want.nodes, shapes, rays, tris, prec)
    gs, gd, guv = bvh.closest_hit(rays, triangles=True)
    same = gs == ws
    # identical hits are identical to the bit (same Moeller-Trumbore arithmetic): distance, u, v
    assert np.array_equal(gd[same], wd[same]) and np.array_equal(guv[same], wuv[same])
    # the stated contract (tests/prunedcheck.py): a different triangle wins only where the reference's winner has a distance more
    # than 2^-16 in front of its own box entry, and then its exact intersection lies behind the device's hit
    assert (~same).mean() < 1e-3, (~same).mean()
    PC.check_closest(gs, gd, guv, ws, wd, tris, shapes, rays, prec)
    bvh.free()
    return int((ws != O.U32_MAX).sum())


def test_closest_hit_triangles_cubes(api):
    shapes, tris = O.create_n_cubes(2000, want_tris=True)
    rays = rays_for(shapes, 20000, seed=23)
    # aim a good part of the rays at cube centres so that many of them hit something
    rng = np.random.default_rng(5)
    centres = (shapes["min"][::12] + shapes["max"][::12]) * 0.5
    tgt = centres[rng.integers(0, len(centres), 10000)].astype(np.float64) + rng.uniform(-0.4, 0.4, (10000, 3))
    org = tgt + rng.normal(0, 1, (10000, 3)) * 3000
    rays[:10000] = O.ray_new(org, tgt - org)
    nhit = _check_triangle_closest(api, shapes, tris, rays)
    assert nhit > 5000


def test_closest_hit_triangles_sponza(api):
    """Sponza (66 450 triangles): primary rays from inside the atrium; closest triangle per ray == the caller's loop over Bvh::traverse +
    Ray::intersects_triangle (within the stated tolerance where two hits coincide)."""
    from bvh_b200 import scenes

    z = np.load(os.path.join(ROOT, "tests", "golden", "sponza_tris.npz"))
    tris = z["vertices"][z["triangles"].astype(np.int64)].astype(np.float32)
    shapes = O.tri_aabbs(tris)
    o, d = scenes.pinhole_rays(160, 120)
    rays = O.ray_new(o, d)
    nhit = _check_triangle_closest(api, shapes, tris.reshape(-1, 9), rays)
    assert nhit > 0.5 * len(rays)


def test_closest_hit_f64_and_empty(api):
    shapes, tris = O.create_n_cubes(300, prec="f64", want_tris=True)
    rays = rays_for(shapes, 5000, "f64", seed=29)
    _check_triangle_closest(api, shapes, tris, rays, "f64")
    e = api.Bvh.build(scene("empty"))
    s, dist, _ = e.closest_hit(rays_for(scene("empty"), 7))
    assert np.all(s == O.U32_MAX) and np.all(np.isinf(dist))


# ---- Bvh::update_shapes form: changed indices + their new AABBs ---------------------------------------------------------------
@pytest.mark.parametrize("name,prec,frac", [("cubes1000", "f32", 0.02), ("random5000", "f32", 0.10), ("random3000", "f64", 0.05)])
def test_update_shapes_equals_optimize_with_all_aabbs(api, name, prec, frac):
    """bvhgpu_update_* (only the changed shapes cross the boundary, optimization.rs:304-315's signature) == bvhgpu_optimize_* fed with
    the AABBs of ALL shapes: same node array; and with max_growth <= 0 == bvhgpu_refit_*."""
    shapes = scene(name, prec).copy()
    F = shapes["min"].dtype
    rng = np.random.default_rng(31)
    m = max(1, int(len(shapes) * frac))
    moved = rng.choice(len(shapes), m, replace=False)
    ext = float(shapes["max"].max() - shapes["min"].min())
    delta = rng.uniform(-ext / 8, ext / 8, (m, 3)).astype(F)
    new = shapes.copy()
    new["min"][moved] += delta
    new["max"][moved] += delta
    a, b = api.Bvh.build(shapes, prec=prec), api.Bvh.build(shapes, prec=prec)
    ra = a.optimize(new, 1.5)
    rb = b.update_shapes(moved, new, 1.5)
    assert ra == rb
    assert np.array_equal(a.nodes.view(np.uint8), b.nodes.view(np.uint8)) and np.array_equal(a.node_index, b.node_index)
    assert O.is_consistent(b.nodes, new, prec) and O.is_tight(b.nodes, prec)
    c, d = api.Bvh.build(shapes, prec=prec), api.Bvh.build(shapes, prec=prec)
    c.refit(new)
    assert d.update_shapes(moved, new, 0.0) == 0
    assert np.array_equal(c.nodes.view(np.uint8), d.nodes.view(np.uint8))
    for t in (a, b, c, d):
        t.free()


def test_update_shapes_rejects_bad_input_untouched(api):
    from bvh_b200 import capi

    shapes = scene("cubes1000").copy()
    bvh = api.Bvh.build(shapes)
    before = bvh.nodes.copy()
    bad = shapes.copy()
    bad["max"][10][2] = np.nan
    with pytest.raises(capi.BvhGpuError) as e:
        bvh.update_shapes([3, 10, 11], bad)
    assert e.value.status == capi.ERR_NAN
    idx = np.array([1, len(shapes)], dtype=np.uint32)
    fresh = shapes[[1, 2]]
    with pytest.raises(capi.BvhGpuError) as e:
        capi.check(capi.lib().bvhgpu_update_f32x3(bvh._h, _p(idx), _p(fresh), 2, C.c_double(1.5), None))
    assert e.value.status == capi.ERR_INVALID
    bvh._nodes = None
    assert np.array_equal(before.view(np.uint8), bvh.nodes.view(np.uint8))
    bvh.free()


def test_slow_drift_is_rebuilt_eventually(api):
    """Growth is judged against the surface area a node had when it was last (re)built, not against the previous call: a cluster that
    drifts away by a little per frame (never x1.5 in one step) must still be rebuilt, and the tree must stay as good as the oracle's
    update_shapes on the same frames (SAH cost within the stated 1.10)."""
    shapes = scene("cubes1000").copy()
    bvh = api.Bvh.build(shapes)
    ob = O.build(shapes)
    ref_nodes, ref_index = ob.nodes.copy(), ob.node_index.copy()
    rng = np.random.default_rng(41)
    movers = rng.choice(len(shapes) // 12, 40, replace=False)            # 40 whole cubes (12 triangles each) drift together
    idx = (movers[:, None] * 12 + np.arange(12)[None, :]).reshape(-1).astype(np.uint32)
    direction = rng.normal(0, 1, (len(movers), 3)).astype(np.float32)
    direction /= np.linalg.norm(direction, axis=1, keepdims=True)
    total_rebuilt, per_call = 0, []
    for frame in range(40):
        step = np.repeat(direction * np.float32(400.0), 12, axis=0)      # << scene extent (200 000) per frame
        shapes["min"][idx] += step
        shapes["max"][idx] += step
        r = bvh.update_shapes(idx, shapes, 1.5)
        per_call.append(r)
        total_rebuilt += r
        ref_nodes, ref_index = O.update_shapes(ref_nodes, ref_index, shapes, idx)
    assert total_rebuilt > 0, per_call
    nodes = bvh.nodes
    assert O.is_consistent(nodes, shapes) and O.is_tight(nodes)
    c_gpu, c_ref = bvh.sah_cost()[0], O.sah_cost(ref_nodes)[0]
    c_fresh = O.sah_cost(O.build(shapes).nodes)[0]
    assert c_gpu <= 1.10 * c_ref, (c_gpu, c_ref, c_fresh, per_call)
    bvh.free()


# ---- D = 2 (SURVEY 8f N4) ------------------------------------------------------------------------------------------------------
def _scene2d(kind, n, F, rng):
    from bvh_b200.dtypes import BY_PREC_2D

    a = np.zeros(n, dtype=BY_PREC_2D["f32" if F == np.float32 else "f64"]["aabb"])
    if kind == "random":
        mn = rng.uniform(-100, 100, (n, 2))
        a["min"], a["max"] = mn, mn + rng.uniform(0, 8, (n, 2)) ** 2 / 8
    elif kind == "points":                      # coincident degenerate boxes: the halving branch
        base = rng.integers(-4, 4, (max(n // 6, 1), 2)).astype(float)
        mn = base[rng.integers(0, len(base), n)]
        a["min"], a["max"] = mn, mn
    elif kind == "line":                        # all centres on one axis
        x = rng.integers(0, max(n // 3, 2), n).astype(float)
        a["min"][:, 0], a["max"][:, 0] = x - 0.25, x + 0.25
        a["min"][:, 1], a["max"][:, 1] = -0.25, 0.25
    return a


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("kind,n", [("random", 1), ("random", 2), ("random", 33), ("random", 700), ("points", 300), ("line", 200)])
def test_two_dimensional_bvh_matches_the_2d_restatement(api, kind, n, prec):
    """Bvh<T,2>: build, flatten and both traversals against tests/pyref.py run in TWO dimensions (an independent restatement of the
    reference's generic code: 2-term dot in surface_area, largest_axis over 2 components, 2-D slab test) -- node for node, bit for bit."""
    from tests import pyref
    from bvh_b200 import capi
    from bvh_b200.dtypes import BY_PREC_2D

    F = np.float32 if prec == "f32" else np.float64
    rng = np.random.default_rng(n * 7 + len(kind))
    a = _scene2d(kind, n, F, rng)
    want_nodes, want_index = pyref.build(a, F)
    bvh = api.Bvh2.build(a, prec=prec)
    nodes, index = bvh.nodes_and_index()
    assert list(index) == list(want_index)
    for i, w in enumerate(want_nodes):
        if w[0] == "leaf":
            assert nodes["child_l"][i] == O.U32_MAX and nodes["parent"][i] == w[1] and nodes["shape"][i] == w[2]
        else:
            assert (nodes["parent"][i], nodes["child_l"][i], nodes["child_r"][i]) == (w[1], w[2], w[3])
            for side, box in (("l_aabb", w[4]), ("r_aabb", w[5])):
                assert np.array_equal(nodes[side]["min"][i], np.array(box[0], dtype=F)) and np.array_equal(nodes[side]["max"][i], np.array(box[1], dtype=F))
    flat = bvh.flatten()
    wflat = pyref.flatten(want_nodes)
    assert len(flat) == len(wflat)
    for i, (box, entry, exit_, shape) in enumerate(wflat):
        assert (flat["entry_index"][i], flat["exit_index"][i], flat["shape_index"][i]) == (entry, exit_, shape)
        if box is not None:
            assert np.array_equal(flat["aabb"]["min"][i], np.array(box[0], dtype=F)) and np.array_equal(flat["aabb"]["max"][i], np.array(box[1], dtype=F))
    # rays: random + axis-aligned ones that start on box edges (0 * inf = NaN rule)
    m = 300
    org = rng.uniform(-120, 120, (m, 2)); tgt = rng.uniform(-100, 100, (m, 2))
    dirs = tgt - org
    for i in range(40):
        dirs[i] = [1.0, 0.0] if i % 2 else [0.0, -1.0]
        if i % 4 < 2:
            org[i] = a["min"][rng.integers(0, n)]
    rays = np.zeros(m, dtype=BY_PREC_2D[prec]["ray"])
    prs = [pyref.ray_new(F, org[i], dirs[i]) for i in range(m)]
    for i, (o, d, inv) in enumerate(prs):
        rays["origin"][i], rays["direction"][i], rays["inv_direction"][i] = o, d, inv
    off, hits = bvh.traverse_batch(rays, mode=capi.TRAVERSE_BVH)
    off2, hits2 = bvh.traverse_batch(rays, mode=capi.TRAVERSE_FLAT)
    for i in range(m):
        want = pyref.traverse_recursive(want_nodes, a, (prs[i][0], prs[i][2]), F)
        assert hits[off[i]:off[i + 1]].tolist() == want, i
        assert hits2[off2[i]:off2[i + 1]].tolist() == want, i        # tight trees: the FLAT leaf re-test agrees
    bvh.free()


# ---- nearest_to with the triangle's own PointDistance on the device ---------------------------------------------------------------
@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_nearest_to_with_native_triangle_distance(api, prec):
    """bvhgpu_nearest_triangles_*: the reference's nearest_to walk (bvh_node.rs:327-372 / flat_bvh.rs:513-562) with
    Triangle::distance_squared (closest_point_triangle, testbase.rs:353-443) at the leaves, evaluated on the device: same triangle (ties
    included) and bit-identical distance as the oracle -- and as brute force over all triangles."""
    from bvh_b200 import capi

    shapes, tris = O.create_n_cubes(400, prec=prec, want_tris=True)
    want = O.build(shapes, prec)
    bvh = api.Bvh.build(shapes, prec=prec)
    bvh.set_triangles(tris)
    rng = np.random.default_rng(77)
    centres = (shapes["min"][::12] + shapes["max"][::12]) * 0.5
    pts = np.concatenate([centres[rng.integers(0, len(centres), 1500)] + rng.normal(0, 3.0, (1500, 3)), rng.uniform(-1.2e5, 1.2e5, (1500, 3))])
    ws, wd = O.nearest_to(want.nodes, shapes, pts, prec, flat=False, kind=O.DIST_TRIANGLE, tris=tris)
    gs, gd = bvh.nearest_triangles_batch(pts, mode=capi.TRAVERSE_BVH)
    assert np.array_equal(gs, ws) and np.array_equal(gd, wd)
    flat = O.flatten(want.nodes, prec)
    ws2, wd2 = O.nearest_to(flat, shapes, pts, prec, flat=True, kind=O.DIST_TRIANGLE, tris=tris)
    gs2, gd2 = bvh.nearest_triangles_batch(pts, mode=capi.TRAVERSE_FLAT)
    assert np.array_equal(gs2, ws2) and np.array_equal(gd2, wd2)
    for i in range(0, len(pts), 211):                                    # brute force (nearest_to_some_bh, testbase.rs:270-312)
        d2 = O.shape_distances_squared(shapes, pts[i], prec, kind=O.DIST_TRIANGLE, tris=tris)
        assert d2[gs[i]] == d2.min()
    bvh.free()


@pytest.mark.parametrize("name", ["cubes1", "boxes21", "cubes1000", "cubes10000", "random5000", "points500", "huge300", "skew3000", "line200"])
def test_shared_memory_top_tree_walk_is_bit_identical(api, name):
    """Option traverse_top = 1 (walk_top_kernel: top records in shared memory) == the plain walk == the oracle, BVH and FLAT
    modes, also after a refit (the top records follow the traversal records)."""
    from bvh_b200 import capi

    shapes = scene(name, "f32")
    bvh = api.Bvh.build(shapes, prec="f32")
    rays = rays_for(shapes, 20000, "f32", seed=5, axis_aligned=500)
    ctx = bvh.ctx
    try:
        ctx.set_option("traverse_persistent", 1); ctx.set_option("traverse_stream", 0)
        for round_ in range(2):
            nodes = bvh.nodes
            for mode, omode in ((capi.TRAVERSE_BVH, O.MODE_RECURSIVE), (capi.TRAVERSE_FLAT, O.MODE_FLAT)):
                tree = nodes if omode == O.MODE_RECURSIVE else O.flatten(nodes, "f32")
                r = O.traverse(tree, shapes, rays, omode, "f32")
                visits = []
                for top in (0, 1, 64, 500):                      # off, full budget, tiny budgets (64: skew3000 gets no top records at all)
                    ctx.set_option("traverse_top", top)
                    off, hits = bvh.traverse_batch(rays, mode=mode)
                    visits.append(bvh.traverse_stats()[0])
                    assert np.array_equal(off.astype(np.uint64), r.offsets) and np.array_equal(hits, r.hits), (mode, top, round_)
                assert len(set(visits)) == 1, visits
            if name == "huge300":
                break
            rng = np.random.default_rng(1)
            dl = rng.uniform(-3, 3, (len(shapes), 3)).astype(np.float32)
            shapes = shapes.copy(); shapes["min"] += dl; shapes["max"] += dl
            bvh.refit(shapes)
    finally:
        ctx.set_option("traverse_top", -1); ctx.set_option("traverse_persistent", 2); ctx.set_option("traverse_stream", -1)
        bvh.free()


@pytest.mark.parametrize("mode_name", ["bvh", "flat"])
def test_streamed_host_path_with_the_shared_memory_top(api, mode_name):
    """The host-pointer path streams the rays into the running walk_top_kernel<.., STREAM> (forced: traverse_stream = 1,
    traverse_top = 1): same CSR as the oracle; the metric says the call was streamed."""
    from bvh_b200 import capi

    shapes = O.create_n_cubes(3000)
    want = O.build(shapes)
    rays, _ = O.create_rays(400_000)
    mode, omode = (capi.TRAVERSE_BVH, O.MODE_RECURSIVE) if mode_name == "bvh" else (capi.TRAVERSE_FLAT, O.MODE_FLAT)
    tree = want.nodes if omode == O.MODE_RECURSIVE else O.flatten(want.nodes)
    r = O.traverse(tree, shapes, rays, omode, threads=O.hardware_threads())
    bvh = api.Bvh.build(shapes)
    ctx = bvh.ctx
    try:
        ctx.set_option("traverse_top", 1); ctx.set_option("traverse_stream", 1)
        for compact in (False, True):
            off, hits = bvh.traverse_batch(rays, mode=mode, compact=compact)
            assert ctx.get_metric("host_streamed") == 1.0
            assert np.array_equal(off.astype(np.uint64), r.offsets) and np.array_equal(hits, r.hits), compact
    finally:
        ctx.set_option("traverse_top", -1); ctx.set_option("traverse_stream", -1)
        bvh.free()
