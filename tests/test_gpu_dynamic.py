"""Batched add / remove of shapes on the device (bvhgpu_add_shapes_* / bvhgpu_remove_shapes_*) against the oracle's sequential
Bvh::add_shape / Bvh::remove_shape re-emitted in preorder (tests/dynoracle.py).  Run on an H100:  python -m pytest tests -m gpu"""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O
from tests import dynoracle as D
from tests.scenes import rays_for, scene

pytestmark = pytest.mark.gpu
SCENES = ["cubes1000", "random5000", "points700", "huge300"]


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A

    return A


def _fresh_shapes(rng, k, prec, far=False):
    mn = rng.uniform(-1000, 1000, (k, 3)) * (1e4 if far else 1.0)
    return O.make_aabbs(mn, mn + rng.uniform(0, 30, (k, 3)), prec)


def _check_walks(api, bvh, nodes, shapes, prec, nrays=2000):
    """flatten and the traversal CSR (BVH and FLAT modes; f32 also with the shared-memory top walk on and off) == the oracle's."""
    from bvh_b200 import capi

    if len(shapes) == 0:
        return
    flat = O.flatten(nodes, prec)
    g = bvh.flatten().nodes
    for f in ("entry_index", "exit_index", "shape_index"):
        assert np.array_equal(g[f], flat[f])
    rays = rays_for(shapes, nrays, prec, seed=len(shapes))
    ctx = bvh.ctx
    for mode, tree, omode in ((capi.TRAVERSE_BVH, nodes, O.MODE_RECURSIVE), (capi.TRAVERSE_FLAT, flat, O.MODE_FLAT)):
        r = O.traverse(tree, shapes, rays, omode, prec)
        for top in ((0, 1) if prec == "f32" else (-1,)):
            ctx.set_option("traverse_top", top)
            try:
                off, hits = bvh.traverse_batch(rays, mode=mode)
            finally:
                ctx.set_option("traverse_top", -1)
            assert np.array_equal(off.astype(np.uint64), r.offsets) and np.array_equal(hits, r.hits), (mode, top)


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("name", SCENES)
def test_remove_is_exact(api, name, prec):
    shapes0 = scene(name, prec)
    n = len(shapes0)
    want0 = O.build(shapes0, prec)
    # f32 "huge": the builder stores empty child boxes where surface areas overflow.  The reference refits only until a box stops
    # changing, the device refits every affected node: the boxes agree on tight trees, the topology always.
    tight = O.is_tight(want0.nodes, prec)
    rng = np.random.default_rng(5)
    for k in sorted({1, 2, max(1, n // 100), (30 * n) // 100, n - 1, n}):
        idx = rng.choice(n, k, replace=False).astype(np.uint32)
        bvh = api.Bvh.build(shapes0, prec=prec)
        bvh.flatten_dev()                                       # have_flat: the flat array must follow
        moves = bvh.remove_shapes(idx)
        wn, wi, ws = D.remove_shapes(want0.nodes, want0.node_index, shapes0, idx, prec)
        assert np.array_equal(moves, D.swap_moves(n, idx).astype(np.uint32))
        assert bvh.num_shapes == n - k
        if n - k:
            g = bvh.nodes
            for f in ("parent", "child_l", "child_r", "shape"):
                assert np.array_equal(g[f], wn[f]), (k, f)
            assert np.array_equal(bvh.node_index, wi)
            if tight:
                assert D.same_tree(g, wn), k
        if tight:
            _check_walks(api, bvh, wn, ws, prec, 1000)
        bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_single_add_is_the_reference_tree(api, prec):
    """200 add_shapes(k=1, max_growth=0) == the oracle's add_shape after every call: boxes inside the scene, far away (merge branch),
    degenerate boxes and f32-overflowing surface areas."""
    rng = np.random.default_rng(2)
    shapes = scene("random5000", prec)[:800]
    want = O.build(shapes, prec)
    nodes, ni = want.nodes, want.node_index
    bvh = api.Bvh.build(shapes, prec=prec)
    for step in range(200):
        kind = step % 4
        if kind == 0:
            new = _fresh_shapes(rng, 1, prec)
        elif kind == 1:
            new = _fresh_shapes(rng, 1, prec, far=True)
        elif kind == 2:
            p = rng.integers(-5, 5, (1, 3)).astype(float)
            new = O.make_aabbs(p, p, prec)
        else:
            mn = rng.uniform(-1e30, 1e30, (1, 3))
            new = O.make_aabbs(mn, mn + 1e29, prec)
        shapes = np.concatenate([shapes, new])
        assert bvh.add_shapes(new, max_growth=0.0) == 0
        nodes, ni = D.add_shapes(nodes, ni, shapes, 1, prec)
        assert D.same_tree(bvh.nodes, nodes), step
        assert np.array_equal(bvh.node_index, ni), step
    _check_walks(api, bvh, nodes, shapes, prec)
    bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("name", SCENES)
def test_batched_add(api, name, prec):
    from bvh_b200 import capi

    base = scene(name, prec)
    n = len(base)
    rng = np.random.default_rng(9)
    pool = np.concatenate([base[rng.permutation(n)], _fresh_shapes(rng, n, prec)])    # duplicates of scene boxes + new ones
    for k in sorted({2, max(2, n // 100), n // 10, n}):
        new = pool[rng.choice(len(pool), k, replace=False)]
        shapes = np.concatenate([base, new])
        for mg in (0.0, 1.5):
            bvh = api.Bvh.build(base, prec=prec)
            rb = bvh.add_shapes(new, max_growth=mg)
            assert bvh.num_shapes == n + k and (mg > 0 or rb == 0)
            nodes = bvh.nodes
            # f32 "huge": overflowing areas leave empty child boxes in built trees, so neither invariants nor hit sets are comparable
            tight = O.is_tight(O.build(base, prec).nodes, prec)
            if tight:
                assert O.is_consistent(nodes, shapes, prec) and O.is_tight(nodes, prec), (k, mg)
            assert np.array_equal(nodes["shape"][bvh.node_index], np.arange(n + k))
            rt = api.Bvh.from_nodes(nodes, shapes, prec=prec)         # validates the preorder layout
            assert D.same_tree(rt.nodes, nodes) and np.array_equal(rt.node_index, bvh.node_index)
            rays = rays_for(shapes, 1500, prec, seed=k)
            fresh = O.build(shapes, prec)
            r = O.traverse(fresh.nodes, shapes, rays, O.MODE_RECURSIVE, prec)
            off, hits = bvh.traverse_batch(rays, mode=capi.TRAVERSE_BVH)
            got = O.per_ray_lists(off, hits)
            exp = O.per_ray_lists(r.offsets, r.hits)
            assert not tight or all(sorted(a) == sorted(b) for a, b in zip(got, exp))
            if mg > 0 and k <= n // 10 and name.startswith(("cubes", "random")):      # zero-area (points) / overflowing (huge) roots have no SAH ratio
                b0 = O.build(base, prec)
                wn, _ = D.add_shapes(b0.nodes, b0.node_index, shapes, k, prec)
                assert bvh.sah_cost()[0] <= 1.10 * O.sah_cost(wn, prec)[0], (k, bvh.sah_cost(), O.sah_cost(wn, prec))
            rt.free(); bvh.free()
    empty = api.Bvh.build(base[:0], prec=prec)                  # adding to an empty tree == build
    empty.add_shapes(base, max_growth=1.5)
    ref = api.Bvh.build(base, prec=prec)
    assert D.same_tree(empty.nodes, ref.nodes) and np.array_equal(empty.node_index, ref.node_index)
    empty.free(); ref.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_churn(api, prec):
    """40 frames of remove 1 % + add 1 %: consistent, tight, SAH within 10 % of the oracle applying the same sequence; every query
    equals a from_nodes tree over the same nodes; update_shapes still works afterwards."""
    from bvh_b200 import capi

    rng = np.random.default_rng(4)
    shapes = scene("random5000", prec)
    bvh = api.Bvh.build(shapes, prec=prec)
    want = O.build(shapes, prec)
    wn, wi = want.nodes, want.node_index
    for frame in range(40):
        k = len(shapes) // 100
        idx = rng.choice(len(shapes), k, replace=False)
        bvh.remove_shapes(idx)
        wn, wi, shapes = D.remove_shapes(wn, wi, shapes, idx, prec)
        new = _fresh_shapes(rng, k, prec)
        shapes = np.concatenate([shapes, new])
        bvh.add_shapes(new, max_growth=1.5)
        wn, wi = D.add_shapes(wn, wi, shapes, k, prec)
    nodes = bvh.nodes
    assert O.is_consistent(nodes, shapes, prec) and O.is_tight(nodes, prec)
    assert bvh.sah_cost()[0] <= 1.10 * O.sah_cost(wn, prec)[0]
    ref = api.Bvh.from_nodes(nodes, shapes, prec=prec)
    rays = rays_for(shapes, 3000, prec, seed=8)
    for mode in (capi.TRAVERSE_BVH, capi.TRAVERSE_FLAT):
        a, b = bvh.traverse_batch(rays, mode=mode), ref.traverse_batch(rays, mode=mode)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    fa, fb = bvh.flatten().nodes, ref.flatten().nodes
    for f in ("entry_index", "exit_index", "shape_index"):
        assert np.array_equal(fa[f], fb[f])
    assert np.array_equal(fa["aabb"]["min"], fb["aabb"]["min"]) and np.array_equal(fa["aabb"]["max"], fb["aabb"]["max"])
    for x, y in zip(bvh.closest_hit(rays), ref.closest_hit(rays)):
        assert np.array_equal(x, y)
    q = np.concatenate([shapes["min"][:300], shapes["max"][:300]], axis=1)
    for x, y in zip(bvh.query_batch(capi.QUERY_AABB, q), ref.query_batch(capi.QUERY_AABB, q)):
        assert np.array_equal(x, y)
    pts = shapes["min"][::7].astype(float)
    for x, y in zip(bvh.nearest_to_batch(pts), ref.nearest_to_batch(pts)):
        assert np.array_equal(x, y)
    for x, y in zip(bvh.traverse_ordered(rays), ref.traverse_ordered(rays)):
        assert np.array_equal(x, y)
    moved = rng.choice(len(shapes), 50, replace=False)
    dl = rng.uniform(-5, 5, (50, 3))
    shapes = shapes.copy(); shapes["min"][moved] += dl; shapes["max"][moved] += dl
    bvh.update_shapes(moved, shapes, 1.5)
    assert O.is_consistent(bvh.nodes, shapes, prec) and O.is_tight(bvh.nodes, prec)
    ref.free(); bvh.free()


def test_bad_input_leaves_the_tree_untouched(api):
    from bvh_b200 import capi

    shapes = scene("random5000", "f32")
    bvh = api.Bvh.build(shapes)
    before = bvh.nodes.tobytes()
    bad = _fresh_shapes(np.random.default_rng(0), 3, "f32")
    bad["max"][1][2] = np.nan
    L = capi.lib()
    for call in (lambda: bvh.add_shapes(bad), lambda: bvh.remove_shapes([3, 5000]), lambda: bvh.remove_shapes([3, 4, 3])):
        with pytest.raises(capi.BvhGpuError):
            call()
        assert bvh.nodes.tobytes() == before and bvh.num_shapes == 5000
    rb = C.c_size_t(0)
    assert L.bvhgpu_add_shapes_f32x3(bvh._h, bad.ctypes.data_as(C.c_void_p), (1 << 30), C.c_double(0), C.byref(rb)) == capi.ERR_INVALID
    assert L.bvhgpu_remove_shapes_f32x3(bvh._h, np.arange(5001, dtype=np.uint32).ctypes.data_as(C.c_void_p), 5001) == capi.ERR_INVALID
    bvh._nodes = None
    assert bvh.nodes.tobytes() == before and bvh.num_shapes == 5000
    bvh.free()


def test_dev_forms_replicas_and_triangles(api):
    """_dev_ forms == host forms byte for byte; two trees fed the same calls are byte-identical; triangles follow a removal and
    are dropped by an add."""
    import torch
    from bvh_b200 import capi

    tris_all = O.create_n_cubes(300, want_tris=True)
    shapes, tris = tris_all if isinstance(tris_all, tuple) else (tris_all, None)
    if tris is None:
        pytest.skip("create_n_cubes does not return triangles")
    tris = np.asarray(tris, dtype=np.float32).reshape(-1, 9)
    L = capi.lib()
    rng = np.random.default_rng(6)
    a, b, c = (api.Bvh.build(shapes) for _ in range(3))
    for t in (a, b, c):
        t.set_triangles(tris)
    idx = rng.choice(len(shapes), 97, replace=False).astype(np.uint32)
    a.remove_shapes(idx); b.remove_shapes(idx)
    di = torch.from_numpy(idx.astype(np.int32)).cuda()
    torch.cuda.synchronize()
    capi.check(L.bvhgpu_remove_shapes_dev_f32x3(c._h, C.c_void_p(di.data_ptr()), len(idx)))
    c.ctx.synchronize(); c._nodes = None
    assert a.nodes.tobytes() == b.nodes.tobytes() == c.nodes.tobytes()
    rest = D.apply_moves(shapes, idx)
    rtris = D.apply_moves(tris, idx)
    rays = rays_for(rest, 2000, "f32", seed=3)
    ws, wd, _ = O.closest_hit(a.nodes, rest, rays, tris=rtris)
    gs, gd, _ = a.closest_hit(rays, triangles=True)
    assert np.array_equal(gs, ws) and np.array_equal(gd, wd)
    new = _fresh_shapes(rng, 40, "f32")
    dn = torch.from_numpy(new.view(np.uint8)).cuda()
    torch.cuda.synchronize()
    a.add_shapes(new); b.add_shapes(new)
    rb = C.c_size_t(0)
    capi.check(L.bvhgpu_add_shapes_dev_f32x3(c._h, C.c_void_p(dn.data_ptr()), len(new), C.c_double(1.5), C.byref(rb)))
    c._nodes = None
    assert a.nodes.tobytes() == b.nodes.tobytes() == c.nodes.tobytes()
    assert np.array_equal(a.node_index, c.node_index)
    with pytest.raises(capi.BvhGpuError) as e:
        a.closest_hit(rays, triangles=True)
    assert e.value.status == capi.ERR_INVALID
    for t in (a, b, c):
        t.free()


def _pool_used_bytes():
    """Bytes in use in device 0's default memory pool (the library allocates everything stream-ordered from it)."""
    cu = C.CDLL("libcuda.so.1")
    dev, pool, used = C.c_int(0), C.c_void_p(), C.c_uint64(0)
    assert cu.cuDeviceGet(C.byref(dev), 0) == 0
    assert cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0
    assert cu.cuMemPoolGetAttribute(pool, 7, C.byref(used)) == 0          # CU_MEMPOOL_ATTR_USED_MEM_CURRENT
    return used.value


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_update_then_add_does_not_grow_device_memory(api, prec):
    """The per-frame workflow update_shapes(.., 1.5) + add_shapes(.., 1.5) + remove_shapes at a steady shape count: after the first frames
    the pool's used memory stays exactly flat (every per-tree array is released or reused when the node count changes)."""
    rng = np.random.default_rng(12)
    shapes = scene("random5000", prec)
    bvh = api.Bvh.build(shapes, prec=prec)
    used = []
    for frame in range(8):
        moved = rng.choice(len(shapes), 50, replace=False)
        dl = rng.uniform(-40, 40, (50, 3))
        shapes = shapes.copy(); shapes["min"][moved] += dl; shapes["max"][moved] += dl
        bvh.update_shapes(moved, shapes, 1.5)
        new = _fresh_shapes(rng, 25, prec)
        bvh.add_shapes(new, max_growth=1.5)
        shapes = np.concatenate([shapes, new])
        idx = rng.choice(len(shapes), 25, replace=False)
        bvh.remove_shapes(idx)
        shapes = D.apply_moves(shapes, idx)
        bvh.ctx.synchronize()
        used.append(_pool_used_bytes())
    assert O.is_consistent(bvh.nodes, shapes, prec) and O.is_tight(bvh.nodes, prec)
    assert used[2:] == [used[2]] * len(used[2:]), used
    bvh.free()
