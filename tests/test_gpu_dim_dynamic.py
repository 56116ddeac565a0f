"""add_shapes and remove_shapes of Bvh<T,2> and Bvh<T,4> on the device:
- 4-D through a constant fourth axis equals the 3-D device path node for node (removes of 1 .. n shapes, batched adds with and
  without the growth rebuild, the scenes of test_gpu_dynamic.py);
- 2-D equals the 3-D device path on the z = [0, 0] lift;
- genuinely 2-D and 4-D scenes against the dimension-generic restatement of the reference's add_shape / remove_shape
  (tests/dimdyn.py): 200 single adds equal it after every call, batched removes equal it exactly, batched adds and 40 churn frames
  stay within 1.10x its SAH cost, and the reference's invariants (tests/dimcheck.py) hold throughout;
- traversal records and flat arrays built before a call follow the new tree (4-D, and 2-D where FLAT reads the lifted boxes);
- the contract: refusals leave the tree untouched, k = 0, empty trees, the device-pointer forms on a side stream, determinism,
  device memory."""

import numpy as np
import pytest

from tests import dimcheck, dimdyn, dimref
from tests import test_gpu_dim_update as U
from tests.dynoracle import swap_moves
from tests.scenes import scene

pytestmark = pytest.mark.gpu
PRECS = ("f32", "f64")
SCENES = ["cubes1000", "random5000", "points700", "huge300"]


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A

    return A


def _fresh3(rng, k, prec):
    from oracle import oracle as O

    mn = rng.uniform(-1000, 1000, (k, 3))
    return O.make_aabbs(mn, mn + rng.uniform(0, 30, (k, 3)), prec)


def _bytes(b):
    nodes, idx = b.nodes_and_index()
    return nodes.tobytes() + idx.tobytes()


def _invariants(b, a, tight=True):
    nodes, idx = b.nodes_and_index()
    assert b.n == len(a) == len(idx)
    assert dimcheck.layout_ok(nodes, idx)
    if tight:
        assert dimcheck.is_consistent(nodes, a) and dimcheck.is_tight(nodes)
    return nodes, idx


def _apply_moves(a, moves, k):
    """The shape list after remove_shapes: the survivors that move take their new index, the last k entries go."""
    a = a.copy()
    if len(moves):
        a[moves[:, 0]] = a[moves[:, 1]]
    return a[: len(a) - k]


# ---- 1. D = 4 through a constant fourth axis = D = 3 ------------------------------------------------------------------------
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("name", SCENES)
def test_lifted_4d_remove_equals_3d(api, name, prec):
    a = scene(name, prec)
    n = len(a)
    rng = np.random.default_rng(n)
    for k in sorted({1, 2, max(1, n // 100), n // 10, (30 * n) // 100, n - 1, n}):
        idx = rng.choice(n, k, replace=False).astype(np.uint32)
        b3, b4 = api.Bvh.build(a, prec=prec), api.Bvh4.build(U._lift(a, prec), prec=prec)
        m3, m4 = b3.remove_shapes(idx), b4.remove_shapes(idx)
        assert np.array_equal(m3, m4) and np.array_equal(m4, swap_moves(n, idx).astype(np.uint32))
        assert b4.n == b3.num_shapes == n - k
        if n - k:
            U._same34(b3, b4)
        b3.free(); b4.free()


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("name", SCENES)
def test_lifted_4d_add_equals_3d(api, name, prec):
    base = scene(name, prec)
    n = len(base)
    rng = np.random.default_rng(9)
    pool = np.concatenate([base[rng.permutation(n)], _fresh3(rng, n, prec)])    # duplicates of scene boxes + new ones
    for k in sorted({1, 2, max(2, n // 100), n // 10, (30 * n) // 100, n - 1, n}):
        new = pool[rng.choice(len(pool), k, replace=False)]
        for growth in (0.0, 1.5):
            b3, b4 = api.Bvh.build(base, prec=prec), api.Bvh4.build(U._lift(base, prec), prec=prec)
            r3 = b3.add_shapes(new, max_growth=growth)
            r4 = b4.add_shapes(U._lift(new, prec), max_growth=growth)
            assert r3 == r4 and (growth > 0 or r4 == 0)
            assert b4.n == b3.num_shapes == n + k
            U._same34(b3, b4)
            b3.free(); b4.free()


@pytest.mark.parametrize("prec", PRECS)
def test_lifted_4d_churn_equals_3d(api, prec):
    """Growth rebuilds through the level loop (a 60 000-shape scene, far-away additions) and removes, interleaved."""
    rng = np.random.default_rng(31)
    a = U._scene3("random5000", prec)
    a = np.concatenate([a] + [U._scene3("random5000", prec) for _ in range(11)])
    b3, b4 = api.Bvh.build(a, prec=prec), api.Bvh4.build(U._lift(a, prec), prec=prec)
    rebuilt = 0
    for step in range(6):
        idx = rng.choice(len(a), len(a) // 50, replace=False).astype(np.uint32)
        moves = b3.remove_shapes(idx)
        assert np.array_equal(moves, b4.remove_shapes(idx))
        a = _apply_moves(a, moves, len(idx))
        new = _fresh3(rng, len(a) // 25, prec)
        new["min"] *= 3; new["max"] *= 3
        r = b3.add_shapes(new, max_growth=1.5)
        assert r == b4.add_shapes(U._lift(new, prec), max_growth=1.5)
        rebuilt += r
        U._same34(b3, b4)
        a = np.concatenate([a, new])
    assert rebuilt > 256
    b3.free(); b4.free()


# ---- 2. D = 2 equals the 3-D path on the lift ---------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", PRECS)
def test_2d_add_and_remove_equal_3d_on_the_lift(api, prec):
    from bvh_b200.dtypes import BY_PREC_2D

    F = U._F(prec)
    rng = np.random.default_rng(22)
    mn, mx = dimref.scene("random", 5000, 2, F, rng)
    a = U._boxes(mn, mx, BY_PREC_2D[prec]["aabb"])
    b2, b3 = api.Bvh2.build(a, prec=prec), api.Bvh.build(U._lift2(a, prec), prec=prec)

    def same():
        n2, i2 = b2.nodes_and_index()
        n3 = b3.nodes
        assert np.array_equal(i2, b3.node_index)
        for f in ("parent", "child_l", "child_r", "shape"):
            assert np.array_equal(n2[f], n3[f]), f
        for side in ("l_aabb", "r_aabb"):
            for mm in ("min", "max"):
                assert np.array_equal(n2[side][mm], n3[side][mm][:, :2])

    for step, (k_rm, k_add, growth) in enumerate(((50, 1, 0.0), (500, 700, 1.5), (1, 2000, 1.5), (1200, 50, 0.0))):
        idx = rng.choice(len(a), k_rm, replace=False).astype(np.uint32)
        moves = b2.remove_shapes(idx)
        assert np.array_equal(moves, b3.remove_shapes(idx))
        a = _apply_moves(a, moves, k_rm)
        same()
        mn, mx = dimref.scene("random", k_add, 2, F, rng)
        new = U._boxes(mn * (1 + step), mx * (1 + step), BY_PREC_2D[prec]["aabb"])
        assert b2.add_shapes(new, max_growth=growth) == b3.add_shapes(U._lift2(new, prec), max_growth=growth)
        a = np.concatenate([a, new])
        same()
        _invariants(b2, a)
    b2.free(); b3.free()


# ---- 3. genuinely 2-D and 4-D scenes ------------------------------------------------------------------------------------------
def _cls(api, D):
    return api.Bvh2 if D == 2 else api.Bvh4


def _scene_d(api, kind, n, D, prec, rng):
    mn, mx = dimref.scene(kind, n, D, U._F(prec), rng)
    return U._boxes(mn, mx, _cls(api, D)._TABLE[prec]["aabb"])


def _same_as(b, dyn):
    """The device tree equals the restatement's, re-emitted in preorder, node for node (boxes with ==)."""
    want, want_ni = dyn.canonical()
    nodes, idx = b.nodes_and_index()
    assert np.array_equal(idx, want_ni)
    for f in ("parent", "child_l", "child_r", "shape"):
        assert np.array_equal(nodes[f], want[f]), f
    for side in ("l_aabb", "r_aabb"):
        for mm in ("min", "max"):
            assert np.array_equal(nodes[side][mm], want[side][mm]), (side, mm)
    return nodes


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("D", [2, 4])
def test_single_adds_equal_the_restatement(api, D, prec):
    """200 add_shapes(k = 1, max_growth = 0) == the reference's add_shape after every call: boxes inside the scene, far away (the merge
    branch), degenerate points and overflow-scale boxes, with every axis (w included) in play."""
    F = U._F(prec)
    rng = np.random.default_rng(200 + D)
    a = _scene_d(api, "random", 500, D, prec, rng)
    b = _cls(api, D).build(a, prec=prec)
    nodes, idx = b.nodes_and_index()
    dyn = dimdyn.Dyn(nodes, idx, a)
    for step in range(200):
        kind = step % 4
        if kind == 0:
            mn = rng.uniform(-100, 100, D); mx = mn + rng.uniform(0, 8, D)
        elif kind == 1:
            mn = rng.uniform(-100, 100, D) * 1e4; mx = mn + rng.uniform(0, 8, D)
        elif kind == 2:
            mn = mx = rng.integers(-5, 5, D).astype(float)
        else:
            mn = rng.uniform(-1e30, 1e30, D); mx = mn + 1e29
        new = U._boxes(mn[None, :].astype(F), mx[None, :].astype(F), _cls(api, D)._TABLE[prec]["aabb"])
        assert b.add_shapes(new, max_growth=0.0) == 0
        dyn.add(new["min"][0], new["max"][0])
        _same_as(b, dyn)
    assert dyn.merges > 0 and b.n == 700
    b.free()


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("kind", ["random", "coincident", "axis", "peel"])
@pytest.mark.parametrize("D", [2, 4])
def test_batched_add_and_remove_keep_the_invariants(api, D, kind, prec):
    """Batched removes equal the restatement exactly; batched adds keep the invariants and, with the growth rebuild, stay within
    1.10x the SAH cost of the same boxes added one by one by the reference's add_shape."""
    rng = np.random.default_rng(D * 10 + len(kind))
    n = 300 if kind == "peel" else 3000
    a = _scene_d(api, kind, n, D, prec, rng)
    b = _cls(api, D).build(a, prec=prec)
    for step, growth in enumerate((0.0, 1.5, 1.5)):
        new = _scene_d(api, kind if kind != "peel" else "random", max(1, n // (3 - step) // 10), D, prec, rng)
        nodes, idx = b.nodes_and_index()
        dyn = dimdyn.Dyn(nodes, idx, a)
        b.add_shapes(new, max_growth=growth)
        a = np.concatenate([a, new])
        nodes, _ = _invariants(b, a)
        if growth > 0 and kind != "coincident":               # coincident boxes: a zero-area root has no SAH ratio
            dyn.add_many(new)
            assert dimcheck.sah_cost(nodes) <= 1.10 * dimcheck.sah_cost(dyn.canonical()[0]), step
        idx = rng.choice(len(a), len(a) // 4, replace=False).astype(np.uint32)
        nodes, ni = b.nodes_and_index()
        dyn = dimdyn.Dyn(nodes, ni, a)
        moves = b.remove_shapes(idx)
        assert np.array_equal(moves, dyn.remove(idx))
        a = _apply_moves(a, moves, len(idx))
        _same_as(b, dyn)
        _invariants(b, a)                                     # every node's box is the join of what is left below it
    b.free()


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("D", [2, 4])
def test_churn_keeps_the_invariants_and_update_still_works(api, D, prec):
    """40 frames of 1 % remove + 1 % add: the invariants hold, the SAH cost stays within 1.10x that of the restatement applying the
    same sequence, and update_shapes and refit work afterwards."""
    rng = np.random.default_rng(40 + D)
    n = 10000
    a = _scene_d(api, "random", n, D, prec, rng)
    b = _cls(api, D).build(a, prec=prec)
    nodes, idx = b.nodes_and_index()
    dyn = dimdyn.Dyn(nodes, idx, a)
    for frame in range(40):
        idx = rng.choice(len(a), n // 100, replace=False).astype(np.uint32)
        moves = b.remove_shapes(idx)
        assert np.array_equal(moves, dyn.remove(idx))
        a = _apply_moves(a, moves, len(idx))
        new = _scene_d(api, "random", n // 100, D, prec, rng)
        b.add_shapes(new, max_growth=1.5)
        dyn.add_many(new)
        a = np.concatenate([a, new])
        if frame % 10 == 9:
            nodes, _ = _invariants(b, a)
            assert dimcheck.sah_cost(nodes) <= 1.10 * dimcheck.sah_cost(dyn.canonical()[0]), frame
    changed, a = U._move(a, rng, 0.05, 60.0)
    b.update_shapes(changed, a, max_growth=1.5)
    _invariants(b, a)
    b.refit(a)
    _invariants(b, a)
    b.free()


# ---- 4. cached device state follows the new tree -------------------------------------------------------------------------------
def _check_caches(api, D, prec, op):
    from bvh_b200 import capi

    cls = _cls(api, D)
    F = U._F(prec)
    rng = np.random.default_rng(D + (op == "add"))
    n = 1500
    a = _scene_d(api, "random", n, D, prec, rng)
    b, plain = cls.build(a, prec=prec), cls.build(a, prec=prec)
    if op == "add":
        new = _scene_d(api, "random", 400, D, prec, rng)
        a2 = np.concatenate([a, new])
    else:
        idx = rng.choice(n, 500, replace=False).astype(np.uint32)
        a2 = _apply_moves(a, swap_moves(n, idx), len(idx))
    ray_dtype = cls._TABLE[prec]["ray"]
    centre = (a2["min"].astype(np.float64) + a2["max"].astype(np.float64)) / 2
    prs = U._rays(a2, 120, D, F, rng, centre[rng.permutation(len(a2))])
    rays_np = np.zeros(len(prs), dtype=ray_dtype)
    for i, (o, d, inv) in enumerate(prs):
        rays_np["origin"][i], rays_np["direction"][i], rays_np["inv_direction"][i] = o, d, inv
    recs = {k: dimref.queries(k, a2["min"], a2["max"], 120, F, rng, nan=False) for k in (dimref.AABB, dimref.POINT, dimref.BALL)}
    pts = dimref.points(a2["min"], a2["max"], 80, F, rng)
    U._everything(b, D, F, rays_np, recs, pts)                # traversal records and the flat array exist from here on
    for t in (b, plain):
        if op == "add":
            t.add_shapes(new, max_growth=1.5)
        else:
            t.remove_shapes(idx)
    assert _bytes(b) == _bytes(plain)
    nodes, _ = b.nodes_and_index()
    new_res = U._everything(b, D, F, rays_np, recs, pts)
    pf = plain.flatten()                                      # field by field: the 2-D f64 record's padding is not part of it
    for f in ("entry_index", "exit_index", "shape_index"):
        assert np.array_equal(new_res["flat"][f], pf[f]), f
    for mm in ("min", "max"):
        assert np.array_equal(new_res["flat"]["aabb"][mm], pf["aabb"][mm]), mm
    flat, ex = U._expected(nodes, a2, D, F, prs, recs, pts)
    assert len(flat) == len(new_res["flat"])
    for key, want in ex.items():
        if key[0] == "near":
            shape, dist = new_res[key]
            assert shape.tolist() == [w[0] for w in want], key
            assert np.array_equal(dist, np.array([w[1] for w in want], dtype=F)), key
        else:
            got = U._csr_lists(*new_res[key])
            assert got == want, key
            if op == "add" and key[1] == capi.TRAVERSE_FLAT:
                assert any(s >= n for hits in got for s in hits), key     # the new shapes are found
    b.free(); plain.free()


@pytest.mark.parametrize("op", ["add", "remove"])
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("D", [2, 4])
def test_caches_follow_the_new_tree(api, D, prec, op):
    _check_caches(api, D, prec, op)


# ---- 5. contract -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("D", [2, 4])
def test_refusals_leave_the_tree_untouched(api, D, prec):
    from bvh_b200 import capi

    rng = np.random.default_rng(D)
    a = _scene_d(api, "random", 2000, D, prec, rng)
    b = _cls(api, D).build(a, prec=prec)
    b.update_shapes(np.arange(10, dtype=np.uint32), a)        # the baseline exists: a refusal must not disturb it either
    before = _bytes(b)
    bad = a[:3].copy()
    bad["max"][1, D - 1] = np.nan
    for call, status in ((lambda: b.add_shapes(bad), capi.ERR_NAN),
                         (lambda: b.add_shapes(a[:3], max_growth=0.5), capi.ERR_INVALID),
                         (lambda: b.remove_shapes(np.array([5, 2000], np.uint32)), capi.ERR_INVALID),
                         (lambda: b.remove_shapes(np.array([5, 7, 5], np.uint32)), capi.ERR_INVALID),
                         (lambda: b.remove_shapes(np.arange(2001, dtype=np.uint32) % 2000), capi.ERR_INVALID)):
        with pytest.raises(capi.BvhGpuError) as e:
            call()
        assert e.value.status == status
        assert _bytes(b) == before and b.n == 2000
    assert b.add_shapes(a[:0]) == 0                           # k = 0: no-ops
    assert len(b.remove_shapes(np.zeros(0, np.uint32))) == 0
    assert _bytes(b) == before
    b.add_shapes(a[:100])                                     # the tree still works after the refusals
    _invariants(b, np.concatenate([a, a[:100]]))
    b.free()


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("D", [2, 4])
def test_empty_trees_and_determinism(api, D, prec):
    rng = np.random.default_rng(7 + D)
    cls = _cls(api, D)
    a = _scene_d(api, "random", 3000, D, prec, rng)
    empty = cls.build(a[:0], prec=prec)
    empty.add_shapes(a, max_growth=1.5)                       # an add to an empty tree is build
    built = cls.build(a, prec=prec)
    assert _bytes(empty) == _bytes(built) and empty.n == len(a)
    moves = empty.remove_shapes(rng.permutation(len(a)).astype(np.uint32))    # every shape: the tree of an n = 0 build
    assert len(moves) == 0 and empty.n == 0 and _bytes(empty) == b""
    assert len(empty.flatten()) == 0
    empty.add_shapes(a[:500])
    assert _bytes(empty) == _bytes(cls.build(a[:500], prec=prec))
    for k in (1, 2):                                          # tiny trees
        t = cls.build(a[:k], prec=prec)
        t.add_shapes(a[k:k + 3])
        _invariants(t, a[:k + 3])
        t.remove_shapes(np.arange(k + 2, dtype=np.uint32))
        _invariants(t, a[k + 2:k + 3])
        t.free()
    t1, t2 = cls.build(a, prec=prec), cls.build(a, prec=prec)     # two trees given the same calls are byte-identical
    for step in range(3):
        idx = rng.choice(t1.n, 300, replace=False).astype(np.uint32)
        new = _scene_d(api, "random", 400, D, prec, rng)
        for t in (t1, t2):
            t.remove_shapes(idx)
            t.add_shapes(new, max_growth=1.5)
        assert _bytes(t1) == _bytes(t2)
    empty.free(); built.free(); t1.free(); t2.free()


@pytest.mark.parametrize("prec", PRECS)
def test_device_pointer_forms_on_a_side_stream_equal_the_host_forms(api, prec):
    import torch

    from bvh_b200 import capi

    rng = np.random.default_rng(11)
    a = U._scene4("random", 30000, prec, rng)
    host, dev = api.Bvh4.build(a, prec=prec), api.Bvh4.build(a, prec=prec)
    ctx = dev.ctx
    s = torch.cuda.Stream()
    ctx.set_stream(s.cuda_stream)
    try:
        for step in range(3):
            idx = rng.choice(host.n, 600, replace=False).astype(np.uint32)
            new = U._scene4("random", 900, prec, rng)
            m_host = host.remove_shapes(idx)
            r_host = host.add_shapes(new)
            with torch.cuda.stream(s):                        # the inputs are produced on the side stream, behind a busy kernel
                torch.cuda._sleep(50_000_000)
                d_idx = torch.from_numpy(idx.view(np.int32)).to("cuda")
                d_box = torch.from_numpy(np.ascontiguousarray(new).view(np.uint8)).to("cuda")
            assert np.array_equal(dev.remove_shapes_dev(d_idx.data_ptr(), len(idx), indices=idx), m_host)
            assert dev.add_shapes_dev(d_box.data_ptr(), len(new)) == r_host
            s.synchronize()
            assert _bytes(dev) == _bytes(host) and dev.n == host.n
        bad = torch.tensor([host.n], dtype=torch.int32, device="cuda")
        with pytest.raises(capi.BvhGpuError) as e:
            dev.remove_shapes_dev(bad.data_ptr(), 1)
        assert e.value.status == capi.ERR_INVALID
        assert _bytes(dev) == _bytes(host)
    finally:
        ctx.set_stream(None)
    host.free(); dev.free()


def test_device_memory_returns_to_its_level_over_update_add_remove_frames(api):
    import torch

    rng = np.random.default_rng(3)
    a = U._scene4("random", 20000, "f32", rng)
    a2 = _scene_d(api, "random", 20000, 2, "f32", rng)
    b, b2 = api.Bvh4.build(a, prec="f32"), api.Bvh2.build(a2, prec="f32")
    b.flatten(); b2.flatten()

    def frame():
        nonlocal a, a2
        for t, x, D in ((b, a, 4), (b2, a2, 2)):
            changed, x = U._move(x, rng, 0.05, 40.0)
            t.update_shapes(changed, x)
            idx = rng.choice(len(x), 200, replace=False).astype(np.uint32)
            x = _apply_moves(x, t.remove_shapes(idx), len(idx))
            new = _scene_d(api, "random", 200, D, "f32", rng)
            t.add_shapes(new)
            x = np.concatenate([x, new])
            t.flatten()
            if D == 4:
                a = x
            else:
                a2 = x

    frame()
    api.Context.default().synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(20):
        frame()
    api.Context.default().synchronize()
    assert free0 - torch.cuda.mem_get_info()[0] < 16 << 20
    b.free(); b2.free()
