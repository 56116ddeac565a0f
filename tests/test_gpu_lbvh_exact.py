"""The LBVH builders (BVHGPU_BUILD_LBVH = 1, BVHGPU_BUILD_LBVH_TREELET = 2) equal tests/lbvhref.py node for node: integers bit for bit,
coordinates with ==, node_index; f32 and f64, D = 3 and D = 2, on ordinary scenes, at the TILE boundaries, on scenes of identical
centroids, on a comb of single-bit codes that builds root paths of 80 edges, on boxes that mix -0.0 and +0.0 in one coordinate, on
f64 centroids spanning more than DBL_MAX, and on a 500 k f64 treelet build that defers its small subtrees.  Then the dynamic calls
started from LBVH trees (refit, optimize, update_shapes, add_shapes, remove_shapes) against their restatements, and one query sweep
per LBVH tree against the oracle or brute force on the device's own node array.
Run on an H100:  python -m pytest tests/test_gpu_lbvh_exact.py -m gpu"""
import ctypes as C
import itertools

import numpy as np
import pytest

from oracle import oracle as O
from tests import dimdyn, dimorder, dimref
from tests import dynoracle as DY
from tests import lbvhref as LR
from tests import rebuildref as RR
from tests.edge_inputs import edge_scene, empty_child_boxes
from tests.scenes import scene

pytestmark = pytest.mark.gpu
PRECS = ("f32", "f64")
MODES = (1, 2)
U32_MAX = 0xFFFFFFFF
LBVH_SCENES = ["cubes1", "random2", "random3", "random33", "random257", "random1000", "cubes1000", "points3000", "line700", "skew3000",
               "huge300", "edge:huge", "edge:mixed"]


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A

    return A


def _cls(api, D):
    return api.Bvh if D == 3 else api.Bvh2


def _state(b, D):
    if D == 3:
        b._nodes = b._node_index = None
        return b.nodes, b.node_index
    return b.nodes_and_index()


def _assert_same(nodes, idx, wn, wi, what):
    assert len(nodes) == len(wn), what
    assert np.array_equal(idx, wi), (what, "node_index")
    for f in ("parent", "child_l", "child_r", "shape"):
        bad = np.flatnonzero(nodes[f] != wn[f])
        assert len(bad) == 0, (what, f, bad[:8].tolist())
    for side in ("l_aabb", "r_aabb"):
        for mm in ("min", "max"):                             # == : only the sign of a zero may differ (DESIGN §2)
            bad = np.flatnonzero(np.any(nodes[side][mm] != wn[side][mm], axis=1))
            assert len(bad) == 0, (what, side, mm, bad[:8].tolist())


def _build_and_check(api, a, prec, mode, what, D=None):
    """Builds on the device, asserts equality with the restatement; returns (bvh, nodes, node_index, info)."""
    D = D or a["min"].shape[1]
    wn, wi, info = LR.restate(a, prec, mode)
    b = _cls(api, D).build(a, prec=prec, mode=mode)
    nodes, idx = _state(b, D)
    _assert_same(nodes, idx, wn, wi, what)
    return b, nodes, idx, info


def _named(name, prec):
    if name.startswith("edge:"):
        return edge_scene(name[5:], 2000, prec)
    return scene(name, prec)


# ---- the build -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("name", LBVH_SCENES)
def test_named_scenes(api, name, prec, mode):
    a = _named(name, prec)
    b, nodes, _, _ = _build_and_check(api, a, prec, mode, (name, prec, mode))
    if name == "points3000" and mode == 2:                    # the halving branch inside treelets sees the Morton order
        assert RR.halving_pairs(nodes, a, [{"root": 0, "count": len(a)}]) > 0
    b.free()


SIZES = [(n, D) for D in (3, 2) for n in (2, 3, 511, 512, 513, 1024, 1025, 20000)] + [(200000, 3)]     # (2-D treelets: tests/pyref.py)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("n,D", SIZES)
def test_sizes(api, n, D, prec, mode):
    a = RR.random_scene(n, D, prec, np.random.default_rng(n + 7 * D))
    b, nodes, _, info = _build_and_check(api, a, prec, mode, (n, D, prec, mode))
    if mode == 2:
        assert (info["treelets"] == [0]) == (n <= LR.TILE)
    b.free()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("D,prec", [(3, "f32"), (3, "f64"), (2, "f32")])
def test_identical_centroids(api, D, prec, mode):
    a = LR.identical_scene(1025, D, prec, np.random.default_rng(D))
    b, _, _, info = _build_and_check(api, a, prec, mode, (D, prec, mode))
    assert np.all(info["code"] == 0)
    b.free()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("D,prec", [(3, "f32"), (3, "f64"), (2, "f32")])
def test_comb_of_single_bit_codes(api, D, prec, mode):
    """Root paths of >= 80 edges (D = 3): path_kernel's pointer jumping must cover them, and every quantum must land on its bit."""
    a = LR.comb_scene(D, prec)
    b, nodes, _, info = _build_and_check(api, a, prec, mode, (D, prec, mode))
    if mode == 1:
        assert LR.depth(nodes) >= (80 if D == 3 else 55)
    assert len(np.unique(info["code"])) == (65 if D == 3 else 44)
    b.free()


@pytest.mark.parametrize("D", [3, 2])
@pytest.mark.parametrize("prec", PRECS)
def test_signed_zeros_are_deterministic(api, D, prec):
    """Children with -0.0 and +0.0 in one coordinate: the stored sign is that of min_t / max_t whatever the arrival order, so LBVH
    node arrays equal the restatement byte for byte, two builds give the same bytes, and a refit with unchanged boxes is a no-op."""
    a = LR.signed_zero_scene(20000, D, prec, np.random.default_rng(11))
    for mode in MODES:
        b, nodes, idx, _ = _build_and_check(api, a, prec, mode, (D, prec, mode))
        assert LR.mixed_zero_signs(nodes) > 100 and empty_child_boxes(nodes) == 0
        if mode == 1:
            wn, wi, _ = LR.restate(a, prec, 1)
            assert nodes.tobytes() == wn.tobytes()
        again = _cls(api, D).build(a, prec=prec, mode=mode)
        assert _state(again, D)[0].tobytes() == nodes.tobytes()
        again.free()
        b.refit(a)
        assert _state(b, D)[0].tobytes() == nodes.tobytes(), ("refit", mode)
        b.free()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("D", [3, 2])
def test_refit_with_unchanged_boxes_keeps_the_bytes(api, D, mode):
    for prec in PRECS:
        a = RR.random_scene(20000, D, prec, np.random.default_rng(31))
        b, nodes, _, _ = _build_and_check(api, a, prec, mode, (D, prec, mode))
        b.refit(a)
        assert _state(b, D)[0].tobytes() == nodes.tobytes()
        b.free()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("D", [3, 2])
def test_centroid_extent_beyond_dbl_max(api, D, mode):
    """hi - lo overflows: the operands are halved, so the x quanta still spread the shapes and no NaN reaches the conversion."""
    a = LR.overflow_centroid_scene(3000, D, np.random.default_rng(12))
    b, nodes, idx, info = _build_and_check(api, a, "f64", mode, (D, mode))
    assert info["morton"][0]["overflow"] and info["morton"][0]["nan_u_unhalved"] > 0
    assert len(np.unique(info["code"] >> np.uint64(62))) == 2
    if mode == 1 and D == 3:
        assert O.is_consistent(nodes, a, "f64") and O.is_tight(nodes, "f64")
    b.free()


@pytest.mark.parametrize("prec,n,name", [("f32", 20000, "random"), ("f64", 20000, "random"), ("f32", 3000, "points3000")])
def test_treelets_under_every_builder_strategy(api, prec, n, name):
    a = RR.random_scene(n, 3, prec, np.random.default_rng(5)) if name == "random" else scene(name, prec)
    wn, wi, _ = LR.restate(a, prec, 2)
    ctx = api.Context.default()
    try:
        for small, subtree, gang in itertools.product((-1, 0, 1), repeat=3):
            ctx.set_option("build_small", small); ctx.set_option("build_subtree", subtree); ctx.set_option("build_gang", gang)
            b = api.Bvh.build(a, prec=prec, mode=2)
            nodes, idx = _state(b, 3)
            _assert_same(nodes, idx, wn, wi, (small, subtree, gang))
            b.free()
    finally:
        ctx.set_option("build_small", -1); ctx.set_option("build_subtree", -1); ctx.set_option("build_gang", -1)


def test_f64_treelets_of_a_500k_scene_defer_their_small_subtrees(api):
    """f64 with n >= 400 000: treelet_begin defers ranges of <= 16 shapes to the thread-per-range kernel by default."""
    a = RR.random_scene(500_000, 3, "f64", np.random.default_rng(50))
    b, _, _, info = _build_and_check(api, a, "f64", 2, "500k")
    assert len(info["treelets"]) > 900
    b.free()


# ---- dynamic calls on LBVH trees --------------------------------------------------------------------------------------------------
class _Dev:
    """A device tree built in an LBVH mode behind the forms of the update step (the template of test_gpu_rebuild_exact.py)."""

    def __init__(self, api, D, a, prec, mode):
        self.D, self.prec = D, prec
        self.b = _cls(api, D).build(a, prec=prec, mode=mode)

    def state(self):
        return _state(self.b, self.D)

    def step(self, form, changed, a, mg):
        import torch

        from bvh_b200 import capi

        if form == "optimize":
            return self.b.optimize(a, mg)
        if form == "update":
            return self.b.update_shapes(changed, a, max_growth=mg)
        d_idx = torch.from_numpy(np.ascontiguousarray(changed, dtype=np.uint32).view(np.int32)).to("cuda")
        d_box = torch.from_numpy(np.ascontiguousarray(a[changed]).view(np.uint8)).to("cuda")
        torch.cuda.synchronize()
        rb = C.c_size_t(0)
        capi.check(getattr(capi.lib(), f"bvhgpu_update_dev_{self.b._d['suffix']}")(self.b._h, C.c_void_p(d_idx.data_ptr()), C.c_void_p(d_box.data_ptr()),
                                                                                  len(changed), C.c_double(mg), C.byref(rb)))
        return int(rb.value)


def _treelet_ranges(nodes, roots):
    return [(r, r + 2 * int(nodes["shape"][r]) - 1) for r in roots]


FORMS = {2: ("update",), 3: ("optimize", "update", "update_dev")}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("D,prec", [(3, "f32"), (3, "f64"), (2, "f32"), (2, "f64")])
def test_refit_optimize_and_update_from_lbvh_trees(api, D, prec, mode):
    """Every form, max_growth 0 and 1.5, two calls each, against rebuildref.Tree started from the LBVH tree's nodes and node_index;
    the treelet trees rebuild roots inside treelets and above them."""
    rng = np.random.default_rng(60 + D + mode)
    a0 = RR.random_scene(20000, D, prec, rng)
    _, _, info = LR.restate(a0, prec, mode)
    for form in FORMS[D]:
        for mg in ((1.5,) if form == "optimize" else (0.0, 1.5)):
            a = a0
            dev = _Dev(api, D, a, prec, mode)
            nodes, idx = dev.state()
            t = RR.Tree(nodes, idx)
            tl = _treelet_ranges(nodes, info["treelets"])
            inside = above = 0
            for call in range(2):
                changed, a = RR.mixed_motion(a, rng)
                want = t.optimize(a, mg) if form == "optimize" else t.update(changed, a, mg)
                got = dev.step(form, changed, a, mg)
                assert got == want, (form, mg, call, got, want)
                nodes, idx = dev.state()
                _assert_same(nodes, idx, t.nodes, t.node_index, (form, mg, call))
                for r in t.facts.get("roots", []):
                    inside += any(lo < r["root"] < hi for lo, hi in tl)
                    above += r["count"] > LR.TILE
            if mg > 0:
                assert above > 0 and (mode == 1 or inside > 0), (form, inside, above)
            dev.b.free()
    b = _cls(api, D).build(a0, prec=prec, mode=mode)           # refit with new boxes: the full climb over the LBVH tree
    t = RR.Tree(*_state(b, D))
    _, a1 = RR.mixed_motion(a0, rng)
    b.refit(a1)
    t.update(np.arange(len(a1)), a1, 0.0)
    _assert_same(*_state(b, D), t.nodes, t.node_index, "refit")
    b.free()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("prec", PRECS)
def test_remove_and_add_from_lbvh_trees_3d(api, prec, mode):
    """remove_shapes == the oracle's sequential remove_shape on the LBVH node array (one removal set empties the left subtree of a
    treelet root, which contracts that root); add_shapes (max_growth 0) == the oracle's add_shape, one shape per call."""
    rng = np.random.default_rng(70 + mode)
    a = RR.random_scene(5000, 3, prec, rng)
    _, _, info = LR.restate(a, prec, mode)
    b = api.Bvh.build(a, prec=prec, mode=mode)
    nodes0, idx0 = _state(b, 3)
    b.free()
    sets = [rng.choice(len(a), 50, replace=False), rng.choice(len(a), 2500, replace=False)]
    if mode == 2:
        r = info["treelets"][len(info["treelets"]) // 2]
        left = LR.subtree_shapes(nodes0, int(nodes0["child_l"][r]))
        sets.append(np.unique(np.concatenate([left, rng.choice(len(a), 30, replace=False)])))
    for idx in sets:
        idx = idx.astype(np.uint32)
        b = api.Bvh.build(a, prec=prec, mode=mode)
        b.remove_shapes(idx)
        wn, wi, _ = DY.remove_shapes(nodes0, idx0, a, idx, prec)
        _assert_same(*_state(b, 3), wn, wi, ("remove", len(idx)))
        b.free()
    b = api.Bvh.build(a, prec=prec, mode=mode)
    nodes, ni, shapes = nodes0, idx0, a
    for step in range(60):
        mn = rng.uniform(-100, 100, (1, 3)) * (1e3 if step % 3 == 1 else 1.0)
        new = RR.make_boxes(mn, mn + rng.uniform(0, 8, (1, 3)), 3, prec)
        shapes = np.concatenate([shapes, new])
        assert b.add_shapes(new, max_growth=0.0) == 0
        nodes, ni = DY.add_shapes(nodes, ni, shapes, 1, prec)
    _assert_same(*_state(b, 3), nodes, ni, "add")
    b.free()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("prec", PRECS)
def test_remove_and_add_from_lbvh_trees_2d(api, prec, mode):
    rng = np.random.default_rng(80 + mode)
    a = RR.random_scene(3000, 2, prec, rng)
    b = api.Bvh2.build(a, prec=prec, mode=mode)
    nodes0, idx0 = _state(b, 2)
    b.free()
    b = api.Bvh2.build(a, prec=prec, mode=mode)
    dyn = dimdyn.Dyn(nodes0, idx0, a)
    idx = rng.choice(len(a), 700, replace=False).astype(np.uint32)
    b.remove_shapes(idx)
    dyn.remove(idx)
    want, wi = dyn.canonical()
    _assert_same(*_state(b, 2), want, wi, "remove")
    for step in range(40):
        mn = rng.uniform(-100, 100, 2)
        new = RR.make_boxes(mn[None], (mn + rng.uniform(0, 8, 2))[None], 2, prec)
        assert b.add_shapes(new, max_growth=0.0) == 0
        dyn.add(new["min"][0], new["max"][0])
    want, wi = dyn.canonical()
    _assert_same(*_state(b, 2), want, wi, "add")
    b.free()


# ---- one query sweep per LBVH tree -----------------------------------------------------------------------------------------------
def _csr_equal(off, hits, want_lists, what):
    got = O.per_ray_lists(off, hits)
    assert len(got) == len(want_lists), what
    for i, (g, w) in enumerate(zip(got, want_lists)):
        assert [int(x) for x in g] == [int(x) for x in w], (what, i)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("D,prec", [(3, "f32"), (3, "f64"), (2, "f32"), (2, "f64")])
def test_query_sweep(api, D, prec, mode):
    from bvh_b200 import capi
    from tests import anyhit as H
    from tests import knnref as K

    F = RR._F(prec)
    rng = np.random.default_rng(90 + D + mode)
    a = RR.random_scene(3000, D, prec, rng)
    b, nodes, _, _ = _build_and_check(api, a, prec, mode, (D, prec, mode))
    mn, mx = np.asarray(a["min"], dtype=F), np.asarray(a["max"], dtype=F)
    flat = b.flatten().nodes if D == 3 else b.flatten()
    if D == 3:                                                 # flatten == the reference recursion over the same node array
        want = O.flatten(nodes, prec)
        for f in ("entry_index", "exit_index", "shape_index"):
            assert np.array_equal(flat[f], want[f]), f
        assert np.array_equal(flat["aabb"]["min"], want["aabb"]["min"]) and np.array_equal(flat["aabb"]["max"], want["aabb"]["max"])
    T = dimorder.Tree(nodes, a, flat)
    # rays: traverse (BVH and FLAT), ordered traversal, closest hit, any hit
    o, d, inv = dimorder.rays(mn, mx, 200, F, rng)
    tab = b._d if D == 2 else O._DT[prec]
    rays = np.zeros(len(o), dtype=tab["ray"])
    rays["origin"], rays["direction"], rays["inv_direction"] = o, d, inv
    if D == 3:
        for mode_t, tree, om in ((capi.TRAVERSE_BVH, nodes, O.MODE_RECURSIVE), (capi.TRAVERSE_FLAT, O.flatten(nodes, prec), O.MODE_FLAT)):
            r = O.traverse(tree, a, rays, om, prec)
            off, hits = b.traverse_batch(rays, mode=mode_t)
            assert np.array_equal(off.astype(np.uint64), r.offsets) and np.array_equal(hits, r.hits), mode_t
    else:
        off, hits = b.traverse_batch(rays, mode=capi.TRAVERSE_BVH)
        _csr_equal(off, hits, [[s for s, _ in T._candidates((list(o[i]), list(inv[i])))] for i in range(len(o))], "traverse")
    for asc in (True, False):
        off, hits, dist = b.traverse_ordered(rays, asc)
        for i in range(len(o)):
            w = T.ordered((list(o[i]), list(inv[i])), asc)
            assert hits[off[i]:off[i + 1]].tolist() == [s for s, _ in w], ("ordered", asc, i)
            assert np.array_equal(dist[off[i]:off[i + 1]], np.array([x for _, x in w], dtype=F)), ("ordered", asc, i)
    ch = b.closest_hit(rays)
    cs, cd = ch[0], ch[1]
    for i in range(len(o)):
        s, x = T.closest((list(o[i]), list(inv[i])))
        assert cs[i] == s and (x is None and np.isinf(cd[i]) or cd[i] == x), ("closest", i)
    assert np.array_equal(b.any_hit(rays), H.aabb_batch(nodes, a, o, inv, None))
    lim = np.where(np.isfinite(cd), cd, F(1)).astype(F)
    assert np.array_equal(b.any_hit(rays, lim), H.aabb_batch(nodes, a, o, inv, lim))
    # Aabb / Point / Ball queries, BVH and FLAT
    for kind in (capi.QUERY_AABB, capi.QUERY_POINT, capi.QUERY_BALL):
        q = dimref.queries(kind, mn, mx, 150, F, rng)
        for mode_q in (capi.TRAVERSE_BVH, capi.TRAVERSE_FLAT):
            off, hits = b.query_batch(kind, q, mode_q)
            ref = T.query_bvh if mode_q == capi.TRAVERSE_BVH else T.query_flat
            _csr_equal(off, hits, [ref(kind, rec) for rec in q], ("query", kind, mode_q))
    # nearest (BVH and FLAT) and knn
    p = dimref.points(mn, mx, 150, F, rng)
    for mode_q, ref in ((capi.TRAVERSE_BVH, T.nearest_bvh), (capi.TRAVERSE_FLAT, T.nearest_flat)):
        s, dd = b.nearest_to_batch(p, mode=mode_q)
        for i in range(len(p)):
            ws, wd = ref(p[i])
            assert s[i] == ws and dd[i] == wd, ("nearest", mode_q, i)
    bs, bd = K.brute(mn, mx, p, 17)
    for k in (1, 5, 17):
        s, dd = b.knn(p, k)
        assert np.array_equal(s, bs[:, :k]) and dd.tobytes() == np.ascontiguousarray(bd[:, :k]).tobytes(), k
    b.free()
