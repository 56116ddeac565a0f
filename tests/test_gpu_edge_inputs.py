"""GPU parity on the edge-case inputs of tests/edge_inputs.py: "no split wins" trees (overflowing surface areas, empty child boxes)
walked by finite unit rays, the f64 no-split branch of every build strategy, f64 LBVH builds, -0.0 direction components and
subnormal coordinates / directions.  Source of truth everywhere: the C++ oracle, which tests/test_edge_inputs_cpu.py pins to
tests/pyref.py on the same inputs.  Every test first asserts that its inputs contain what it is about.
Run on an H100:  python -m pytest tests -m gpu"""
import numpy as np
import pytest

from oracle import oracle as O
from tests import dynoracle as D
from tests.edge_inputs import FAMILIES, HUGE, SCENE_KINDS, edge_ray_batch, edge_scene, empty_child_boxes, ray_facts
from tests.scenes import rays_for, scene

pytestmark = pytest.mark.gpu
PRECS = ("f32", "f64")
EDGE = [(k, p) for p in PRECS for k in SCENE_KINDS]
UINT = {"f32": np.uint32, "f64": np.uint64}


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A

    return A


def _nodes_equal(a, b):
    """Integers bit for bit; AABB coordinates with == (DESIGN §2: only the sign of a zero may differ)."""
    if len(a) != len(b):
        return False
    for f in ("parent", "child_l", "child_r", "shape"):
        if not np.array_equal(a[f], b[f]):
            return False
    return all(np.array_equal(a[f][g], b[f][g]) for f in ("l_aabb", "r_aabb") for g in ("min", "max"))


def _flat_equal(a, b):
    if len(a) != len(b):
        return False
    for f in ("entry_index", "exit_index", "shape_index"):
        if not np.array_equal(a[f], b[f]):
            return False
    return np.array_equal(a["aabb"]["min"], b["aabb"]["min"]) and np.array_equal(a["aabb"]["max"], b["aabb"]["max"])


def _assert_csr(off, hits, want, fam, what):
    """CSR == the oracle's; on a mismatch, name the ray families that differ."""
    off = np.asarray(off).astype(np.uint64)
    if np.array_equal(off, want.offsets) and np.array_equal(hits, want.hits):
        return
    bad = np.arange(len(fam))
    if len(off) == len(want.offsets) and int(off[-1]) == len(hits):
        got, exp = O.per_ray_lists(off, hits), O.per_ray_lists(want.offsets, want.hits)
        bad = np.array([i for i in range(len(fam)) if not np.array_equal(got[i], exp[i])], dtype=np.int64)
    pytest.fail(f"{what}: {len(bad)} of {len(fam)} rays differ; families {sorted(set(fam[bad].tolist()))}; first {bad[:5].tolist()}")


def _assert_tree_preconditions(kind, shapes, built):
    if kind in ("huge", "mixed"):
        assert built.nosplit_fallthrough > 0 and empty_child_boxes(built.nodes) == built.nosplit_fallthrough
    else:
        assert built.degenerate_splits == len(shapes) - 1


def _assert_ray_preconditions(kind, shapes, rays, fam):
    """Every family is present, no ray is a point-in-box test, and the batch reaches the arithmetic it is meant for."""
    assert all((fam == f).sum() > 0 for f in FAMILIES)
    facts = ray_facts(rays, shapes)
    assert facts["nonzero_direction"] == len(rays), facts
    for key in ("neg_zero", "inv_neg_inf", "face_plane_nan", "subnormal_dir_finite_inv", "subnormal_dir_inf_inv"):
        assert facts[key] > 0, (key, facts)
    assert facts["subnormal_differences" if kind == "subnormal" else "overflowing_products"] > 0, facts


def _edge_case(kind, prec, n=2000, per_family=300, seed=0):
    shapes = edge_scene(kind, n, prec)
    built = O.build(shapes, prec)
    _assert_tree_preconditions(kind, shapes, built)
    rays, fam = edge_ray_batch(shapes, per_family, prec, seed)
    _assert_ray_preconditions(kind, shapes, rays, fam)
    return shapes, built, rays, fam


# ---- exact builder ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [300, 2000, 5000])
@pytest.mark.parametrize("kind,prec", EDGE)
def test_exact_build_is_bit_identical(api, kind, prec, n):
    shapes = edge_scene(kind, n, prec)
    want = O.build(shapes, prec)
    _assert_tree_preconditions(kind, shapes, want)
    bvh = api.Bvh.build(shapes, prec=prec)
    assert _nodes_equal(bvh.nodes, want.nodes)
    assert np.array_equal(bvh.node_index, want.node_index)
    assert _flat_equal(bvh.flatten().nodes, O.flatten(want.nodes, prec))
    bvh.free()


@pytest.mark.parametrize("kind,prec", [("huge", "f64"), ("mixed", "f64"), ("subnormal", "f64"), ("mixed", "f32"), ("subnormal", "f32")])
def test_builder_strategies_are_bit_identical(api, kind, prec):
    """The six build_small / build_subtree / build_gang combinations of test_gpu_parity's strategy test, on the no-split and
    all-degenerate scenes: every strategy's copy of the "no split wins" and halving branches must produce the reference's bits."""
    shapes = edge_scene(kind, 2000, prec)
    want = O.build(shapes, prec)
    _assert_tree_preconditions(kind, shapes, want)
    wflat = O.flatten(want.nodes, prec)
    ctx = api.Context.default()
    try:
        for small, subtree, gang in ((0, 0, 0), (0, 1, 0), (0, 0, 1), (0, 1, 1), (1, 1, 1), (1, 0, 1)):
            ctx.set_option("build_small", small); ctx.set_option("build_subtree", subtree); ctx.set_option("build_gang", gang)
            bvh = api.Bvh.build(shapes, prec=prec)
            assert _nodes_equal(bvh.nodes, want.nodes), (small, subtree, gang)
            assert np.array_equal(bvh.node_index, want.node_index), (small, subtree, gang)
            assert _flat_equal(bvh.flatten().nodes, wflat), (small, subtree, gang)
            bvh.free()
    finally:
        ctx.set_option("build_small", -1); ctx.set_option("build_subtree", -1); ctx.set_option("build_gang", -1)


def test_forced_gangs_on_a_large_f64_mixed_scene(api):
    """300 k shapes: gangs (normally off at this size) forced on, next to the queue-mode tile tasks, through the f64 no-split branch."""
    shapes = edge_scene("mixed", 300_000, "f64")
    want = O.build(shapes, "f64", threads=O.hardware_threads())
    _assert_tree_preconditions("mixed", shapes, want)
    ctx = api.Context.default()
    ctx.set_option("build_gang", 1)
    try:
        bvh = api.Bvh.build(shapes, prec="f64")
        assert _nodes_equal(bvh.nodes, want.nodes)
        assert np.array_equal(bvh.node_index, want.node_index)
        bvh.free()
    finally:
        ctx.set_option("build_gang", -1)


# ---- traversal --------------------------------------------------------------------------------------------------------------
def _tiled(r, reps):
    """The oracle's CSR of a ray batch repeated `reps` times."""
    counts = np.tile(np.diff(r.offsets.astype(np.int64)), reps)
    return O.TraverseResult(np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64), np.tile(r.hits, reps), 0, 0, 0, False)


@pytest.mark.parametrize("kind,prec", EDGE)
def test_traversal_parity(api, kind, prec):
    """BVH and FLAT CSR == the oracle for every ray family: single-pass / two-pass / forced-overflow re-walk x both pass-1 kernels,
    both ray layouts, the device-pointer entry point; f32 also the shared-memory top walk at four budgets (same visit count) and
    the streamed host path."""
    import torch

    from bvh_b200 import capi

    shapes, built, rays, fam = _edge_case(kind, prec)
    nodes, flat = built.nodes, O.flatten(built.nodes, prec)
    want = {capi.TRAVERSE_BVH: O.traverse(nodes, shapes, rays, O.MODE_RECURSIVE, prec),
            capi.TRAVERSE_FLAT: O.traverse(flat, shapes, rays, O.MODE_FLAT, prec)}
    if kind != "subnormal":
        assert len(want[capi.TRAVERSE_BVH].hits) > len(want[capi.TRAVERSE_FLAT].hits)      # the two semantics really differ here
    bvh = api.Bvh.build(shapes, prec=prec)
    ctx = bvh.ctx
    try:
        for mode, r in want.items():
            for slots, pers in ((4, 2), (0, 1), (1, 0), (-1, 1)):
                ctx.set_option("traverse_slots", slots); ctx.set_option("traverse_persistent", pers)
                for compact in (False, True):
                    off, hits = bvh.traverse_batch(rays, mode=mode, compact=compact)
                    _assert_csr(off, hits, r, fam, f"mode {mode} slots {slots} persistent {pers} compact {compact}")
            ctx.set_option("traverse_slots", -1); ctx.set_option("traverse_persistent", 2)
            dev = torch.device("cuda", 0)
            ctx.set_stream(torch.cuda.current_stream().cuda_stream)
            try:
                d_rays = torch.from_numpy(rays.view(np.uint8).reshape(-1)).to(dev)
                d_off = torch.empty(len(rays) + 1, dtype=torch.int32, device=dev)
                d_hits = torch.empty(len(r.hits) + 16, dtype=torch.int32, device=dev)
                total = bvh.traverse_dev(d_rays.data_ptr(), len(rays), d_off.data_ptr(), d_hits.data_ptr(), d_hits.numel(), mode=mode, want_total=True)
                assert total == len(r.hits)
                _assert_csr(d_off.cpu().numpy().view(np.uint32), d_hits[:total].cpu().numpy().view(np.uint32), r, fam, f"traverse_dev mode {mode}")
            finally:
                ctx.set_stream(None)
            if prec == "f32":
                ctx.set_option("traverse_persistent", 1); ctx.set_option("traverse_stream", 0)
                visits = []
                for top in (0, 1, 64, 500):
                    ctx.set_option("traverse_top", top)
                    off, hits = bvh.traverse_batch(rays, mode=mode)
                    visits.append(bvh.traverse_stats()[0])
                    _assert_csr(off, hits, r, fam, f"mode {mode} traverse_top {top}")
                assert len(set(visits)) == 1, visits
                ctx.set_option("traverse_persistent", 2)
                ctx.set_option("traverse_top", 1); ctx.set_option("traverse_stream", 1)
                reps = 240_000 // len(rays) + 1                  # the host path streams from 240 000 rays up
                big = np.tile(rays, reps)
                for compact in (False, True):
                    off, hits = bvh.traverse_batch(big, mode=mode, compact=compact)
                    assert ctx.get_metric("host_streamed") == 1.0
                    _assert_csr(off, hits, _tiled(r, reps), np.tile(fam, reps), f"streamed mode {mode} compact {compact}")
                ctx.set_option("traverse_top", -1); ctx.set_option("traverse_stream", -1)
    finally:
        ctx.set_option("traverse_slots", -1); ctx.set_option("traverse_persistent", 2)
        ctx.set_option("traverse_top", -1); ctx.set_option("traverse_stream", -1)
        bvh.free()


def _stored_box(nodes, node_index, shape, prec):
    """The child box a leaf's parent stores for it: what the distance-ordered walk slices (src/bvh/distance_traverse.rs:100-116)."""
    leaf = int(node_index[shape])
    p = int(nodes["parent"][leaf])
    side = "l_aabb" if int(nodes["child_l"][p]) == leaf else "r_aabb"
    return np.array([(nodes[side]["min"][p], nodes[side]["max"][p])], dtype=O._DT[prec]["aabb"])


@pytest.mark.parametrize("kind,prec", EDGE)
def test_ordered_traversal(api, kind, prec):
    """traverse_ordered: the set of Bvh::traverse, sorted by the slice of the child box the tree stores for each leaf (the shape's own
    AABB only on tight trees; an empty box on "no split wins" nodes), ties in DFS order, distances bit for bit."""
    shapes, built, rays, fam = _edge_case(kind, prec, per_family=60, seed=1)
    F = O._DT[prec]["f"]
    nodes, node_index = built.nodes, built.node_index
    ref = O.traverse(nodes, shapes, rays, O.MODE_RECURSIVE, prec)
    lists = O.per_ray_lists(ref.offsets, ref.hits)
    bvh = api.Bvh.build(shapes, prec=prec)
    boxes = {int(s): _stored_box(nodes, node_index, int(s), prec) for s in np.unique(ref.hits)}
    empty = sum(1 for b in boxes.values() if b["min"][0][0] > b["max"][0][0])
    assert (empty > 0) == (kind != "subnormal")                 # keys really come from empty stored boxes on no-split trees
    slices = [[O.ray_slice(ray, boxes[int(h)], prec) for h in lst] for ray, lst in zip(rays, lists)]
    assert all(s is not None for sl in slices for s in sl)
    for ascending in (True, False):
        off, hits, dists = bvh.traverse_ordered(rays, ascending)
        assert np.array_equal(off.astype(np.uint64), ref.offsets), ascending
        for i, (lst, sl) in enumerate(zip(lists, slices)):
            key = [s[0] if ascending else -s[1] for s in sl]
            order = sorted(range(len(lst)), key=lambda j: key[j])          # stable: ties keep DFS order
            assert hits[off[i]:off[i + 1]].tolist() == [int(lst[j]) for j in order], (ascending, i, fam[i])
            wd = np.array([sl[j][0] if ascending else sl[j][1] for j in order], dtype=F)
            assert np.array_equal(dists[off[i]:off[i + 1]].view(UINT[prec]), wd.view(UINT[prec])), (ascending, i, fam[i])
    bvh.free()


@pytest.mark.parametrize("kind,prec", EDGE)
def test_closest_hit_aabb_mode(api, kind, prec):
    """closest_hit (AABB mode) == O.closest_hit bit for bit: the shape whose own AABB is entered first among Bvh::traverse's
    candidates, also where empty stored boxes make those candidates a superset of the shapes the ray hits."""
    shapes, built, rays, fam = _edge_case(kind, prec, seed=2)
    ws, wd, _ = O.closest_hit(built.nodes, shapes, rays, prec=prec)
    assert (ws != O.U32_MAX).sum() > len(rays) // 10
    bvh = api.Bvh.build(shapes, prec=prec)
    gs, gd, _ = bvh.closest_hit(rays)
    bad = np.flatnonzero((gs != ws) | (gd.view(UINT[prec]) != wd.view(UINT[prec])))
    assert len(bad) == 0, (len(bad), sorted(set(fam[bad].tolist())), bad[:5].tolist())
    bvh.free()


@pytest.mark.parametrize("kind,prec", EDGE)
def test_query_parity(api, kind, prec):
    """POINT / AABB / BALL queries in BVH and FLAT modes == O.query, with points and query boxes on box corners and with -0.0
    coordinates."""
    from bvh_b200 import capi

    shapes = edge_scene(kind, 2000, prec)
    want = O.build(shapes, prec)
    _assert_tree_preconditions(kind, shapes, want)
    flat = O.flatten(want.nodes, prec)
    bvh = api.Bvh.build(shapes, prec=prec)
    rng = np.random.default_rng(31)
    mn, mx = shapes["min"].astype(np.float64), shapes["max"].astype(np.float64)
    lo, hi = mn.min(axis=0), mx.max(axis=0)
    ext = hi - lo
    n = 3000
    pick = rng.integers(0, len(shapes), n)
    pts = rng.uniform(lo - 0.05 * ext, hi + 0.05 * ext, (n, 3))
    pts[:400] = mn[pick[:400]]                                 # on box corners
    pts[400:800] = mx[pick[400:800]]
    pts[800:1000] = -0.0                                       # the origin as -0.0 / +0.0 and mixed signs
    pts[1000:1200] = 0.0
    pts[1200:1400, 1] = -0.0
    amin = rng.uniform(lo, hi, (n, 3))
    aab = np.concatenate([amin, amin + rng.uniform(0, 0.2, (n, 3)) * ext], axis=1)
    aab[:400] = np.concatenate([mn[pick[:400]], mx[pick[:400]]], axis=1)            # exactly a shape's box
    aab[400:600] = np.concatenate([mx[pick[400:600]], mx[pick[400:600]]], axis=1)   # a shape's max corner as a point box
    aab[600:800, 3:] = -0.0                                                          # max = -0.0 ...
    aab[600:800, :3] = np.minimum(aab[600:800, :3], 0.0)
    aab[800:1000, :3] = -0.0                                                         # ... and min = -0.0
    aab[800:1000, 3:] = np.maximum(aab[800:1000, 3:], 0.0)
    balls = np.concatenate([rng.uniform(lo, hi, (n, 3)), rng.uniform(0, 0.15, (n, 1)) * ext.max()], axis=1)
    balls[:400, :3] = mn[pick[:400]]                                                 # centred on a corner
    balls[400:600] = np.concatenate([np.full((200, 3), -0.0), rng.uniform(0, 0.15, (200, 1)) * ext.max()], axis=1)
    assert np.any(np.signbit(pts) & (pts == 0)) and np.any(np.signbit(aab) & (aab == 0)) and np.any(np.signbit(balls) & (balls == 0))
    balls[600:1500, 3] = rng.uniform(0, 10, 900)                                    # radius**2 finite at every scale
    # Unlike the slab test, contains / overlap with Aabb::empty() is false: a no-split root hides the whole tree from point and box
    # queries in both semantics, although they touch many shapes (a device walk that let an empty box pass would report hits).  A
    # ball passes an empty box exactly when radius**2 overflows to inf (ball.rs:85-99 clamps to inf, then -inf: distance**2 = inf).
    root_hidden = kind != "subnormal"
    if root_hidden:
        r = want.nodes[0]
        assert r["l_aabb"]["min"][0] > r["l_aabb"]["max"][0] and r["r_aabb"]["min"][0] > r["r_aabb"]["max"][0]
    p = pts.astype(shapes["min"].dtype)
    assert np.any(np.all((p[:, None] >= shapes["min"][None]) & (p[:, None] <= shapes["max"][None]), axis=2))   # corner points lie in boxes
    for kind_q, q in ((capi.QUERY_POINT, pts), (capi.QUERY_AABB, aab), (capi.QUERY_BALL, balls)):
        for mode, fl in ((capi.TRAVERSE_BVH, None), (capi.TRAVERSE_FLAT, flat)):
            off, hits = bvh.query_batch(kind_q, q, mode)
            woff, whits = O.query(kind_q, q, want.nodes, shapes, fl, prec)
            assert (len(whits) == 0) == (root_hidden and kind_q != capi.QUERY_BALL), (kind_q, mode, len(whits))
            assert np.array_equal(off.astype(np.uint64), woff) and np.array_equal(hits, whits), (kind_q, mode)
    bvh.free()


# ---- LBVH and LBVH + treelet in f64 -----------------------------------------------------------------------------------------
LBVH_SCENES = ["cubes1", "random2", "random3", "random33", "random257", "random1000", "cubes1000", "points3000", "line700", "skew3000",
               "huge300", "edge:huge", "edge:mixed"]


@pytest.mark.parametrize("mode", [1, 2], ids=["lbvh", "lbvh_treelet"])
@pytest.mark.parametrize("name", LBVH_SCENES)
def test_lbvh_f64_is_a_valid_reference_layout_bvh(api, name, mode):
    """test_gpu_parity's LBVH checks in f64 (Morton quantisation of f64 centroids up to 1e160).  The consistency / tightness check
    is relaxed only for the treelet mode on the overflow-scale scenes, whose SAH-rebuilt treelets store empty child boxes; the
    hit-set comparison with the exact tree only where the exact tree has empty child boxes (different semantics, not a bug)."""
    from bvh_b200 import capi

    edge = name.startswith("edge:")
    if edge:
        shapes = edge_scene(name[5:], 2000, "f64")
        rays, _ = edge_ray_batch(shapes, 300, "f64", seed=8)
    else:
        shapes = scene(name, "f64")
        rays = rays_for(shapes, 2000, "f64", seed=8)
    exact = O.build(shapes, "f64")
    assert (empty_child_boxes(exact.nodes) > 0) == edge                 # f64 at 1e30 ("huge300") has no overflow; 1e160 has
    bvh = api.Bvh.build(shapes, prec="f64", mode=mode)
    nodes, idx = bvh.nodes, bvh.node_index
    n = len(shapes)
    assert len(nodes) == 2 * n - 1
    leaves = nodes["child_l"] == O.U32_MAX
    assert leaves.sum() == n and np.array_equal(np.sort(nodes["shape"][leaves]), np.arange(n))
    assert np.array_equal(nodes["shape"][idx], np.arange(n))
    if mode == capi.BUILD_LBVH_TREELET and n <= 512 and name.startswith("random"):
        assert _nodes_equal(nodes, exact.nodes)
    has_empty = empty_child_boxes(nodes) > 0
    assert has_empty == (edge and mode == capi.BUILD_LBVH_TREELET)
    if not has_empty:
        assert O.is_consistent(nodes, shapes, "f64") and O.is_tight(nodes, "f64")
    again = api.Bvh.from_nodes(nodes, shapes, prec="f64")
    assert np.array_equal(again.node_index, idx)
    again.free()
    assert _flat_equal(bvh.flatten().nodes, O.flatten(nodes, "f64"))
    r = O.traverse(nodes, shapes, rays, O.MODE_RECURSIVE, "f64")
    off, hits = bvh.traverse_batch(rays)
    assert np.array_equal(off.astype(np.uint64), r.offsets) and np.array_equal(hits, r.hits)
    if not edge:
        rr = O.traverse(exact.nodes, shapes, rays, O.MODE_RECURSIVE, "f64")
        for a, b in zip(O.per_ray_lists(r.offsets, r.hits), O.per_ray_lists(rr.offsets, rr.hits)):
            assert sorted(a.tolist()) == sorted(b.tolist())
    bvh.free()


# ---- trees that differ from the oracle's by design ----------------------------------------------------------------------------
def _walks_match_own_nodes(api, bvh, shapes, prec, what, seed):
    """After refit / add / remove on a no-split tree the device's boxes may differ from the reference's (DESIGN §2, header notes of
    bvhgpu_add_shapes_*), so the source of truth is the oracle run on the device's own node array: flatten == O.flatten(nodes),
    CSR (BVH and FLAT; f32 with the shared-memory top walk off and on) == O.traverse of those nodes."""
    from bvh_b200 import capi

    nodes = bvh.nodes
    flat = O.flatten(nodes, prec)
    assert _flat_equal(bvh.flatten().nodes, flat), what
    rays, fam = edge_ray_batch(shapes, 150, prec, seed)
    assert ray_facts(rays, shapes)["nonzero_direction"] == len(rays)
    ctx = bvh.ctx
    for mode, tree, omode in ((capi.TRAVERSE_BVH, nodes, O.MODE_RECURSIVE), (capi.TRAVERSE_FLAT, flat, O.MODE_FLAT)):
        r = O.traverse(tree, shapes, rays, omode, prec)
        for top in ((0, 1) if prec == "f32" else (-1,)):
            ctx.set_option("traverse_top", top)
            try:
                off, hits = bvh.traverse_batch(rays, mode=mode)
            finally:
                ctx.set_option("traverse_top", -1)
            _assert_csr(off, hits, r, fam, f"{what}: mode {mode} top {top}")


def _far_or_near(rng, k, prec):
    """New shapes for add: alternately overflow-scale and unit-scale boxes."""
    s = HUGE[prec]
    mn = np.where((np.arange(k) % 2 == 0)[:, None], rng.uniform(-s, s, (k, 3)), rng.uniform(-50, 50, (k, 3)))
    size = np.where((np.arange(k) % 2 == 0)[:, None], rng.uniform(0, s / 10, (k, 3)), rng.uniform(0.05, 2.0, (k, 3)))
    return O.make_aabbs(mn, mn + size, prec)


@pytest.mark.parametrize("kind,prec", [(k, p) for p in PRECS for k in ("huge", "mixed")])
def test_dynamic_updates_of_no_split_trees(api, kind, prec):
    shapes0 = edge_scene(kind, 2000, prec)
    n = len(shapes0)
    want0 = O.build(shapes0, prec)
    _assert_tree_preconditions(kind, shapes0, want0)
    rng = np.random.default_rng(17)
    # refit after a small motion
    bvh = api.Bvh.build(shapes0, prec=prec)
    moved = shapes0.copy()
    dl = (rng.uniform(-1, 1, (n, 3)) * (np.abs(shapes0["max"].astype(np.float64)) + 1.0) * 1e-3).astype(shapes0["min"].dtype)
    moved["min"] += dl
    moved["max"] += dl
    bvh.refit(moved)
    assert np.array_equal(bvh.nodes[["parent", "child_l", "child_r", "shape"]], want0.nodes[["parent", "child_l", "child_r", "shape"]])
    _walks_match_own_nodes(api, bvh, moved, prec, "refit", 1)
    bvh.free()
    # remove k = 1, 1 %, 30 %: topology == the reference's remove_shape sequence, walks == the oracle on the device's nodes
    for k in (1, n // 100, (30 * n) // 100):
        idx = rng.choice(n, k, replace=False).astype(np.uint32)
        bvh = api.Bvh.build(shapes0, prec=prec)
        bvh.flatten_dev()
        bvh.remove_shapes(idx)
        wn, wi, rest = D.remove_shapes(want0.nodes, want0.node_index, shapes0, idx, prec)
        g = bvh.nodes
        for f in ("parent", "child_l", "child_r", "shape"):
            assert np.array_equal(g[f], wn[f]), (k, f)
        assert np.array_equal(bvh.node_index, wi)
        if k < (30 * n) // 100:
            assert empty_child_boxes(g) > 0, k                       # still a no-split tree
        _walks_match_own_nodes(api, bvh, rest, prec, f"remove {k}", 2 + k)
        bvh.free()
    # 50 single adds (k = 1, no rebuild: the reference's own topology), then one batched add with rebuilds
    bvh = api.Bvh.build(shapes0, prec=prec)
    shapes, nodes, ni = shapes0, want0.nodes, want0.node_index
    for step in range(50):
        new = _far_or_near(rng, 1, prec)
        shapes = np.concatenate([shapes, new])
        assert bvh.add_shapes(new, max_growth=0.0) == 0
        nodes, ni = D.add_shapes(nodes, ni, shapes, 1, prec)
        g = bvh.nodes
        for f in ("parent", "child_l", "child_r", "shape"):
            assert np.array_equal(g[f], nodes[f]), (step, f)
        assert np.array_equal(bvh.node_index, ni), step
    assert empty_child_boxes(bvh.nodes) > 0
    _walks_match_own_nodes(api, bvh, shapes, prec, "50 single adds", 3)
    new = _far_or_near(rng, n // 10, prec)
    shapes = np.concatenate([shapes, new])
    bvh.add_shapes(new, max_growth=1.5)
    assert bvh.num_shapes == len(shapes)
    assert np.array_equal(bvh.nodes["shape"][bvh.node_index], np.arange(len(shapes)))
    assert empty_child_boxes(bvh.nodes) > 0
    _walks_match_own_nodes(api, bvh, shapes, prec, "batched add", 4)
    bvh.free()
