"""Pins tests/rebuildref.py, the restatement of the update step that tests/test_gpu_rebuild_exact.py holds the device to, without a
device: global motion gives Bvh::build, no motion changes nothing, every step keeps the builder's layout and the reference's
invariants, the two builders agree on rebuilt subsets in leaf order, and the scenes of the GPU file contain what that file claims."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import dimcheck, pyref
from tests import rebuildref as RR

PRECS = ("f32", "f64")


def _same(nodes, idx, want_nodes, want_idx):
    assert np.array_equal(idx, want_idx)
    for f in ("parent", "child_l", "child_r", "shape"):
        assert np.array_equal(nodes[f], want_nodes[f]), f
    for side in ("l_aabb", "r_aabb"):
        for mm in ("min", "max"):
            assert np.array_equal(nodes[side][mm], want_nodes[side][mm]), (side, mm)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("D", [2, 3, 4])
def test_global_motion_rebuilds_the_root_into_build(D, prec):
    rng = np.random.default_rng(D)
    n = 3000 if D == 3 else 1200
    a = RR.random_scene(n, D, prec, rng)
    t = RR.Tree(*RR.build(a, prec))
    g = a.copy()
    g["min"] = (a["min"].astype(np.float64) * 3 + 50).astype(a["min"].dtype)
    g["max"] = g["min"] + (a["max"] - a["min"])
    idx = np.arange(n, dtype=np.uint32)
    rebuilt = t.optimize(g, 1.5) if D == 3 else t.update(idx, g, 1.5)
    assert rebuilt == n and [r["root"] for r in t.facts["roots"]] == [0]
    _same(t.nodes, t.node_index, *RR.build(g, prec))


@pytest.mark.parametrize("D", [2, 3, 4])
def test_no_motion_rebuilds_nothing_and_max_growth_0_only_climbs(D):
    rng = np.random.default_rng(10 + D)
    a = RR.random_scene(2000, D, "f32", rng)
    nodes, idx = RR.build(a, "f32")
    t = RR.Tree(nodes, idx)
    assert t.update(np.arange(0, 2000, 3), a, 1.5) == 0
    if D == 3:
        assert t.optimize(a, 1.5) == 0
    assert t.nodes.tobytes() == nodes.tobytes() and np.array_equal(t.node_index, idx)
    changed = np.sort(rng.choice(2000, 200, replace=False))
    b = RR.jitter(a, changed, 60.0, rng)
    assert t.update(changed, b, 0.0) == 0 and t.facts["roots"] == []
    for f in ("parent", "child_l", "child_r", "shape"):
        assert np.array_equal(t.nodes[f], nodes[f])
    assert dimcheck.is_consistent(t.nodes, b) and dimcheck.is_tight(t.nodes)
    assert t.nodes.tobytes() != nodes.tobytes()


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("D,scene", [(2, "random"), (3, "random"), (4, "random"), (3, "clusters"), (3, "mixed"), (4, "overflow")])
def test_every_restated_step_keeps_the_layout_and_the_invariants(D, scene, prec):
    rng = np.random.default_rng(len(scene) + D)
    if scene == "mixed":
        from tests.edge_inputs import edge_scene

        a = np.ascontiguousarray(edge_scene("mixed", 2000, prec), dtype=RR.aabb_dtype(3, prec))
    elif scene == "overflow":
        from tests import dimref

        a = RR.make_boxes(*dimref.scene("overflow", 1500, 4, RR._F(prec), rng), 4, prec)
    elif scene == "clusters":
        a = RR.clustered_scene(3000, D, prec, rng)
    else:
        a = RR.random_scene(3000 if D == 3 else 1500, D, prec, rng)
    no_split = scene in ("mixed", "overflow")                # "no split wins" nodes: empty child boxes, neither consistent nor tight
    t = RR.Tree(*RR.build(a, prec))
    for frame in range(6):
        changed, a = RR.mixed_motion(a, rng, regions=(200, 40), singles=20) if not no_split else \
            (lambda c: (c, RR.jitter(a, c, float(np.median((a["max"] - a["min"]).astype(np.float64))) * 3, rng)))(
                np.sort(rng.choice(len(a), 60, replace=False)))
        mg = (1.5, 1.0, 0.0, 1e30, 1.5, 1.5)[frame]
        rebuilt = t.optimize(a, max(mg, 1.0)) if D == 3 and frame % 2 else t.update(changed, a, mg)
        assert rebuilt == sum(r["count"] for r in t.facts["roots"])
        assert dimcheck.layout_ok(t.nodes, t.node_index)
        if not no_split:
            assert dimcheck.is_consistent(t.nodes, a) and dimcheck.is_tight(t.nodes)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("scene", ["random", "clusters"])
def test_pyref_and_the_oracle_build_rebuilt_subsets_alike(scene, prec):
    """For D = 3 the restatement takes the oracle's build; tests/pyref.py must give the same subtree for every root's shapes in leaf
    order, including subsets of coincident centres, where the halving branch makes the result depend on that order."""
    rng = np.random.default_rng(3)
    a = RR.random_scene(4000, 3, prec, rng) if scene == "random" else RR.clustered_scene(4000, 3, prec, rng)
    t = RR.Tree(*RR.build(a, prec))
    changed, a = RR.mixed_motion(a, rng, regions=(300, 40), singles=20)
    assert t.update(changed, a, 1.5) > 50
    if scene == "clusters":
        assert RR.halving_pairs(t.nodes, a, t.facts["roots"]) > 0
    F = RR._F(prec)
    for ro in t.facts["roots"]:
        r, k = ro["root"], ro["count"]
        rng_ = np.arange(r, r + 2 * k - 1)
        order = t.nodes["shape"][rng_[t.nodes["child_l"][rng_] == RR.U32_MAX]].astype(np.int64)
        for sub in (order, order[::-1]):
            want = O.build(np.ascontiguousarray(a[sub], dtype=O._DT[prec]["aabb"]), prec)
            pn, pidx = pyref.build([{"min": x["min"], "max": x["max"]} for x in a[sub]], F)
            got = RR.Tree(np.zeros(len(pn), dtype=RR.node_dtype(3, prec)), np.zeros(len(pidx), np.uint32))
            got._place(0, pn, pidx, np.arange(len(pidx)), 0)
            _same(got.nodes, got.node_index, np.array(want.nodes, dtype=RR.node_dtype(3, prec)), want.node_index)


def test_the_seed_box_enters_the_split_costs():
    """The root box only divides the split costs, yet an empty seed box (SA = inf) makes every finite cost 0 and the first candidate
    win: pyref.build(root_aabb=...) must follow it, or the restated overflow-scale rebuilds would not pin the device's seed."""
    F = np.float32
    rng = np.random.default_rng(1)
    mn = rng.uniform(-50, 50, (64, 3))
    pa = [{"min": [F(v) for v in m], "max": [F(v + 1) for v in m]} for m in mn]
    plain, _ = pyref.build(pa, F)
    seeded, _ = pyref.build(pa, F, root_aabb=([F(np.inf)] * 3, [F(-np.inf)] * 3))
    assert plain != seeded


# ---- the scenes of tests/test_gpu_rebuild_exact.py contain what it claims (the 1.2 M-shape 4-D case asserts its own) ------------
@pytest.mark.parametrize("D,form", [(2, "update"), (3, "optimize"), (3, "update"), (3, "update_dev"), (4, "update"), (4, "update_dev")])
def test_gpu_scene_roots_of_every_size(D, form):
    from tests.test_gpu_rebuild_exact import REGIONS, _assert_root_sizes

    rng = np.random.default_rng(100 * D + len(form))
    n = 8000 if D == 4 else 20000
    a = RR.random_scene(n, D, "f32", rng, w_scale=3.0)
    t = RR.Tree(*RR.build(a, "f32"))
    seen = []
    for call in range(2):
        changed, a = RR.mixed_motion(a, rng, regions=REGIONS[D])
        t.optimize(a, 1.5) if form == "optimize" else t.update(changed, a, 1.5)
        seen.append(t.facts)
    _assert_root_sizes(D, seen)


@pytest.mark.parametrize("D", [2, 3, 4])
def test_gpu_scene_clusters_halve(D):
    from tests.test_gpu_rebuild_exact import FORMS

    rng = np.random.default_rng(D)
    a = RR.clustered_scene(6000, D, "f32", rng)
    t = RR.Tree(*RR.build(a, "f32"))
    for form in FORMS[D]:
        changed, a = RR.mixed_motion(a, rng, regions=(400, 60), singles=30, single_scale=3.0)
        t.optimize(a, 1.5) if form == "optimize" else t.update(changed, a, 1.5)
        assert RR.halving_pairs(t.nodes, a, t.facts["roots"]) > 0


@pytest.mark.parametrize("kind,D,prec", [("huge", 3, "f32"), ("huge", 3, "f64"), ("mixed", 3, "f32"), ("mixed", 3, "f64"), ("overflow", 4, "f32")])
def test_gpu_scene_overflow_frames(kind, D, prec):
    """The mixed scenes reach incremental roots whose seed is not the joint box of their shapes; a full refit never does."""
    from tests.test_gpu_rebuild_exact import overflow_frames

    def step(dev, t, form, changed, b, mg, what):
        t.optimize(b, mg) if form == "optimize" else t.update(changed, b, mg)
        return t.facts

    differs = overflow_frames(kind, D, prec, lambda form, b: (None, RR.Tree(*RR.build(b, prec))), step)
    assert kind != "mixed" or differs > 0
