"""CPU checks of the edge-case inputs (tests/edge_inputs.py) before any GPU result is compared with them:
- each scene and each ray family contains what it claims (no-split nodes, degenerate splits, -0.0 components, inv = -inf, subnormal
  directions, overflowing slab products), so the GPU tests cannot quietly turn into point-in-box tests;
- the C++ oracle equals the independent numpy-scalar restatement (tests/pyref.py) on these inputs, node for node and hit list for
  hit list, so "GPU == oracle" means "GPU == the reference's arithmetic"."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import pyref
from tests.edge_inputs import FAMILIES, SCENE_KINDS, edge_ray_batch, edge_scene, empty_child_boxes, ray_facts

PRECS = ("f32", "f64")
FT = {"f32": np.float32, "f64": np.float64}


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("kind", SCENE_KINDS)
def test_scene_preconditions(kind, prec):
    n = 400
    s = edge_scene(kind, n, prec)
    F = FT[prec]
    c = s["min"] * F(0.5) + s["max"] * F(0.5)
    assert np.all(np.isfinite(c.max(axis=0) - c.min(axis=0)))                 # centroid extents stay finite (no NaN bucket)
    b = O.build(s, prec)
    if kind in ("huge", "mixed"):
        assert b.nosplit_fallthrough > 0
        assert empty_child_boxes(b.nodes) == b.nosplit_fallthrough           # each such node stores Aabb::empty() children
        assert not O.is_tight(b.nodes, prec)
    if kind == "mixed":                                                       # ordinary SAH splits below the no-split top
        assert b.nosplit_fallthrough + b.degenerate_splits < n - 1
    if kind == "subnormal":
        tiny = np.finfo(F).tiny
        assert np.all(np.abs(s["min"]) < tiny) and np.all(np.abs(s["max"]) < tiny) and np.any(s["max"] != 0)
        assert b.degenerate_splits == n - 1 and b.nosplit_fallthrough == 0    # every inner node halves
        assert O.is_tight(b.nodes, prec)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("kind", SCENE_KINDS)
def test_ray_family_preconditions(kind, prec):
    s = edge_scene(kind, 400, prec)
    rays, fam = edge_ray_batch(s, 200, prec)
    F = FT[prec]
    assert np.all(np.isfinite(rays["direction"])) and np.all(np.isfinite(rays["origin"]))
    b = O.build(s, prec)
    counts = np.diff(O.traverse(b.nodes, s, rays, O.MODE_RECURSIVE, prec).offsets.astype(np.int64))
    for f in FAMILIES:
        m = fam == f
        facts = ray_facts(rays[m], s)
        assert facts["nonzero_direction"] == m.sum(), f                       # no zero-direction (point-in-box) rays
        assert counts[m].sum() > 0, f
        if f in ("axis", "face"):
            assert facts["neg_zero"] > 0 and facts["pos_zero"] > 0 and facts["inv_neg_inf"] > 0 and facts["inv_pos_inf"] > 0, (f, facts)
        if f == "face":
            assert facts["face_plane_nan"] > 0, facts
        if f == "inside":
            o = rays["origin"][m]
            inside = np.any(np.all((o[:, None, :] >= s["min"][None]) & (o[:, None, :] <= s["max"][None]), axis=2), axis=1)
            assert inside.all()
        if f == "tiny" and kind != "subnormal":
            assert facts["overflowing_products"] > 0, facts
        if f == "subdir":
            assert facts["subnormal_dir_finite_inv"] > 0 and facts["subnormal_dir_inf_inv"] > 0, facts
            d, inv = rays["direction"][m], rays["inv_direction"][m]
            sub = (d != 0) & (np.abs(d) < np.finfo(F).tiny)
            assert np.all(np.abs(inv[sub & np.isfinite(inv)]) > np.finfo(F).max / 4)
        if kind == "subnormal":
            assert facts["subnormal_differences"] > 0, f


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("kind", ["huge", "mixed"])
def test_bvh_and_flat_semantics_differ_on_no_split_trees(kind, prec):
    """An empty child box passes the slab test for every ray; only FlatBvh::traverse re-tests the shape, so the two hit lists differ."""
    s = edge_scene(kind, 400, prec)
    b = O.build(s, prec)
    rays, _ = edge_ray_batch(s, 100, prec)
    rr = O.traverse(b.nodes, s, rays, O.MODE_RECURSIVE, prec)
    rf = O.traverse(O.flatten(b.nodes, prec), s, rays, O.MODE_FLAT, prec)
    assert len(rr.hits) > len(rf.hits) > 0


def _assert_nodes_equal_pyref(nodes, index, want_nodes, want_index, F):
    assert list(index) == list(want_index)
    assert len(nodes) == len(want_nodes)
    for i, w in enumerate(want_nodes):
        if w[0] == "leaf":
            assert (nodes["parent"][i], nodes["child_l"][i], nodes["child_r"][i], nodes["shape"][i]) == (w[1], O.U32_MAX, O.U32_MAX, w[2]), i
        else:
            assert (nodes["parent"][i], nodes["child_l"][i], nodes["child_r"][i]) == (w[1], w[2], w[3]), i
            for side, box in (("l_aabb", w[4]), ("r_aabb", w[5])):
                assert np.array_equal(nodes[side]["min"][i], np.array(box[0], dtype=F)), (i, side)
                assert np.array_equal(nodes[side]["max"][i], np.array(box[1], dtype=F)), (i, side)


@pytest.mark.parametrize("n", [64, 400])
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("kind", SCENE_KINDS)
def test_oracle_build_and_flatten_equal_pyref(kind, prec, n):
    F = FT[prec]
    s = edge_scene(kind, n, prec)
    b = O.build(s, prec)
    want_nodes, want_index = pyref.build(s, F)
    _assert_nodes_equal_pyref(b.nodes, b.node_index, want_nodes, want_index, F)
    flat, wflat = O.flatten(b.nodes, prec), pyref.flatten(want_nodes)
    assert len(flat) == len(wflat)
    for i, (box, entry, exit_, shape) in enumerate(wflat):
        assert (flat["entry_index"][i], flat["exit_index"][i], flat["shape_index"][i]) == (entry, exit_, shape), i
        if box is not None:
            assert np.array_equal(flat["aabb"]["min"][i], np.array(box[0], dtype=F)) and np.array_equal(flat["aabb"]["max"][i], np.array(box[1], dtype=F))


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("kind", SCENE_KINDS)
def test_oracle_traversal_equals_pyref(kind, prec):
    """Both reference semantics on every ray family: O.traverse MODE_RECURSIVE == pyref.traverse_recursive (Bvh::traverse) and
    O.traverse MODE_FLAT == pyref.traverse_flat (FlatBvh::traverse), hit list for hit list."""
    F = FT[prec]
    s = edge_scene(kind, 400, prec)
    b = O.build(s, prec)
    rays, fam = edge_ray_batch(s, 40, prec, seed=3)
    r = O.traverse(b.nodes, s, rays, O.MODE_RECURSIVE, prec)
    rr = O.per_ray_lists(r.offsets, r.hits)
    r = O.traverse(O.flatten(b.nodes, prec), s, rays, O.MODE_FLAT, prec)
    rf = O.per_ray_lists(r.offsets, r.hits)
    want_nodes, _ = pyref.build(s, F)
    wflat = pyref.flatten(want_nodes)
    for i, r in enumerate(rays):
        ray = ([F(v) for v in r["origin"]], [F(v) for v in r["inv_direction"]])
        assert rr[i].tolist() == pyref.traverse_recursive(want_nodes, s, ray, F), (i, fam[i])
        assert rf[i].tolist() == pyref.traverse_flat(wflat, s, ray, F), (i, fam[i])
