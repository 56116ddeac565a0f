"""The limited-walk model of tests/crosswalk.py without a GPU, on the oracle's exact-SAH trees of the scenes the device is held to in
tests/test_gpu_crossings_edges.py:
- without a limit it is the loop over the oracle's Bvh::traverse CSR (crossings.counts_csr), and the per-node restatement agrees;
- with a limit (the families around each ray's k-th crossing) it equals the loop on every bounded row, never exceeds it, and the
  per-node restatement agrees on every row;
- positive controls: rows where the limited walk and the loop differ exist (grazing f32, stale triangles in f32 and f64), so a walk
  that ignores its limit when entering children is told apart from the model;
- the analytic scenes meet their closed forms: the layer stack's 2048 / 2048 crossings and j + 1 below a limit, the EVEN_ODD / NONZERO
  truths of overlapping and nested shells, and a 1e-4 icosphere that is invisible in f32 (|det| < eps) and exact in f64."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import crossings as X
from tests import crosswalk as W
from tests.test_crossings_cpu import sphere_points

FT = {"f32": np.float32, "f64": np.float64}


def _tree(tris, prec):
    shapes = O.tri_aabbs(tris, prec)
    return O.build(shapes, prec).nodes, shapes


def _eq(a, b):
    return np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def _differ(a, b):
    return (a[0] != b[0]) | (a[1] != b[1])


def _all_scenes(prec):
    F = FT[prec]
    out = dict(W.triangle_scenes(prec))
    for name, (t, p, _, _) in W.ball_pairs(F, m=100).items():
        out[name] = (t.reshape(-1, 9), X.point_rays(p, F))
    return out


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_model_is_the_loop_without_a_limit_and_bounded_rows_with_one(prec):
    F = FT[prec]
    rng = np.random.default_rng(12)
    report = {}
    for name, (tris, rays) in _all_scenes(prec).items():
        nodes, shapes = _tree(tris, prec)
        cand = W.candidates(nodes, shapes, rays)
        tr = O.traverse(nodes, shapes, rays, O.MODE_RECURSIVE, prec)
        loop = X.counts_csr(rays, tris, tr.offsets, tr.hits)
        got = W.model(nodes, shapes, tris, rays, None, cand)
        assert _eq(got, loop), name
        assert _eq(W.model_preorder(nodes, shapes, tris, rays), loop), name
        unbounded = 0
        for lname, tm in W.kth_limits(rays, tris, cand, rng).items():
            want = X.counts_csr(rays, tris, tr.offsets, tr.hits, tm)
            ok = X.bounded_rows(rays, tris, nodes, shapes, tr.offsets, tr.hits, tm)
            got = W.model(nodes, shapes, tris, rays, tm, cand)
            assert np.array_equal(got[0][ok], want[0][ok]) and np.array_equal(got[1][ok], want[1][ok]), (name, lname)
            assert np.all(got[0] <= want[0]) and np.all(got[1] <= want[1]), (name, lname)
            assert not _differ(got, want)[ok].any(), (name, lname)
            assert _eq(W.unlimited_walk(nodes, shapes, tris, rays, tm, cand), want), (name, lname)
            if lname in ("above", "below", "random", "above_last", "negzero"):
                assert _eq(W.model_preorder(nodes, shapes, tris, rays, tm), got), (name, lname)
            if lname in ("zero", "negzero", "negative", "nan", "subnormal"):
                assert not got[0].any() and not got[1].any(), (name, lname)
            if lname in ("inf", "max_finite"):
                assert _eq(got, loop), (name, lname)
            unbounded += int((~ok).sum())
        report[name] = (int(loop[0].sum()), int(loop[1].sum()), unbounded)
    print(prec, "scene: (front, back, unbounded rows over the limits)", report)


def test_grazing_f32_has_rows_the_limit_decides():
    """The grazing family in f32 with the limit just above each ray's last crossing: the limited walk misses the grazing triangle B,
    entered only at fl(d_B * (1 + 2^-16)) < its box entry, on at least 40 rows; the loop (and a walk that ignores the limit when
    entering children) counts it.  In f64 the same limits leave every row bounded."""
    for prec, least in (("f32", 40), ("f64", 0)):
        tris, rays = W.triangle_scenes(prec)["grazing"]
        nodes, shapes = _tree(tris, prec)
        cand = W.candidates(nodes, shapes, rays)
        tm = W.kth_limits(rays, tris, cand, np.random.default_rng(0))["above_last"]
        got = W.model(nodes, shapes, tris, rays, tm, cand)
        mutant = W.unlimited_walk(nodes, shapes, tris, rays, tm, cand)
        diff = _differ(got, mutant)
        print(prec, "grazing rows the limit decides:", int(diff.sum()), "of", len(rays))
        if least:
            assert diff.sum() >= least
            assert np.all((got[0].astype(np.int64) + got[1])[diff] < (mutant[0].astype(np.int64) + mutant[1])[diff])
        else:
            assert not diff.any()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_stale_triangles_have_rows_the_limit_decides(prec):
    F = FT[prec]
    tris, own, moved, rays = W.stale(F)
    nodes = O.build(moved, prec).nodes
    cand = W.candidates(nodes, moved, rays)
    fam = W.kth_limits(rays, tris, cand, np.random.default_rng(3))
    for lname in ("above_last", "above", "random"):
        tm = fam[lname]
        got = W.model(nodes, moved, tris, rays, tm, cand)
        mutant = W.unlimited_walk(nodes, moved, tris, rays, tm, cand)
        diff = _differ(got, mutant)
        assert diff.sum() >= 100, lname
        assert np.all((got[0] <= mutant[0]) & (got[1] <= mutant[1])), lname
        assert _eq(W.model_preorder(nodes, moved, tris, rays, tm), got), lname
    # without a limit the moved boxes only change which triangles are candidates
    loop = W.unlimited_walk(nodes, moved, tris, rays, None, cand)
    assert _eq(W.model(nodes, moved, tris, rays, None, cand), loop) and loop[0].sum() + loop[1].sum() > len(rays) // 2


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_layer_stack_counts_are_closed_form(prec):
    F = FT[prec]
    tris, rays, _ = W.layer_stack(F)
    nodes, shapes = _tree(tris, prec)
    cand = W.candidates(nodes, shapes, rays)
    f, b = W.model(nodes, shapes, tris, rays, None, cand)
    assert np.all(f == W.LAYERS // 2) and np.all(b == W.LAYERS // 2)
    assert _eq((f, b), X.counts_brute(rays, tris))
    j = np.random.default_rng(2).integers(0, W.LAYERS, len(rays))
    j[:4] = [0, 1, W.LAYERS - 2, W.LAYERS - 1]
    f, b = W.model(nodes, shapes, tris, rays, W.layer_limits(rays, j), cand)
    assert np.array_equal(f.astype(np.int64) + b, j + 1)
    assert np.array_equal(b.astype(np.int64) - f, (j + 2) // 2 - (j + 1) // 2)     # layers 0, 2, ... through the back face


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_shell_truths_under_both_rules(prec):
    F = FT[prec]
    for name, (t, p, eo, nz) in W.ball_pairs(F, m=1500).items():
        nodes, shapes = _tree(t.reshape(-1, 9), prec)
        assert eo.sum() > 100 and (~eo).sum() > 100, name
        assert np.array_equal(eo, nz) == (name == "nested_flipped"), name
        for rule, truth in ((X.EVEN_ODD, eo), (X.NONZERO, nz)):
            got = W.contains_model(nodes, shapes, t.reshape(-1, 9), p, rule)
            assert np.array_equal(got, truth), (name, rule, int((got != truth).sum()))


def test_tiny_icosphere_is_invisible_in_f32_only():
    rng = np.random.default_rng(4)
    p, truth = sphere_points(rng, 2000)
    for prec in ("f32", "f64"):
        F = FT[prec]
        t = (X.icosphere(3, np.float64) * 1e-4).astype(F).reshape(-1, 9)
        nodes, shapes = _tree(t, prec)
        for rule in (X.EVEN_ODD, X.NONZERO):
            got = W.contains_model(nodes, shapes, t, (p * 1e-4).astype(F), rule)
            if prec == "f32":
                assert not got.any()
            else:
                assert np.array_equal(got, truth)


def test_model_on_root_leaf_and_empty_trees():
    for prec in ("f32", "f64"):
        F = FT[prec]
        one = np.array([[0, 0, 0, 1, 0, 0, 0, 1, 0]], dtype=F)
        rays = O.ray_new(np.array([[0.25, 0.25, 2], [0.25, 0.25, -2], [5, 5, 2]]), np.array([[0, 0, -1], [0, 0, 1], [0, 0, -1]]), prec)
        nodes, shapes = _tree(one, prec)
        for tm in (None, F(0.5), F(3)):
            got = W.model(nodes, shapes, one, rays, tm)
            assert _eq(got, W.model_preorder(nodes, shapes, one, rays, tm))
            assert got[0].tolist() == [0 if tm == F(0.5) else 1, 0, 0] and got[1].tolist() == [0, 0 if tm == F(0.5) else 1, 0]
        nodes, shapes = _tree(one[:0], prec)
        assert not any(x.any() for x in W.model(nodes, shapes, one[:0], rays))


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_mixed_edge_scene_counts_below_empty_child_boxes(prec):
    """The huge and mixed edge trees store Aabb::empty() child boxes ("no split wins"); the slab test passes on them, and on the mixed
    scene counted triangles lie below them, so a walk that skipped boxes with min > max would count less there."""
    from tests import edge_dims as ED

    scenes = W.triangle_scenes(prec)
    for kind in ED.SCENE_KINDS:
        tris, rays = scenes[f"edge_{kind}"]
        nodes, shapes = _tree(tris, prec)
        got = W.model(nodes, shapes, tris, rays)
        skip = W.model(nodes, shapes, tris, rays, skip_empty=True)
        assert (ED.empty_child_boxes(nodes) > 0) == (kind != "subnormal"), kind
        assert _differ(got, skip).any() == (kind == "mixed"), kind
        assert (got[0].sum() + got[1].sum() > 0) == (kind == "mixed"), kind
