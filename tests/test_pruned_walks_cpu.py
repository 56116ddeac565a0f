"""CPU side of the distance-pruned walks: tests/exactref.py and tests/prunedmodel.py pinned to the C++ oracle on benign inputs, and
proof that every adversarial family of tests/adversarial.py reaches the case it is meant to reach."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import adversarial as A, dimref, exactref as E, prunedcheck as PC, prunedmodel as M, pyref

FT = {"f32": np.float32, "f64": np.float64}


def _rel(a, b):
    a, b = E.fr(a), E.fr(b) if not isinstance(b, type(E.fr(0))) else b
    return abs(a - b) / max(abs(b), E.fr(1e-300))


def nodes_dim(shapes, F):
    """pyref.build's tree (the reference's build in any dimension) as a structured node array in the C-ABI field names."""
    D = shapes["min"].shape[1]
    tree, _ = pyref.build(shapes, F)
    box = np.dtype([("min", F, (D,)), ("max", F, (D,))])
    out = np.zeros(len(tree), dtype=[("parent", "<u4"), ("child_l", "<u4"), ("child_r", "<u4"), ("shape", "<u4"), ("l_aabb", box), ("r_aabb", box)])
    for i, nd in enumerate(tree):
        out[i]["parent"] = nd[1] if nd[1] is not None else M.U32_MAX
        if nd[0] == "leaf":
            out[i]["child_l"] = out[i]["child_r"] = M.U32_MAX
            out[i]["shape"] = nd[2]
            for s in ("l_aabb", "r_aabb"):
                out[i][s]["min"], out[i][s]["max"] = np.inf, -np.inf
        else:
            out[i]["child_l"], out[i]["child_r"] = nd[2], nd[3]
            (out[i]["l_aabb"]["min"], out[i]["l_aabb"]["max"]), (out[i]["r_aabb"]["min"], out[i]["r_aabb"]["max"]) = nd[4], nd[5]
    return out


def shapes_dim(mn, mx):
    F = mn.dtype.type
    a = np.zeros(len(mn), dtype=[("min", F, (mn.shape[1],)), ("max", F, (mn.shape[1],))])
    a["min"], a["max"] = mn, mx
    return a


def tree_for(mn, mx, prec):
    """(nodes, shapes) of a box scene: the oracle's build in 3-D, pyref's in 2-D and 4-D."""
    shapes = shapes_dim(mn, mx)
    if mn.shape[1] == 3:
        shapes = O.make_aabbs(mn, mx, prec)
        return O.build(shapes, prec).nodes, shapes
    return nodes_dim(shapes, FT[prec]), shapes


# ---- exactref against the oracle on benign inputs -------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_exactref_agrees_with_oracle_on_benign_inputs(prec):
    F = FT[prec]
    ulp = float(np.finfo(F).eps)
    shapes, tris = O.create_n_cubes(40, prec=prec, want_tris=True)
    tris = tris.reshape(-1, 9)
    rng = np.random.default_rng(1)
    hits = 0
    for k in rng.choice(len(tris), 120, replace=False):
        tri = tris[k].reshape(3, 3).astype(np.float64)
        tgt = tri.T @ rng.dirichlet([2, 2, 2])
        org = tgt + rng.normal(size=3) * 50
        ray = O.ray_new(org, tgt - org, prec)[0]
        t, u, v = O.ray_triangle(ray, tris[k], prec)
        ex = E.ray_triangle(ray["origin"], ray["direction"], *tris[k].reshape(3, 3))
        assert np.isfinite(t) == (ex is not None and ex[0] > 0)
        if np.isfinite(t):
            hits += 1
            assert _rel(t, ex[0]) < 64 * ulp                      # u and v cancel in o - a: looser
            assert abs(E.fr(u) - ex[1]) < 4096 * ulp and abs(E.fr(v) - ex[2]) < 4096 * ulp
        sl = O.ray_slice(ray, shapes[k], prec)
        es = E.slab_entry(ray["origin"], ray["direction"], shapes["min"][k], shapes["max"][k])
        assert (sl is None) == (es is None)
        if sl is not None:
            assert abs(E.fr(max(sl[0], F(0))) - es[0]) <= 8 * ulp * max(abs(es[0]), 1)
    assert hits > 40                                            # the rest are back faces
    pts = rng.uniform(-1.2e5, 1.2e5, (20, 3)).astype(F)
    for p in pts:
        for kind in (O.DIST_AABB, O.DIST_TRIANGLE):
            d2 = O.shape_distances_squared(shapes, p, prec, kind=kind, tris=tris)
            for j in range(0, len(shapes), 37):
                ex = E.box_lower_d2(p, shapes["min"][j], shapes["max"][j]) if kind == O.DIST_AABB else E.point_triangle_d2(p, *tris[j].reshape(3, 3))
                assert _rel(d2[j], ex) < 1e3 * ulp
                assert E.box_far_d2(p, shapes["min"][j], shapes["max"][j]) >= ex
    for D in (2, 4):                                            # the box distance in other dimensions, against dimref
        mn = rng.uniform(-100, 100, (30, D)).astype(F)
        mx = (mn + rng.uniform(0, 10, (30, D))).astype(F)
        p = rng.uniform(-120, 120, D).astype(F)
        for a, b in zip(mn, mx):
            assert _rel(dimref.min_distance_sq(list(p), list(a), list(b)), E.box_lower_d2(p, a, b)) < 64 * ulp or E.box_lower_d2(p, a, b) == 0
        tri = rng.uniform(-10, 10, (3, D)).astype(F)
        assert E.point_triangle_d2(p, *tri) <= min(E.box_lower_d2(p, v, v) for v in tri)


def test_exactref_edges():
    """Back faces, rays in the triangle's plane and zero direction components, in exact arithmetic."""
    a, b, c = [0.0, 0, 0], [1.0, 0, 0], [0.0, 1, 0]
    assert E.ray_triangle([0.25, 0.25, 1], [0, 0, -1.0], a, b, c) == (1, 0.25, 0.25)
    assert E.ray_triangle([0.25, 0.25, 1], [0, 0, -1.0], a, c, b) is None          # back face
    assert E.ray_triangle([-1, 0.25, 0], [1.0, 0, 0], a, b, c) is None             # in the plane: det = 0
    assert E.ray_triangle([0.5, 0.5, 1], [0, 0, -1.0], a, b, c)[1:] == (0.5, 0.5)  # on the edge u + v = 1
    assert E.slab_entry([0, 0.5, 0.5], [1.0, 0, 0], [1, 0, 0], [2, 1, 1]) == (1, 2)
    assert E.slab_entry([0, 1.5, 0.5], [1.0, 0, 0], [1, 0, 0], [2, 1, 1]) is None
    assert E.point_triangle_d2([0, 0, 1], a, a, a) == 1 and E.point_triangle_d2([2, 0, 0], a, b, [0.5, 0, 0]) == 1


# ---- the model against the oracle on benign inputs ------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_model_agrees_with_oracle_on_benign_inputs(prec):
    """Moeller-Trumbore and the slab entry of the model are the oracle's bit for bit; on a cube scene the pruned walk gives the
    oracle's closest triangle (the contract holds where it does not), and the candidate lists hold the oracle's nearest shape."""
    F = FT[prec]
    shapes, tris = O.create_n_cubes(60, prec=prec, want_tris=True)
    tris = tris.reshape(-1, 9)
    rng = np.random.default_rng(2)
    centres = (shapes["min"][::12].astype(np.float64) + shapes["max"][::12]) / 2
    tgt = centres[rng.integers(0, len(centres), 300)] + rng.uniform(-0.4, 0.4, (300, 3))
    org = tgt + rng.normal(size=(300, 3)) * 3000
    rays = O.ray_new(org, tgt - org, prec)
    for r in range(0, 300, 7):
        for k in rng.integers(0, len(tris), 5):
            mt = M.moeller_trumbore(list(rays["origin"][r]), list(rays["direction"][r]), *tris[k].reshape(3, 3))
            assert np.array(mt, dtype=F).tobytes() == np.array(O.ray_triangle(rays[r], tris[k], prec), dtype=F).tobytes()
            sl, ms = O.ray_slice(rays[r], shapes[k], prec), M.slice_entry(rays["origin"][r], rays["inv_direction"][r], shapes["min"][k], shapes["max"][k])
            assert (sl is not None) == ms[0] and (sl is None or max(sl[0], F(0)) == ms[1])
    b = O.build(shapes, prec)
    ws, wd, wuv = O.closest_hit(b.nodes, shapes, rays, tris, prec)
    ms, md, muv = M.closest_triangles(b.nodes, shapes, tris, rays)
    assert (ws != O.U32_MAX).sum() > 100
    assert PC.check_closest(ms, md, muv, ws, wd, tris, shapes, rays, prec) <= 1
    pts = np.concatenate([centres[:20] + rng.normal(size=(20, 3)) * 30, rng.uniform(-1e5, 1e5, (10, 3))]).astype(F)
    tree = M.Tree(b.nodes, shapes)
    ws, _ = O.nearest_to(b.nodes, shapes, pts, prec)
    for i, p in enumerate(pts):
        lst = tree.candidates(list(p))
        assert int(ws[i]) in lst and len(lst) < 50
        assert lst == tree.candidates(list(p), slack=False) or set(tree.candidates(list(p), slack=False)) <= set(lst)


# ---- every family reaches its case ------------------------------------------------------------------------------------------------
def test_grazing_family_breaks_the_old_tolerance():
    """f32 grazing hits with a blocker: the pruned walk (the model) and the unpruned loop disagree, by far more than the 2e-5 the
    triangle mode used to state, and every disagreement satisfies the contract."""
    tris, o, d, ratio = A.grazing(np.float32)
    assert (ratio > float(A.MARGIN) * (1 + 1e-4)).sum() >= 20
    rays = O.ray_new(o, d, "f32")
    shapes = O.tri_aabbs(tris, "f32")
    nodes = O.build(shapes, "f32").nodes
    ws, wd, wuv = O.closest_hit(nodes, shapes, rays, tris, "f32")
    ms, md, muv = M.closest_triangles(nodes, shapes, tris, rays)
    diff = ms != ws
    assert diff.sum() >= 20
    assert np.max(np.abs(md[diff].astype(np.float64) - wd[diff]) / wd[diff]) > 1e-2
    PC.check_closest(ms, md, muv, ws, wd, tris, shapes, rays, "f32")


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("family", ["shared", "degenerate", "offset"])
def test_triangle_families_on_the_model(family, prec):
    """Each family yields hits, and its own case: ties between neighbours (shared), misses by det = 0 / back face / t <= eps and
    zero-area triangles (degenerate), or coordinates where an ulp is large (offset); the contract holds on all of them."""
    F = FT[prec]
    if family == "shared":
        tris, o, d = A.shared_edges(F)
    elif family == "degenerate":
        tris, o, d = A.degenerate(F)
    else:
        tris, o, d = A.offset_scene(F, 1e6 if prec == "f32" else 1e13)
    rays = O.ray_new(o, d, prec)
    shapes = O.tri_aabbs(tris, prec)
    nodes = O.build(shapes, prec).nodes
    ws, wd, wuv = O.closest_hit(nodes, shapes, rays, tris, prec)
    ms, md, muv = M.closest_triangles(nodes, shapes, tris, rays)
    assert (ws != O.U32_MAX).sum() > len(rays) // 5
    PC.check_closest(ms, md, muv, ws, wd, tris, shapes, rays, prec)
    if family == "shared":                    # rays aimed at shared vertices / edges hit several triangles at one distance
        nt = 0
        for r in range(len(rays)):
            ts = [O.ray_triangle(rays[r], t, prec)[0] for t in tris]
            best = min(ts)
            nt += np.isfinite(best) and sum(t == best for t in ts) > 1
        assert nt >= 10
    if family == "degenerate":
        hits = set(ws[ws != O.U32_MAX].tolist())
        assert hits and all(k % 5 == 0 for k in hits)   # only the plain front faces are hit: not back faces, slivers or zero area


def test_issue_example_excluded_by_the_old_bound():
    """The concrete 3-D f32 case: under the reference's rounded distance box X is the nearest shape, but the bound without slack
    leaves it out of the list; the bound with slack lists it."""
    mn = np.array([A.ISSUE_X[0], np.array(A.ISSUE_P) + [0.5, 0, 0.5]], dtype=np.float32)
    mx = np.array([A.ISSUE_X[1], np.array(A.ISSUE_P) + [0.5, 0, 0.5]], dtype=np.float32)
    p = np.array(A.ISSUE_P, dtype=np.float32)
    shapes = O.make_aabbs(mn, mx)
    d2 = O.shape_distances_squared(shapes, p)
    assert d2[0] == 0.25 and d2[1] == 0.5
    assert E.box_lower_d2(p, mn[0], mx[0]) == 1
    nodes = O.build(shapes).nodes
    tree = M.Tree(nodes, shapes)
    assert tree.candidates(list(p), slack=False) == [1]
    assert sorted(tree.candidates(list(p))) == [0, 1]


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("D", [2, 3, 4])
@pytest.mark.parametrize("family", sorted(A.BOX_FAMILIES))
def test_box_families_on_the_model(family, D, prec):
    """The model's candidate lists meet the contract on every family; each family shows its case: the reference's rounding picks
    a shape that is not an exact nearest (large), ties at the minimal exact distance (ties), subnormal extents (mixed), U = inf and
    every shape listed (overflow).  In 3-D f32 the old bound loses the reference's nearest shape on the large family."""
    F = FT[prec]
    mn, mx, pts = A.BOX_FAMILIES[family](F, D)
    nodes, shapes = tree_for(mn, mx, prec)
    tree = M.Tree(nodes, shapes)
    lists = [tree.candidates(list(p)) for p in pts]
    ties, rounded = PC.check_candidates(lists, nodes, shapes, pts, prec)
    if family == "large" and prec == "f32" and D == 3:
        assert rounded > 0
        old = [tree.candidates(list(p), slack=False) for p in pts]
        with pytest.raises(AssertionError):
            PC.check_candidates(old, nodes, shapes, pts, prec)
    if family == "ties":
        assert ties > 5
    if family == "mixed":
        assert np.any((mx - mn > 0) & (mx - mn < np.finfo(F).tiny))
    if family == "overflow":
        assert all(sorted(lst) == list(range(len(mn))) for lst in lists)
    sizes = [len(lst) for lst in lists]
    if family in ("large", "mixed"):
        assert np.mean(sizes) < len(mn) / 2, np.mean(sizes)
