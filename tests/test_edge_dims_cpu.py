"""CPU checks of the edge inputs in every dimension (tests/edge_dims.py) before any GPU result is compared with them:
- each (scene, family, D, prec) reaches its case: "no split wins" trees with empty stored child boxes in f32 and f64, subnormal
  coordinates, -0.0 components and inv = +-inf on every axis, slab products (b - o) * inv that overflow, subnormal directions with a
  finite and an infinite inverse, slab entries that are exactly -0 before the clamp, knn keys that are exactly 0, a few subnormal steps
  and +inf, radii whose r * r overflows, underflows or rounds up onto a key, and limits at 0, -0, the smallest subnormal, +inf and each
  ray's own entry and exit;
- at D = 3 the dimension-generic restatements equal the C++ oracle on these inputs: dimorder (ordered and closest, through O.traverse,
  O.ray_slice and O.closest_hit), anyhit.aabb and multihit.aabb (through O.closest_hit and O.traverse), knnref (keys through
  O.shape_distances_squared, the walk equal to the brute force on the oracle's tree), dimref.nearest (O.nearest_to, BVH and FLAT), the
  triangle keys of knntri and prunedmodel.moeller_trumbore (O.shape_distances_squared and O.ray_triangle) on the edge triangles.
That makes them the oracles of tests/test_gpu_edge_dims.py at these scales."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import oracle as O
from tests import anyhit as H, dimorder, dimref, edge_dims as ED, knnref as K, knntri as KT, multihit as MH, prunedcheck as PC, prunedmodel as M
from tests.edge_inputs import FAMILIES
from tests.test_pruned_walks_cpu import tree_for

FT = ED.FT
UINT = {np.float32: np.uint32, np.float64: np.uint64}
CASES = [(kind, D, prec) for kind in ED.SCENE_KINDS for D in ED.DIMS for prec in ED.PRECS]


def _bits(a):
    a = np.ascontiguousarray(np.asarray(a))
    return a.view(UINT[a.dtype.type])


def _fb(x, F):
    return np.array([x], dtype=F).view(UINT[F])[0]


def _shapes3(mn, mx, prec):
    return O.make_aabbs(mn, mx, prec)


def _rays3(o, d, inv, prec):
    r = np.zeros(len(o), dtype=O._DT[prec]["ray"])
    r["origin"], r["direction"], r["inv_direction"] = o, d, inv
    return r


@pytest.mark.parametrize("kind,D,prec", CASES)
def test_scene_preconditions(kind, D, prec):
    F = FT[prec]
    mn, mx = ED.scene(kind, 300, D, prec)
    c = mn * F(0.5) + mx * F(0.5)
    assert np.all(np.isfinite(c.max(axis=0) - c.min(axis=0)))                # centroid extents stay finite (no NaN bucket)
    nodes, _ = tree_for(mn, mx, prec)
    if kind in ("huge", "mixed"):                                             # surface areas overflow in f32 and in f64
        assert ED.empty_child_boxes(nodes) > 0
    if kind == "mixed":
        assert ED.empty_child_boxes(nodes) < len(mn) // 2
    if kind == "subnormal":
        tiny = np.finfo(F).tiny
        assert np.all(np.abs(mn) < tiny) and np.all(np.abs(mx) < tiny) and np.any(mx != 0)
        assert ED.empty_child_boxes(nodes) == 0


def _neg_zero_entries(o, inv, mn, mx):
    """Rays with some box whose folded slab tmin is exactly -0 (the clamp turns it into +0) and that the slab test accepts."""
    F = o.dtype.type
    cnt = 0
    with np.errstate(all="ignore"):
        l = (mn[None] - o[:, None]) * inv[:, None]
        r = (mx[None] - o[:, None]) * inv[:, None]
        lo = np.minimum(l, r)
        tmin = lo[..., 0]
        for k in range(1, o.shape[1]):
            tmin = np.where(tmin >= lo[..., k], tmin, lo[..., k])
        tmax = np.maximum(l, r).min(axis=-1)
        ok = ~np.isnan(l).any(-1) & ~np.isnan(r).any(-1) & (tmax >= F(0))
    cnt = int(np.sum(np.any(ok & (tmin == 0) & np.signbit(tmin), axis=1)))
    return cnt


@pytest.mark.parametrize("kind,D,prec", CASES)
def test_ray_family_preconditions(kind, D, prec):
    F = FT[prec]
    mn, mx = ED.scene(kind, 300, D, prec)
    o, d, inv, fam = ED.ray_batch(mn, mx, 48, prec)
    assert np.all(np.isfinite(o)) and np.all(np.isfinite(d))
    nodes, shapes = tree_for(mn, mx, prec)
    tree = dimorder.Tree(nodes, shapes)
    for f in FAMILIES:
        m = np.flatnonzero(fam == f)
        facts = ED.ray_facts(o[m], d[m], inv[m], mn, mx)
        assert facts["nonzero_direction"] == len(m), f                        # no zero-direction (point-in-box) rays
        assert sum(len(tree._candidates((list(o[i]), list(inv[i])))) for i in m) > 0, f
        if f in ("axis", "face"):
            assert facts["neg_zero"] > 0 and facts["pos_zero"] > 0 and facts["inv_neg_inf"] > 0 and facts["inv_pos_inf"] > 0, facts
            assert facts["axes_special"] == list(range(D)), facts
        if f == "face":
            assert facts["face_plane_nan"] > 0, facts
        if f == "inside":
            inside = np.any(np.all((o[m][:, None] >= mn[None]) & (o[m][:, None] <= mx[None]), axis=2), axis=1)
            assert inside.all()
            assert _neg_zero_entries(o[m], inv[m], mn, mx) > 0                # origins on a face: entry -0 before the clamp
        if f == "tiny" and kind != "subnormal":
            assert facts["overflowing_products"] > 0, facts
        if f == "subdir":
            assert facts["subnormal_dir_finite_inv"] > 0 and facts["subnormal_dir_inf_inv"] > 0, facts
            assert facts["axes_special"] == list(range(D)), facts
            sub = (d[m] != 0) & (np.abs(d[m]) < np.finfo(F).tiny)
            assert np.all(np.abs(inv[m][sub & np.isfinite(inv[m])]) > np.finfo(F).max / 4)
            on = (o[m][:, None, :] == mn[None]) | (o[m][:, None, :] == mx[None])      # on a face plane along a finite-inverse axis
            assert np.any(on & (sub & np.isfinite(inv[m]))[:, None, :])
        if kind == "subnormal":
            assert facts["subnormal_differences"] > 0, f


@pytest.mark.parametrize("kind,D,prec", CASES)
def test_point_radius_and_limit_preconditions(kind, D, prec):
    F = FT[prec]
    fi = np.finfo(F)
    mn, mx = ED.scene(kind, 300, D, prec)
    pts, pk = ED.points(mn, mx, 100, prec)
    keys = np.array([K.keys(mn, mx, p) for p in pts])
    assert np.all(~np.isnan(keys))
    assert np.sum(keys == 0) > 0                                              # on faces / inside, and underflowed squares
    assert np.any(np.signbit(pts[pk == "zero"]) & (pts[pk == "zero"] == 0))   # -0 components
    if kind == "huge":
        assert np.sum(np.isposinf(keys)) > 0                                  # squared distances overflow T, f64 too
    if kind == "subnormal":
        assert np.sum((keys > 0) & (keys < fi.tiny)) > 0                      # a few subnormal steps
        assert np.all(keys[pk != "near"] == 0)                                # every other square underflows to 0
    r, rk = ED.radii(mn, mx, pts, prec)
    with np.errstate(all="ignore"):
        rr = r * r
    assert np.all(np.isposinf(rr[rk == "overflow"]))
    assert np.all((rr[rk == "underflow"] == 0) & (r[rk == "underflow"] > 0))
    up = np.flatnonzero(rk == "roundup")
    below = 0
    for i in up:
        pos = keys[i][(keys[i] > 0) & np.isfinite(keys[i])]
        if len(pos) and ED._roundup_radius(pos.min(), F) is not None:     # otherwise no r rounds onto that key
            assert rr[i] == pos.min(), i
            below += Fraction(float(r[i])) ** 2 < Fraction(float(pos.min()))
    if kind == "subnormal":
        assert below > 0                                                      # d2 <= r * r holds in T, not in exact arithmetic
    nodes, shapes = tree_for(mn, mx, prec)
    o, d, inv, fam = ED.ray_batch(mn, mx, 8, prec)
    lim, dstar = ED.limits(dimorder.Tree(nodes, shapes), o, inv, prec)
    assert np.any(np.isfinite(dstar)) and np.any(np.isinf(dstar))
    assert np.any(dstar == 0)                                                 # entries exactly 0
    assert lim["subnormal"][0] == fi.smallest_subnormal and np.all(lim["exit"] >= np.where(np.isfinite(dstar), dstar, np.inf))
    assert np.signbit(lim["negzero"]).all() and np.isposinf(lim["inf"]).all()


# ---- D = 3: the restatements against the C++ oracle -----------------------------------------------------------------------------
def _setup3(kind, prec, n=200, per=16):
    mn, mx = ED.scene(kind, n, 3, prec)
    shapes = _shapes3(mn, mx, prec)
    nodes = O.build(shapes, prec).nodes
    o, d, inv, fam = ED.ray_batch(mn, mx, per, prec, seed=3)
    return mn, mx, shapes, nodes, _rays3(o, d, inv, prec), o, inv, fam


@pytest.mark.parametrize("prec", ED.PRECS)
@pytest.mark.parametrize("kind", ED.SCENE_KINDS)
def test_dimorder_equals_the_oracle_in_3d(kind, prec):
    F = FT[prec]
    mn, mx, shapes, nodes, rays, o, inv, fam = _setup3(kind, prec)
    tree = dimorder.Tree(nodes, shapes)
    ref = O.traverse(nodes, shapes, rays, O.MODE_RECURSIVE, prec)
    lists = O.per_ray_lists(ref.offsets, ref.hits)
    leaf_box = {}
    for nd in nodes:
        if nd["child_l"] != O.U32_MAX:
            leaf_box[int(nd["child_l"])] = nd["l_aabb"]; leaf_box[int(nd["child_r"])] = nd["r_aabb"]
    node_of = {int(nd["shape"]): i for i, nd in enumerate(nodes) if nd["child_l"] == O.U32_MAX}
    ws, wd, _ = O.closest_hit(nodes, shapes, rays, prec=prec)
    for i, lst in enumerate(lists):
        ray = (list(o[i]), list(inv[i]))
        sl = [O.ray_slice(rays[i], np.array([(leaf_box[node_of[int(s)]]["min"], leaf_box[node_of[int(s)]]["max"])], dtype=shapes.dtype), prec)
              for s in lst]
        for ascending in (True, False):
            key = [s[0] if ascending else -s[1] for s in sl]
            order = sorted(range(len(lst)), key=lambda j: key[j])
            want = [(int(lst[j]), _fb(sl[j][0] if ascending else sl[j][1], F)) for j in order]
            assert [(int(s), _fb(x, F)) for s, x in tree.ordered(ray, ascending)] == want, (i, fam[i], ascending)
        s, e = tree.closest(ray)
        assert s == ws[i] and _fb(np.inf if e is None else e, F) == _fb(wd[i], F), (i, fam[i])
    assert (ws != O.U32_MAX).sum() > 0


@pytest.mark.parametrize("prec", ED.PRECS)
@pytest.mark.parametrize("kind", ED.SCENE_KINDS)
def test_any_hit_and_multi_hit_aabb_models_equal_the_oracle_in_3d(kind, prec):
    """anyhit.aabb reports a hit iff the oracle's closest AABB distance is < tmax, with a witness from O.traverse's set entered before
    tmax; multihit.aabb equals its brute force, whose rows are O.traverse's set with O.ray_slice entries, stably sorted."""
    F = FT[prec]
    mn, mx, shapes, nodes, rays, o, inv, fam = _setup3(kind, prec, per=10)
    ref = O.traverse(nodes, shapes, rays, O.MODE_RECURSIVE, prec)
    lists = O.per_ray_lists(ref.offsets, ref.hits)
    ws, wd, _ = O.closest_hit(nodes, shapes, rays, prec=prec)
    tree = dimorder.Tree(nodes, shapes)
    lim_fams, _ = ED.limits(tree, o, inv, prec)
    node_of = {int(nd["shape"]): i for i, nd in enumerate(nodes) if nd["child_l"] == O.U32_MAX}
    for name, tm in lim_fams.items():
        got = H.aabb_batch(nodes, shapes, o, inv, tm)
        lim = np.full(len(rays), np.inf, dtype=F) if tm is None else tm
        assert np.array_equal(got != H.U32_MAX, wd < lim), name
        for r in np.flatnonzero(got != H.U32_MAX):
            w = int(got[r])
            assert w in set(lists[r].tolist()), (name, r)
            sl = O.ray_slice(rays[r], shapes[w], prec)
            assert sl is not None and max(sl[0], F(0)) < lim[r], (name, r)
        if name in ("exact", "zero", "negzero", "negative", "nan"):
            assert np.all(got == H.U32_MAX), name
        for k in (1, 3, 64) if name in ("null", "exact", "exit", "subnormal") else (3,):
            model = MH.aabb_batch(nodes, shapes, o, inv, k, tm)
            brute = MH.brute_aabb_batch(nodes, shapes, o, inv, k, tm)
            assert np.array_equal(model[0], brute[0]) and np.array_equal(_bits(model[1]), _bits(brute[1])), (name, k)
            for r in range(len(rays)):
                q = []
                for s in lists[r]:
                    sl = O.ray_slice(rays[r], shapes[int(s)], prec)
                    if sl is not None and (tm is None or max(sl[0], F(0)) < tm[r]):
                        q.append((max(sl[0], F(0)), node_of[int(s)], int(s)))
                q.sort(key=lambda t: (t[0], t[1]))
                want = [s for _, _, s in q[:k]]
                assert brute[0][r, :len(want)].tolist() == want and np.all(brute[0][r, len(want):] == O.U32_MAX), (name, k, r)
                assert [_fb(e, F) for e, _, _ in q[:k]] == [_fb(x, F) for x in brute[1][r, :len(want)]], (name, k, r)


@pytest.mark.parametrize("prec", ED.PRECS)
@pytest.mark.parametrize("kind", ED.SCENE_KINDS)
def test_knn_and_nearest_models_equal_the_oracle_in_3d(kind, prec):
    F = FT[prec]
    mn, mx = ED.scene(kind, 200, 3, prec)
    shapes = _shapes3(mn, mx, prec)
    nodes = O.build(shapes, prec).nodes
    pts, _ = ED.points(mn, mx, 60, prec)
    for p in pts:                                                            # the key: Aabb::min_distance_squared
        assert np.array_equal(_bits(K.keys(mn, mx, p)), _bits(O.shape_distances_squared(shapes, p, prec))), p
    r, _ = ED.radii(mn, mx, pts, prec)
    walk = K.Walk(nodes, mn, mx)
    for k in (1, 5, 17, 64):
        for md in (None, r):
            ws, wd, _ = walk.rows(pts, k, md)
            bs, bd = K.brute(mn, mx, pts, k, md)
            assert np.array_equal(ws, bs) and wd.tobytes() == bd.tobytes(), (k, md is None)
    t = dimref.Tree(nodes, shapes, O.flatten(nodes, prec))
    for flat in (False, True):
        os_, od = O.nearest_to(O.flatten(nodes, prec) if flat else nodes, shapes, pts, prec, flat=flat)
        for i, p in enumerate(pts):
            s, dd = (t.nearest_flat if flat else t.nearest_bvh)(list(p))
            assert s == os_[i] and _fb(dd, F) == _fb(od[i], F), (flat, i)


@pytest.mark.parametrize("prec", ED.PRECS)
@pytest.mark.parametrize("kind", ED.SCENE_KINDS)
def test_triangle_models_equal_the_oracle_in_3d(kind, prec):
    """On the edge triangles: knntri's Triangle::distance_squared equals the oracle's, and prunedmodel.moeller_trumbore equals
    O.ray_triangle (distance and uv bits) for every family's rays; at subnormal scale det < eps, so every ray misses."""
    F = FT[prec]
    mn, mx = ED.scene(kind, 120, 3, prec)
    tris = ED.triangles(mn, mx, prec)
    shapes = O.tri_aabbs(tris, prec)
    assert np.all(shapes["min"] >= mn) and np.all(shapes["max"] <= mx)
    pts, _ = ED.points(mn, mx, 30, prec)
    t3 = tris.reshape(-1, 3, 3)
    for p in pts:
        got = KT.keys(p, t3)
        want = O.shape_distances_squared(shapes, p, prec, kind=O.DIST_TRIANGLE, tris=tris)
        assert np.array_equal(_bits(got), _bits(want)), p
    o, d, inv, fam = ED.ray_batch(shapes["min"], shapes["max"], 8, prec)
    rays = _rays3(o, d, inv, prec)
    hits = 0
    for r in range(len(rays)):
        for s in range(0, len(tris), 3):
            got = M.moeller_trumbore(list(o[r]), list(d[r]), *t3[s])
            want = O.ray_triangle(rays[r], tris[s], prec)
            assert _fb(got[0], F) == _fb(want[0], F), (r, s)
            if np.isfinite(want[0]):
                hits += 1
                assert _fb(got[1], F) == _fb(want[1], F) and _fb(got[2], F) == _fb(want[2], F), (r, s)
    if kind == "subnormal":
        assert hits == 0


@pytest.mark.parametrize("prec", ED.PRECS)
@pytest.mark.parametrize("kind", ED.SCENE_KINDS)
def test_queries_equal_the_oracle_in_3d(kind, prec):
    """dimref.Tree.query_bvh / query_flat equal O.query (Bvh::traverse / FlatBvh::traverse) for Aabb, Point and Ball records at these
    scales; the ball radii reach r * r overflowing, underflowing and rounding up onto a ball distance."""
    F = FT[prec]
    mn, mx = ED.scene(kind, 160, 3, prec)
    shapes = _shapes3(mn, mx, prec)
    nodes = O.build(shapes, prec).nodes
    flat = O.flatten(nodes, prec)
    t = dimref.Tree(nodes, shapes, flat)
    for qk in (dimref.AABB, dimref.POINT, dimref.BALL):
        q = ED.queries(qk, mn, mx, 60, prec)
        for fl in (None, flat):
            off, hits = O.query(qk, q, nodes, shapes, flat=fl, prec=prec)
            fn = t.query_bvh if fl is None else t.query_flat
            for i in range(len(q)):
                assert hits[off[i]:off[i + 1]].tolist() == fn(qk, [F(v) for v in q[i]]), (qk, fl is None, i)
        if qk == dimref.BALL:
            with np.errstate(all="ignore"):
                rr = q[:, -1] * q[:, -1]
            assert np.any(np.isposinf(rr)) and np.any((rr == 0) & (q[:, -1] > 0))
            on_key = sum(rr[i] in set(ED.ball_keys(mn, mx, q[i, :-1])[np.isfinite(ED.ball_keys(mn, mx, q[i, :-1]))].tolist()) and rr[i] > 0
                         for i in range(len(q)))
            assert on_key > 0 or kind == "huge"                                 # fl(r * r) lands on a ball distance (huge: all 0 or +inf)


@pytest.mark.parametrize("kind,D,prec", CASES)
def test_nearest_candidates_model_meets_the_contract(kind, D, prec):
    """prunedmodel.Tree.candidates (the device's nearest_bound + QUERY_WITHIN passes) on these scenes: every list holds every shape at the
    minimal exact distance (exactref), Bvh::nearest_to's shape and the brute-force minimum of the rounded keys (prunedcheck)."""
    mn, mx = ED.scene(kind, 160, D, prec)
    nodes, shapes = tree_for(mn, mx, prec)
    pts, _ = ED.points(mn, mx, 40, prec)
    tree = M.Tree(nodes, shapes)
    lists = [tree.candidates(list(p)) for p in pts]
    PC.check_candidates(lists, nodes, shapes, pts, prec)
    sizes = [len(lst) for lst in lists]
    assert min(sizes) > 0
    if kind == "mixed":
        assert min(sizes) < len(mn)                                            # the bound prunes below the no-split top
