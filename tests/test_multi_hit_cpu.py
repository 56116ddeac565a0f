"""CPU checks behind the multi-hit queries (bvhgpu_multi_hit_*):
- the header declares the 10 entry points and the binding sees them, typed;
- the restatement of tests/multihit.py at D = 3 stands on the C++ oracle: its traversal set is O.traverse's (BVH semantics) and its
  triangle distances are O.ray_triangle's, bit for bit, on a cube scene and every triangle family of tests/adversarial.py;
- triangle mode, for every limit of anyhit.tmax_families and k in {1, 3, 16, 64}: the model equals the brute force (the stable sort of
  the loop over Bvh::traverse) on every row whose brute-force row is bounded, and meets the weaker guarantee (real qualifying hits in
  ascending order) on the others; the grazing family really has unbounded rows in f32, the other families have none;
- the identities on the model: k = 1 without a limit is prunedmodel.closest_triangles, and a row is empty exactly where anyhit reports
  no hit;
- AABB mode: the model equals the brute force on every row in D = 2, 3 and 4, on the dimref scenes and the adversarial box families
  (overflow-scale "no split wins" trees included), and at D = 3 without a limit it is the head of dimorder's ordered traversal.
That makes the restatement the oracle of tests/test_gpu_multi_hit.py."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import adversarial as A, anyhit as H, dimorder, dimref, multihit as MH, prunedmodel as PM, rebuildref

FT = {"f32": np.float32, "f64": np.float64}
UINT = {np.float32: np.uint32, np.float64: np.uint64}
KS = (1, 3, 16, 64)
NEW = [f"bvhgpu_multi_hit_{p}x{d}" for d in (2, 3, 4) for p in ("f32", "f64")]
NEW += [f"bvhgpu_multi_hit_dev_{p}x{d}" for d in (3, 4) for p in ("f32", "f64")]


def test_header_declares_the_new_entry_points():
    from bvh_b200 import capi

    assert len(NEW) == 10
    assert set(NEW) <= set(capi.declared_symbols())
    L = capi.lib()
    for s in NEW:
        assert getattr(L, s).argtypes, s


def _bits(a):
    a = np.asarray(a)
    return a.view(UINT[a.dtype.type]) if a.dtype.type in UINT else a


def _same(x, y):
    return all(np.array_equal(_bits(a), _bits(b)) for a, b in zip(x, y) if a is not None or b is not None)


# ---- triangle mode, D = 3 -----------------------------------------------------------------------------------------------------------
def _cube_scene(prec):
    shapes, tris = O.create_n_cubes(40, prec=prec, want_tris=True)
    rng = np.random.default_rng(11)
    centres = (shapes["min"][::6].astype(np.float64) + shapes["max"][::6]) / 2
    tgt = centres[rng.integers(0, len(centres), 96)] + rng.uniform(-0.6, 0.6, (96, 3))
    org = tgt + rng.normal(size=(96, 3)) * 4000
    return tris.reshape(-1, 9), O.ray_new(org, tgt - org, prec)


def _tri_scene(family, prec):
    F = FT[prec]
    if family == "cubes":
        return _cube_scene(prec)
    if family == "grazing":
        tris, o, d, _ = A.grazing(F)
    elif family == "shared":
        tris, o, d = A.shared_edges(F)
    elif family == "degenerate":
        tris, o, d = A.degenerate(F)
    else:
        tris, o, d = A.offset_scene(F, 1e6 if prec == "f32" else 1e13, m=120)
    return tris, O.ray_new(o, d, prec)


TRI_FAMILIES = ["cubes", "grazing", "shared", "degenerate", "offset"]


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("family", TRI_FAMILIES)
def test_triangle_model_against_the_oracle_and_the_brute_force(family, prec):
    F = FT[prec]
    tris, rays = _tri_scene(family, prec)
    shapes = O.tri_aabbs(tris, prec)
    nodes = O.build(shapes, prec).nodes
    # the model's primitives are the oracle's: the traversal set and the Moeller-Trumbore distances, bit for bit
    ref = O.traverse(nodes, shapes, rays, O.MODE_RECURSIVE, prec)
    cand = [sorted(int(x) for x in lst) for lst in O.per_ray_lists(ref.offsets, ref.hits)]
    t = MH._Tris(nodes, shapes, tris)
    for r in range(len(rays)):
        o, d, inv = t.ray(rays, r)
        assert sorted(t.sh[i] for i in MH._tri_leaves(t, o, inv)) == cand[r], r
        for s in cand[r]:
            got = PM.moeller_trumbore(o, d, *t.tr[s])[0]
            assert _bits(np.array([got], F)) == _bits(np.array([O.ray_triangle(rays[r], tris[s], prec)[0]], F)), (r, s)
    candset = [set(c) for c in cand]
    ws, wd, _ = O.closest_hit(nodes, shapes, rays, tris, prec)
    assert (ws != O.U32_MAX).sum() > 0
    unbounded = 0
    for name, tm in H.tmax_families(wd, F, np.random.default_rng(4)).items():
        empty = H.triangles(nodes, shapes, tris, rays, tm) == H.U32_MAX
        for k in KS:
            got = MH.triangles(nodes, shapes, tris, rays, k, tm)
            bs, bd, buv, bounded = MH.brute_triangles(nodes, shapes, tris, rays, k, tm)
            for r in np.flatnonzero(bounded):
                assert _same((got[0][r], got[1][r], got[2][r]), (bs[r], bd[r], buv[r])), (name, k, r)
            assert MH.weak_ok(got[0], got[1], tris, rays, tm, candset) == [], (name, k)
            assert np.array_equal(got[0][:, 0] == MH.U32_MAX, empty), (name, k)           # identity 2 (and 1 for tm None below)
            unbounded += int((~bounded).sum())
            if name in ("zero", "negzero", "negative", "nan"):
                assert np.all(got[0] == MH.U32_MAX), (name, k)
        if name == "null":
            cs, cd, cuv = PM.closest_triangles(nodes, shapes, tris, rays)
            got = MH.triangles(nodes, shapes, tris, rays, 1, None)
            assert _same((got[0][:, 0], got[1][:, 0], got[2][:, 0]), (cs, cd, cuv))
    if family == "grazing" and prec == "f32":
        assert unbounded > 0                                     # the case the weaker guarantee exists for is reached
    elif family != "grazing":
        assert unbounded == 0


# ---- AABB mode, D = 2, 3, 4 ---------------------------------------------------------------------------------------------------------
def _box_scene(kind, D, prec, rng):
    F = FT[prec]
    if kind == "adv_overflow":
        mn, mx, _ = A.overflow(F, D)
    elif kind in A.BOX_FAMILIES:
        mn, mx, _ = A.BOX_FAMILIES[kind](F, D)
    else:
        mn, mx = dimref.scene(kind, 120, D, F, rng)
    a = np.zeros(len(mn), dtype=rebuildref.node_dtype(D, prec)["l_aabb"])
    a["min"], a["max"] = mn, mx
    nodes, _ = rebuildref.build(a, prec)
    o, _, inv = dimorder.rays(mn, mx, 20, F, rng)
    return nodes, a, o, inv


BOX_SCENES = list(dimref.SCENES) + ["large", "ties", "mixed", "adv_overflow"]


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("kind", BOX_SCENES)
@pytest.mark.parametrize("D", [2, 3, 4])
def test_aabb_model_equals_the_brute_force(D, kind, prec):
    F = FT[prec]
    rng = np.random.default_rng(40 + D)
    nodes, shapes, o, inv = _box_scene(kind, D, prec, rng)
    tree = dimorder.Tree(nodes, shapes)
    dstar = np.array([np.inf if c[1] is None else c[1] for c in (tree.closest((list(o[r]), list(inv[r]))) for r in range(len(o)))], dtype=F)
    if kind == "overflow" and prec == "f32":
        assert np.any(~np.isfinite(nodes["l_aabb"]["min"][:, 0]))             # "no split wins" nodes: empty child boxes
    hits = 0
    for name, tm in H.tmax_families(dstar, F, np.random.default_rng(3)).items():
        for k in KS:
            got = MH.aabb_batch(nodes, shapes, o, inv, k, tm)
            want = MH.brute_aabb_batch(nodes, shapes, o, inv, k, tm)
            assert _same(got[:2], want[:2]), (name, k)
            hits += int((got[0] != MH.U32_MAX).sum())
            if tm is not None:                                                      # identity 2
                assert np.array_equal(got[0][:, 0] == MH.U32_MAX, H.aabb_batch(nodes, shapes, o, inv, tm) == H.U32_MAX), (name, k)
        if name == "null":
            got = MH.aabb_batch(nodes, shapes, o, inv, 1, None)
            c = [tree.closest((list(o[r]), list(inv[r]))) for r in range(len(o))]
            assert np.array_equal(got[0][:, 0], np.array([s for s, _ in c], dtype=np.uint32))            # identity 1
            assert _same((got[1][:, 0],), (np.array([np.inf if e is None else e for _, e in c], dtype=F),))
    assert hits > 0 or kind in ("coincident", "peel")             # point boxes: only exact aims can hit


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_aabb_model_is_the_head_of_the_ordered_traversal_in_3d(prec):
    """Identity 3 on a built tree without "no split wins" nodes: the stored leaf box is the shape's own box."""
    F = FT[prec]
    rng = np.random.default_rng(9)
    nodes, shapes, o, inv = _box_scene("random", 3, prec, rng)
    inner = nodes["child_l"] != MH.U32_MAX
    assert np.all(np.isfinite(nodes["l_aabb"]["min"][inner])) and np.all(np.isfinite(nodes["r_aabb"]["min"][inner]))
    tree = dimorder.Tree(nodes, shapes)
    for k in KS:
        sh, di, _ = MH.aabb_batch(nodes, shapes, o, inv, k, None)
        for r in range(len(o)):
            want = tree.ordered((list(o[r]), list(inv[r])), True)[:k]
            n = len(want)
            assert sh[r, :n].tolist() == [s for s, _ in want] and np.all(sh[r, n:] == MH.U32_MAX), (k, r)
            assert _same((di[r, :n],), (np.array([e for _, e in want], dtype=F),)), (k, r)
