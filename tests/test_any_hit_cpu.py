"""CPU checks behind the any-hit (occlusion) queries:
- the header declares the 10 entry points and the binding sees them;
- the restatement of tests/anyhit.py meets the any-hit contract against the C++ oracle at D = 3, on a random cube scene and on every
  triangle family of tests/adversarial.py, for every family of per-ray limits (NULL, +inf, the ray's own closest distance d* and its
  neighbours, 0, -0, negative, NaN, random):
    AABB mode      a witness exists iff the oracle's closest AABB distance is < tmax; the witness is in O.traverse's set (BVH
                   semantics) and its own AABB is entered at < tmax;
    triangle mode  a witness's Moeller-Trumbore distance (the oracle's) is < tmax; where the model reports no hit but the oracle's
                   unpruned loop has one, every qualifying triangle is a grazing one: the slab entry of its stored box exceeds
                   fl(tmax * (1 + 2^-16)), and in exact arithmetic its intersection lies beyond tmax.
That makes the restatement the oracle of tests/test_gpu_any_hit.py."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import adversarial as A, anyhit as H, exactref as E, prunedcheck as PC

FT = {"f32": np.float32, "f64": np.float64}
NEW = [f"bvhgpu_any_hit_{p}x{d}" for d in (2, 3, 4) for p in ("f32", "f64")]
NEW += [f"bvhgpu_any_hit_dev_{p}x{d}" for d in (3, 4) for p in ("f32", "f64")]


def test_header_declares_the_new_entry_points():
    from bvh_b200 import capi

    assert len(NEW) == 10
    assert set(NEW) <= set(capi.declared_symbols())


def _cube_scene(prec):
    shapes, tris = O.create_n_cubes(40, prec=prec, want_tris=True)
    rng = np.random.default_rng(11)
    centres = (shapes["min"][::6].astype(np.float64) + shapes["max"][::6]) / 2
    tgt = centres[rng.integers(0, len(centres), 160)] + rng.uniform(-0.6, 0.6, (160, 3))
    org = tgt + rng.normal(size=(160, 3)) * 4000
    return tris.reshape(-1, 9), O.ray_new(org, tgt - org, prec)


def _scene(family, prec):
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
        tris, o, d = A.offset_scene(F, 1e6 if prec == "f32" else 1e13, m=200)
    return tris, O.ray_new(o, d, prec)


FAMILIES = ["cubes", "grazing", "shared", "degenerate", "offset"]


def _setup(family, prec):
    tris, rays = _scene(family, prec)
    shapes = O.tri_aabbs(tris, prec)
    nodes = O.build(shapes, prec).nodes
    ref = O.traverse(nodes, shapes, rays, O.MODE_RECURSIVE, prec)
    cand = [set(int(x) for x in lst) for lst in O.per_ray_lists(ref.offsets, ref.hits)]
    return tris, rays, shapes, nodes, cand


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("family", FAMILIES)
def test_aabb_mode_model_meets_the_contract(family, prec):
    F = FT[prec]
    tris, rays, shapes, nodes, cand = _setup(family, prec)
    ws, wd, _ = O.closest_hit(nodes, shapes, rays, prec=prec)
    assert (ws != O.U32_MAX).sum() > 0
    o, inv = rays["origin"], rays["inv_direction"]
    seen = 0
    for name, tm in H.tmax_families(wd, F, np.random.default_rng(3)).items():
        got = H.aabb_batch(nodes, shapes, o, inv, tm)
        lim = np.full(len(rays), np.inf, dtype=F) if tm is None else tm
        assert np.array_equal(got != H.U32_MAX, wd < lim), name          # exact: a hit iff the closest distance is < tmax
        for r in np.flatnonzero(got != H.U32_MAX):
            w = int(got[r])
            assert w in cand[r], (name, r, w)
            sl = O.ray_slice(rays[r], shapes[w], prec)
            assert sl is not None and max(sl[0], F(0)) < lim[r], (name, r, w)
        seen += int((got != H.U32_MAX).sum())
        if name in ("exact", "zero", "negzero", "negative", "nan"):
            assert np.all(got == H.U32_MAX), name
        if name == "above":
            assert np.array_equal(got != H.U32_MAX, np.isfinite(wd)), name
    assert seen > 0


def _stored_boxes(nodes, shapes):
    """The box the walk tests last before shape s's leaf: the child box its parent stores (the own box at a root leaf)."""
    if len(nodes) == 1:
        return {int(nodes[0]["shape"]): shapes[int(nodes[0]["shape"])]}
    leaf_of = {i: int(nd["shape"]) for i, nd in enumerate(nodes) if nd["child_l"] == O.U32_MAX}
    out = {}
    for nd in nodes:
        if nd["child_l"] != O.U32_MAX:
            for c, box in ((int(nd["child_l"]), nd["l_aabb"]), (int(nd["child_r"]), nd["r_aabb"])):
                if c in leaf_of:
                    out[leaf_of[c]] = np.array([(box["min"], box["max"])], dtype=shapes.dtype)[0]
    return out


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("family", FAMILIES)
def test_triangle_mode_model_meets_the_contract(family, prec):
    F = FT[prec]
    tris, rays, shapes, nodes, cand = _setup(family, prec)
    ws, wd, _ = O.closest_hit(nodes, shapes, rays, tris, prec)            # the unpruned loop over Bvh::traverse
    assert (ws != O.U32_MAX).sum() > 0
    stored = _stored_boxes(nodes, shapes)
    margin = PC.MARGIN[prec]
    grazing = 0
    for name, tm in H.tmax_families(wd, F, np.random.default_rng(4)).items():
        got = H.triangles(nodes, shapes, tris, rays, tm)
        lim = np.full(len(rays), np.inf, dtype=F) if tm is None else tm
        for r in np.flatnonzero(got != H.U32_MAX):
            w = int(got[r])
            assert w in cand[r] and O.ray_triangle(rays[r], tris[w], prec)[0] < lim[r], (name, r, w)
        for r in np.flatnonzero((got == H.U32_MAX) & (wd < lim)):        # the unpruned loop has a hit: only the grazing case
            grazing += 1
            for s in cand[r]:
                t = O.ray_triangle(rays[r], tris[s], prec)[0]
                if not t < lim[r]:
                    continue
                sl = O.ray_slice(rays[r], stored[s], prec)
                assert sl is not None and max(sl[0], F(0)) > lim[r] * margin, (name, r, s)
                ex = E.ray_triangle(rays["origin"][r], rays["direction"][r], *tris[s].reshape(3, 3))
                assert ex is None or ex[0] > E.fr(lim[r]), (name, r, s)
        if name in ("zero", "negzero", "negative", "nan"):
            assert np.all(got == H.U32_MAX), name
    if family == "grazing" and prec == "f32":
        assert grazing > 0                                                # the case the clause exists for is reached
