"""CPU side of the k-nearest-triangles query (bvhgpu_knn_triangles_*, DESIGN.md section 4.17).
- tests/knntri.py's closest_point_triangle gives the oracle's Triangle::distance_squared bit for bit, f32 and f64, on cubes, Sponza,
  random soups and every adversarial family;
- the restated walk (knn_walk with the triangle key) equals the brute-force row wherever every qualifying triangle is bounded;
- each family contains what it claims, and the number of unbounded (point, triangle) pairs is pinned at what the model measures;
- a triangle left outside its box (a stale triangle after a refit) is unbounded, and the weaker guarantee holds on it."""
import os

import numpy as np
import pytest

from bvh_b200 import scenes
from oracle import oracle as O
from tests import knntri as KT
from tests.test_pruned_walks_cpu import tree_for

FT = {"f32": np.float32, "f64": np.float64}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def sponza_tris(F):
    z = np.load(os.path.join(ROOT, "tests", "golden", "sponza_tris.npz"))
    return z["vertices"][z["triangles"].astype(np.int64)].astype(F)


def scene(name, F, rng):
    if name == "cubes":
        return scenes.create_n_cubes_tris(40, "f32" if F == np.float32 else "f64")
    if name == "soup":
        return KT.soup(F, 150, rng)
    return KT.family(name, F)[0]


def limits(tris, pts, rng):
    """One limit per point as tests/test_knn_cpu.limits draws them (0, -1, -0, NaN, +inf, random, a key's exact square root), with the
    triangle keys in place of the box keys."""
    F = tris.dtype.type
    out = np.zeros(len(pts), dtype=F)
    for i, p in enumerate(pts):
        kind = i % 7
        if kind < 5:
            out[i] = [0.0, -1.0, -0.0, np.nan, np.inf][kind]
            continue
        key = KT.keys(p, tris)
        key = key[np.isfinite(key)]
        if kind == 5 or len(key) == 0:
            out[i] = F(rng.uniform(0, 2) * np.sqrt(float(np.median(key)))) if len(key) else F(1)
            continue
        key = key[rng.integers(0, len(key))]
        r = F(np.sqrt(key))
        for c in (r, np.nextafter(r, F(np.inf)), np.nextafter(r, F(0))):
            with np.errstate(all="ignore"):
                if c * c == key:
                    r = c
                    break
        out[i] = r
    return out


SCENES = ["cubes", "soup"] + sorted(KT.FAMILIES)
# unbounded (point, triangle) pairs the model measures on each family's 60 points x 80 triangles: none, in f32 and f64
UNBOUNDED = {name: 0 for name in KT.FAMILIES}


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("name", SCENES + ["sponza"])
def test_model_keys_equal_the_oracle(name, prec):
    F = FT[prec]
    rng = np.random.default_rng(7)
    tris = sponza_tris(F) if name == "sponza" else scene(name, F, rng)
    shapes = O.tri_aabbs(tris, prec)
    pts = KT.near_points(tris, 6 if name == "sponza" else 30, rng)
    if name != "sponza":
        pts = np.concatenate([pts, KT.family(name, F)[1][:10] if name in KT.FAMILIES else pts[:0]])
    for p in pts:
        want = O.shape_distances_squared(shapes, p, prec, kind=O.DIST_TRIANGLE, tris=tris)
        got = KT.keys(p, tris)
        assert got.tobytes() == want.tobytes(), (name, p)


def test_cube_triangles_equal_the_oracle():
    """bvh_b200.scenes.create_n_cubes_tris (the probe's 120 k-triangle scene, configs[1]) is create_n_cubes' vertices, with the same
    boxes as create_n_cubes_aabbs."""
    for prec in ("f32", "f64"):
        shapes, tris = O.create_n_cubes(300, prec=prec, want_tris=True)
        got = scenes.create_n_cubes_tris(300, prec)
        assert got.dtype == tris.dtype and got.tobytes() == tris.tobytes()
        assert O.tri_aabbs(got, prec).tobytes() == scenes.create_n_cubes_aabbs(300, prec).tobytes()


def test_vectorised_bound_equals_prunedmodel():
    from tests.prunedmodel import box_lower_d2

    rng = np.random.default_rng(5)
    for F in (np.float32, np.float64):
        tris = np.concatenate([KT.soup(F, 50, rng), KT.family("tiny_far", F)[0], KT.family("subnormal", F)[0]])
        mn, mx = KT.boxes(tris)
        for p in np.concatenate([KT.near_points(tris, 8, rng), KT.odd_points(F)]):
            got = KT.box_lower_d2(p, mn, mx)
            want = np.array([box_lower_d2(list(p), list(a), list(b)) for a, b in zip(mn, mx)], dtype=F)
            assert got.tobytes() == want.tobytes()


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("name", SCENES)
def test_walk_equals_brute_force_where_bounded(name, prec):
    F = FT[prec]
    rng = np.random.default_rng(11 + SCENES.index(name))
    tris = scene(name, F, rng)
    mn, mx = KT.boxes(tris)
    nodes, _ = tree_for(mn, mx, prec)
    pts = KT.family(name, F)[1][:21] if name in KT.FAMILIES else KT.near_points(tris, 21, rng)
    pts = np.concatenate([pts, KT.odd_points(F)])
    assert all(KT.bounded(p, tris, mn, mx).all() for p in pts)
    walk = KT.Walk(nodes, tris)
    lim = limits(tris, pts, rng)
    for k in (1, 5, 17, 64):
        for md in (None, lim):
            ws, wd, _ = walk.rows(pts, k, md)
            bs, bd, _ = KT.brute(tris, pts, k, md)
            assert np.array_equal(ws, bs), (k, md is None)
            assert wd.tobytes() == bd.tobytes(), (k, md is None)


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("name", sorted(KT.FAMILIES))
def test_family_contains_what_it_claims(name, prec):
    F = FT[prec]
    tris, pts = KT.family(name, F)
    mn, mx = KT.boxes(tris)
    keys = np.array([KT.keys(p, tris) for p in pts])
    branches = np.array([KT.branch(p, tris) for p in pts])
    unbounded = sum(int((~KT.bounded(p, tris, mn, mx)).sum()) for p in pts)
    assert unbounded == UNBOUNDED[name]
    a, b, c = tris[:, 0], tris[:, 1], tris[:, 2]
    if name == "overflow":
        assert np.isnan(keys).sum() > 1000 and np.isposinf(keys).sum() > 10
        assert np.isfinite(tris).all() and np.isfinite(pts).all()
    else:
        assert np.isfinite(keys).all()
    if name == "repeated":
        assert all((branches == j).any() for j in range(4))
    if name == "collinear":
        ab, ac = (b - a).astype(np.float64), (c - a).astype(np.float64)
        assert (np.cross(ab, ac) == 0).all() and not (a == b).all(1).any()
    if name == "near_collinear":
        assert (branches == 10).any() and (branches == 9).any()
    if name == "slivers":
        assert (branches == 10).any() and (branches >= 7).sum() > 1000
    if name == "subnormal":
        assert (np.abs(tris) < np.finfo(F).tiny).all() and (tris != 0).any()
    if name == "tiny_far":
        assert (np.abs(tris) > (1e5 if F == np.float32 else 1e13)).all() and (branches < 4).any()


def test_stale_triangle_is_a_witness_of_the_weaker_guarantee():
    """A triangle moved outside the box the tree holds for it (a refit with stale boxes) has a key below its box's bound: the walk
    prunes it although brute force ranks it first.  The row still lists real (s, key_s) in ascending order and every bounded
    qualifying triangle that sorts before its last entry."""
    F = np.float32
    rng = np.random.default_rng(3)
    tris = KT.soup(F, 120, rng)
    mn, mx = KT.boxes(tris)
    nodes, _ = tree_for(mn, mx, "f32")
    moved = tris.copy()
    moved[0] = tris[0] - tris[0].mean(0) + np.array([200.0, 0, 0], dtype=F)          # far outside every box
    p = np.array([200.0, 0.5, 0], dtype=F)
    assert not KT.bounded(p, moved, mn, mx)[0] and KT.bounded(p, moved, mn, mx)[1:].all()
    walk = KT.Walk(nodes, moved)
    for k in (1, 8):
        s, d, _ = walk.row(p, k)
        bs, _, _ = KT.brute(moved, p[None], k)
        assert bs[0, 0] == 0 and 0 not in s
        key = KT.keys(p, moved)
        filled = s[s != KT.U32_MAX]
        assert d[: len(filled)].tobytes() == np.sqrt(key[filled]).astype(F).tobytes()
        assert all((key[x], x) <= (key[y], y) for x, y in zip(filled, filled[1:]))
        ok = KT.bounded(p, moved, mn, mx)
        last = (key[filled[-1]], filled[-1])
        want = [j for j in np.argsort(key, kind="stable") if ok[j] and (key[j], j) <= last]
        assert list(filled) == want
