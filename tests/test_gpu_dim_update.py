"""refit and update_shapes of Bvh<T,2> and Bvh<T,4> on the device:
- 4-D through a constant fourth axis equals the 3-D refit / update node for node (rebuilds with the 4-D builder seeded from many
  roots, 1.2 M shapes, global motion, 40 frames of drift, an overflow-scale scene);
- genuinely 4-D scenes keep the reference's invariants (tests/dimcheck.py), cost no more than a refit, and a global motion rebuilds
  the tree Bvh4.build makes;
- traversal records and flat arrays built before an update follow the new boxes (4-D, and 2-D where FLAT reads the lifted boxes);
- 2-D equals the 3-D path on the z = [0, 0] lift and stays within 10 % of the oracle's update_shapes cost;
- the contract: refusals leave the tree untouched, m = 0, the device-pointer forms on a side stream, device memory."""

import numpy as np
import pytest

from tests import dimcheck, dimref, pyref

pytestmark = pytest.mark.gpu
U32_MAX = 0xFFFFFFFF
PRECS = ("f32", "f64")


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A

    return A


def _F(prec):
    return np.float32 if prec == "f32" else np.float64


def _lift(a3, prec, c=1.5):
    from bvh_b200.dtypes import BY_PREC_4D

    a4 = np.zeros(len(a3), dtype=BY_PREC_4D[prec]["aabb"])
    a4["min"][:, :3], a4["max"][:, :3] = a3["min"], a3["max"]
    a4["min"][:, 3], a4["max"][:, 3] = c, c
    return a4


def _boxes(mn, mx, dtype):
    a = np.zeros(len(mn), dtype=dtype)
    a["min"], a["max"] = mn, mx
    return a


def _move(a, rng, frac, scale):
    """(sorted changed indices, all boxes after moving them by uniform offsets in [-scale, scale])."""
    n, D = a["min"].shape
    F = a["min"].dtype.type
    changed = np.sort(rng.choice(n, max(1, int(n * frac)), replace=False)).astype(np.uint32)
    b = a.copy()
    off = rng.uniform(-scale, scale, (len(changed), D))
    b["min"][changed] = (b["min"][changed].astype(np.float64) + off).astype(F)
    b["max"][changed] = (b["max"][changed].astype(np.float64) + off).astype(F)
    return changed, b


def _same34(b3, b4):
    n3, i3 = b3.nodes, b3.node_index
    n4, i4 = b4.nodes_and_index()
    assert np.array_equal(i4, i3)
    for f in ("parent", "child_l", "child_r", "shape"):
        assert np.array_equal(n4[f], n3[f]), f
    for side in ("l_aabb", "r_aabb"):
        for mm in ("min", "max"):
            assert np.array_equal(n4[side][mm][:, :3], n3[side][mm]), (side, mm)
    inner = n3["child_l"] != U32_MAX
    for side in ("l_aabb", "r_aabb"):
        assert np.all(n4[side]["min"][~inner, 3] == np.inf) and np.all(n4[side]["max"][~inner, 3] == -np.inf)   # leaves keep Aabb::empty()


def _scene3(name, prec):
    from bvh_b200 import scenes
    from bvh_b200.dtypes import BY_PREC
    from tests.edge_inputs import edge_scene

    if name == "cubes":
        return scenes.create_n_cubes_aabbs(10000, prec)
    if name == "huge":
        return np.ascontiguousarray(edge_scene("huge", 20000, prec), dtype=BY_PREC[prec]["aabb"])
    n = {"random5000": 5000, "random1m": 1_200_000}[name]
    rng = np.random.default_rng(n)
    mn = rng.uniform(-1000, 1000, (n, 3))
    return _boxes(mn, mn + rng.uniform(0, 3, (n, 3)), BY_PREC[prec]["aabb"])


# ---- 1. D = 4 through a constant fourth axis = D = 3 ------------------------------------------------------------------------
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("scene", ["cubes", "random5000", "random1m"])
def test_lifted_4d_refit_and_update_equal_3d(api, scene, prec):
    rng = np.random.default_rng(len(scene))
    a = _scene3(scene, prec)
    span = 2000.0 if scene.startswith("random") else 2e5
    b3, b4 = api.Bvh.build(a, prec=prec), api.Bvh4.build(_lift(a, prec), prec=prec)
    _, a = _move(a, rng, 1.0, span * 1e-4)                    # every shape jitters: refit
    b3.refit(a); b4.refit(_lift(a, prec))
    _same34(b3, b4)
    for frac, scale, growth in ((0.05, span / 4, 1.5), (0.05, span / 4, 0.0), (0.01, span / 50, 1.5)):
        changed, a = _move(a, rng, frac, scale)
        r3 = b3.update_shapes(changed, a, max_growth=growth)
        r4 = b4.update_shapes(changed, _lift(a, prec), max_growth=growth)
        assert r3 == r4
        if growth > 0 and frac == 0.05:
            assert r4 > 0 and (scene != "random1m" or r4 > 256)   # large rebuild roots go through the level loop
        if growth == 0:
            assert r4 == 0
        _same34(b3, b4)
    rep = np.array([3, 3, 7, 3], dtype=np.uint32)             # a repeated index with an identical box
    a["min"][rep] += 1.0; a["max"][rep] += 1.0
    assert b3.update_shapes(rep, a) == b4.update_shapes(rep, _lift(a, prec))
    _same34(b3, b4)
    if scene == "random1m":                                   # global motion: every shape moves, the root is rebuilt from 1.2 M shapes
        g = a.copy()
        g["min"] = (a["min"].astype(np.float64) * 2.0).astype(a["min"].dtype)
        g["max"] = g["min"] + (a["max"] - a["min"])
        idx = np.arange(len(a), dtype=np.uint32)
        r3, r4 = b3.update_shapes(idx, g), b4.update_shapes(idx, _lift(g, prec))
        assert r3 == r4 == len(a)
        _same34(b3, b4)
    b3.free(); b4.free()


@pytest.mark.parametrize("prec", PRECS)
def test_lifted_4d_drift_over_40_frames_equals_3d(api, prec):
    """Slow drift accumulates against the baseline of the first update and is rebuilt eventually, identically in 3-D and 4-D."""
    rng = np.random.default_rng(40)
    a = _scene3("random5000", prec)
    b3, b4 = api.Bvh.build(a, prec=prec), api.Bvh4.build(_lift(a, prec), prec=prec)
    vel = rng.uniform(-6, 6, (len(a), 3))
    total = 0
    for frame in range(40):
        changed = np.sort(rng.choice(len(a), 500, replace=False)).astype(np.uint32)
        F = a["min"].dtype.type
        a["min"][changed] = (a["min"][changed] + vel[changed]).astype(F)
        a["max"][changed] = (a["max"][changed] + vel[changed]).astype(F)
        r3, r4 = b3.update_shapes(changed, a), b4.update_shapes(changed, _lift(a, prec))
        assert r3 == r4, frame
        total += r4
        _same34(b3, b4)
    assert total > 0
    b3.free(); b4.free()


def test_lifted_4d_update_of_an_overflow_scale_scene_equals_3d(api):
    rng = np.random.default_rng(2)
    a = _scene3("huge", "f32")
    b3, b4 = api.Bvh.build(a, prec="f32"), api.Bvh4.build(_lift(a, "f32"), prec="f32")
    for growth in (1.5, 0.0):
        changed, a = _move(a, rng, 0.1, 1e29)
        assert b3.update_shapes(changed, a, max_growth=growth) == b4.update_shapes(changed, _lift(a, "f32"), max_growth=growth)
        _same34(b3, b4)
    b3.refit(a); b4.refit(_lift(a, "f32"))
    _same34(b3, b4)
    b3.free(); b4.free()


# ---- 2. genuinely 4-D scenes ------------------------------------------------------------------------------------------------
def _scene4(kind, n, prec, rng):
    from bvh_b200.dtypes import BY_PREC_4D

    F = _F(prec)
    axis = int(kind[-1]) if kind.startswith("axis") else 0
    mn, mx = dimref.scene("axis" if kind.startswith("axis") else kind, n, 4, F, rng, axis=axis)
    return _boxes(mn, mx, BY_PREC_4D[prec]["aabb"])


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("kind", ["random", "coincident", "axis0", "axis1", "axis2", "axis3", "peel", "overflow"])
def test_4d_update_keeps_the_invariants(api, kind, prec):
    rng = np.random.default_rng(len(kind) * 7)
    n = 300 if kind == "peel" else 3000                      # geometric centres: 1.12 ** n stays finite in f32
    a = _scene4(kind, n, prec, rng)
    lo, hi = a["min"].astype(np.float64).min(), a["max"].astype(np.float64).max()
    scale = (hi - lo) / 3 if kind != "coincident" else 5.0
    b, ref = api.Bvh4.build(a, prec=prec), api.Bvh4.build(a, prec=prec)
    before = b.nodes_and_index()[0]
    assert b.update_shapes(np.arange(0, n, 7, dtype=np.uint32), a) == 0          # no motion: nothing changes
    if kind != "overflow":                                    # (the climb replaces the empty boxes of "no split wins" nodes by joins)
        assert b.nodes_and_index()[0].tobytes() == before.tobytes()
    for step in range(3):
        changed, a = _move(a, rng, 0.2, scale)
        rebuilt = b.update_shapes(changed, a, max_growth=1.5)
        assert ref.update_shapes(changed, a, max_growth=0.0) == 0               # the same motion, boxes only
        nodes, idx = b.nodes_and_index()
        assert dimcheck.layout_ok(nodes, idx)
        assert np.array_equal(nodes["shape"][idx], np.arange(n))
        if kind != "overflow":                                # rebuilt "no split wins" subtrees store empty boxes again
            assert dimcheck.is_consistent(nodes, a) and dimcheck.is_tight(nodes)
            rn = ref.nodes_and_index()[0]
            assert dimcheck.is_consistent(rn, a) and dimcheck.is_tight(rn)
            if kind not in ("coincident",):
                assert dimcheck.sah_cost(nodes) <= dimcheck.sah_cost(rn) * (1 + 1e-9), step
        if kind == "random":
            assert rebuilt > 0
    b.refit(a)                                                # a full refit makes every box tight, overflow scenes included
    nodes, _ = b.nodes_and_index()
    assert dimcheck.is_consistent(nodes, a) and dimcheck.is_tight(nodes)
    b.free(); ref.free()


@pytest.mark.parametrize("prec", PRECS)
def test_4d_global_motion_rebuilds_the_tree_build_makes(api, prec):
    rng = np.random.default_rng(4)
    n = 20000
    a = _scene4("random", n, prec, rng)
    b = api.Bvh4.build(a, prec=prec)
    g = _scene4("random", n, prec, rng)
    g["min"] = (g["min"].astype(np.float64) * 3).astype(g["min"].dtype)
    g["max"] = g["min"] + (g["max"] - g["min"]) / 3
    assert b.update_shapes(np.arange(n, dtype=np.uint32), g) == n
    want_nodes, want_idx = api.Bvh4.build(g, prec=prec).nodes_and_index()
    nodes, idx = b.nodes_and_index()
    assert nodes.tobytes() == want_nodes.tobytes() and np.array_equal(idx, want_idx)
    b.free()


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("n", [0, 1, 2, 3])
def test_4d_tiny_trees(api, n, prec):
    from bvh_b200 import capi

    rng = np.random.default_rng(n)
    a = _scene4("random", n, prec, rng)
    b = api.Bvh4.build(a, prec=prec)
    q = np.zeros((1, 8), dtype=_F(prec))
    b.query_batch(capi.QUERY_AABB, q)                         # builds the traversal records
    changed, a = _move(a, rng, 1.0, 500.0) if n else (np.zeros(0, np.uint32), a)
    assert b.update_shapes(changed, a) == 0 or n == 3        # one or two shapes: nothing a rebuild could change
    if n:
        b.refit(a)
        nodes, idx = b.nodes_and_index()
        assert dimcheck.layout_ok(nodes, idx) and dimcheck.is_consistent(nodes, a) and dimcheck.is_tight(nodes)
        rec = np.concatenate([a["min"][-1], a["max"][-1]])[None, :]             # the last shape's new box
        off, hits = b.query_batch(capi.QUERY_AABB, rec)
        want = dimref.Tree(nodes, a).query_bvh(dimref.AABB, list(rec[0]))
        assert hits.tolist() == want and (n - 1) in want
    b.free()


# ---- 3. cached device state follows the boxes ---------------------------------------------------------------------------------
def _flat_of(nodes, F, D):
    """flatten() of a preorder node array (closed form, flatten.cu): nav(i) = (i - 1) + leaves before i."""
    nn = len(nodes)
    leaf = nodes["child_l"] == U32_MAX
    if nn == 0:
        return []
    empty = ([F(np.inf)] * D, [F(-np.inf)] * D)
    if nn == 1:
        return [(None, U32_MAX, 1, int(nodes["shape"][0]))]
    start = np.concatenate([[0], np.cumsum(leaf)[:-1]])
    cnt = dimcheck.counts(nodes)
    out = [None] * (3 * ((nn + 1) // 2) - 2)
    for i in range(1, nn):
        p = int(nodes["parent"][i])
        side = "l_aabb" if nodes["child_l"][p] == i else "r_aabb"
        nav = (i - 1) + int(start[i])
        out[nav] = ((list(nodes[side]["min"][p]), list(nodes[side]["max"][p])), nav + 1, nav + 3 * int(cnt[i]) - 1, U32_MAX)
        if leaf[i]:
            out[nav + 1] = (empty, U32_MAX, nav + 2, int(nodes["shape"][i]))
    return out


def _pyref_nodes(nodes):
    out = []
    for nd in nodes:
        if nd["child_l"] == U32_MAX:
            out.append(("leaf", int(nd["parent"]), int(nd["shape"])))
        else:
            out.append(("node", int(nd["parent"]), int(nd["child_l"]), int(nd["child_r"]),
                        (list(nd["l_aabb"]["min"]), list(nd["l_aabb"]["max"])), (list(nd["r_aabb"]["min"]), list(nd["r_aabb"]["max"]))))
    return out


def _rays(a, m, D, F, rng, targets):
    """m rays from around the scene, aimed at the given points in turn (in 4-D a random ray rarely meets a box)."""
    lo, hi = a["min"].astype(np.float64).min(axis=0), a["max"].astype(np.float64).max(axis=0)
    span = np.maximum(hi - lo, 1.0)
    org = lo - 0.2 * span + rng.uniform(0, 1.4, (m, D)) * span
    tgt = targets[np.arange(m) % len(targets)]
    return [pyref.ray_new(F, org[i], tgt[i] - org[i]) for i in range(m)]


def _everything(b, D, F, rays_np, recs, pts):
    from bvh_b200 import capi

    out = {"flat": b.flatten()}
    for mode in (capi.TRAVERSE_BVH, capi.TRAVERSE_FLAT):
        out[("ray", mode)] = b.traverse_batch(rays_np, mode=mode)
        for kind in (dimref.AABB, dimref.POINT, dimref.BALL):
            out[(kind, mode)] = b.query_batch(kind, recs[kind], mode=mode)
        out[("near", mode)] = b.nearest_to_batch(pts, mode=mode)
    return out


def _csr_lists(off, hits):
    return [hits[off[i]:off[i + 1]].tolist() for i in range(len(off) - 1)]


def _expected(nodes, a, D, F, prs, recs, pts):
    from bvh_b200 import capi

    flat = _flat_of(nodes, F, D)
    pn = _pyref_nodes(nodes)
    tree = dimref.Tree(nodes, a)
    tree.flat = [(box[0] if box else None, box[1] if box else None, e, x, s) for box, e, x, s in flat]
    ex = {}
    ex[("ray", capi.TRAVERSE_BVH)] = [pyref.traverse_recursive(pn, a, (o, inv), F) for o, _, inv in prs]
    ex[("ray", capi.TRAVERSE_FLAT)] = [pyref.traverse_flat([(b, e, x, s) for b, e, x, s in flat], a, (o, inv), F) for o, _, inv in prs]
    for kind in (dimref.AABB, dimref.POINT, dimref.BALL):
        ex[(kind, capi.TRAVERSE_BVH)] = [tree.query_bvh(kind, list(r)) for r in recs[kind]]
        ex[(kind, capi.TRAVERSE_FLAT)] = [tree.query_flat(kind, list(r)) for r in recs[kind]]
    ex[("near", capi.TRAVERSE_BVH)] = [tree.nearest_bvh(list(p)) for p in pts]
    ex[("near", capi.TRAVERSE_FLAT)] = [tree.nearest_flat(list(p)) for p in pts]
    return flat, ex


def _check_caches(api, cls, D, prec, dtype_ray):
    from bvh_b200 import capi

    F = _F(prec)
    rng = np.random.default_rng(D)
    n = 1500
    mn, mx = dimref.scene("random", n, D, F, rng)
    a = _boxes(mn, mx, cls._TABLE[prec]["aabb"])
    b = cls.build(a, prec=prec)
    changed, a2 = _move(a, rng, 0.3, 60.0)
    centre = lambda x: (x["min"][changed].astype(np.float64) + x["max"][changed].astype(np.float64)) / 2
    prs = _rays(a, 120, D, F, rng, np.concatenate([centre(a), centre(a2)])[rng.permutation(2 * len(changed))])   # old and new places
    rays_np = np.zeros(len(prs), dtype=dtype_ray)
    for i, (o, d, inv) in enumerate(prs):
        rays_np["origin"][i], rays_np["direction"][i], rays_np["inv_direction"][i] = o, d, inv
    recs = {k: dimref.queries(k, mn, mx, 120, F, rng, nan=False) for k in (dimref.AABB, dimref.POINT, dimref.BALL)}
    pts = dimref.points(mn, mx, 80, F, rng)
    old = _everything(b, D, F, rays_np, recs, pts)            # traversal records and the flat array exist from here on
    b.update_shapes(changed, a2, max_growth=1.5)
    nodes, _ = b.nodes_and_index()
    new = _everything(b, D, F, rays_np, recs, pts)
    flat, ex = _expected(nodes, a2, D, F, prs, recs, pts)
    _, ex_old = _expected(nodes, a, D, F, prs, recs, pts)     # the new tree read with the OLD shape boxes
    for i, (box, e, x, s) in enumerate(flat):
        f = new["flat"][i]
        assert (f["entry_index"], f["exit_index"], f["shape_index"]) == (e, x, s), i
        if box is not None:
            assert np.array_equal(f["aabb"]["min"], np.array(box[0], dtype=F)) and np.array_equal(f["aabb"]["max"], np.array(box[1], dtype=F)), i
    assert new["flat"].tobytes() != old["flat"].tobytes()
    flat_differs = False                                      # some FLAT answer changes with the shape boxes alone (d_aabb / d_aabb_trav)
    for key, want in ex.items():
        if key[0] == "near":
            shape, dist = new[key]
            assert shape.tolist() == [w[0] for w in want], key
            assert np.array_equal(dist, np.array([w[1] for w in want], dtype=F)), key
            assert [w[0] for w in want] != [w[0] for w in ex_old[key]] or key[1] == capi.TRAVERSE_BVH   # FLAT reads shape boxes
            assert new[key][0].tolist() != old[key][0].tolist()
        else:
            got = _csr_lists(*new[key])
            assert got == want, key
            assert got != _csr_lists(*old[key]), key          # precondition: the motion changed the answer
            if key[1] == capi.TRAVERSE_FLAT:
                flat_differs |= want != ex_old[key]           # FLAT leaves re-test the new shape boxes
    assert flat_differs
    b.free()


@pytest.mark.parametrize("prec", PRECS)
def test_4d_caches_follow_the_boxes(api, prec):
    from bvh_b200.dtypes import BY_PREC_4D

    _check_caches(api, api.Bvh4, 4, prec, BY_PREC_4D[prec]["ray"])


@pytest.mark.parametrize("prec", PRECS)
def test_2d_caches_follow_the_boxes(api, prec):
    from bvh_b200.dtypes import BY_PREC_2D

    _check_caches(api, api.Bvh2, 2, prec, BY_PREC_2D[prec]["ray"])


# ---- 4. D = 2 -----------------------------------------------------------------------------------------------------------------
def _lift2(a2, prec):
    from bvh_b200.dtypes import BY_PREC

    a3 = np.zeros(len(a2), dtype=BY_PREC[prec]["aabb"])
    a3["min"][:, :2], a3["max"][:, :2] = a2["min"], a2["max"]
    return a3


@pytest.mark.parametrize("prec", PRECS)
def test_2d_update_equals_3d_on_the_lift_and_the_oracle_cost(api, prec):
    from bvh_b200.dtypes import BY_PREC_2D
    from oracle import oracle as O

    F = _F(prec)
    rng = np.random.default_rng(22)
    n = 5000
    mn, mx = dimref.scene("random", n, 2, F, rng)
    a = _boxes(mn, mx, BY_PREC_2D[prec]["aabb"])
    b2, b3 = api.Bvh2.build(a, prec=prec), api.Bvh.build(_lift2(a, prec), prec=prec)

    def same():
        n2, i2 = b2.nodes_and_index()
        n3 = b3.nodes
        assert np.array_equal(i2, b3.node_index)
        for f in ("parent", "child_l", "child_r", "shape"):
            assert np.array_equal(n2[f], n3[f]), f
        for side in ("l_aabb", "r_aabb"):
            for mm in ("min", "max"):
                assert np.array_equal(n2[side][mm], n3[side][mm][:, :2])
        return n2, i2

    _, a = _move(a, rng, 1.0, 0.05)
    b2.refit(a); b3.refit(_lift2(a, prec))
    same()
    want0 = O.build(_lift2(a, prec), prec)                    # the oracle's tree of the same boxes: refit keeps build's tree here
    changed, a = _move(a, rng, 0.1, 60.0)
    r2 = b2.update_shapes(changed, a, max_growth=1.5)
    assert r2 == b3.update_shapes(changed, _lift2(a, prec), max_growth=1.5) and r2 > 0
    n2, i2 = same()
    assert dimcheck.layout_ok(n2, i2) and dimcheck.is_consistent(n2, a) and dimcheck.is_tight(n2)
    # the oracle's z = 0 arithmetic is exact: its update_shapes on the lift is the reference's 2-D update
    ref_nodes, _ = O.update_shapes(want0.nodes, want0.node_index, _lift2(a, prec), changed, prec)
    assert dimcheck.sah_cost(n2) <= 1.10 * O.sah_cost(ref_nodes, prec)[0]
    changed, a = _move(a, rng, 0.1, 60.0)
    assert b2.update_shapes(changed, a, max_growth=0.0) == 0 == b3.update_shapes(changed, _lift2(a, prec), max_growth=0.0)
    same()
    b2.free(); b3.free()


# ---- 5. contract -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("D", [2, 4])
def test_refusals_leave_the_tree_untouched(api, D, prec):
    from bvh_b200 import capi

    cls = api.Bvh2 if D == 2 else api.Bvh4
    F = _F(prec)
    rng = np.random.default_rng(D)
    mn, mx = dimref.scene("random", 2000, D, F, rng)
    a = _boxes(mn, mx, cls._TABLE[prec]["aabb"])
    b = cls.build(a, prec=prec)
    b.update_shapes(np.arange(10, dtype=np.uint32), a)        # the baseline exists: a refusal must not disturb it either
    before = b.nodes_and_index()
    bad = a.copy()
    bad["max"][17, D - 1] = np.nan
    for call, status in ((lambda: b.update_shapes(np.array([5, 17], np.uint32), bad), capi.ERR_NAN),
                         (lambda: b.update_shapes(np.array([5, 2000], np.uint32), np.concatenate([a, a[:1]])), capi.ERR_INVALID),
                         (lambda: b.update_shapes(np.array([5], np.uint32), a, max_growth=0.5), capi.ERR_INVALID),
                         (lambda: b.refit(bad), capi.ERR_NAN),
                         (lambda: b.refit(a[:-1]), capi.ERR_INVALID)):
        with pytest.raises(capi.BvhGpuError) as e:
            call()
        assert e.value.status == status
        after = b.nodes_and_index()
        assert after[0].tobytes() == before[0].tobytes() and np.array_equal(after[1], before[1])
    assert b.update_shapes(np.zeros(0, np.uint32), a) == 0    # m = 0: a no-op
    assert b.nodes_and_index()[0].tobytes() == before[0].tobytes()
    changed, a2 = _move(a, rng, 0.2, 50.0)                    # the tree still works after the refusals
    b.update_shapes(changed, a2)
    nodes, idx = b.nodes_and_index()
    assert dimcheck.layout_ok(nodes, idx) and dimcheck.is_consistent(nodes, a2) and dimcheck.is_tight(nodes)
    b.free()


@pytest.mark.parametrize("prec", PRECS)
def test_device_pointer_forms_on_a_side_stream_equal_the_host_forms(api, prec):
    import torch

    from bvh_b200 import capi

    rng = np.random.default_rng(11)
    a = _scene4("random", 30000, prec, rng)
    host, dev = api.Bvh4.build(a, prec=prec), api.Bvh4.build(a, prec=prec)
    ctx = dev.ctx
    s = torch.cuda.Stream()
    ctx.set_stream(s.cuda_stream)
    try:
        for step in range(3):
            changed, a = _move(a, rng, 0.05, 60.0)
            r_host = host.update_shapes(changed, a)
            with torch.cuda.stream(s):                        # the inputs are produced on the side stream, behind a busy kernel
                torch.cuda._sleep(50_000_000)
                d_idx = torch.from_numpy(changed.view(np.int32)).to("cuda", non_blocking=False)
                d_box = torch.from_numpy(np.ascontiguousarray(a[changed]).view(np.uint8)).to("cuda")
            r_dev = dev.update_dev(d_idx.data_ptr(), d_box.data_ptr(), len(changed), want_rebuilt=(step != 1))
            assert r_dev is None or r_dev == r_host
            assert dev.nodes_and_index()[0].tobytes() == host.nodes_and_index()[0].tobytes()
        _, a = _move(a, rng, 1.0, 1.0)
        host.refit(a)
        with torch.cuda.stream(s):
            torch.cuda._sleep(50_000_000)
            d_all = torch.from_numpy(a.view(np.uint8).copy()).to("cuda")
        dev.refit_dev(d_all.data_ptr(), len(a))
        s.synchronize()
        assert dev.nodes_and_index()[0].tobytes() == host.nodes_and_index()[0].tobytes()
        bad = torch.tensor([len(a)], dtype=torch.int32, device="cuda")
        with pytest.raises(capi.BvhGpuError) as e:
            dev.update_dev(bad.data_ptr(), d_all.data_ptr(), 1)
        assert e.value.status == capi.ERR_INVALID
    finally:
        ctx.set_stream(None)
    host.free(); dev.free()


def test_device_memory_returns_to_its_level_over_update_frames(api):
    import torch

    rng = np.random.default_rng(3)
    a = _scene4("random", 20000, "f32", rng)
    a2 = _boxes(*dimref.scene("random", 20000, 2, np.float32, rng), api.Bvh2._TABLE["f32"]["aabb"])
    b, b2 = api.Bvh4.build(a, prec="f32"), api.Bvh2.build(a2, prec="f32")
    b.flatten(); b2.flatten()

    def frame():
        nonlocal a, a2
        changed, a = _move(a, rng, 0.05, 40.0)
        b.update_shapes(changed, a)
        changed, a2 = _move(a2, rng, 0.05, 40.0)
        b2.update_shapes(changed, a2)

    frame()
    api.Context.default().synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(20):
        frame()
    api.Context.default().synchronize()
    assert free0 - torch.cuda.mem_get_info()[0] < 16 << 20
    b.free(); b2.free()
