"""Crossing counts, point-in-mesh and signed distance on the device against the exact walk model of tests/crosswalk.py, on every row,
f32 and f64, host form and _dev with FULL and OD rays.  The model reads the device's own node array (bvh.nodes):
- adversarial triangle families (grazing, shared edges, degenerate, offset scenes at two offsets), the huge / mixed / subnormal edge
  scenes with the edge ray families, the layer stack and stale triangles (boxes moved by refit away from their triangles), under the
  limits around each ray's k-th crossing (anyhit.tmax_families plus the last crossing's nextafter, the smallest subnormal, the largest
  finite value and a scalar); the rows where the limited walk and the loop differ are counted and reported;
- LBVH and LBVH+treelet trees, and trees after update_shapes, add_shapes and remove_shapes down to one shape and to none;
- contains against the model's vote on every point (NaN, infinite, subnormal and overflow-scale points included), and against the truth
  on overlapping and nested shells, offset meshes (reported) and a 1e-4 icosphere (invisible in f32);
- signed_distance against knn_triangles(k = 1) and contains, and -0 for a point on a vertex of an inner shell;
- the three calls after set_triangles_dev on a stream the context then leaves (tests/test_gpu_stream_switch.py's Switch).
Run on an H100:  python -m pytest -s tests/test_gpu_crossings_edges.py -m gpu"""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O
from tests import crossings as X
from tests import crosswalk as W
from tests import edge_dims as ED
from tests.knntri import odd_points
from tests.test_crossings_cpu import sphere_points, torus_points
from tests.test_gpu_crossings import _bits, _forms

pytestmark = pytest.mark.gpu
FT = {"f32": np.float32, "f64": np.float64}
RULES = {"even_odd": X.EVEN_ODD, "nonzero": X.NONZERO}
LIMITS_SHORT = ("null", "above", "below", "random", "above_last", "negzero", "max_finite")     # on the larger or repeated scenes


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A_

    return A_


def _eq(a, b):
    return np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def _differ(a, b):
    return (a[0] != b[0]) | (a[1] != b[1])


def _mesh(api, tris, prec, mode=None):
    from bvh_b200 import capi

    tris = np.ascontiguousarray(tris, dtype=FT[prec]).reshape(-1, 9)
    shapes = O.tri_aabbs(tris, prec)
    bvh = api.Bvh.build(shapes, prec=prec, mode=capi.BUILD_EXACT_SAH if mode is None else mode)
    bvh.set_triangles(tris)
    return bvh, shapes, tris


def _check_counts(bvh, shapes, tris, rays, prec, name, rng, families=None):
    """Every form equals the model on every row, without a limit and under every limit family; returns (rows where the limited walk
    and the loop differ, the unlimited counts)."""
    nodes = bvh.nodes
    cand = W.candidates(nodes, shapes, rays)
    loop = W.unlimited_walk(nodes, shapes, tris, rays, None, cand)
    for i, got in enumerate(_forms(bvh, rays, None, prec)):
        assert _eq(got, loop), (name, "unlimited", i)
    unbounded = 0
    for lname, tm in W.kth_limits(rays, tris, cand, rng).items():
        if families is not None and lname not in families:
            continue
        want = W.model(nodes, shapes, tris, rays, tm, cand)
        for i, got in enumerate(_forms(bvh, rays, tm, prec)):
            assert _eq(got, want), (name, lname, i, int(_differ(got, want).sum()))
        unbounded += int(_differ(want, W.unlimited_walk(nodes, shapes, tris, rays, tm, cand)).sum())
    return unbounded, loop


def _points(rays, shapes, F, rng, m=200):
    """Ray origins, points around the scene, NaN / infinite points, subnormal points and overflow-scale points."""
    lo, hi = shapes["min"].min(axis=0).astype(np.float64), shapes["max"].max(axis=0).astype(np.float64)
    with np.errstate(all="ignore"):
        around = rng.uniform(0, 1, (m, 3)) * (hi - lo) + lo
    fi = np.finfo(F)
    parts = [rays["origin"][:m].astype(np.float64), around, odd_points(np.float64),
             rng.uniform(-64, 64, (8, 3)) * float(fi.smallest_subnormal),
             rng.uniform(-1, 1, (8, 3)) * float(fi.max), np.array([[0.0, -0.0, 0.0], [-0.0, -0.0, -0.0]])]
    with np.errstate(all="ignore"):
        return np.ascontiguousarray(np.concatenate(parts).astype(F))


def _check_contains(bvh, shapes, tris, points, name):
    nodes = bvh.nodes
    pr = X.point_rays(points, shapes["min"].dtype.type)
    cand = W.candidates(nodes, shapes, pr)
    out = {}
    for rule, code in RULES.items():
        want = W.contains_model(nodes, shapes, tris, points, code, cand)
        got = bvh.contains(points, rule)
        assert np.array_equal(got, want), (name, rule, int((got != want).sum()))
        out[rule] = got
    return out


def _check_signed(bvh, points, inside, name):
    s, d, q = bvh.knn_triangles(points, 1, closest=True)
    for rule in RULES:
        gs, gd, gq = bvh.signed_distance(points, rule, closest=True)
        assert np.array_equal(gs, s[:, 0]) and np.array_equal(_bits(gq), _bits(q[:, 0])), (name, rule)
        assert np.array_equal(_bits(gd), _bits(X.signed(s[:, 0], d[:, 0], inside[rule]))), (name, rule)


# ---- triangle families and edge scenes ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_families_and_edge_scenes_equal_the_model(api, prec):
    F = FT[prec]
    rng = np.random.default_rng(61)
    report = {}
    for name, (tris, rays) in W.triangle_scenes(prec).items():
        bvh, shapes, tris = _mesh(api, tris, prec)
        try:
            unb, loop = _check_counts(bvh, shapes, tris, rays, prec, name, rng)
            # the oracle's own exact-SAH tree gives the same loop
            ref = O.build(shapes, prec).nodes
            tr = O.traverse(ref, shapes, rays, O.MODE_RECURSIVE, prec)
            assert _eq(loop, X.counts_csr(rays, tris, tr.offsets, tr.hits)), name
            empty = ED.empty_child_boxes(bvh.nodes)
            if name.startswith("edge_"):
                assert (empty > 0) == (name != "edge_subnormal"), (name, empty)
                assert (loop[0].sum() + loop[1].sum() > 0) == (name == "edge_mixed"), name
                if name == "edge_mixed":                        # counted triangles below Aabb::empty() child boxes
                    assert _differ(loop, W.model(bvh.nodes, shapes, tris, rays, skip_empty=True)).any()
            if name == "grazing" and prec == "f32":
                assert unb >= 40, unb
            inside = _check_contains(bvh, shapes, tris, _points(rays, shapes, F, rng), name)
            report[name] = dict(crossings=int(loop[0].sum() + loop[1].sum()), unbounded_matched=unb, empty_child_boxes=empty,
                                inside=int(inside["even_odd"].sum()))
        finally:
            bvh.free()
    for name, r in report.items():
        print(f"{prec} {name}: {r}")


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_layer_stack_and_stale_triangles(api, prec):
    F = FT[prec]
    rng = np.random.default_rng(62)
    tris, rays, _ = W.layer_stack(F, m=48)
    bvh, shapes, tris = _mesh(api, tris, prec)
    try:
        unb, loop = _check_counts(bvh, shapes, tris, rays, prec, "layers", rng, LIMITS_SHORT)
        assert np.all(loop[0] == W.LAYERS // 2) and np.all(loop[1] == W.LAYERS // 2)
        j = rng.integers(0, W.LAYERS, len(rays))
        j[:4] = [0, 1, W.LAYERS - 2, W.LAYERS - 1]
        for i, (f, b) in enumerate(_forms(bvh, rays, W.layer_limits(rays, j), prec)):
            assert np.array_equal(f.astype(np.int64) + b, j + 1), i
            assert np.array_equal(b.astype(np.int64) - f, (j + 2) // 2 - (j + 1) // 2), i
        print(f"{prec} layers: {unb} unbounded rows matched")
    finally:
        bvh.free()
    # stale triangles: boxes moved by twice their x extent with refit, triangles kept, rays mostly along +x
    tris, own, moved, rays = W.stale(F)
    bvh, _, tris = _mesh(api, tris, prec)
    try:
        bvh.refit(moved)
        unb, loop = _check_counts(bvh, moved, tris, rays, prec, "stale", rng)
        assert unb > 0 and loop[0].sum() + loop[1].sum() > 0
        p = _points(rays, moved, F, rng)
        _check_contains(bvh, moved, tris, p, "stale")
        print(f"{prec} stale: {unb} unbounded rows matched, {int(loop[0].sum() + loop[1].sum())} crossings")
    finally:
        bvh.free()


# ---- build modes and dynamic trees ------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("mode", ["lbvh", "lbvh_treelet"])
def test_lbvh_trees_equal_the_model(api, prec, mode):
    from bvh_b200 import capi

    F = FT[prec]
    rng = np.random.default_rng(63)
    m = {"lbvh": capi.BUILD_LBVH, "lbvh_treelet": capi.BUILD_LBVH_TREELET}[mode]
    ps, _ = sphere_points(rng, 1000)
    pt, _ = torus_points(rng, 1000)
    g_tris, g_rays = W.triangle_scenes(prec)["grazing"]
    meshes = [("icosphere", X.icosphere(3, F), ps), ("torus", X.torus(F=F), pt), ("grazing", g_tris, None)]
    for name, tris, p in meshes:
        bvh, shapes, tris = _mesh(api, tris, prec, m)
        try:
            pts = p.astype(F) if p is not None else _points(g_rays, shapes, F, rng)
            rays = X.point_rays(pts[:300], F) if name != "grazing" else g_rays
            unb, _ = _check_counts(bvh, shapes, tris, rays, prec, f"{mode} {name}", rng, LIMITS_SHORT)
            _check_contains(bvh, shapes, tris, pts, f"{mode} {name}")
            print(f"{prec} {mode} {name}: {unb} unbounded rows matched")
        finally:
            bvh.free()


def _apply_moves(shapes, tris, moves, k):
    s2, t2 = shapes.copy(), tris.copy()
    for new_i, old_i in moves:
        s2[new_i], t2[new_i] = shapes[old_i], tris[old_i]
    return s2[:len(shapes) - k], t2[:len(tris) - k]


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_dynamic_trees_equal_the_model(api, prec):
    F = FT[prec]
    rng = np.random.default_rng(64)
    tris = np.concatenate([X.icosphere(2, F), (X.torus(F=F) * F(0.5) + F(3)).astype(F)]).reshape(-1, 9)
    bvh, shapes, tris = _mesh(api, tris, prec)
    p = np.concatenate([rng.uniform(-1.5, 1.5, (400, 3)), rng.uniform(2, 4, (400, 3))]).astype(F)
    rays = X.point_rays(p[:200], F)
    tm_rays = O.ray_new(rng.uniform(-5, 5, (300, 3)), rng.normal(size=(300, 3)), prec)
    rays = np.concatenate([rays, tm_rays])

    def check(label):
        unb, _ = _check_counts(bvh, shapes, tris, rays, prec, label, rng, LIMITS_SHORT)
        _check_contains(bvh, shapes, tris, p, label)
        return unb

    try:
        # update_shapes of a third of the shapes: their triangles move, the rest stay
        idx = rng.choice(len(shapes), len(shapes) // 3, replace=False)
        t2 = tris.copy()
        t2[idx] = (t2[idx].astype(np.float64) + rng.normal(0, 0.05, (len(idx), 1)) + np.tile(rng.normal(0, 0.2, (len(idx), 3)), 3)).astype(F)
        s2 = O.tri_aabbs(t2, prec)
        bvh.update_shapes(idx, s2)
        bvh.set_triangles(t2)
        shapes, tris = s2, t2
        check("update_shapes")
        # add_shapes of a second mesh
        extra = (X.icosphere(2, F) * F(0.7) + F(-3)).astype(F).reshape(-1, 9)
        bvh.add_shapes(O.tri_aabbs(extra, prec))
        shapes, tris = np.concatenate([shapes, O.tri_aabbs(extra, prec)]), np.concatenate([tris, extra])
        bvh.set_triangles(tris)
        check("add_shapes")
        # remove_shapes down to one shape (the root-leaf walk), then to none
        gone = rng.choice(len(shapes), len(shapes) - 1, replace=False)
        moves = bvh.remove_shapes(gone)
        shapes, tris = _apply_moves(shapes, tris, moves, len(gone))
        bvh.set_triangles(tris)
        assert bvh.num_shapes == 1 and len(bvh.nodes) == 1
        hit = O.ray_new(tris.reshape(-1, 3, 3).astype(np.float64).mean(axis=1) - [[0, 0, 2]], [[0, 0, 1]], prec)
        one_rays = np.concatenate([rays, hit, O.ray_new(hit["origin"] + [[0, 0, 4]], [[0, 0, -1]], prec)])
        r_save = rays
        rays = one_rays
        check("one shape")
        f, b = bvh.count_hits(rays[-2:])
        assert f.sum() + b.sum() == 2, (f, b)
        rays = r_save
        bvh.remove_shapes([0])
        assert bvh.num_shapes == 0
        f, b = bvh.count_hits(rays)
        assert not f.any() and not b.any()
        for rule in RULES:
            assert not bvh.contains(p, rule).any()
    finally:
        bvh.free()


# ---- contains and signed distance against the truth ---------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_shells_contain_their_truth_under_both_rules(api, prec):
    F = FT[prec]
    for name, (t, p, eo, nz) in W.ball_pairs(F).items():
        bvh, shapes, tris = _mesh(api, t, prec)
        try:
            inside = _check_contains(bvh, shapes, tris, p, name)
            assert np.array_equal(inside["even_odd"], eo), (name, int((inside["even_odd"] != eo).sum()))
            assert np.array_equal(inside["nonzero"], nz), (name, int((inside["nonzero"] != nz).sum()))
            _check_signed(bvh, p, inside, name)
        finally:
            bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_offset_and_tiny_meshes(api, prec):
    """At 1e4 (f32) / 1e12 (f64) the vote equals the model on every point and its agreement with the truth is reported (the vote is
    not watertight there); an icosphere scaled by 1e-4 has |det| < eps in f32, so nothing is inside, and is exact in f64."""
    F = FT[prec]
    rng = np.random.default_rng(65)
    off = 1e4 if prec == "f32" else 1e12
    ps, ts = sphere_points(rng, 3000)
    pt, tt = torus_points(rng, 3000)
    for name, tris, p, truth in (("icosphere", X.icosphere(3, np.float64), ps, ts), ("torus", X.torus(), pt, tt)):
        t = (tris + off).astype(F)
        q = (p + off).astype(F)
        bvh, shapes, t = _mesh(api, t, prec)
        try:
            inside = _check_contains(bvh, shapes, t, q, f"offset {name}")
            _check_signed(bvh, q, inside, f"offset {name}")
            agree = {rule: float(np.mean(inside[rule] == truth)) for rule in RULES}
            print(f"{prec} {name} at offset {off:g}: agreement with the truth {agree}")
        finally:
            bvh.free()
    t = (X.icosphere(3, np.float64) * 1e-4).astype(F)
    q = (ps * 1e-4).astype(F)
    bvh, shapes, t = _mesh(api, t, prec)
    try:
        inside = _check_contains(bvh, shapes, t, q, "tiny icosphere")
        for rule in RULES:
            if prec == "f32":
                assert not inside[rule].any(), rule
            else:
                assert np.array_equal(inside[rule], ts), rule
        _check_signed(bvh, q, inside, "tiny icosphere")
    finally:
        bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_signed_distance_is_negative_zero_on_an_inner_vertex(api, prec):
    """Two nested outward icospheres; a point exactly on a vertex of the inner one is at distance 0 and, under NONZERO, inside: the
    triangles through the vertex give Moeller-Trumbore distance 0, which is rejected, so back - front is 1 or 2 on every ray."""
    F = FT[prec]
    ico = X.icosphere(2, np.float64)
    t = np.concatenate([ico, 0.5 * ico]).astype(F)
    bvh, shapes, t = _mesh(api, t, prec)
    try:
        inner = t.reshape(-1, 3, 3)[len(ico):]
        v = np.unique(inner.reshape(-1, 3), axis=0)[:: 7]
        f, b = bvh.count_hits(X.point_rays(v, F))
        w = (b.astype(np.int64) - f).reshape(-1, 3)
        assert np.all((w == 1) | (w == 2)), w
        assert bvh.contains(v, "nonzero").all()
        s, d = bvh.signed_distance(v, "nonzero")
        assert np.all(d == 0) and np.all(np.signbit(d)), d
        s, d = bvh.signed_distance(np.array([[0.0, 0.0, 0.0]], dtype=F), "nonzero")
        assert d[0] < 0
    finally:
        bvh.free()


# ---- the three calls after set_triangles_dev on a stream the context leaves ---------------------------------------------------------
@pytest.fixture(scope="module")
def twin_ctx(api):
    ctx = api.Context()
    yield ctx
    ctx.close()


def _crossing_consumers(prec):
    """(name, host(tree, rays, pts) -> arrays, prepare(rays, pts) -> launch(tree) -> read() for the _dev form)."""
    import torch

    from tests.test_gpu_stream_switch import _dev, _host

    dt = torch.float32 if prec == "f32" else torch.float64

    def count_dev(rays, pts):
        d_r = _dev(rays)
        f = torch.full((len(rays),), 7, dtype=torch.int32, device="cuda")
        b = torch.full((len(rays),), 7, dtype=torch.int32, device="cuda")

        def launch(tree):
            tree.count_hits_dev(d_r.data_ptr(), len(rays), 0, f.data_ptr(), b.data_ptr())
            return lambda: (_host(f, np.uint32), _host(b, np.uint32))
        return launch

    def contains_dev(rays, pts):
        d_p = _dev(pts)
        out = torch.full((len(pts),), 7, dtype=torch.uint8, device="cuda")

        def launch(tree):
            tree.contains_dev(d_p.data_ptr(), len(pts), out.data_ptr(), "nonzero")
            return lambda: (out.cpu().numpy().astype(bool),)
        return launch

    def signed_dev(rays, pts):
        d_p = _dev(pts)
        s = torch.full((len(pts),), 7, dtype=torch.int32, device="cuda")
        d = torch.full((len(pts),), 7, dtype=dt, device="cuda")
        q = torch.full((3 * len(pts),), 7, dtype=dt, device="cuda")

        def launch(tree):
            tree.signed_distance_dev(d_p.data_ptr(), len(pts), s.data_ptr(), d.data_ptr(), q.data_ptr(), "nonzero")
            return lambda: (_host(s, np.uint32), d.cpu().numpy(), q.cpu().numpy().reshape(-1, 3))
        return launch

    return [("count_hits", lambda t, r, p: t.count_hits(r), count_dev),
            ("contains", lambda t, r, p: (t.contains(p, "nonzero"),), contains_dev),
            ("signed_distance", lambda t, r, p: t.signed_distance(p, "nonzero", closest=True), signed_dev)]


def _winding_scene(prec, k=6, seed=5, m=1500):
    """(tris, other, rays, points): a k^3 lattice of unit cubes at spacing 2, outward; `other` is the same triangles with both
    triangles of a random half of the faces reversed (the boxes are the same).  Rays and points lie in and around the lattice, so
    most rays cross several cubes and an outside point's NONZERO vote changes where one face of a crossed cube is reversed."""
    F = FT[prec]
    rng = np.random.default_rng(seed)
    c = np.stack(np.meshgrid(*[np.arange(k) * 2.0] * 3, indexing="ij"), -1).reshape(-1, 3)
    corners = np.array([[x, y, z] for x in (-0.5, 0.5) for y in (-0.5, 0.5) for z in (-0.5, 0.5)])
    unit = []
    for ax in range(3):
        for side in (-0.5, 0.5):
            q = corners[corners[:, ax] == side][[0, 1, 3, 2]]
            for t in (q[[0, 1, 2]], q[[0, 2, 3]]):
                n = np.cross(t[1] - t[0], t[2] - t[0])
                unit.append(t if n @ t.mean(axis=0) > 0 else t[[0, 2, 1]])
    tris = (c[:, None, None, :] + np.array(unit)[None]).reshape(-1, 3, 3)
    flip = np.repeat(rng.random(len(c) * 6) < 0.5, 2)
    other = tris.copy()
    other[flip] = other[flip][:, [0, 2, 1]]
    lo, hi = -1.0, 2.0 * (k - 1) + 1.0
    org = rng.uniform(lo - 5, hi + 5, (m, 3))
    rays = O.ray_new(org, rng.uniform(lo, hi, (m, 3)) - org, prec)
    pts = rng.uniform(lo, hi, (m, 3)).astype(F)
    return tris.reshape(-1, 9).astype(F), other.reshape(-1, 9).astype(F), rays, pts


@pytest.mark.parametrize("direction", ["own_to_torch", "torch_to_own", "torch_a_to_b", "torch_to_legacy"])
@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_crossing_calls_after_set_triangles_dev_then_switch(api, twin_ctx, direction, prec):
    """set_triangles_dev (a witness: it returns while P is still busy) replaces the cube faces by a set with half the faces' windings
    reversed: the boxes stay, front / back, the NONZERO vote and the sign change.  count_hits, contains and signed_distance, host and
    _dev forms, on Q equal a twin's host calls after the same change."""
    from bvh_b200 import capi
    from tests.test_gpu_stream_switch import Switch, _dev, _drain, _free, _same, _sfx

    tris, other, rays, pts = _winding_scene(prec)
    shapes = O.tri_aabbs(tris, prec)
    assert O.tri_aabbs(other, prec).tobytes() == shapes.tobytes()
    consumers = _crossing_consumers(prec)
    twin = api.Bvh.build(shapes, prec=prec, ctx=twin_ctx)
    sw = Switch(api, direction)
    tree = api.Bvh.build(shapes, prec=prec, ctx=sw.ctx)
    try:
        twin.set_triangles(tris)
        before = {name: host(twin, rays, pts) for name, host, _ in consumers}
        twin.set_triangles(other)
        after = {name: host(twin, rays, pts) for name, host, _ in consumers}
        tree.set_triangles(tris)
        launches = {name: prep(rays, pts) for name, _, prep in consumers}
        d_other = _dev(other)
        _drain()
        pending = sw.spin()
        capi.check(getattr(capi.lib(), f"bvhgpu_tree_set_triangles_dev_{_sfx(3, prec)}")(tree._h, C.c_void_p(d_other.data_ptr()), len(other)))
        assert not pending.query()
        sw.switch()
        reads = {}
        for name, host, _ in consumers:
            res = host(tree, rays, pts)
            reads[name] = (lambda r=res: r)
            reads[name + "_dev"] = launches[name](tree)
        _drain()
        for name, read in reads.items():
            base = name.removesuffix("_dev")
            assert not _same(before[base], after[base]), name
            assert _same(read(), after[base]), name
    finally:
        _free(tree, twin)
        sw.close()
