"""Crossing counts, point-in-mesh and signed distance on the device (bvhgpu_count_hits_*, bvhgpu_contains_points_*,
bvhgpu_signed_distance_* and their _dev forms), f32 and f64, against the restatement of tests/crossings.py:
- count_hits without a limit equals the loop over traverse_batch's CSR with both windings, on the configs[1] 120 k-triangle cube scene
  (10^5 rays aimed at its cubes) and on Sponza (an open mesh), host form and _dev with FULL and OD rays; the difference to the brute
  force over every triangle is reported, and the device never counts more;
- with per-ray and scalar limits (0, -0, NaN, +inf, random) the counts equal the limited-walk model of tests/crosswalk.py on every
  row and the loop on every bounded row, never exceed the loop elsewhere, and the number of unbounded rows is reported;
- contains equals the vote on the device's own counts and on restated counts, and the truth on the cube scene, an icosphere, a torus
  and (EVEN_ODD) an icosphere with flipped triangles; signed_distance is knn_triangles(k = 1) with the sign of contains;
- the contract: empty tree, n = 1, n = 0, NaN points and rays, refusals that write nothing, the sticky build before missing triangles,
  triangles after add_shapes / remove_shapes / a refit with stale triangles, batch sizes at the grid edges, the _dev forms on a
  non-default stream without host synchronisation."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import crossings as X
from tests import crosswalk as W
from tests.test_crossings_cpu import cube_points, flip_some, sphere_points, torus_points
from tests.test_knn_triangles_cpu import sponza_tris

pytestmark = pytest.mark.gpu
U32_MAX = 0xFFFFFFFF
FT = {"f32": np.float32, "f64": np.float64}
RULES = {"even_odd": X.EVEN_ODD, "nonzero": X.NONZERO}


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A_

    return A_


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({np.float32: np.uint32, np.float64: np.uint64}[a.dtype.type]) if a.dtype.type in (np.float32, np.float64) else a


def _mesh(api, tris, prec):
    tris = np.ascontiguousarray(tris, dtype=FT[prec]).reshape(-1, 3, 3)
    shapes = O.tri_aabbs(tris, prec)
    bvh = api.Bvh.build(shapes, prec=prec)
    bvh.set_triangles(tris.reshape(-1, 9))
    return bvh, shapes, tris


def _dev_counts(bvh, rays, tmax, layout, prec):
    import torch

    from bvh_b200 import capi

    n = len(rays)
    src = rays if layout == capi.RAYS_FULL else np.ascontiguousarray(np.concatenate([rays["origin"], rays["direction"]], axis=1))
    d_rays = torch.from_numpy(np.frombuffer(src.tobytes(), dtype=np.uint8).copy()).cuda()
    tm = None if tmax is None else np.array(np.broadcast_to(np.asarray(tmax, dtype=FT[prec]), (n,)))
    d_tm = None if tm is None else torch.from_numpy(tm).cuda()
    f = torch.full((n,), 7, dtype=torch.int32, device="cuda")
    b = torch.full((n,), 7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    bvh.count_hits_dev(d_rays.data_ptr(), n, d_tm.data_ptr() if d_tm is not None else 0, f.data_ptr(), b.data_ptr(), layout=layout)
    bvh.ctx.synchronize()
    return f.cpu().numpy().view(np.uint32), b.cpu().numpy().view(np.uint32)


def _forms(bvh, rays, tmax, prec):
    from bvh_b200 import capi

    return [bvh.count_hits(rays, tmax)] + [_dev_counts(bvh, rays, tmax, lay, prec) for lay in (capi.RAYS_FULL, capi.RAYS_OD)]


def _cube_scene(api, prec, n_rays, seed=8):
    from bvh_b200 import scenes

    F = FT[prec]
    tris = scenes.create_n_cubes_tris(10_000, prec)
    bvh, shapes, tris = _mesh(api, tris, prec)
    rng = np.random.default_rng(seed)
    tgt = shapes["min"][rng.integers(0, len(shapes), n_rays)].astype(np.float64) + rng.uniform(0, 1, (n_rays, 3))
    org = rng.uniform(-1.1e5, 1.1e5, (n_rays, 3))
    rays = api.Ray.new(org.astype(F), (tgt - org).astype(F), prec=prec)
    return bvh, shapes, tris, rays


def _sponza_scene(api, prec, n_rays, seed=9):
    F = FT[prec]
    bvh, shapes, tris = _mesh(api, sponza_tris(F), prec)
    rng = np.random.default_rng(seed)
    lo, hi = shapes["min"].min(axis=0).astype(np.float64), shapes["max"].max(axis=0).astype(np.float64)
    org = rng.uniform(lo, hi, (n_rays, 3))
    rays = api.Ray.new(org.astype(F), rng.normal(0, 1, (n_rays, 3)).astype(F), prec=prec)
    return bvh, shapes, tris, rays


@pytest.fixture(scope="module", params=[("cubes", "f32"), ("cubes", "f64"), ("sponza", "f32"), ("sponza", "f64")], ids=lambda p: "-".join(p))
def scene(api, request):
    name, prec = request.param
    bvh, shapes, tris, rays = (_cube_scene(api, prec, 100_000) if name == "cubes" else _sponza_scene(api, prec, 20_000))
    off, hits = bvh.traverse_batch(rays)
    yield name, prec, bvh, shapes, tris, rays, off, hits
    bvh.free()


def test_count_hits_equals_the_loop_over_traverse(scene):
    name, prec, bvh, shapes, tris, rays, off, hits = scene
    want = X.counts_csr(rays, tris, off, hits)
    assert want[0].sum() > 1000 and want[1].sum() > 1000, name
    for i, got in enumerate(_forms(bvh, rays, None, prec)):
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), (name, i)
    # the brute force over every triangle on a sample: reported, and never below the device
    pick = np.random.default_rng(1).choice(len(rays), 200, replace=False)
    bf = X.counts_brute(rays[pick], tris)
    diff = int((bf[0] != want[0][pick]).sum() + (bf[1] != want[1][pick]).sum())
    assert np.all(want[0][pick] <= bf[0]) and np.all(want[1][pick] <= bf[1])
    print(f"{name} {prec}: {len(rays)} rays, {int(want[0].sum())} front / {int(want[1].sum())} back crossings, "
          f"brute force differs on {diff} of {2 * len(pick)} sampled counts")


def _limit_families(rays, bvh, F, rng):
    d = bvh.closest_hit(rays, triangles=True)[1]
    fin = np.isfinite(d)
    scale = d[fin].max() if fin.any() else F(1)
    rnd = (rng.uniform(0, 3, len(rays)) * np.where(fin, d, scale)).astype(F)
    return {"random": rnd, "d*": d.astype(F), "zero": F(0), "-zero": F(-0.0), "nan": F(np.nan), "inf": F(np.inf), "scalar": F(scale / 2)}


def test_count_hits_with_limits_on_bounded_rows(scene):
    name, prec, bvh, shapes, tris, rays, off, hits = scene
    F = FT[prec]
    sub = slice(0, 20_000)
    r = rays[sub]
    o2, h2 = bvh.traverse_batch(r)
    cand = W.candidates(bvh.nodes, shapes, r)
    for lname, tm in _limit_families(r, bvh, F, np.random.default_rng(4)).items():
        want = X.counts_csr(r, tris, o2, h2, tm)
        ok = X.bounded_rows(r, tris, bvh.nodes, shapes, o2, h2, tm)
        model = W.model(bvh.nodes, shapes, tris, r, tm, cand)
        for i, got in enumerate(_forms(bvh, r, tm, prec)):
            assert np.array_equal(got[0], model[0]) and np.array_equal(got[1], model[1]), (name, lname, i)
            assert np.array_equal(got[0][ok], want[0][ok]) and np.array_equal(got[1][ok], want[1][ok]), (name, lname, i)
            assert np.all(got[0] <= want[0]) and np.all(got[1] <= want[1]), (name, lname, i)
        if lname in ("zero", "-zero", "nan"):
            assert not want[0].any() and not want[1].any()
        if lname == "inf":
            nolim = X.counts_csr(r, tris, o2, h2)
            assert np.array_equal(want[0], nolim[0]) and np.array_equal(want[1], nolim[1])
        print(f"{name} {prec} tmax={lname}: {int((~ok).sum())} unbounded rows of {len(r)}")


def _contains_checks(bvh, tris, points, prec, truth=None, rules=("even_odd", "nonzero")):
    """contains equals the vote on the device's own counts and on restated counts (traverse_batch's CSR), and the truth if given."""
    F = FT[prec]
    pr = X.point_rays(points, F)
    dev_counts = bvh.count_hits(pr)
    o, h = bvh.traverse_batch(pr)
    restated = X.counts_csr(pr, tris, o, h)
    assert np.array_equal(dev_counts[0], restated[0]) and np.array_equal(dev_counts[1], restated[1])
    for rule in rules:
        got = bvh.contains(points, rule)
        assert np.array_equal(got, X.vote(*dev_counts, RULES[rule])), rule
        assert np.array_equal(got, X.vote(*restated, RULES[rule])), rule
        if truth is not None:
            assert np.array_equal(got, truth), (rule, int((got != truth).sum()))
    return restated


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_contains_on_analytic_meshes(api, prec):
    from bvh_b200 import scenes

    F = FT[prec]
    rng = np.random.default_rng(21)
    cubes = scenes.create_n_cubes_tris(2000, prec)
    ico = X.icosphere(3, F)
    meshes = [("cubes", cubes, *cube_points(cubes, F, rng, 5000), ("even_odd",)),
              ("icosphere", ico, *sphere_points(rng, 5000), ("even_odd", "nonzero")),
              ("torus", X.torus(F=F), *torus_points(rng, 5000), ("even_odd", "nonzero"))]
    flipped, _ = flip_some(ico, rng, 0.5)
    ps, ts = sphere_points(rng, 5000)
    meshes.append(("flipped icosphere", flipped, ps, ts, ("even_odd",)))
    for name, tris, p, truth, rules in meshes:
        bvh, _, tr = _mesh(api, tris, prec)
        try:
            assert truth.sum() > 100 and (~truth).sum() > 100, name
            _contains_checks(bvh, tr, p.astype(F), prec, truth, rules)
            if name == "flipped icosphere":             # NONZERO needs oriented shells: it is wrong on some outside points here
                wrong = bvh.contains(p.astype(F), "nonzero") != truth
                assert wrong.any() and not truth[wrong].any(), name
        finally:
            bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_contains_and_signed_distance_on_the_scenes(api, prec):
    """The vote on the 120 k-triangle cube scene and on Sponza (open: the vote is whatever its rays count), and signed_distance:
    shape, |dist| and closest are knn_triangles(k = 1) bit for bit, the sign is contains'."""
    F = FT[prec]
    rng = np.random.default_rng(5)
    for build in (_cube_scene, _sponza_scene):
        bvh, shapes, tris, rays = build(api, prec, 10)
        try:
            if build is _cube_scene:
                p, truth = cube_points(tris.reshape(-1, 9), F, rng, 20_000)
            else:
                lo, hi = shapes["min"].min(axis=0), shapes["max"].max(axis=0)
                p, truth = rng.uniform(lo, hi, (20_000, 3)).astype(F), None
            _contains_checks(bvh, tris, p, prec, truth, ("even_odd",) if truth is not None else ("even_odd", "nonzero"))
            s, d, q = bvh.knn_triangles(p, 1, closest=True)
            for rule in ("even_odd", "nonzero"):
                inside = bvh.contains(p, rule)
                gs, gd, gq = bvh.signed_distance(p, rule, closest=True)
                assert np.array_equal(gs, s[:, 0]) and np.array_equal(_bits(np.abs(gd)), _bits(d[:, 0])) and np.array_equal(_bits(gq), _bits(q[:, 0]))
                assert np.array_equal(_bits(gd), _bits(X.signed(s[:, 0], d[:, 0], inside))), rule
                assert np.array_equal(np.signbit(gd), inside), rule
                gs2, gd2 = bvh.signed_distance(p, rule)
                assert np.array_equal(gs2, gs) and np.array_equal(_bits(gd2), _bits(gd))
            assert bvh.contains(p).sum() > 100
        finally:
            bvh.free()


def _dev_points(p):
    import torch

    return torch.from_numpy(np.ascontiguousarray(p)).cuda()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_edges(api, prec):
    import torch

    F = FT[prec]
    ico = X.icosphere(1, F)
    # empty tree: zeros, +inf / INVALID / NaN
    b0 = api.Bvh.build(O.tri_aabbs(ico[:0], prec), prec=prec)
    rays = O.ray_new(np.zeros((5, 3)), np.ones((5, 3)), prec)
    f, b = b0.count_hits(rays)
    assert not f.any() and not b.any()
    assert not b0.contains(np.zeros((7, 3), dtype=F)).any()
    s, d, q = b0.signed_distance(np.zeros((7, 3), dtype=F), closest=True)
    assert np.all(s == U32_MAX) and np.all(np.isposinf(d)) and np.all(np.isnan(q))
    b0.free()
    # n = 1: the shape's own box decides
    one = np.array([[[0, 0, 0], [1, 0, 0], [0, 1, 0]]], dtype=F)
    b1, shapes1, t1 = _mesh(api, one, prec)
    o = np.array([[0.25, 0.25, 2], [0.25, 0.25, -2], [5, 5, 2]])
    r1 = O.ray_new(o, np.array([[0, 0, -1], [0, 0, 1], [0, 0, -1]]), prec)
    f, b = b1.count_hits(r1)
    assert f.tolist() == [1, 0, 0] and b.tolist() == [0, 1, 0]
    want = X.counts_csr(r1, t1, *b1.traverse_batch(r1))
    assert np.array_equal(f, want[0]) and np.array_equal(b, want[1])
    b1.free()
    # n = 0 calls, NaN points and rays
    bvh, _, tr = _mesh(api, ico, prec)
    assert bvh.count_hits(rays[:0])[0].shape == (0,) and bvh.contains(np.zeros((0, 3), dtype=F)).shape == (0,)
    assert bvh.signed_distance(np.zeros((0, 3), dtype=F))[0].shape == (0,)
    p = np.array([[0, 0, 0], [np.nan, 0, 0], [0, 0, np.nan], [3, 3, 3]], dtype=F)
    for rule in ("even_odd", "nonzero"):
        assert bvh.contains(p, rule).tolist() == [True, False, False, False]
    nan_rays = O.ray_new(np.array([[np.nan, 0, 0], [0, 0, 0]]), np.array([[1, 0.1, 0.2], [np.nan, 1, 0]]), prec)
    f, b = bvh.count_hits(nan_rays)
    want = X.counts_csr(nan_rays, tr, *bvh.traverse_batch(nan_rays))
    assert np.array_equal(f, want[0]) and np.array_equal(b, want[1]) and not f.any() and not b.any()
    # a point at the centre is at depth -(distance); a point on nothing keeps its sign positive
    s, d = bvh.signed_distance(p)
    assert d[0] < 0 and d[3] > 0 and s[1] == U32_MAX and np.isposinf(d[1])
    torch.cuda.synchronize()
    bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_refusals_write_nothing(api, prec):
    import torch

    from bvh_b200 import capi

    F = FT[prec]
    L = capi.lib()
    suf = f"{prec}x3"
    ico = X.icosphere(1, F)
    bvh = api.Bvh.build(O.tri_aabbs(ico, prec), prec=prec)             # triangles never set
    n = 50
    rays = O.ray_new(np.zeros((n, 3)), np.ones((n, 3)), prec)
    pts = np.zeros((n, 3), dtype=F)
    g_u32 = np.full(n + 8, 7, dtype=np.uint32)
    g_u32b = np.full(n + 8, 7, dtype=np.uint32)
    g_u8 = np.full(n + 8, 7, dtype=np.uint8)
    g_f = np.full(5 * n + 8, 7, dtype=F)
    cnt, cdev = getattr(L, f"bvhgpu_count_hits_{suf}"), getattr(L, f"bvhgpu_count_hits_dev_{suf}")
    con, condev = getattr(L, f"bvhgpu_contains_points_{suf}"), getattr(L, f"bvhgpu_contains_points_dev_{suf}")
    sd, sddev = getattr(L, f"bvhgpu_signed_distance_{suf}"), getattr(L, f"bvhgpu_signed_distance_dev_{suf}")
    u, ub, u8, fl = g_u32.ctypes.data, g_u32b.ctypes.data, g_u8.ctypes.data, g_f.ctypes.data
    d_rays = torch.from_numpy(rays.view(np.uint8).copy()).cuda()
    d_pts = torch.from_numpy(pts).cuda()
    d_out = torch.full((4 * n + 8,), 7, dtype=torch.int32, device="cuda")
    do = d_out.data_ptr()
    E = capi.ERR_INVALID
    refused = [
        cnt(bvh._h, rays.ctypes.data, n, None, u, ub),                                        # missing triangles
        cnt(None, rays.ctypes.data, n, None, u, ub), cnt(bvh._h, None, n, None, u, ub), cnt(bvh._h, rays.ctypes.data, n, None, None, ub),
        cnt(bvh._h, rays.ctypes.data, n, None, u, None), cnt(bvh._h, rays.ctypes.data, 1 << 31, None, u, ub),
        cdev(bvh._h, d_rays.data_ptr(), 2, n, None, do, do + 4 * n),                          # unknown layout
        cdev(bvh._h, d_rays.data_ptr(), capi.RAYS_FULL, n, None, do, do + 4 * n),             # missing triangles
        cdev(bvh._h, None, capi.RAYS_FULL, n, None, do, do), cdev(bvh._h, d_rays.data_ptr(), capi.RAYS_OD, 1 << 31, None, do, do),
        con(bvh._h, pts.ctypes.data, n, 0, u8), con(bvh._h, pts.ctypes.data, n, 2, u8), con(bvh._h, pts.ctypes.data, n, -1, u8),
        con(bvh._h, None, n, 0, u8), con(bvh._h, pts.ctypes.data, n, 0, None), con(bvh._h, pts.ctypes.data, 1 << 31, 0, u8),
        condev(bvh._h, d_pts.data_ptr(), n, 0, do), condev(bvh._h, d_pts.data_ptr(), n, 5, do), condev(bvh._h, None, n, 0, do),
        sd(bvh._h, pts.ctypes.data, n, 0, u, fl, fl + n * g_f.itemsize), sd(bvh._h, pts.ctypes.data, n, 3, u, fl, None),
        sd(bvh._h, pts.ctypes.data, n, 0, None, fl, None), sd(bvh._h, pts.ctypes.data, n, 0, u, None, None),
        sddev(bvh._h, d_pts.data_ptr(), n, 0, do, do + 4 * n, None), sddev(bvh._h, d_pts.data_ptr(), n, 2, do, do + 4 * n, None),
        sddev(bvh._h, d_pts.data_ptr(), n, 0, None, do, None),
    ]
    assert all(rc == E for rc in refused), refused
    torch.cuda.synchronize()
    assert np.all(g_u32 == 7) and np.all(g_u32b == 7) and np.all(g_u8 == 7) and np.all(g_f == 7)
    assert np.all(d_out.cpu().numpy() == 7)
    # n = 0 with everything null is a no-op for every form
    assert cnt(bvh._h, None, 0, None, None, None) == capi.OK and cdev(bvh._h, None, capi.RAYS_OD, 0, None, None, None) == capi.OK
    assert con(bvh._h, None, 0, 0, None) == capi.OK and condev(bvh._h, None, 0, 1, None) == capi.OK
    assert sd(bvh._h, None, 0, 0, None, None, None) == capi.OK and sddev(bvh._h, None, 0, 0, None, None, None) == capi.OK
    # missing triangles after add_shapes dropped them
    bvh.set_triangles(ico)
    bvh.count_hits(rays)
    bvh.add_shapes(O.tri_aabbs(ico[:2], prec))
    for call in (lambda: bvh.count_hits(rays), lambda: bvh.contains(pts), lambda: bvh.signed_distance(pts)):
        with pytest.raises(capi.BvhGpuError) as e:
            call()
        assert e.value.status == E
    bvh.free()


def test_failed_build_is_sticky_before_missing_triangles(api):
    import torch

    from bvh_b200 import capi

    shapes, _ = O.create_n_cubes(100, want_tris=True)
    shapes = shapes.copy()
    shapes["min"][33][1] = np.nan
    d = torch.from_numpy(shapes.view(np.uint8).reshape(-1)).cuda()
    torch.cuda.synchronize()
    bvh = api.Bvh.build_dev(d.data_ptr(), len(shapes))
    rays = O.ray_new(np.zeros((10, 3)), np.ones((10, 3)))
    pts = np.zeros((10, 3), dtype=np.float32)
    for _ in range(2):
        for call in (lambda: bvh.count_hits(rays), lambda: _dev_counts(bvh, rays, None, capi.RAYS_FULL, "f32"), lambda: bvh.contains(pts),
                     lambda: bvh.signed_distance(pts)):
            with pytest.raises(capi.BvhGpuError) as e:
                call()
            assert e.value.status == capi.ERR_NAN
    bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_triangles_follow_remove_and_stale_refit(api, prec):
    F = FT[prec]
    rng = np.random.default_rng(31)
    tris = np.concatenate([X.icosphere(2, F), X.torus(F=F) * F(0.5) + F(3)])
    bvh, shapes, tr = _mesh(api, tris, prec)
    p = np.concatenate([rng.uniform(-1.5, 1.5, (2000, 3)), rng.uniform(2, 4, (2000, 3))]).astype(F)
    gone = rng.choice(len(shapes), len(shapes) // 7, replace=False)
    moves = bvh.remove_shapes(gone)
    s2, t2 = shapes.copy(), tr.copy()
    for new_i, old_i in moves:
        s2[new_i], t2[new_i] = shapes[old_i], tr[old_i]
    m = len(shapes) - len(gone)
    s2, t2 = s2[:m], t2[:m]
    _contains_checks(bvh, t2, p, prec)
    rays = X.point_rays(p[:500], F)
    want = X.counts_csr(rays, t2, *bvh.traverse_batch(rays))
    got = bvh.count_hits(rays)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    # refit the boxes to moved triangles but keep the old triangles: the walk reads the stale triangles through the new boxes
    t3 = (t2 + F(0.25)).astype(F)
    bvh.refit(O.tri_aabbs(t3, prec))
    want = X.counts_csr(rays, t2, *bvh.traverse_batch(rays))
    got = bvh.count_hits(rays)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    bvh.set_triangles(t3)
    _contains_checks(bvh, t3, p, prec)
    bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_batch_sizes_at_the_grid_edges(api, prec):
    import torch

    F = FT[prec]
    bvh, _, tr = _mesh(api, X.icosphere(2, F), prec)
    rng = np.random.default_rng(41)
    allp = rng.uniform(-1.5, 1.5, (400, 3)).astype(F)
    full_inside = bvh.contains(allp)
    full_sd = bvh.signed_distance(allp)
    rays = X.point_rays(allp, F)
    full_counts = bvh.count_hits(rays)
    for n in (0, 1, 2, 127, 128, 129, 255, 256, 257, 3 * 43 - 1, 3 * 43 + 1, 384, 385):
        inside = bvh.contains(allp[:n])
        assert np.array_equal(inside, full_inside[:n]), n
        s, d = bvh.signed_distance(allp[:n])
        assert np.array_equal(s, full_sd[0][:n]) and np.array_equal(_bits(d), _bits(full_sd[1][:n])), n
        f, b = bvh.count_hits(rays[:n])
        assert np.array_equal(f, full_counts[0][:n]) and np.array_equal(b, full_counts[1][:n]), n
        # guarded device outputs: nothing past n is written
        d_p = _dev_points(allp[:n] if n else allp[:1])
        g = torch.full((n + 64,), 9, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        bvh.contains_dev(d_p.data_ptr(), n, g.data_ptr())
        bvh.ctx.synchronize()
        gh = g.cpu().numpy()
        assert np.array_equal(gh[:n].astype(bool), full_inside[:n]) and np.all(gh[n:] == 9), n
    bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_dev_forms_on_a_side_stream(api, prec):
    """Every _dev form on a non-default stream installed with set_stream, no host synchronisation between the calls; results equal the
    host forms."""
    import torch

    F = FT[prec]
    rng = np.random.default_rng(51)
    bvh, _, tr = _mesh(api, X.torus(F=F), prec)
    p = rng.uniform([-1.6, -1.6, -0.6], [1.6, 1.6, 0.6], (30_000, 3)).astype(F)
    rays = X.point_rays(p[:10_000], F)
    tm = rng.uniform(0, 3, len(rays)).astype(F)
    hf, hb = bvh.count_hits(rays, tm)
    hin = bvh.contains(p, "nonzero")
    hs, hd, hq = bvh.signed_distance(p, "nonzero", closest=True)
    dev = torch.device("cuda", 0)
    side = torch.cuda.Stream(device=dev)
    dt = torch.float32 if prec == "f32" else torch.float64
    with torch.cuda.stream(side):
        d_rays = torch.from_numpy(rays.view(np.uint8).copy()).to(dev)
        d_tm = torch.from_numpy(tm).to(dev)
        d_p = torch.from_numpy(p).to(dev)
        f = torch.full((len(rays),), 7, dtype=torch.int32, device=dev)
        b = torch.full((len(rays),), 7, dtype=torch.int32, device=dev)
        ins = torch.full((len(p),), 7, dtype=torch.uint8, device=dev)
        s = torch.full((len(p),), 7, dtype=torch.int32, device=dev)
        d = torch.full((len(p),), 7, dtype=dt, device=dev)
        q = torch.full((3 * len(p),), 7, dtype=dt, device=dev)
        bvh.ctx.set_stream(side.cuda_stream)
        try:
            bvh.count_hits_dev(d_rays.data_ptr(), len(rays), d_tm.data_ptr(), f.data_ptr(), b.data_ptr())
            bvh.contains_dev(d_p.data_ptr(), len(p), ins.data_ptr(), "nonzero")
            bvh.signed_distance_dev(d_p.data_ptr(), len(p), s.data_ptr(), d.data_ptr(), q.data_ptr(), "nonzero")
        finally:
            bvh.ctx.set_stream(None)
        side.synchronize()
    assert np.array_equal(f.cpu().numpy().view(np.uint32), hf) and np.array_equal(b.cpu().numpy().view(np.uint32), hb)
    assert np.array_equal(ins.cpu().numpy().astype(bool), hin)
    assert np.array_equal(s.cpu().numpy().view(np.uint32), hs) and np.array_equal(_bits(d.cpu().numpy()), _bits(hd))
    assert np.array_equal(_bits(q.cpu().numpy().reshape(-1, 3)), _bits(hq))
    assert hin.sum() > 100 and (~hin).sum() > 100 and hf.sum() > 0
    bvh.free()
