"""The k nearest shapes of a batch of points on the device (bvhgpu_knn_* / bvhgpu_knn_dev_*).  Every comparison is exact: indices
equal, distances bit-equal.
- against the brute force of tests/knnref.py in D = 2, 3, 4 and f32 / f64, on every dimref scene, the skew3000 scene, a ~90-level-deep
  tree and the large-coordinates family, for k across every bucket boundary (1, 2, 5, 16, 17, 32, 33, 64), with and without per-point limits
  (0, -1, -0, NaN, +inf, random, and radii whose square is a shape's key exactly), points with NaN / infinite coordinates included;
- at scale: the 120 k-triangle-box scene of BASELINE.json configs[1] and 20 k points of its seed chain, k = 8, against a torch brute
  force in the same operation order;
- the contract: empty and one-shape trees, k > n, refusals with the output buffers untouched, n = 0, the sticky failed build,
  NULL limits equal to +inf limits;
- the current boxes after refit, update_shapes (loose boxes and rebuilds), add_shapes and remove_shapes, in D = 2, 3 and 4;
- the device forms on a torch side stream equal the host forms (D = 3, 4); the 2-D rows equal the 3-D rows of the lifted scene and
  4-D rows with a constant fourth axis equal the 3-D rows; k = 1 distances equal bvhgpu_nearest_* distances on random scenes."""
import numpy as np
import pytest

from bvh_b200 import scenes
from oracle import oracle as O
from tests import adversarial as A, dimref, knnref as K
from tests.test_knn_cpu import limits, odd_points

pytestmark = pytest.mark.gpu
U32_MAX = 0xFFFFFFFF
FT = {"f32": np.float32, "f64": np.float64}
CASES = [(D, p) for D in (2, 3, 4) for p in ("f32", "f64")]
KS = (1, 2, 5, 16, 17, 32, 33, 64)


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A_

    return A_


def _cls(api, D):
    return {2: api.Bvh2, 3: api.Bvh, 4: api.Bvh4}[D]


def _aabbs(api, D, prec, mn, mx):
    from bvh_b200.dtypes import BY_PREC

    t = BY_PREC[prec] if D == 3 else _cls(api, D)._TABLE[prec]
    a = np.zeros(len(mn), dtype=t["aabb"])
    a["min"], a["max"] = mn, mx
    return a


def _build(api, D, prec, mn, mx):
    return _cls(api, D).build(_aabbs(api, D, prec, mn, mx), prec=prec)


def _check(bvh, mn, mx, pts, lim, ks=KS):
    """bvh.knn equals the brute force for every k, with no limit, with `lim`, and NULL equals all +inf."""
    for md in (None, lim):
        bs, bd = K.brute(mn, mx, pts, 64, md)
        for k in ks:
            s, d = bvh.knn(pts, k, md)
            assert np.array_equal(s, bs[:, :k]), (k, md is None)
            assert d.tobytes() == np.ascontiguousarray(bd[:, :k]).tobytes(), (k, md is None)
    s0, d0 = bvh.knn(pts, 5)
    s1, d1 = bvh.knn(pts, 5, np.inf)
    assert np.array_equal(s0, s1) and d0.tobytes() == d1.tobytes()


@pytest.mark.parametrize("scene", dimref.SCENES)
@pytest.mark.parametrize("D,prec", CASES)
def test_against_brute_force(api, D, prec, scene):
    F = FT[prec]
    rng = np.random.default_rng(10 * D + (prec == "f64") + 100 * dimref.SCENES.index(scene))
    mn, mx = dimref.scene(scene, 300, D, F, rng)
    pts = np.concatenate([dimref.points(mn, mx, 60, F, rng), odd_points(D, F)])
    bvh = _build(api, D, prec, mn, mx)
    _check(bvh, mn, mx, pts, limits(mn, mx, pts, rng))
    if scene == "random":                                      # k = 1 and Bvh::nearest_to agree on the distance here
        p = dimref.points(mn, mx, 200, F, rng)
        _, nd = bvh.nearest_to_batch(p)
        _, kd = bvh.knn(p, 1)
        assert kd[:, 0].tobytes() == nd.tobytes()
    bvh.free()


@pytest.mark.parametrize("D,prec", CASES)
def test_large_coordinates(api, D, prec):
    """The reference's cancellation, the concrete X / Y / p case in 3-D f32 included."""
    F = FT[prec]
    mn, mx, pts = A.large_coordinates(F, D)
    bvh = _build(api, D, prec, mn, mx)
    _check(bvh, mn, mx, pts, limits(mn, mx, pts, np.random.default_rng(1)), ks=(1, 2, 17, 64))
    bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_skew_and_deep_trees(api, prec):
    """The skew3000 scene of the parity tests (one far outlier per level), and 3 000 point boxes at geometric positions 1.05^i on one
    axis, whose f64 tree is about 90 levels deep: the walk climbs by parent links and keeps no stack."""
    from tests import scenes as S

    F = FT[prec]
    shapes = S.scene("skew3000", prec)
    c = np.zeros((3000, 3)); c[:, 0] = (1.05 if prec == "f64" else 1.02) ** np.arange(3000)
    c[:, 1:] = np.random.default_rng(4).uniform(-1, 1, (3000, 2))
    for mn, mx in ((shapes["min"], shapes["max"]), (c, c)):
        mn, mx = np.ascontiguousarray(mn).astype(F), np.ascontiguousarray(mx).astype(F)
        bvh = _build(api, 3, prec, mn, mx)
        if prec == "f64" and mn[1, 0] == F(1.05):
            assert max(_depths(bvh.nodes)) > 60
        pts = dimref.points(mn, mx, 60, F, np.random.default_rng(2))
        _check(bvh, mn, mx, pts, limits(mn, mx, pts, np.random.default_rng(3)))
        bvh.free()


def _depths(nodes):
    depth = np.zeros(len(nodes), dtype=np.int64)
    for i in range(1, len(nodes)):
        depth[i] = depth[int(nodes["parent"][i])] + 1
    return depth


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_configs1_scene_at_scale(api, prec):
    """120 k triangle boxes (create_n_cubes_aabbs(10 000)), 20 k points of the create_ray chain, k = 8: equal to a torch brute force
    (elementwise ops rounding once each, squares summed left to right, a stable sort by key then index) in chunks of points."""
    import torch

    F = FT[prec]
    aabbs = scenes.create_n_cubes_aabbs(10_000, prec)
    pts, _ = scenes.ray_endpoints(20_000, prec=prec)
    bvh = api.Bvh.build(aabbs, prec=prec)
    s, d = bvh.knn(pts, 8)
    dev = torch.device("cuda", 0)
    mn, mx = torch.from_numpy(np.ascontiguousarray(aabbs["min"])).to(dev), torch.from_numpy(np.ascontiguousarray(aabbs["max"])).to(dev)
    hs = (mx - mn) * 0.5
    c = mn + hs
    for a in range(0, len(pts), 128):
        p = torch.from_numpy(pts[a:a + 128]).to(dev)[:, None, :]
        q = torch.abs(p - c[None]) - hs[None]
        o = torch.where(q > 0, q, torch.zeros_like(q))
        d2 = o[..., 0] * o[..., 0] + o[..., 1] * o[..., 1] + o[..., 2] * o[..., 2]
        key, idx = torch.sort(d2, dim=1, stable=True)
        assert np.array_equal(s[a:a + 128], idx[:, :8].cpu().numpy().astype(np.uint32))
        assert d[a:a + 128].tobytes() == torch.sqrt(key[:, :8]).cpu().numpy().astype(F).tobytes()
    bvh.free()


@pytest.mark.parametrize("D,prec", CASES)
def test_contract(api, D, prec):
    from bvh_b200 import capi

    F = FT[prec]
    rng = np.random.default_rng(40 + D)
    mn, mx = dimref.scene("random", 50, D, F, rng)
    pts = dimref.points(mn, mx, 20, F, rng)
    bvh = _build(api, D, prec, mn, mx)
    s, d = bvh.knn(pts, 64)                                    # k > n: padding
    assert (s[:, 50:] == U32_MAX).all() and np.isinf(d[:, 50:]).all() and (s[:, :50] != U32_MAX).all()
    s, d = bvh.knn(pts[:0], 4)                                 # n = 0: a no-op
    assert s.shape == (0, 4)
    fn = getattr(capi.lib(), f"bvhgpu_knn_{bvh._d['suffix']}")
    P = api._ptr
    for k, pp, ps, pd, tree in ((0, pts, True, True, bvh._h), (65, pts, True, True, bvh._h), (4, None, True, True, bvh._h),
                                (4, pts, False, True, bvh._h), (4, pts, True, False, bvh._h), (4, pts, True, True, None)):
        s = np.full((len(pts), 65), 7, dtype=np.uint32)
        d = np.full((len(pts), 65), 7, dtype=F)
        st = fn(tree, P(pp) if pp is not None else None, len(pts), k, None, P(s) if ps else None, P(d) if pd else None)
        assert st == capi.ERR_INVALID and (s == 7).all() and (d == 7).all(), (k, pp is None, ps, pd, tree is None)
    bvh.free()
    for n in (0, 1):                                           # empty tree: padding; one shape: its own box decides
        bvh = _build(api, D, prec, mn[:n], mx[:n])
        s, d = bvh.knn(pts, 3, np.full(len(pts), 60, dtype=F))
        bs, bd = K.brute(mn[:n], mx[:n], pts, 3, np.full(len(pts), 60, dtype=F))
        assert np.array_equal(s, bs) and d.tobytes() == bd.tobytes()
        bvh.free()


def test_failed_build_is_sticky(api):
    import torch

    from bvh_b200 import capi

    shapes, _ = O.create_n_cubes(100, want_tris=True)
    shapes = shapes.copy()
    shapes["min"][33][1] = np.nan
    d = torch.from_numpy(shapes.view(np.uint8).reshape(-1)).cuda()
    torch.cuda.synchronize()
    bvh = api.Bvh.build_dev(d.data_ptr(), len(shapes))
    out_s = torch.zeros(10 * 4, dtype=torch.int32, device="cuda")
    out_d = torch.zeros(10 * 4, dtype=torch.float32, device="cuda")
    pts = torch.zeros(30, dtype=torch.float32, device="cuda")
    for _ in range(2):
        with pytest.raises(capi.BvhGpuError) as e:
            bvh.knn(np.zeros((10, 3), dtype=np.float32), 4)
        assert e.value.status == capi.ERR_NAN
        with pytest.raises(capi.BvhGpuError) as e:
            bvh.knn_dev(pts.data_ptr(), 10, 4, 0, out_s.data_ptr(), out_d.data_ptr())
        assert e.value.status == capi.ERR_NAN
    bvh.free()


@pytest.mark.parametrize("D,prec", CASES)
def test_current_boxes_after_refit_update_add_and_remove(api, D, prec):
    F = FT[prec]
    rng = np.random.default_rng(60 + D)
    mn, mx = dimref.scene("random", 400, D, F, rng)
    pts = np.concatenate([dimref.points(mn, mx, 40, F, rng), odd_points(D, F)])
    aabbs = _aabbs(api, D, prec, mn, mx)
    bvh = _cls(api, D).build(aabbs, prec=prec)

    def check(a):
        lim = limits(a["min"], a["max"], pts, rng)
        _check(bvh, np.ascontiguousarray(a["min"]), np.ascontiguousarray(a["max"]), pts, lim, ks=(1, 17, 64))

    check(aabbs)
    shift = rng.uniform(-3, 3, (len(aabbs), D)).astype(F)
    aabbs["min"], aabbs["max"] = (aabbs["min"] + shift).astype(F), (aabbs["max"] + shift).astype(F)
    bvh.refit(aabbs)
    check(aabbs)
    for growth in (0.0, 1.5):                                  # loose boxes (refit of the changed paths only), then rebuilds
        changed = rng.choice(len(aabbs), 60, replace=False)
        shift = rng.uniform(-40, 40, (60, D)).astype(F)
        aabbs["min"][changed] = (aabbs["min"][changed] + shift).astype(F)
        aabbs["max"][changed] = (aabbs["max"][changed] + shift).astype(F)
        bvh.update_shapes(changed, aabbs, max_growth=growth)
        check(aabbs)
    nmn, nmx = dimref.scene("random", 40, D, F, rng)
    new = _aabbs(api, D, prec, nmn, nmx)
    bvh.add_shapes(new)
    aabbs = np.concatenate([aabbs, new])
    check(aabbs)
    gone = rng.choice(len(aabbs), 70, replace=False)
    moves = bvh.remove_shapes(gone)
    after = aabbs.copy()
    for new_i, old_i in moves:
        after[new_i] = aabbs[old_i]
    check(after[: len(aabbs) - len(gone)])
    bvh.free()


@pytest.mark.parametrize("D,prec", [(3, "f32"), (3, "f64"), (4, "f32"), (4, "f64")])
def test_knn_dev_on_a_side_stream_equals_the_host_form(api, D, prec):
    import torch

    F = FT[prec]
    rng = np.random.default_rng(5 + D)
    mn, mx = dimref.scene("random", 3000, D, F, rng)
    pts = dimref.points(mn, mx, 5000, F, rng)
    lim = (rng.uniform(0, 1, len(pts)) * 30).astype(F)
    bvh = _build(api, D, prec, mn, mx)
    dev = torch.device("cuda", 0)
    side = torch.cuda.Stream(device=dev)
    for k, md in ((1, None), (8, lim), (40, lim)):
        hs, hd = bvh.knn(pts, k, md)
        with torch.cuda.stream(side):
            d_p = torch.from_numpy(pts).to(dev)
            d_r = torch.from_numpy(md).to(dev) if md is not None else None
            d_s = torch.full((len(pts) * k,), 7, dtype=torch.int32, device=dev)
            d_d = torch.full((len(pts) * k,), 7, dtype=torch.float32 if prec == "f32" else torch.float64, device=dev)
            bvh.ctx.set_stream(side.cuda_stream)
            try:
                bvh.knn_dev(d_p.data_ptr(), len(pts), k, d_r.data_ptr() if d_r is not None else 0, d_s.data_ptr(), d_d.data_ptr())
            finally:
                bvh.ctx.set_stream(None)
            side.synchronize()
        assert np.array_equal(d_s.cpu().numpy().view(np.uint32).reshape(-1, k), hs)
        assert d_d.cpu().numpy().tobytes() == hd.tobytes()
        assert (hs != U32_MAX).any() and (md is None or (hs == U32_MAX).any())
    bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_lifts(api, prec):
    """2-D rows equal the 3-D rows of the scene lifted to z = 0; 4-D rows with a constant fourth axis equal the 3-D rows."""
    F = FT[prec]
    rng = np.random.default_rng(70)
    mn2, mx2 = dimref.scene("random", 500, 2, F, rng)
    p2 = np.concatenate([dimref.points(mn2, mx2, 100, F, rng), odd_points(2, F)])
    lim = limits(mn2, mx2, p2, rng)
    z = lambda a, v: np.concatenate([a, np.full((len(a), 1), v, dtype=F)], axis=1).astype(F)   # noqa: E731
    b2, b3 = _build(api, 2, prec, mn2, mx2), _build(api, 3, prec, z(mn2, 0), z(mx2, 0))
    b4 = _build(api, 4, prec, z(z(mn2, 0), 3.5), z(z(mx2, 0), 3.5))
    for k in (1, 9, 64):
        for md in (None, lim):
            s2, d2 = b2.knn(p2, k, md)
            s3, d3 = b3.knn(z(p2, 0), k, md)
            s4, d4 = b4.knn(z(z(p2, 0), 3.5), k, md)
            assert np.array_equal(s2, s3) and d2.tobytes() == d3.tobytes()
            assert np.array_equal(s4, s3) and d4.tobytes() == d3.tobytes()
    for b in (b2, b3, b4):
        b.free()
