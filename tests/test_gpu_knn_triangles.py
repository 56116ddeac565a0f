"""The k nearest triangles of a batch of points on the device (bvhgpu_knn_triangles_* / _dev_*).  Every comparison is exact: indices
equal, distances and closest points bit-equal to tests/knntri.py's brute force (whose keys equal the oracle's
Triangle::distance_squared, tests/test_knn_triangles_cpu.py), on scenes where every triangle is bounded (DESIGN.md section 4.17):
- cubes, Sponza, random soups and every adversarial family, f32 and f64, k across every bucket boundary, with and without per-point
  limits (0, -0, -1, NaN, +inf, random, radii whose square is a key exactly), points with NaN / infinite coordinates;
- empty and one-triangle trees, refusals with the outputs untouched, a sticky failed build;
- after remove_shapes (the triangles follow their shapes), and after refit with the triangles set again;
- the _dev form on a side stream equals the host form;
- k = 1 distances equal nearest_triangles' where that returns the brute-force minimum (cubes, Sponza);
- the 120 k-triangle configs[1] scene on a few thousand points."""
import os

import numpy as np
import pytest

from bvh_b200 import scenes
from oracle import oracle as O
from tests import knntri as KT
from tests.test_knn_triangles_cpu import limits, sponza_tris

pytestmark = pytest.mark.gpu
U32_MAX = 0xFFFFFFFF
FT = {"f32": np.float32, "f64": np.float64}
KS = (1, 4, 5, 8, 9, 16, 17, 32, 33, 64)


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A_

    return A_


def _build(api, tris, prec):
    bvh = api.Bvh.build(O.tri_aabbs(tris, prec), prec=prec)
    bvh.set_triangles(tris)
    return bvh


def _check(bvh, tris, pts, lim, ks=KS):
    mn, mx = KT.boxes(tris)
    assert all(KT.bounded(p, tris, mn, mx).all() for p in pts)
    for md in (None, lim):
        bs, bd, bq = KT.brute(tris, pts, 64, md)
        for k in ks:
            s, d, q = bvh.knn_triangles(pts, k, md, closest=True)
            assert np.array_equal(s, bs[:, :k]), (k, md is None)
            assert d.tobytes() == np.ascontiguousarray(bd[:, :k]).tobytes(), (k, md is None)
            assert q.tobytes() == np.ascontiguousarray(bq[:, :k]).tobytes(), (k, md is None)
            s2, d2 = bvh.knn_triangles(pts, k, md)
            assert np.array_equal(s2, s) and d2.tobytes() == d.tobytes()


def _scene(name, F, rng):
    if name == "cubes":
        return scenes.create_n_cubes_tris(60, "f32" if F == np.float32 else "f64"), None
    if name == "soup":
        return KT.soup(F, 300, rng), None
    return KT.family(name, F)


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("name", ["cubes", "soup"] + sorted(KT.FAMILIES))
def test_against_brute_force(api, name, prec):
    F = FT[prec]
    rng = np.random.default_rng(31)
    tris, pts = _scene(name, F, rng)
    if pts is None:
        pts = KT.near_points(tris, 60, rng)
    pts = np.concatenate([pts, KT.odd_points(F)])
    bvh = _build(api, tris, prec)
    _check(bvh, tris, pts, limits(tris, pts, rng))
    bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_sponza_and_k1_equals_nearest_triangles(api, prec):
    """k = 1 is the brute-force minimum; on cubes and Sponza nearest_triangles returns it too (checked first), so the distances agree."""
    F = FT[prec]
    rng = np.random.default_rng(9)
    for tris in (scenes.create_n_cubes_tris(400, prec), sponza_tris(F)):
        pts = KT.near_points(tris, 300, rng, spread=3.0)
        bvh = _build(api, tris, prec)
        ns, nd = bvh.nearest_triangles_batch(pts)
        bs, bd, _ = KT.brute(tris, pts, 8)
        assert np.array_equal(nd, bd[:, 0])
        s, d = bvh.knn_triangles(pts, 1)
        assert d[:, 0].tobytes() == nd.tobytes() and np.array_equal(s[:, 0], bs[:, 0])
        s, d, q = bvh.knn_triangles(pts, 8, closest=True)
        assert np.array_equal(s, bs) and d.tobytes() == bd.tobytes()
        bvh.free()


def test_contract(api):
    from bvh_b200 import capi

    F = np.float32
    rng = np.random.default_rng(4)
    tris = KT.soup(F, 50, rng)
    pts = KT.near_points(tris, 20, rng)
    bvh = _build(api, tris, "f32")
    s, d, q = bvh.knn_triangles(pts, 64, closest=True)                 # k > n: padding
    assert (s[:, 50:] == U32_MAX).all() and np.isposinf(d[:, 50:]).all() and np.isnan(q[:, 50:]).all() and (s[:, :50] != U32_MAX).all()
    assert bvh.knn_triangles(pts[:0], 4)[0].shape == (0, 4)            # n = 0: a no-op
    fn = getattr(capi.lib(), "bvhgpu_knn_triangles_f32x3")
    P = api._ptr
    for k, pp, ps, pd, tree in ((0, pts, True, True, bvh._h), (65, pts, True, True, bvh._h), (4, None, True, True, bvh._h),
                                (4, pts, False, True, bvh._h), (4, pts, True, False, bvh._h), (4, pts, True, True, None)):
        s = np.full((len(pts), 65), 7, dtype=np.uint32)
        d = np.full((len(pts), 65), 7, dtype=F)
        q = np.full((len(pts), 65, 3), 7, dtype=F)
        st = fn(tree, P(pp) if pp is not None else None, len(pts), k, None, P(s) if ps else None, P(d) if pd else None, P(q))
        assert st == capi.ERR_INVALID and (s == 7).all() and (d == 7).all() and (q == 7).all(), (k, pp is None, ps, pd, tree is None)
    bvh.free()
    plain = api.Bvh.build(O.tri_aabbs(tris, "f32"))                     # no triangles set
    with pytest.raises(capi.BvhGpuError) as e:
        plain.knn_triangles(pts, 4)
    assert e.value.status == capi.ERR_INVALID
    plain.free()
    bvh = _build(api, tris, "f32")
    bvh.add_shapes(O.tri_aabbs(tris[:3], "f32"))                        # add_shapes drops the triangles
    with pytest.raises(capi.BvhGpuError) as e:
        bvh.knn_triangles(pts, 4)
    assert e.value.status == capi.ERR_INVALID
    bvh.free()
    for n in (0, 1):                                                   # empty tree: padding; one triangle
        bvh = _build(api, tris[:n], "f32")
        s, d, q = bvh.knn_triangles(pts, 3, np.full(len(pts), 60, dtype=F), closest=True)
        bs, bd, bq = KT.brute(tris[:n], pts, 3, np.full(len(pts), 60, dtype=F))
        assert np.array_equal(s, bs) and d.tobytes() == bd.tobytes() and q.tobytes() == bq.tobytes()
        bvh.free()


def test_failed_build_is_sticky(api):
    import torch

    from bvh_b200 import capi

    shapes, tris = O.create_n_cubes(100, want_tris=True)
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
            bvh.knn_triangles(np.zeros((10, 3), dtype=np.float32), 4)
        assert e.value.status == capi.ERR_NAN
        with pytest.raises(capi.BvhGpuError) as e:
            bvh.knn_triangles_dev(pts.data_ptr(), 10, 4, 0, out_s.data_ptr(), out_d.data_ptr())
        assert e.value.status == capi.ERR_NAN
    bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_after_remove_shapes_and_refit(api, prec):
    F = FT[prec]
    rng = np.random.default_rng(21)
    tris = KT.soup(F, 400, rng)
    pts = KT.near_points(tris, 40, rng)
    bvh = _build(api, tris, prec)
    gone = rng.choice(len(tris), 70, replace=False)
    moves = bvh.remove_shapes(gone)                                     # the triangles follow their shapes
    after = tris.copy()
    for new_i, old_i in moves:
        after[new_i] = tris[old_i]
    after = after[: len(tris) - len(gone)]
    _check(bvh, after, pts, limits(after, pts, rng), ks=(1, 9, 64))
    moved = (after + rng.uniform(-3, 3, (len(after), 1, 3))).astype(F)
    bvh.refit(O.tri_aabbs(moved, prec))
    bvh.set_triangles(moved)
    _check(bvh, moved, pts, limits(moved, pts, rng), ks=(1, 9, 64))
    bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_dev_form_on_a_side_stream_equals_the_host_form(api, prec):
    import torch

    F = FT[prec]
    rng = np.random.default_rng(8)
    tris = scenes.create_n_cubes_tris(500, prec)
    pts = KT.near_points(tris, 5000, rng, spread=5.0)
    lim = (rng.uniform(0, 1, len(pts)) * 3).astype(F)
    bvh = _build(api, tris, prec)
    dev = torch.device("cuda", 0)
    side = torch.cuda.Stream(device=dev)
    dt = torch.float32 if prec == "f32" else torch.float64
    for k, md in ((1, None), (8, lim), (40, lim)):
        hs, hd, hq = bvh.knn_triangles(pts, k, md, closest=True)
        with torch.cuda.stream(side):
            d_p = torch.from_numpy(pts).to(dev)
            d_r = torch.from_numpy(md).to(dev) if md is not None else None
            d_s = torch.full((len(pts) * k,), 7, dtype=torch.int32, device=dev)
            d_d = torch.full((len(pts) * k,), 7, dtype=dt, device=dev)
            d_q = torch.full((len(pts) * k * 3,), 7, dtype=dt, device=dev)
            bvh.ctx.set_stream(side.cuda_stream)
            try:
                bvh.knn_triangles_dev(d_p.data_ptr(), len(pts), k, d_r.data_ptr() if d_r is not None else 0, d_s.data_ptr(), d_d.data_ptr(),
                                      d_q.data_ptr())
            finally:
                bvh.ctx.set_stream(None)
            side.synchronize()
        assert np.array_equal(d_s.cpu().numpy().view(np.uint32).reshape(-1, k), hs)
        assert d_d.cpu().numpy().tobytes() == hd.tobytes() and d_q.cpu().numpy().tobytes() == hq.tobytes()
        assert (hs != U32_MAX).any() and (md is None or (hs == U32_MAX).any())
    bvh.free()


def test_configs1_scene_at_scale(api):
    """The 120 k triangles of configs[1] (create_n_cubes(10 000)), 3 000 points near them and uniform in the bounds, k = 8, f32."""
    rng = np.random.default_rng(12)
    tris = scenes.create_n_cubes_tris(10_000, "f32")
    pts = np.concatenate([KT.near_points(tris, 1500, rng, spread=5.0), rng.uniform(-1e5, 1e5, (500, 3)).astype(np.float32)])
    bvh = _build(api, tris, "f32")
    s, d, q = bvh.knn_triangles(pts, 8, closest=True)
    bs, bd, bq = KT.brute(tris, pts, 8)
    assert np.array_equal(s, bs) and d.tobytes() == bd.tobytes() and q.tobytes() == bq.tobytes()
    bvh.free()
