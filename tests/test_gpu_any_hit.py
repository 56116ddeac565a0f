"""Any-hit (occlusion) queries with a per-ray distance limit on the device (bvhgpu_any_hit_* / bvhgpu_any_hit_dev_*):
- the device equals the restatement of tests/anyhit.py bit for bit, run over the device's own nodes:
    AABB mode in D = 2, 3, 4 and f32 / f64, random and overflow-scale scenes, host forms, the 3-D device form with FULL and OD rays
    and the 4-D device form;
    triangle mode in D = 3 on the triangle families of tests/adversarial.py and on a 120 k-triangle cube scene, host form and device
    form with both layouts;
  for the limits of anyhit.tmax_families: NULL, +inf, the ray's own closest distance d* (AABB mode: no hit), nextafter(d*, +inf) (a hit)
  and nextafter(d*, 0), 0, -0, negative, NaN and random values in (0, 2 d*);
- the contract: empty trees, n = 1 (hit and miss) and n = 2, refusals, the sticky failed build, triangle mode before set_triangles and
  after add_shapes, two calls byte-identical, the device form on a side stream, the model after refit, update_shapes, add_shapes and
  remove_shapes;
- a 4-D brute force at 200 k shapes: a hit exactly where some shape's own box is entered before tmax."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O
from tests import adversarial as A, anyhit as H, dimorder, dimref

pytestmark = pytest.mark.gpu
U32_MAX = 0xFFFFFFFF
FT = {"f32": np.float32, "f64": np.float64}
CASES = [(D, p) for D in (2, 3, 4) for p in ("f32", "f64")]


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A_

    return A_


def _cls(api, D):
    return {2: api.Bvh2, 3: api.Bvh, 4: api.Bvh4}[D]


def _table(api, D, prec):
    from bvh_b200.dtypes import BY_PREC

    return BY_PREC[prec] if D == 3 else _cls(api, D)._TABLE[prec]


def _aabbs(api, D, prec, mn, mx):
    a = np.zeros(len(mn), dtype=_table(api, D, prec)["aabb"])
    a["min"], a["max"] = mn, mx
    return a


def _rays(api, D, prec, o, d, inv):
    r = np.zeros(len(o), dtype=_table(api, D, prec)["ray"])
    r["origin"], r["direction"], r["inv_direction"] = o, d, inv
    return r


def _nodes(bvh, D):
    return bvh.nodes if D == 3 else bvh.nodes_and_index()[0]


def _closest(bvh, rays, triangles=False):
    """(shape, distance) of closest_hit in any D."""
    out = bvh.closest_hit(rays, triangles=triangles) if triangles else bvh.closest_hit(rays)
    return out[0], out[1]


def _dev3(bvh, rays, tmax, layout, triangles, prec):
    """bvhgpu_any_hit_dev_*x3 on device copies of the rays (FULL: the Ray structs, OD: origin + direction) and the limits."""
    import torch

    from bvh_b200 import capi

    n = len(rays)
    src = rays if layout == capi.RAYS_FULL else np.ascontiguousarray(np.concatenate([rays["origin"], rays["direction"]], axis=1))
    d_rays = torch.from_numpy(np.frombuffer(src.tobytes(), dtype=np.uint8).copy()).cuda()
    d_tmax = None if tmax is None else torch.from_numpy(np.ascontiguousarray(tmax)).cuda()
    sh = torch.full((n,), 7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    fn = getattr(capi.lib(), f"bvhgpu_any_hit_dev_{'f32x3' if prec == 'f32' else 'f64x3'}")
    capi.check(fn(bvh._h, C.c_void_p(d_rays.data_ptr()), layout, n, C.c_void_p(d_tmax.data_ptr()) if d_tmax is not None else None,
                  1 if triangles else 0, C.c_void_p(sh.data_ptr())))
    bvh.ctx.synchronize()
    return sh.cpu().numpy().view(np.uint32)


def _dev4(bvh, rays, tmax):
    import torch

    d_rays = torch.from_numpy(rays.view(np.uint8)).cuda()
    d_tmax = None if tmax is None else torch.from_numpy(np.ascontiguousarray(tmax)).cuda()
    sh = torch.full((len(rays),), 7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    bvh.any_hit_dev(d_rays.data_ptr(), len(rays), d_tmax.data_ptr() if d_tmax is not None else 0, sh.data_ptr())
    bvh.ctx.synchronize()
    return sh.cpu().numpy().view(np.uint32)


def _forms(bvh, D, rays, tmax, prec, triangles=False):
    """Every form of the call: host, and the device forms (3-D: FULL and OD rays; 4-D)."""
    from bvh_b200 import capi

    if D == 3:
        out = [bvh.any_hit(rays, tmax, triangles=triangles)]
        out += [_dev3(bvh, rays, tmax, lay, triangles, prec) for lay in (capi.RAYS_FULL, capi.RAYS_OD)]
        return out
    out = [bvh.any_hit(rays, tmax)]
    if D == 4:
        out.append(_dev4(bvh, rays, tmax))
    return out


def _check_aabb(bvh, D, shapes, rays, prec, families=None):
    """Every form equals the model for every limit family; returns the number of rays with a hit over all families."""
    F = FT[prec]
    nodes = _nodes(bvh, D)
    o, inv = rays["origin"], rays["inv_direction"]
    _, dstar = _closest(bvh, rays)
    hits = 0
    for name, tm in H.tmax_families(dstar, F, np.random.default_rng(5)).items():
        if families is not None and name not in families:
            continue
        want = H.aabb_batch(nodes, shapes, o, inv, tm)
        for got in _forms(bvh, D, rays, tm, prec):
            assert got.tobytes() == want.tobytes(), name
        lim = np.full(len(rays), np.inf, dtype=F) if tm is None else tm
        assert np.array_equal(want != U32_MAX, dstar < lim), name              # exact
        if name == "exact":
            assert np.all(want == U32_MAX)
        if name == "above":
            assert np.array_equal(want != U32_MAX, np.isfinite(dstar))
        hits += int((want != U32_MAX).sum())
    return hits


@pytest.mark.parametrize("scene", ["random", "overflow"])
@pytest.mark.parametrize("D,prec", CASES)
def test_aabb_mode_equals_the_model(api, D, prec, scene):
    F = FT[prec]
    rng = np.random.default_rng(70 + D)
    mn, mx = dimref.scene(scene, 400, D, F, rng)
    o, d, inv = dimorder.rays(mn, mx, 250, F, rng)
    shapes = _aabbs(api, D, prec, mn, mx)
    bvh = _cls(api, D).build(shapes, prec=prec)
    try:
        assert _check_aabb(bvh, D, shapes, _rays(api, D, prec, o, d, inv), prec) > 0
    finally:
        bvh.free()


def _tri_scene(family, prec):
    F = FT[prec]
    if family == "grazing":
        tris, o, d, _ = A.grazing(F)
    elif family == "shared":
        tris, o, d = A.shared_edges(F)
    elif family == "degenerate":
        tris, o, d = A.degenerate(F)
    elif family == "offset_lo":
        tris, o, d = A.offset_scene(F, 1e4 if prec == "f32" else 1e12)
    else:
        tris, o, d = A.offset_scene(F, 1e7 if prec == "f32" else 1e15)
    return tris, O.ray_new(o, d, prec)


def _check_triangles(bvh, shapes, tris, rays, prec, families=None):
    F = FT[prec]
    nodes = bvh.nodes
    _, dstar = _closest(bvh, rays, triangles=True)
    hits = 0
    for name, tm in H.tmax_families(dstar, F, np.random.default_rng(6)).items():
        if families is not None and name not in families:
            continue
        want = H.triangles(nodes, shapes, tris, rays, tm)
        for got in _forms(bvh, 3, rays, tm, prec, triangles=True):
            assert got.tobytes() == want.tobytes(), name
        if name in ("zero", "negzero", "negative", "nan"):
            assert np.all(want == U32_MAX), name
        hits += int((want != U32_MAX).sum())
    return hits


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("family", ["grazing", "shared", "degenerate", "offset_lo", "offset_hi"])
def test_triangle_mode_equals_the_model(api, family, prec):
    tris, rays = _tri_scene(family, prec)
    shapes = O.tri_aabbs(tris, prec)
    bvh = api.Bvh.build(shapes, prec=prec)
    try:
        bvh.set_triangles(tris)
        assert _check_triangles(bvh, shapes, tris, rays, prec) > 0
    finally:
        bvh.free()


def test_triangle_mode_on_a_120k_cube_scene(api):
    shapes, tris = O.create_n_cubes(10_000, want_tris=True)
    tris = tris.reshape(-1, 9)
    assert len(tris) == 120_000
    rng = np.random.default_rng(8)
    tgt = shapes["min"][rng.integers(0, len(shapes), 1500)].astype(np.float64) + rng.uniform(0, 1, (1500, 3))
    org = rng.uniform(-1.1e5, 1.1e5, (1500, 3))
    rays = O.ray_new(org, tgt - org)
    bvh = api.Bvh.build(shapes)
    try:
        bvh.set_triangles(tris)
        assert _check_triangles(bvh, shapes, tris, rays, "f32", families=("null", "above", "below", "random")) > 0
        # AABB mode on the same scene and rays
        assert _check_aabb(bvh, 3, shapes, rays, "f32", families=("null", "exact", "above", "random")) > 0
    finally:
        bvh.free()


@pytest.mark.parametrize("D,prec", CASES)
def test_contract(api, D, prec):
    from bvh_b200 import capi

    F = FT[prec]
    L = capi.lib()
    rng = np.random.default_rng(90 + D)
    cls = _cls(api, D)
    suf = _table(api, D, prec)["suffix"]
    mn, mx = dimref.scene("random", 300, D, F, rng)
    o, d, inv = dimorder.rays(mn, mx, 200, F, rng)
    rays = _rays(api, D, prec, o, d, inv)
    # n = 0: no hit for every ray, in every form
    b0 = cls.build(_aabbs(api, D, prec, mn[:0], mx[:0]), prec=prec)
    for got in _forms(b0, D, rays, None, prec):
        assert np.all(got == U32_MAX)
    b0.free()
    # n = 1 (the shape's own box decides, hit and miss) and n = 2
    for k in (1, 2):
        ok, dk, ik = dimorder.rays(mn[:k], mx[:k], 100, F, rng)
        rk = _rays(api, D, prec, ok, dk, ik)
        bk = cls.build(_aabbs(api, D, prec, mn[:k], mx[:k]), prec=prec)
        hits = _check_aabb(bk, D, _aabbs(api, D, prec, mn[:k], mx[:k]), rk, prec)
        first = bk.any_hit(rk)
        assert hits > 0 and np.any(first == U32_MAX) and np.any(first != U32_MAX)
        bk.free()
    bvh = cls.build(_aabbs(api, D, prec, mn, mx), prec=prec)
    # refusals write nothing
    fn = getattr(L, f"bvhgpu_any_hit_{suf}")
    out = np.full(len(rays), 7, dtype=np.uint32)
    head = (bvh._h, rays.ctypes.data)
    tail = (None, 0) if D == 3 else (None,)
    assert fn(bvh._h, None, len(rays), *tail, out.ctypes.data) == capi.ERR_INVALID
    assert fn(*head, len(rays), *tail, None) == capi.ERR_INVALID
    assert fn(*head, 1 << 31, *tail, out.ctypes.data) == capi.ERR_INVALID
    assert fn(None, rays.ctypes.data, len(rays), *tail, out.ctypes.data) == capi.ERR_INVALID
    assert np.all(out == 7)
    assert fn(*head, 0, *tail, None) == capi.OK                                 # nrays == 0
    if D == 3:
        dfn = getattr(L, f"bvhgpu_any_hit_dev_{suf}")
        assert dfn(bvh._h, None, capi.RAYS_FULL, 5, None, 0, None) == capi.ERR_INVALID
        assert dfn(bvh._h, 1, 2, 5, None, 0, 1) == capi.ERR_INVALID             # unknown ray layout: nothing is read
        assert dfn(bvh._h, 1, capi.RAYS_FULL, 1 << 31, None, 0, 1) == capi.ERR_INVALID
        assert dfn(bvh._h, None, capi.RAYS_OD, 0, None, 0, None) == capi.OK
        with pytest.raises(capi.BvhGpuError) as e:                             # triangle mode before set_triangles
            bvh.any_hit(rays, triangles=True)
        assert e.value.status == capi.ERR_INVALID
    if D == 4:
        dfn = getattr(L, f"bvhgpu_any_hit_dev_{suf}")
        assert dfn(bvh._h, None, 5, None, None) == capi.ERR_INVALID
        assert dfn(bvh._h, 1, 1 << 31, None, 1) == capi.ERR_INVALID
        assert dfn(bvh._h, None, 0, None, None) == capi.OK
    # two calls, byte-identical
    tm = (rng.uniform(0, 1, len(rays)) * 300).astype(F)
    assert bvh.any_hit(rays, tm).tobytes() == bvh.any_hit(rays, tm).tobytes()
    assert bvh.any_hit(rays, F(150)).tobytes() == bvh.any_hit(rays, np.full(len(rays), 150, dtype=F)).tobytes()
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
    rays = O.ray_new(np.zeros((10, 3)), np.ones((10, 3)))
    for _ in range(2):
        with pytest.raises(capi.BvhGpuError) as e:
            bvh.any_hit(rays)
        assert e.value.status == capi.ERR_NAN
        with pytest.raises(capi.BvhGpuError) as e:
            _dev3(bvh, rays, None, capi.RAYS_FULL, False, "f32")
        assert e.value.status == capi.ERR_NAN
    bvh.free()


def test_triangle_mode_after_add_shapes_is_refused(api):
    from bvh_b200 import capi

    shapes, tris = O.create_n_cubes(50, want_tris=True)
    bvh = api.Bvh.build(shapes)
    bvh.set_triangles(tris)
    rays = O.ray_new(np.full((64, 3), -2e5), np.ones((64, 3)))
    bvh.any_hit(rays, triangles=True)
    bvh.add_shapes(shapes[:3])
    with pytest.raises(capi.BvhGpuError) as e:
        bvh.any_hit(rays, triangles=True)
    assert e.value.status == capi.ERR_INVALID
    with pytest.raises(capi.BvhGpuError) as e:
        _dev3(bvh, rays, None, capi.RAYS_OD, True, "f32")
    assert e.value.status == capi.ERR_INVALID
    bvh.free()


@pytest.mark.parametrize("D,prec", CASES)
def test_model_after_refit_update_add_and_remove(api, D, prec):
    F = FT[prec]
    rng = np.random.default_rng(60 + D)
    mn, mx = dimref.scene("random", 500, D, F, rng)
    o, d, inv = dimorder.rays(mn, mx, 150, F, rng)
    rays = _rays(api, D, prec, o, d, inv)
    aabbs = _aabbs(api, D, prec, mn, mx)
    bvh = _cls(api, D).build(aabbs, prec=prec)
    fam = ("null", "above", "random")
    _check_aabb(bvh, D, aabbs, rays, prec, fam)
    shift = rng.uniform(-3, 3, (len(aabbs), D)).astype(F)
    aabbs["min"], aabbs["max"] = (aabbs["min"] + shift).astype(F), (aabbs["max"] + shift).astype(F)
    bvh.refit(aabbs)
    _check_aabb(bvh, D, aabbs, rays, prec, fam)
    changed = rng.choice(len(aabbs), 60, replace=False)
    shift = rng.uniform(-20, 20, (60, D)).astype(F)
    aabbs["min"][changed] = (aabbs["min"][changed] + shift).astype(F)
    aabbs["max"][changed] = (aabbs["max"][changed] + shift).astype(F)
    bvh.update_shapes(changed, aabbs, max_growth=1.5)
    _check_aabb(bvh, D, aabbs, rays, prec, fam)
    nmn, nmx = dimref.scene("random", 40, D, F, rng)
    new = _aabbs(api, D, prec, nmn, nmx)
    bvh.add_shapes(new)
    aabbs = np.concatenate([aabbs, new])
    _check_aabb(bvh, D, aabbs, rays, prec, fam)
    gone = rng.choice(len(aabbs), 70, replace=False)
    moves = bvh.remove_shapes(gone)
    after = aabbs.copy()
    for new_i, old_i in moves:
        after[new_i] = aabbs[old_i]
    after = after[: len(aabbs) - len(gone)]
    _check_aabb(bvh, D, after, rays, prec, fam)
    bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_any_hit_dev_on_a_side_stream_equals_the_host_form(api, prec):
    import torch

    F = FT[prec]
    rng = np.random.default_rng(5)
    mn, mx = dimref.scene("random", 3000, 4, F, rng)
    o, d, inv = dimorder.rays(mn, mx, 5000, F, rng)
    rays = _rays(api, 4, prec, o, d, inv)
    tm = (rng.uniform(0, 1, len(rays)) * 500).astype(F)
    bvh = api.Bvh4.build(_aabbs(api, 4, prec, mn, mx), prec=prec)
    hs = bvh.any_hit(rays, tm)
    dev = torch.device("cuda", 0)
    side = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(side):
        d_rays = torch.from_numpy(rays.view(np.uint8)).to(dev)
        d_tm = torch.from_numpy(tm).to(dev)
        d_s = torch.full((len(rays),), 7, dtype=torch.int32, device=dev)
        bvh.ctx.set_stream(side.cuda_stream)
        try:
            bvh.any_hit_dev(d_rays.data_ptr(), len(rays), d_tm.data_ptr(), d_s.data_ptr())
        finally:
            bvh.ctx.set_stream(None)
        side.synchronize()
    assert np.array_equal(d_s.cpu().numpy().view(np.uint32), hs)
    assert np.sum(hs != U32_MAX) > 0 and np.sum(hs == U32_MAX) > 0
    bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_4d_against_brute_force_at_scale(api, prec):
    """200 k shapes, 20 k rays, random limits: a hit exactly where the minimum entry over every shape whose own box the ray enters
    (torch elementwise ops, each rounding once as the slab test does) is < tmax, and the witness's own entry is < tmax."""
    import torch

    F = FT[prec]
    rng = np.random.default_rng(17)
    n, m = 200_000, 20_000
    mn = rng.uniform(-1000, 1000, (n, 4)).astype(F)
    mx = (mn + rng.uniform(0, 6, (n, 4))).astype(F)
    o, d, inv = dimorder.rays(mn, mx, m, F, rng)
    tm = rng.uniform(0, 4000, m).astype(F)                     # most first hits of this sparse scene lie 1000 - 3000 away
    bvh = api.Bvh4.build(_aabbs(api, 4, prec, mn, mx), prec=prec)
    ws = bvh.any_hit(_rays(api, 4, prec, o, d, inv), tm)
    dev = torch.device("cuda", 0)
    tmn, tmx = torch.from_numpy(mn).to(dev), torch.from_numpy(mx).to(dev)
    best = np.full(m, np.inf, dtype=F)
    own = np.full(m, np.inf, dtype=F)
    for a in range(0, m, 256):
        to, ti = torch.from_numpy(o[a:a + 256]).to(dev)[:, None, :], torch.from_numpy(inv[a:a + 256]).to(dev)[:, None, :]
        l, r = (tmn[None] - to) * ti, (tmx[None] - to) * ti
        nan = torch.isnan(l).any(-1) | torch.isnan(r).any(-1)
        tmin, tmax = torch.minimum(l, r).amax(-1), torch.maximum(l, r).amin(-1)
        entry = torch.where(tmin > 0, tmin, torch.zeros_like(tmin))
        key = torch.where(~nan & ~(entry > tmax), entry, torch.full_like(entry, float("inf")))
        best[a:a + 256] = key.amin(-1).cpu().numpy()
        w = torch.from_numpy(ws[a:a + 256].astype(np.int64)).to(dev)
        valid = w != U32_MAX
        idx = torch.where(valid, w, torch.zeros_like(w))
        own[a:a + 256] = torch.where(valid, key.gather(1, idx[:, None])[:, 0], torch.full_like(key[:, 0], float("inf"))).cpu().numpy()
    hit = ws != U32_MAX
    assert hit.sum() > m // 50 and (~hit).sum() > m // 50
    assert np.array_equal(hit, best < tm)
    assert np.all(own[hit] < tm[hit])
    bvh.free()
