"""Multi-hit queries with an optional per-ray distance limit on the device (bvhgpu_multi_hit_* / bvhgpu_multi_hit_dev_*):
- the device equals the restatement of tests/multihit.py bit for bit (shapes, distances and uv), run over the device's own nodes:
    AABB mode in D = 2, 3, 4 and f32 / f64, random and overflow-scale scenes; triangle mode in D = 3 on the triangle families of
    tests/adversarial.py; every form: host, the 3-D device form with FULL and OD rays, the 4-D device form;
  k at every K-bucket edge (1, 4, 5, 8, 9, 16, 17, 32, 33, 64) and every limit of anyhit.tmax_families;
- the identities on the 120 k-triangle configs[1] scene with 1 M rays aimed at its cubes: k = 1 without a limit is closest_hit (both
  modes, with uv), a row is empty exactly where any_hit reports no hit (k = 1 and 3), AABB mode is the head of traverse_ordered; and
  the model on a few hundred of those rays;
- the contract: refusals write nothing, n = 0, an empty tree, n = 1 hit and miss, the sticky failed build before missing triangles,
  triangle mode before set_triangles and after add_shapes, the model after refit, update_shapes and remove_shapes (triangles follow
  their shapes), two calls byte-identical, the device form on a side stream."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O
from tests import adversarial as A, anyhit as H, dimorder, dimref, multihit as MH

pytestmark = pytest.mark.gpu
U32_MAX = 0xFFFFFFFF
FT = {"f32": np.float32, "f64": np.float64}
UINT = {np.float32: np.uint32, np.float64: np.uint64}
CASES = [(D, p) for D in (2, 3, 4) for p in ("f32", "f64")]
EDGES = (1, 4, 5, 8, 9, 16, 17, 32, 33, 64)
FAMILY_KS = (1, 9, 64)                     # k swept over every limit family; every edge runs with "null" and "random"


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


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(UINT[a.dtype.type]) if a.dtype.type in UINT else a


def _same(got, want, uv):
    """Shapes and distances bit for bit; uv too when `uv` (the model's uv, or zeros for AABB mode)."""
    ok = np.array_equal(got[0], want[0]) and np.array_equal(_bits(got[1]), _bits(want[1]))
    if uv is not None and got[2] is not None:
        ok = ok and np.array_equal(_bits(got[2]), _bits(uv))
    return ok


def _dev3(bvh, rays, k, tmax, layout, triangles, prec):
    """bvhgpu_multi_hit_dev_*x3 on device copies of the rays (FULL: the Ray structs, OD: origin + direction) and the limits, into
    poisoned outputs."""
    import torch

    from bvh_b200 import capi

    n = len(rays)
    dt = torch.float32 if prec == "f32" else torch.float64
    src = rays if layout == capi.RAYS_FULL else np.ascontiguousarray(np.concatenate([rays["origin"], rays["direction"]], axis=1))
    d_rays = torch.from_numpy(np.frombuffer(src.tobytes(), dtype=np.uint8).copy()).cuda()
    d_tmax = None if tmax is None else torch.from_numpy(np.ascontiguousarray(tmax)).cuda()
    sh = torch.full((n * k,), 7, dtype=torch.int32, device="cuda")
    di = torch.full((n * k,), 7, dtype=dt, device="cuda")
    uv = torch.full((n * k * 2,), 7, dtype=dt, device="cuda")
    torch.cuda.synchronize()
    bvh.multi_hit_dev(d_rays.data_ptr(), n, k, d_tmax.data_ptr() if d_tmax is not None else 0, sh.data_ptr(), di.data_ptr(), uv.data_ptr(),
                      triangles=triangles, layout=layout)
    bvh.ctx.synchronize()
    return sh.cpu().numpy().view(np.uint32).reshape(n, k), di.cpu().numpy().reshape(n, k), uv.cpu().numpy().reshape(n, k, 2)


def _dev4(bvh, rays, k, tmax, prec):
    import torch

    n = len(rays)
    dt = torch.float32 if prec == "f32" else torch.float64
    d_rays = torch.from_numpy(rays.view(np.uint8)).cuda()
    d_tmax = None if tmax is None else torch.from_numpy(np.ascontiguousarray(tmax)).cuda()
    sh = torch.full((n * k,), 7, dtype=torch.int32, device="cuda")
    di = torch.full((n * k,), 7, dtype=dt, device="cuda")
    torch.cuda.synchronize()
    bvh.multi_hit_dev(d_rays.data_ptr(), n, k, d_tmax.data_ptr() if d_tmax is not None else 0, sh.data_ptr(), di.data_ptr())
    bvh.ctx.synchronize()
    return sh.cpu().numpy().view(np.uint32).reshape(n, k), di.cpu().numpy().reshape(n, k), None


def _forms(bvh, D, rays, k, tmax, prec, triangles=False):
    """Every form of the call: host (with uv in 3-D), and the device forms (3-D: FULL and OD rays; 4-D)."""
    from bvh_b200 import capi

    if D == 3:
        out = [bvh.multi_hit(rays, k, tmax, triangles=triangles, uv=True)]
        out += [_dev3(bvh, rays, k, tmax, lay, triangles, prec) for lay in (capi.RAYS_FULL, capi.RAYS_OD)]
        return out
    out = [bvh.multi_hit(rays, k, tmax)]
    if D == 4:
        out.append(_dev4(bvh, rays, k, tmax, prec))
    return out


def _plan(tmax_families):
    """(limit name, limits, k): every edge with the null and random limits, every limit with FAMILY_KS."""
    for name, tm in tmax_families.items():
        for k in EDGES if name in ("null", "random") else FAMILY_KS:
            yield name, tm, k


def _check_aabb(bvh, D, shapes, rays, prec, families=None, ks=None):
    """Every form equals the model for the planned (limit, k); returns the number of filled slots."""
    F = FT[prec]
    nodes = _nodes(bvh, D)
    o, inv = rays["origin"], rays["inv_direction"]
    _, dstar = bvh.closest_hit(rays)[:2]
    filled = 0
    for name, tm, k in _plan(H.tmax_families(dstar, F, np.random.default_rng(5))):
        if (families is not None and name not in families) or (ks is not None and k not in ks):
            continue
        want = MH.aabb_batch(nodes, shapes, o, inv, k, tm)
        zeros = np.zeros((len(rays), k, 2), dtype=F)
        for f, got in enumerate(_forms(bvh, D, rays, k, tm, prec)):
            assert _same(got, want, zeros), (name, k, f)
        filled += int((want[0] != U32_MAX).sum())
    return filled


def _check_triangles(bvh, shapes, tris, rays, prec, families=None, ks=None):
    F = FT[prec]
    nodes = bvh.nodes
    dstar = bvh.closest_hit(rays, triangles=True)[1]
    filled = 0
    for name, tm, k in _plan(H.tmax_families(dstar, F, np.random.default_rng(6))):
        if (families is not None and name not in families) or (ks is not None and k not in ks):
            continue
        want = MH.triangles(nodes, shapes, tris, rays, k, tm)
        for f, got in enumerate(_forms(bvh, 3, rays, k, tm, prec, triangles=True)):
            assert _same(got, want, want[2]), (name, k, f)
        filled += int((want[0] != U32_MAX).sum())
    return filled


@pytest.mark.parametrize("scene", ["random", "overflow"])
@pytest.mark.parametrize("D,prec", CASES)
def test_aabb_mode_equals_the_model(api, D, prec, scene):
    F = FT[prec]
    rng = np.random.default_rng(70 + D)
    mn, mx = dimref.scene(scene, 300, D, F, rng)
    o, d, inv = dimorder.rays(mn, mx, 48, F, rng)
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
    else:
        tris, o, d = A.offset_scene(F, 1e4 if prec == "f32" else 1e12, m=96)
    return tris, O.ray_new(o, d, prec)


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("family", ["grazing", "shared", "degenerate", "offset"])
def test_triangle_mode_equals_the_model(api, family, prec):
    tris, rays = _tri_scene(family, prec)
    shapes = O.tri_aabbs(tris, prec)
    bvh = api.Bvh.build(shapes, prec=prec)
    try:
        bvh.set_triangles(tris)
        assert _check_triangles(bvh, shapes, tris, rays, prec) > 0
    finally:
        bvh.free()


@pytest.fixture(scope="module")
def cubes(api):
    """configs[1]'s 120 k triangles (create_n_cubes_tris(10 000)) and 1 M rays aimed at points of random cubes from random origins
    (the create_ray chain of configs[1] hits almost nothing in triangle mode)."""
    from bvh_b200 import scenes
    from bvh_b200.dtypes import BY_PREC

    tris = scenes.create_n_cubes_tris(10_000)
    a = np.zeros(len(tris), dtype=BY_PREC["f32"]["aabb"])
    a["min"], a["max"] = tris.min(axis=1), tris.max(axis=1)
    rng = np.random.default_rng(8)
    n = 1_000_000
    tgt = a["min"][rng.integers(0, len(a), n)].astype(np.float64) + rng.uniform(0, 1, (n, 3))
    org = rng.uniform(-1.1e5, 1.1e5, (n, 3))
    bvh = api.Bvh.build(a)
    bvh.set_triangles(tris.reshape(-1, 9))
    rays = api.Ray.new(org, tgt - org)
    yield bvh, a, tris.reshape(-1, 9), rays
    bvh.free()


@pytest.mark.parametrize("triangles", [False, True])
def test_identities_on_the_120k_cube_scene(api, cubes, triangles):
    bvh, shapes, tris, rays = cubes
    assert len(tris) == 120_000 and len(rays) == 1_000_000
    # 1: k = 1 without a limit is closest_hit, shape, distance and uv
    cs, cd, cuv = bvh.closest_hit(rays, triangles=triangles)
    ms, md, muv = bvh.multi_hit(rays, 1, triangles=triangles, uv=True)
    assert np.array_equal(ms[:, 0], cs) and np.array_equal(_bits(md[:, 0]), _bits(cd)) and np.array_equal(_bits(muv[:, 0]), _bits(cuv))
    assert (cs != U32_MAX).sum() > 1000
    # 2: with a limit a row is empty exactly where any_hit reports no hit
    rng = np.random.default_rng(12)
    fin = np.isfinite(cd)
    tm = (rng.uniform(0, 2, len(rays)) * np.where(fin, cd, cd[fin].max())).astype(np.float32)
    empty_any = bvh.any_hit(rays, tm, triangles=triangles) == U32_MAX
    for k in (1, 3):
        s, _, _ = bvh.multi_hit(rays, k, tm, triangles=triangles)
        assert np.array_equal(s[:, 0] == U32_MAX, empty_any), k
    assert empty_any.sum() > 1000 and (~empty_any).sum() > 1000
    # 3: AABB mode without a limit is the head of traverse_ordered (ascending) on this tight tree
    if not triangles:
        sub = rays[:20_000]
        off, hits, dists = bvh.traverse_ordered(sub, True)
        for k in (1, 3):
            s, d, _ = bvh.multi_hit(sub, k)
            for r in range(len(sub)):
                n = min(k, int(off[r + 1] - off[r]))
                assert np.array_equal(s[r, :n], hits[off[r]:off[r] + n]) and np.all(s[r, n:] == U32_MAX), (k, r)
                assert np.array_equal(_bits(d[r, :n]), _bits(dists[off[r]:off[r] + n])), (k, r)
    # the model on a few hundred of the rays
    pick = rng.choice(len(rays), 300, replace=False)
    sub = rays[pick]
    for k in (1, 3, 16):
        got = bvh.multi_hit(sub, k, tm[pick], triangles=triangles, uv=True)
        if triangles:
            want = MH.triangles(bvh.nodes, shapes, tris, sub, k, tm[pick])
            assert _same(got, want, want[2]), k
        else:
            want = MH.aabb_batch(bvh.nodes, shapes, sub["origin"], sub["inv_direction"], k, tm[pick])
            assert _same(got, want, np.zeros((len(sub), k, 2), dtype=np.float32)), k


@pytest.mark.parametrize("D,prec", CASES)
def test_contract(api, D, prec):
    from bvh_b200 import capi

    F = FT[prec]
    L = capi.lib()
    rng = np.random.default_rng(90 + D)
    cls = _cls(api, D)
    suf = _table(api, D, prec)["suffix"]
    mn, mx = dimref.scene("random", 300, D, F, rng)
    o, d, inv = dimorder.rays(mn, mx, 120, F, rng)
    rays = _rays(api, D, prec, o, d, inv)
    # an empty tree: rows of padding in every form
    b0 = cls.build(_aabbs(api, D, prec, mn[:0], mx[:0]), prec=prec)
    for got in _forms(b0, D, rays, 5, None, prec):
        assert np.all(got[0] == U32_MAX) and np.all(np.isposinf(got[1]))
        assert got[2] is None or np.all(_bits(got[2]) == 0)
    b0.free()
    # n = 1: the shape's own box decides (hit and miss)
    o1, d1, i1 = dimorder.rays(mn[:1], mx[:1], 100, F, rng)
    r1 = _rays(api, D, prec, o1, d1, i1)
    b1 = cls.build(_aabbs(api, D, prec, mn[:1], mx[:1]), prec=prec)
    assert _check_aabb(b1, D, _aabbs(api, D, prec, mn[:1], mx[:1]), r1, prec, families=("null", "random"), ks=(1, 4, 5)) > 0
    first = b1.multi_hit(r1, 2)[0]
    assert np.any(first[:, 0] == U32_MAX) and np.any(first[:, 0] != U32_MAX) and np.all(first[:, 1] == U32_MAX)
    b1.free()
    bvh = cls.build(_aabbs(api, D, prec, mn, mx), prec=prec)
    # refusals write nothing
    n = len(rays)
    fn = getattr(L, f"bvhgpu_multi_hit_{suf}")
    sh = np.full(n * 64, 7, dtype=np.uint32)
    di = np.full(n * 64, 7, dtype=F)
    uv = np.full(n * 128, 7, dtype=F)
    outs = (sh.ctypes.data, di.ctypes.data, uv.ctypes.data) if D == 3 else (sh.ctypes.data, di.ctypes.data)
    mode = (0,) if D == 3 else ()
    for k in (0, 65, 1 << 31):
        assert fn(bvh._h, rays.ctypes.data, n, k, None, *mode, *outs) == capi.ERR_INVALID, k
    assert fn(bvh._h, None, n, 4, None, *mode, *outs) == capi.ERR_INVALID
    assert fn(bvh._h, rays.ctypes.data, n, 4, None, *mode, None, *outs[1:]) == capi.ERR_INVALID
    assert fn(bvh._h, rays.ctypes.data, n, 4, None, *mode, outs[0], None, *outs[2:]) == capi.ERR_INVALID
    assert fn(bvh._h, rays.ctypes.data, 1 << 31, 4, None, *mode, *outs) == capi.ERR_INVALID
    assert fn(None, rays.ctypes.data, n, 4, None, *mode, *outs) == capi.ERR_INVALID
    if D == 3:
        assert fn(bvh._h, rays.ctypes.data, n, 4, None, 1, *outs) == capi.ERR_INVALID        # triangles never set
    assert np.all(sh == 7) and np.all(di == 7) and np.all(uv == 7)
    assert fn(bvh._h, rays.ctypes.data, 0, 4, None, *mode, *outs) == capi.OK                # nrays == 0
    assert np.all(sh == 7)
    if D == 3:
        dfn = getattr(L, f"bvhgpu_multi_hit_dev_{suf}")
        assert dfn(bvh._h, None, capi.RAYS_FULL, 5, 4, None, 0, 1, 1, None) == capi.ERR_INVALID
        assert dfn(bvh._h, 1, 2, 5, 4, None, 0, 1, 1, None) == capi.ERR_INVALID             # unknown ray layout: nothing is read
        assert dfn(bvh._h, 1, capi.RAYS_FULL, 5, 0, None, 0, 1, 1, None) == capi.ERR_INVALID
        assert dfn(bvh._h, 1, capi.RAYS_FULL, 5, 65, None, 0, 1, 1, None) == capi.ERR_INVALID
        assert dfn(bvh._h, 1, capi.RAYS_FULL, 1 << 31, 4, None, 0, 1, 1, None) == capi.ERR_INVALID
        assert dfn(bvh._h, None, capi.RAYS_OD, 0, 4, None, 0, None, None, None) == capi.OK
        with pytest.raises(capi.BvhGpuError) as e:                                         # triangle mode before set_triangles
            _dev3(bvh, rays, 4, None, capi.RAYS_OD, True, prec)
        assert e.value.status == capi.ERR_INVALID
    if D == 4:
        dfn = getattr(L, f"bvhgpu_multi_hit_dev_{suf}")
        assert dfn(bvh._h, None, 5, 4, None, 1, 1) == capi.ERR_INVALID
        assert dfn(bvh._h, 1, 5, 0, None, 1, 1) == capi.ERR_INVALID
        assert dfn(bvh._h, 1, 1 << 31, 4, None, 1, 1) == capi.ERR_INVALID
        assert dfn(bvh._h, None, 0, 4, None, None, None) == capi.OK
    # two calls, byte-identical; a scalar limit is the same as one per ray
    tm = (rng.uniform(0, 1, n) * 300).astype(F)
    a1, a2 = bvh.multi_hit(rays, 7, tm), bvh.multi_hit(rays, 7, tm)
    assert a1[0].tobytes() == a2[0].tobytes() and a1[1].tobytes() == a2[1].tobytes()
    b1_, b2_ = bvh.multi_hit(rays, 7, F(150)), bvh.multi_hit(rays, 7, np.full(n, 150, dtype=F))
    assert b1_[0].tobytes() == b2_[0].tobytes() and b1_[1].tobytes() == b2_[1].tobytes()
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
    for _ in range(2):
        for tri in (False, True):                               # no triangles were ever set: the failed build is reported first
            with pytest.raises(capi.BvhGpuError) as e:
                bvh.multi_hit(rays, 3, triangles=tri)
            assert e.value.status == capi.ERR_NAN
            with pytest.raises(capi.BvhGpuError) as e:
                _dev3(bvh, rays, 3, None, capi.RAYS_FULL, tri, "f32")
            assert e.value.status == capi.ERR_NAN
    bvh.free()


def test_triangle_mode_after_add_shapes_is_refused(api):
    from bvh_b200 import capi

    shapes, tris = O.create_n_cubes(50, want_tris=True)
    bvh = api.Bvh.build(shapes)
    bvh.set_triangles(tris)
    rays = O.ray_new(np.full((64, 3), -2e5), np.ones((64, 3)))
    bvh.multi_hit(rays, 4, triangles=True)
    bvh.add_shapes(shapes[:3])
    with pytest.raises(capi.BvhGpuError) as e:
        bvh.multi_hit(rays, 4, triangles=True)
    assert e.value.status == capi.ERR_INVALID
    with pytest.raises(capi.BvhGpuError) as e:
        _dev3(bvh, rays, 4, None, capi.RAYS_OD, True, "f32")
    assert e.value.status == capi.ERR_INVALID
    bvh.free()


@pytest.mark.parametrize("D,prec", CASES)
def test_model_after_refit_update_and_remove(api, D, prec):
    F = FT[prec]
    rng = np.random.default_rng(60 + D)
    mn, mx = dimref.scene("random", 400, D, F, rng)
    o, d, inv = dimorder.rays(mn, mx, 60, F, rng)
    rays = _rays(api, D, prec, o, d, inv)
    aabbs = _aabbs(api, D, prec, mn, mx)
    bvh = _cls(api, D).build(aabbs, prec=prec)
    fam, ks = ("null", "random"), (1, 5, 17)
    _check_aabb(bvh, D, aabbs, rays, prec, fam, ks)
    shift = rng.uniform(-3, 3, (len(aabbs), D)).astype(F)
    aabbs["min"], aabbs["max"] = (aabbs["min"] + shift).astype(F), (aabbs["max"] + shift).astype(F)
    bvh.refit(aabbs)
    _check_aabb(bvh, D, aabbs, rays, prec, fam, ks)
    changed = rng.choice(len(aabbs), 60, replace=False)
    shift = rng.uniform(-20, 20, (60, D)).astype(F)
    aabbs["min"][changed] = (aabbs["min"][changed] + shift).astype(F)
    aabbs["max"][changed] = (aabbs["max"][changed] + shift).astype(F)
    bvh.update_shapes(changed, aabbs, max_growth=1.5)
    _check_aabb(bvh, D, aabbs, rays, prec, fam, ks)
    gone = rng.choice(len(aabbs), 70, replace=False)
    moves = bvh.remove_shapes(gone)
    after = aabbs.copy()
    for new_i, old_i in moves:
        after[new_i] = aabbs[old_i]
    after = after[: len(aabbs) - len(gone)]
    assert _check_aabb(bvh, D, after, rays, prec, fam, ks) > 0
    bvh.free()


def test_triangles_follow_their_shapes_after_remove(api):
    tris, rays = _tri_scene("shared", "f32")
    shapes = O.tri_aabbs(tris, "f32")
    bvh = api.Bvh.build(shapes)
    bvh.set_triangles(tris)
    gone = np.random.default_rng(2).choice(len(shapes), len(shapes) // 5, replace=False)
    moves = bvh.remove_shapes(gone)
    s2, t2 = shapes.copy(), tris.copy()
    for new_i, old_i in moves:
        s2[new_i], t2[new_i] = shapes[old_i], tris[old_i]
    s2, t2 = s2[: len(shapes) - len(gone)], t2[: len(shapes) - len(gone)]
    assert _check_triangles(bvh, s2, t2, rays, "f32", families=("null", "random"), ks=(1, 5, 17)) > 0
    bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_multi_hit_dev_on_a_side_stream_equals_the_host_form(api, prec):
    import torch

    F = FT[prec]
    rng = np.random.default_rng(5)
    mn, mx = dimref.scene("random", 3000, 4, F, rng)
    o, d, inv = dimorder.rays(mn, mx, 5000, F, rng)
    rays = _rays(api, 4, prec, o, d, inv)
    tm = (rng.uniform(0, 1, len(rays)) * 500).astype(F)
    k = 6
    bvh = api.Bvh4.build(_aabbs(api, 4, prec, mn, mx), prec=prec)
    hs, hd, _ = bvh.multi_hit(rays, k, tm)
    dev = torch.device("cuda", 0)
    side = torch.cuda.Stream(device=dev)
    dt = torch.float32 if prec == "f32" else torch.float64
    with torch.cuda.stream(side):
        d_rays = torch.from_numpy(rays.view(np.uint8)).to(dev)
        d_tm = torch.from_numpy(tm).to(dev)
        d_s = torch.full((len(rays) * k,), 7, dtype=torch.int32, device=dev)
        d_d = torch.full((len(rays) * k,), 7, dtype=dt, device=dev)
        bvh.ctx.set_stream(side.cuda_stream)
        try:
            bvh.multi_hit_dev(d_rays.data_ptr(), len(rays), k, d_tm.data_ptr(), d_s.data_ptr(), d_d.data_ptr())
        finally:
            bvh.ctx.set_stream(None)
        side.synchronize()
    assert np.array_equal(d_s.cpu().numpy().view(np.uint32).reshape(-1, k), hs)
    assert np.array_equal(_bits(d_d.cpu().numpy().reshape(-1, k)), _bits(hd))
    assert np.sum(hs[:, 0] != U32_MAX) > 0 and np.sum(hs[:, 0] == U32_MAX) > 0 and np.sum(hs[:, 1] != U32_MAX) > 0
    bvh.free()
