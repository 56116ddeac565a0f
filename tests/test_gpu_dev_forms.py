"""The device-pointer (`_dev_`) entry points and their f64 twins through the C ABI, against the host forms and the CPU oracle.

Every `_dev_` call runs on a side torch stream installed as the library's stream.  Its inputs are produced on that stream right
before the call (a spin kernel, then an XOR that decodes a scrambled upload), and its outputs are read back on the same stream.
A `_dev_` form that enqueued on another stream, or read its input before the producer ran, would see the scrambled bytes.
Run on an H100:  python -m pytest tests/test_gpu_dev_forms.py -m gpu"""
import contextlib
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O
from tests import prunedcheck as PC
from tests.scenes import rays_for, scene

pytestmark = pytest.mark.gpu

SPIN = 20_000_000            # torch.cuda._sleep cycles ahead of every producer (~10 ms on an H100)
LONG_SPIN = 200_000_000      # ~0.1 s: long enough to tell a call that returns at once from one that waits for the stream
KEY = 0xA5


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A

    return A


def _sfx(prec):
    return "f32x3" if prec == "f32" else "f64x3"


def _F(prec):
    return np.float32 if prec == "f32" else np.float64


def _vp(t):
    return None if t is None else C.c_void_p(t.data_ptr())


@contextlib.contextmanager
def _side_stream(ctx):
    """A fresh torch stream that is both the library context's stream and torch's current stream."""
    import torch

    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    ctx.set_stream(s.cuda_stream)
    try:
        with torch.cuda.stream(s):
            yield s
    finally:
        s.synchronize()
        ctx.set_stream(None)


def _produce(*arrays, spin=SPIN):
    """The arrays' bytes in device memory (uint8 tensors), produced on the current stream: scrambled uploads, one spin kernel,
    then one XOR per array that restores the bytes.  Whatever reads them must be ordered after the current stream."""
    import torch

    enc = [torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1) ^ np.uint8(KEY)).to("cuda") for a in arrays]
    torch.cuda._sleep(spin)
    out = [torch.bitwise_xor(e, KEY) for e in enc]
    return out[0] if len(out) == 1 else out


def _buf(nbytes, fill=0xFF):
    """A device buffer on the current stream, every byte `fill` (0xFF: U32_MAX / NaN sentinels)."""
    import torch

    return torch.full((max(int(nbytes), 16),), fill, dtype=torch.uint8, device="cuda")


def _host(t, dtype, count=None):
    """Read a device buffer back on the current stream."""
    a = t.cpu().numpy().view(dtype)
    return a if count is None else a[:count]


def _ray_inputs(shapes, n, prec, seed):
    """Origins and directions: rays_for's random and axis-aligned rays (zero direction components +0.0, half of the axis-aligned
    ones starting on a box's min corner), then the same axis-aligned rays again with -0.0 zero components (inv = -inf), half of
    those starting on a box's max corner.  On a face plane (mn - o) * inv is 0 * inf = NaN: the slab test's NaN rule.
    The directions are rays_for's f64 unit vectors: on f32 scenes with coordinates near 1e30 the f32 normalisation overflows to a
    zero direction, which normalised once more is 0 / 0, and the bits of that NaN differ between the host and the device."""
    k = n // 4
    base = rays_for(shapes, n, "f64", seed=seed, axis_aligned=k)
    o, d = base["origin"].astype(np.float64), base["direction"].astype(np.float64)
    ao, ad = o[:k].copy(), d[:k].copy()
    ad[ad == 0] = -0.0
    if len(shapes):
        pick = np.random.default_rng(seed).integers(0, len(shapes), k)
        ao[1::2] = shapes["max"][pick[1::2]].astype(np.float64)
    o, d = np.concatenate([o, ao]), np.concatenate([d, ad])
    assert np.signbit(d[d == 0]).any() and (~np.signbit(d[d == 0])).any()
    return o.astype(_F(prec)), d.astype(_F(prec))


def _dev_rays(ctx, o, d, prec):
    """bvhgpu_rays_new_dev_* on the current stream, its origins and directions produced just before."""
    from bvh_b200 import capi
    from bvh_b200.dtypes import BY_PREC

    to, td = _produce(o, d)
    out = _buf(len(o) * BY_PREC[prec]["ray"].itemsize)
    capi.check(getattr(capi.lib(), f"bvhgpu_rays_new_dev_{_sfx(prec)}")(ctx._h, _vp(to), _vp(td), len(o), _vp(out)))
    return out


def _closest_dev(bvh, rays, layout, use_triangles, with_uv=True):
    """bvhgpu_closest_hit_dev_* on the current stream; `rays` is a device buffer (FULL) or a host array of 6 scalars per ray
    (OD), produced just before the call.  Returns (status, shape, dist, uv or None) read back on the same stream."""
    from bvh_b200 import capi
    from bvh_b200.dtypes import BY_PREC

    F = _F(bvh.prec)
    n = rays.numel() // BY_PREC[bvh.prec]["ray"].itemsize if layout == capi.RAYS_FULL else len(rays)
    d_rays = rays if layout == capi.RAYS_FULL else _produce(rays)
    sh, dist = _buf(4 * n), _buf(F().itemsize * n)
    uv = _buf(2 * F().itemsize * n) if with_uv else None
    st = getattr(capi.lib(), f"bvhgpu_closest_hit_dev_{_sfx(bvh.prec)}")(bvh._h, _vp(d_rays), layout, n, use_triangles, _vp(sh), _vp(dist), _vp(uv))
    return st, _host(sh, np.uint32, n), _host(dist, F, n), (None if uv is None else _host(uv, F, 2 * n).reshape(n, 2))


def test_version_string():
    from bvh_b200 import capi

    v = capi.lib().bvhgpu_version()
    assert isinstance(v, bytes) and v.strip()


# ---- Ray::new and closest hit ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("name", ["cubes1", "boxes21", "random5000", "huge300", "skew3000"])
def test_closest_hit_dev_aabb_mode(api, name, prec):
    """Rays built by bvhgpu_rays_new_dev_* == O.ray_new byte for byte (-0.0 components included); closest_hit_dev in both ray
    layouts (OD recomputes inv on the device) == O.closest_hit bit for bit; dev_uv = NULL leaves shape and distance unchanged."""
    from bvh_b200 import capi

    shapes = scene(name, prec)
    want = O.build(shapes, prec)
    bvh = api.Bvh.build(shapes, prec=prec)
    o, d = _ray_inputs(shapes, 3000, prec, seed=17)
    rays = O.ray_new(o, d, prec)
    ws, wd, _ = O.closest_hit(want.nodes, shapes, rays, prec=prec)
    od = np.concatenate([rays["origin"], rays["direction"]], axis=1)
    try:
        with _side_stream(bvh.ctx):
            d_rays = _dev_rays(bvh.ctx, o, d, prec)
            assert _host(d_rays, np.uint8).tobytes() == rays.tobytes()
            for layout, src in ((capi.RAYS_FULL, None), (capi.RAYS_OD, od)):
                for with_uv in (True, False):
                    if layout == capi.RAYS_FULL:
                        d_rays = _dev_rays(bvh.ctx, o, d, prec)
                    st, gs, gd, _ = _closest_dev(bvh, d_rays if src is None else src, layout, 0, with_uv)
                    assert st == capi.OK
                    assert gs.tobytes() == ws.tobytes() and gd.tobytes() == wd.tobytes(), (layout, with_uv)
    finally:
        bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_closest_hit_dev_edges(api, prec):
    """nrays = 0 writes nothing; an empty tree gives (U32_MAX, +inf, uv 0); ray_layout 2 and triangle mode before any triangles
    were set give BVHGPU_ERR_INVALID and write nothing."""
    from bvh_b200 import capi

    F = _F(prec)
    fn = getattr(capi.lib(), f"bvhgpu_closest_hit_dev_{_sfx(prec)}")
    shapes = scene("boxes21", prec)
    bvh, empty = api.Bvh.build(shapes, prec=prec), api.Bvh.build(scene("empty", prec), prec=prec)
    o, d = _ray_inputs(shapes, 40, prec, seed=3)
    try:
        with _side_stream(bvh.ctx):
            d_rays = _dev_rays(bvh.ctx, o, d, prec)
            n = len(o)
            for tree, count, layout, tri, want_st in ((bvh, 0, capi.RAYS_FULL, 0, capi.OK), (bvh, n, 2, 0, capi.ERR_INVALID),
                                                      (bvh, n, capi.RAYS_FULL, 1, capi.ERR_INVALID)):
                sh, dist, uv = _buf(4 * n), _buf(F().itemsize * n), _buf(2 * F().itemsize * n)
                assert fn(tree._h, _vp(d_rays), layout, count, tri, _vp(sh), _vp(dist), _vp(uv)) == want_st
                for b in (sh, dist, uv):
                    assert bool((b == 0xFF).all())
            for layout in (capi.RAYS_FULL, capi.RAYS_OD):
                src = d_rays if layout == capi.RAYS_FULL else np.concatenate([o, d], axis=1)
                for tri in (0, 1):
                    st, gs, gd, guv = _closest_dev(empty, src, layout, tri)
                    assert st == capi.OK
                    assert np.all(gs == O.U32_MAX) and np.all(np.isposinf(gd)) and np.all(guv == 0)
    finally:
        bvh.free(); empty.free()


def _triangle_scene(prec):
    shapes, tris = O.create_n_cubes(500 if prec == "f32" else 300, prec=prec, want_tris=True)
    tris = np.ascontiguousarray(tris).reshape(-1, 9)
    o, d = _ray_inputs(shapes, 4000, prec, seed=23)
    rng = np.random.default_rng(5)                       # half of the rays aimed at cube centres, so that many hit a triangle
    centres = (shapes["min"][::12] + shapes["max"][::12]).astype(np.float64) * 0.5
    tgt = centres[rng.integers(0, len(centres), 2000)] + rng.uniform(-0.4, 0.4, (2000, 3))
    org = tgt + rng.normal(0, 1, (2000, 3)) * 3000
    o[:2000], d[:2000] = org, tgt - org
    return shapes, tris, o, d


def _assert_stated_tolerance(gs, gd, guv, ws, wd, wuv, tris, shapes, rays, prec):
    """The closest-hit triangle mode's stated contract (include/bvh_b200.h, tests/prunedcheck.py): identical hits agree to the bit;
    a different triangle wins only where the reference's winner lies more than 2^-16 in front of its own box entry."""
    same = gs == ws
    assert np.array_equal(gd[same], wd[same]) and np.array_equal(guv[same], wuv[same])
    assert (~same).mean() < 1e-3, (~same).mean()
    PC.check_closest(gs, gd, guv, ws, wd, tris, shapes, rays, prec)


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_set_triangles_dev_and_closest_hit_dev_triangle_mode(api, prec):
    """Triangles loaded with bvhgpu_tree_set_triangles_dev_* (no stream sync inside): closest_hit_dev in both layouts is
    byte-identical to the host closest_hit after host set_triangles, and within the stated tolerance of the oracle;
    nearest_triangles in BVH and FLAT modes returns the same bytes; a wrong triangle count is refused."""
    from bvh_b200 import capi

    shapes, tris, o, d = _triangle_scene(prec)
    rays = O.ray_new(o, d, prec)
    ref, dev = api.Bvh.build(shapes, prec=prec), api.Bvh.build(shapes, prec=prec)
    ref.set_triangles(tris)
    hs, hd, huv = ref.closest_hit(rays, triangles=True)
    want = O.build(shapes, prec)
    ws, wd, wuv = O.closest_hit(want.nodes, shapes, rays, tris, prec)
    _assert_stated_tolerance(hs, hd, huv, ws, wd, wuv, tris, shapes, rays, prec)
    assert int((ws != O.U32_MAX).sum()) > 500
    fn = getattr(capi.lib(), f"bvhgpu_tree_set_triangles_dev_{_sfx(prec)}")
    rng = np.random.default_rng(77)
    pts = np.concatenate([shapes["min"][rng.integers(0, len(shapes), 1000)] + rng.normal(0, 3.0, (1000, 3)), rng.uniform(-1.2e5, 1.2e5, (1000, 3))])
    try:
        with _side_stream(dev.ctx):
            d_tris = _produce(tris)
            capi.check(fn(dev._h, _vp(d_tris), len(tris)))
            od = np.concatenate([rays["origin"], rays["direction"]], axis=1)
            for layout in (capi.RAYS_FULL, capi.RAYS_OD):
                for with_uv in (True, False):
                    src = _dev_rays(dev.ctx, o, d, prec) if layout == capi.RAYS_FULL else od
                    st, gs, gd, guv = _closest_dev(dev, src, layout, 1, with_uv)
                    assert st == capi.OK
                    assert gs.tobytes() == hs.tobytes() and gd.tobytes() == hd.tobytes(), (layout, with_uv)
                    if with_uv:
                        assert guv.tobytes() == huv.tobytes()
            for mode in (capi.TRAVERSE_BVH, capi.TRAVERSE_FLAT):
                a, b = ref.nearest_triangles_batch(pts, mode), dev.nearest_triangles_batch(pts, mode)
                assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes(), mode
            bad = _produce(tris[:-1])
            assert fn(dev._h, _vp(bad), len(tris) - 1) == capi.ERR_INVALID
            assert fn(dev._h, _vp(d_tris), len(tris) + 1) == capi.ERR_INVALID
            st, gs, gd, _ = _closest_dev(dev, od, capi.RAYS_OD, 1)           # the triangles loaded before are still in place
            assert gs.tobytes() == hs.tobytes() and gd.tobytes() == hd.tobytes()
    finally:
        ref.free(); dev.free()


# ---- Aabb / Point / Ball queries on device pointers --------------------------------------------------------------------------------
def _queries(shapes, n=3000):
    """The generator of test_query_parity: points (200 exactly on box corners), boxes and balls over the scene's bounds."""
    from bvh_b200 import capi

    rng = np.random.default_rng(12)
    lo, hi = shapes["min"].min(axis=0).astype(float), shapes["max"].max(axis=0).astype(float)
    ext = hi - lo + 1e-3
    pts = rng.uniform(lo - 0.05 * ext, hi + 0.05 * ext, (n, 3))
    pts[:200] = shapes["min"][rng.integers(0, len(shapes), 200)]
    amin = rng.uniform(lo, hi, (n, 3))
    aab = np.concatenate([amin, amin + rng.uniform(0, 0.2, (n, 3)) * ext], axis=1)
    balls = np.concatenate([rng.uniform(lo, hi, (n, 3)), (rng.uniform(0, 0.15, (n, 1)) * ext.max())], axis=1)
    return ((capi.QUERY_AABB, aab), (capi.QUERY_POINT, pts), (capi.QUERY_BALL, balls))


def _query_dev(bvh, mode, kind, q, cap, want_total=True, spin=SPIN, hits_len=None):
    """bvhgpu_query_dev_* on the current stream with the queries produced just before.  Returns (status, total or None, offsets,
    hits buffer of max(cap, hits_len) entries, the stream's idle state right after the call returned)."""
    import torch
    from bvh_b200 import capi

    n = len(q)
    d_q = _produce(q, spin=spin)
    d_off, d_hits = _buf(4 * (n + 1)), _buf(4 * max(cap, hits_len or 0))
    tot = C.c_size_t(12345)
    st = getattr(capi.lib(), f"bvhgpu_query_dev_{_sfx(bvh.prec)}")(bvh._h, mode, kind, _vp(d_q), n, _vp(d_off), _vp(d_hits), cap,
                                                                 C.byref(tot) if want_total else None)
    idle = torch.cuda.current_stream().query()
    return st, (tot.value if want_total else None), _host(d_off, np.uint32, n + 1), _host(d_hits, np.uint32), idle


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("name", ["boxes21", "random3000", "points500", "huge300"])
def test_query_dev(api, name, prec):
    """AABB / Point / Ball x BVH / FLAT: the CSR of query_dev == O.query.  total = NULL returns before the stream has run and gives
    the same result; cap below the total: BVHGPU_ERR_CAPACITY, the right *total, complete offsets, hits[:cap] = the prefix of the
    full list, nothing written at or after cap."""
    from bvh_b200 import capi

    F = _F(prec)
    shapes = scene(name, prec)
    want = O.build(shapes, prec)
    flat = O.flatten(want.nodes, prec)
    bvh = api.Bvh.build(shapes, prec=prec)
    checked_async = False
    try:
        with _side_stream(bvh.ctx):
            for kind, q in _queries(shapes):
                q = q.astype(F)
                for mode, fl in ((capi.TRAVERSE_BVH, None), (capi.TRAVERSE_FLAT, flat)):
                    woff, whits = O.query(kind, q, want.nodes, shapes, fl, prec)
                    tot = len(whits)
                    st, total, off, hits, _ = _query_dev(bvh, mode, kind, q, tot)
                    assert st == capi.OK and total == tot, (kind, mode)
                    assert np.array_equal(off.astype(np.uint64), woff) and np.array_equal(hits[:tot], whits), (kind, mode)
                    spin = SPIN if checked_async else LONG_SPIN
                    st, _, off, hits, idle = _query_dev(bvh, mode, kind, q, tot, want_total=False, spin=spin)
                    assert st == capi.OK
                    if not checked_async:
                        assert not idle                  # returned while the producer was still running
                        checked_async = True
                    assert np.array_equal(off.astype(np.uint64), woff) and np.array_equal(hits[:tot], whits), (kind, mode)
                    if tot >= 2:
                        cap = tot // 2
                        st, total, off, hits, _ = _query_dev(bvh, mode, kind, q, cap, hits_len=tot)
                        assert st == capi.ERR_CAPACITY and total == tot, (kind, mode)
                        assert np.array_equal(off.astype(np.uint64), woff)
                        assert np.array_equal(hits[:cap], whits[:cap]) and np.all(hits[cap:] == O.U32_MAX), (kind, mode)
    finally:
        bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_query_dev_edges_and_kinds(api, prec):
    """n = 0 and an empty tree give all-zero offsets and no hits.  A kind outside {AABB, POINT, BALL} is refused with
    BVHGPU_ERR_INVALID and nothing is written; the query buffer holds 6 scalars per query and the hit buffer the full result, so
    that an implementation which accepted the kind would stay inside every buffer."""
    from bvh_b200 import capi

    F = _F(prec)
    shapes = scene("boxes21", prec)
    bvh, empty = api.Bvh.build(shapes, prec=prec), api.Bvh.build(scene("empty", prec), prec=prec)
    q = np.concatenate([shapes["min"], shapes["max"]], axis=1).astype(F)          # 21 boxes: every query hits its own shape
    woff, whits = O.query(O.QUERY_AABB, q, O.build(shapes, prec).nodes, shapes, None, prec)
    full = 64 * len(q)
    assert len(whits) <= full
    try:
        with _side_stream(bvh.ctx):
            st, total, off, _, _ = _query_dev(bvh, capi.TRAVERSE_BVH, capi.QUERY_POINT, q[:0, :3], 16)
            assert st == capi.OK and total == 0 and off.tolist() == [0]
            for kind, stride in ((capi.QUERY_AABB, 6), (capi.QUERY_POINT, 3), (capi.QUERY_BALL, 4)):
                for mode in (capi.TRAVERSE_BVH, capi.TRAVERSE_FLAT):
                    st, total, off, hits, _ = _query_dev(empty, mode, kind, q[:, :stride].copy(), 16)
                    assert st == capi.OK and total == 0 and not off.any() and np.all(hits == O.U32_MAX)
            for kind in (0, 4, 5, -1):
                for mode in (capi.TRAVERSE_BVH, capi.TRAVERSE_FLAT):
                    st, total, off, hits, _ = _query_dev(bvh, mode, kind, q, full)
                    assert st == capi.ERR_INVALID, (kind, mode)
                    assert np.all(off == O.U32_MAX) and np.all(hits == O.U32_MAX), (kind, mode)
            st, total, off, hits, _ = _query_dev(bvh, capi.TRAVERSE_BVH, capi.QUERY_AABB, q, full)      # the tree is still fine
            assert st == capi.OK and np.array_equal(off.astype(np.uint64), woff) and np.array_equal(hits[:total], whits)
    finally:
        bvh.free(); empty.free()


# ---- Bvh::update_shapes on device pointers -----------------------------------------------------------------------------------------
def _motion(shapes, prec, frac=0.05, seed=31):
    F = shapes["min"].dtype
    rng = np.random.default_rng(seed)
    m = max(1, int(len(shapes) * frac))
    moved = rng.choice(len(shapes), m, replace=False).astype(np.uint32)
    ext = float(shapes["max"].max() - shapes["min"].min())
    delta = rng.uniform(-ext / 8, ext / 8, (m, 3)).astype(F)
    new = shapes.copy()
    new["min"][moved] += delta
    new["max"][moved] += delta
    return moved, new


def _update_dev(bvh, idx, fresh, max_growth, want_rebuilt=True):
    from bvh_b200 import capi

    d_idx, d_fresh = _produce(np.ascontiguousarray(idx, dtype=np.uint32), np.ascontiguousarray(fresh))
    rb = C.c_size_t(777)
    st = getattr(capi.lib(), f"bvhgpu_update_dev_{_sfx(bvh.prec)}")(bvh._h, _vp(d_idx), _vp(d_fresh), len(idx), C.c_double(max_growth),
                                                                  C.byref(rb) if want_rebuilt else None)
    bvh._nodes = None
    return st, rb.value


def _tree_bytes(bvh):
    bvh._nodes = None
    return bvh.nodes.tobytes() + bvh.node_index.tobytes()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_update_dev(api, prec):
    """update_dev with max_growth 1.5 and 0 == the host update_shapes on the same motion, byte for byte (nodes and node_index),
    with and without `rebuilt` (NULL: the asynchronous return); a changed list that repeats indices with the same AABBs gives the
    tree of the list without the repeats."""
    from bvh_b200 import capi

    shapes = scene("cubes1000" if prec == "f32" else "random3000", prec)
    moved, new = _motion(shapes, prec)
    rep = np.concatenate([moved, moved[::3], moved[:5]])           # every third index twice, the first five up to three times
    for mg in (1.5, 0.0):
        host = api.Bvh.build(shapes, prec=prec)
        r_host = host.update_shapes(moved, new, mg)
        want = _tree_bytes(host)
        assert (r_host > 0) == (mg > 0)
        trees = [api.Bvh.build(shapes, prec=prec) for _ in range(3)]
        try:
            with _side_stream(trees[0].ctx):
                st, rb = _update_dev(trees[0], moved, new[moved], mg)
                assert st == capi.OK and rb == r_host
                st, _ = _update_dev(trees[1], moved, new[moved], mg, want_rebuilt=False)
                assert st == capi.OK
                st, _ = _update_dev(trees[2], rep, new[rep], mg, want_rebuilt=False)
                assert st == capi.OK
                for i, t in enumerate(trees):
                    assert _tree_bytes(t) == want, (mg, i)
        finally:
            host.free()
            for t in trees:
                t.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_update_dev_rejects_bad_input_untouched(api, prec):
    """An index >= n (BVHGPU_ERR_INVALID) or a NaN coordinate (BVHGPU_ERR_NAN) in the device-side lists is refused before the tree
    is touched: same bytes, and it still traverses like the oracle."""
    from bvh_b200 import capi

    shapes = scene("cubes1000", prec)
    bvh = api.Bvh.build(shapes, prec=prec)
    before = _tree_bytes(bvh)
    nodes = bvh.nodes.copy()
    nan_boxes = shapes[[3, 10, 11]].copy()
    nan_boxes["max"][1][2] = np.nan
    try:
        with _side_stream(bvh.ctx):
            for idx, fresh, want_st in ((np.array([1, len(shapes)]), shapes[[1, 2]], capi.ERR_INVALID),
                                        (np.array([3, 10, 11]), nan_boxes, capi.ERR_NAN)):
                for mg in (1.5, 0.0):
                    st, _ = _update_dev(bvh, idx, fresh, mg)
                    assert st == want_st, (want_st, mg)
                    assert _tree_bytes(bvh) == before
        rays = rays_for(shapes, 1000, prec, seed=5, axis_aligned=100)
        r = O.traverse(nodes, shapes, rays, O.MODE_RECURSIVE, prec)
        off, hits = bvh.traverse_batch(rays)
        assert np.array_equal(off.astype(np.uint64), r.offsets) and np.array_equal(hits, r.hits)
    finally:
        bvh.free()


# ---- refit / optimize / add / remove / OD traversal on device pointers, both precisions ---------------------------------------------
@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_refit_and_optimize_dev(api, prec):
    """bvhgpu_refit_dev_* / bvhgpu_optimize_dev_* == the host forms, byte for byte."""
    from bvh_b200 import capi

    L = capi.lib()
    shapes = scene("cubes1000", prec)
    rng = np.random.default_rng(21)
    moved = rng.choice(len(shapes), 600, replace=False)
    delta = rng.uniform(-3000, 3000, (600, 3)).astype(_F(prec))
    new = shapes.copy()
    new["min"][moved] += delta
    new["max"][moved] += delta
    a, b, a2, b2 = (api.Bvh.build(shapes, prec=prec) for _ in range(4))
    try:
        a.refit(new)
        ra = a2.optimize(new, 1.5)
        with _side_stream(b.ctx):
            capi.check(getattr(L, f"bvhgpu_refit_dev_{_sfx(prec)}")(b._h, _vp(_produce(new)), len(new)))
            assert _tree_bytes(a) == _tree_bytes(b)
            rb = C.c_size_t(0)
            capi.check(getattr(L, f"bvhgpu_optimize_dev_{_sfx(prec)}")(b2._h, _vp(_produce(new)), len(new), C.c_double(1.5), C.byref(rb)))
            assert ra == rb.value and ra > 0
            assert _tree_bytes(a2) == _tree_bytes(b2)
        assert O.is_consistent(b2.nodes, new, prec) and O.is_tight(b2.nodes, prec)
    finally:
        for t in (a, b, a2, b2):
            t.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_add_and_remove_shapes_dev_and_node_counts(api, prec):
    """bvhgpu_remove_shapes_dev_* / bvhgpu_add_shapes_dev_* == the host forms byte for byte (add with and without `rebuilt`);
    bvhgpu_tree_num_nodes_* is 2n-1 after build, add and remove, and 0 for an empty tree."""
    from bvh_b200 import capi

    L = capi.lib()
    num_nodes = getattr(L, f"bvhgpu_tree_num_nodes_{_sfx(prec)}")
    shapes = scene("cubes300", prec)
    n = len(shapes)
    rng = np.random.default_rng(6)
    idx = rng.choice(n, 97, replace=False).astype(np.uint32)
    mn = rng.uniform(-1000, 1000, (40, 3))
    new = O.make_aabbs(mn, mn + rng.uniform(0, 30, (40, 3)), prec)
    host, dev, dev2 = (api.Bvh.build(shapes, prec=prec) for _ in range(3))
    empty = api.Bvh.build(scene("empty", prec), prec=prec)
    try:
        assert num_nodes(host._h) == 2 * n - 1 and num_nodes(empty._h) == 0
        host.remove_shapes(idx)
        with _side_stream(dev.ctx):
            for t in (dev, dev2):
                capi.check(getattr(L, f"bvhgpu_remove_shapes_dev_{_sfx(prec)}")(t._h, _vp(_produce(idx)), len(idx)))
                assert _tree_bytes(t) == _tree_bytes(host)
                assert num_nodes(t._h) == 2 * (n - 97) - 1
            r_host = host.add_shapes(new, max_growth=1.5)
            rb = C.c_size_t(777)
            capi.check(getattr(L, f"bvhgpu_add_shapes_dev_{_sfx(prec)}")(dev._h, _vp(_produce(new)), len(new), C.c_double(1.5), C.byref(rb)))
            assert rb.value == r_host
            capi.check(getattr(L, f"bvhgpu_add_shapes_dev_{_sfx(prec)}")(dev2._h, _vp(_produce(new)), len(new), C.c_double(1.5), None))
            for t in (dev, dev2):
                assert _tree_bytes(t) == _tree_bytes(host)
                assert num_nodes(t._h) == 2 * (n - 97 + 40) - 1
            capi.check(getattr(L, f"bvhgpu_add_shapes_dev_{_sfx(prec)}")(empty._h, _vp(_produce(new)), len(new), C.c_double(0.0), None))
            assert num_nodes(empty._h) == 2 * len(new) - 1
            capi.check(getattr(L, f"bvhgpu_remove_shapes_dev_{_sfx(prec)}")(empty._h, _vp(_produce(np.arange(len(new), dtype=np.uint32))), len(new)))
            assert num_nodes(empty._h) == 0 and empty.num_shapes == 0
        assert num_nodes(host._h) == 2 * host.num_shapes - 1
    finally:
        for t in (host, dev, dev2, empty):
            t.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_traverse_od_dev(api, prec):
    """bvhgpu_traverse_od_dev_* on 100 k rays == the host OD form == the oracle, in BVH and FLAT modes."""
    from bvh_b200 import capi

    shapes = O.create_n_cubes(2000, prec=prec)
    want = O.build(shapes, prec)
    rays, _ = O.create_rays(100_000, prec=prec)
    bvh = api.Bvh.build(shapes, prec=prec)
    od = np.concatenate([rays["origin"], rays["direction"]], axis=1)
    fn = getattr(capi.lib(), f"bvhgpu_traverse_od_dev_{_sfx(prec)}")
    try:
        for mode, tree, omode in ((capi.TRAVERSE_BVH, want.nodes, O.MODE_RECURSIVE), (capi.TRAVERSE_FLAT, O.flatten(want.nodes, prec), O.MODE_FLAT)):
            r = O.traverse(tree, shapes, rays, omode, prec, threads=O.hardware_threads())
            hoff, hhits = bvh.traverse_batch(rays, mode=mode, compact=True)
            assert np.array_equal(hoff.astype(np.uint64), r.offsets) and np.array_equal(hhits, r.hits)
            with _side_stream(bvh.ctx):
                d_od = _produce(od)
                d_off, d_hits = _buf(4 * (len(rays) + 1)), _buf(4 * len(r.hits))
                tot = C.c_size_t(0)
                capi.check(fn(bvh._h, mode, _vp(d_od), len(rays), _vp(d_off), _vp(d_hits), len(r.hits), C.byref(tot)))
                assert tot.value == len(r.hits)
                assert _host(d_off, np.uint32).tobytes() == hoff.tobytes() and _host(d_hits, np.uint32).tobytes() == hhits.tobytes()
    finally:
        bvh.free()


# ---- capacity branches that fetch the retained result --------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_capacity_and_fetch(api, prec):
    """traverse, query and nearest_candidates with `cap` below the total: BVHGPU_ERR_CAPACITY with the needed size, complete
    offsets, then bvhgpu_traverse_fetch_* returns the full list (= the oracle's for traverse and query); a fetch with too small a
    buffer is refused."""
    from bvh_b200 import capi

    L = capi.lib()
    sfx = _sfx(prec)
    fetch = getattr(L, f"bvhgpu_traverse_fetch_{sfx}")
    shapes = scene("random5000", prec)
    want = O.build(shapes, prec)
    bvh = api.Bvh.build(shapes, prec=prec)
    F = _F(prec)

    def p(a):
        return a.ctypes.data_as(C.c_void_p)

    def check_fetch(off, woff, whits, total):
        assert total.value == len(whits) > 8 and np.array_equal(off.astype(np.uint64), woff)
        assert fetch(bvh._h, p(np.zeros(8, dtype=np.uint32)), 8) == capi.ERR_CAPACITY
        full = np.zeros(total.value, dtype=np.uint32)
        capi.check(fetch(bvh._h, p(full), total.value))
        assert np.array_equal(full, whits)

    try:
        rays = rays_for(shapes, 2000, prec, seed=2, axis_aligned=200)
        r = O.traverse(want.nodes, shapes, rays, O.MODE_RECURSIVE, prec)
        small = np.zeros(8, dtype=np.uint32)
        for name in ("traverse", "traverse_od"):
            src = rays if name == "traverse" else np.ascontiguousarray(np.concatenate([rays["origin"], rays["direction"]], axis=1))
            off, total = np.zeros(len(rays) + 1, dtype=np.uint32), C.c_size_t(0)
            st = getattr(L, f"bvhgpu_{name}_{sfx}")(bvh._h, capi.TRAVERSE_BVH, p(src), len(rays), p(off), p(small), 8, C.byref(total))
            assert st == capi.ERR_CAPACITY, name
            check_fetch(off, r.offsets, r.hits, total)
        for kind, q in _queries(shapes, 1000):
            q = np.ascontiguousarray(q, dtype=F)
            woff, whits = O.query(kind, q, want.nodes, shapes, None, prec)
            off, total = np.zeros(len(q) + 1, dtype=np.uint32), C.c_size_t(0)
            st = getattr(L, f"bvhgpu_query_{sfx}")(bvh._h, capi.TRAVERSE_BVH, kind, p(q), len(q), p(off), p(small), 8, C.byref(total))
            assert st == capi.ERR_CAPACITY, kind
            check_fetch(off, woff, whits, total)
        pts = np.ascontiguousarray(_queries(shapes, 1000)[1][1], dtype=F)
        off_ok, cand_ok = bvh.nearest_candidates(pts)
        ws, _ = O.nearest_to(want.nodes, shapes, pts, prec)
        for i in range(len(pts)):                                        # every list holds the nearest shape
            assert ws[i] in cand_ok[off_ok[i]:off_ok[i + 1]]
        off, total = np.zeros(len(pts) + 1, dtype=np.uint32), C.c_size_t(0)
        st = getattr(L, f"bvhgpu_nearest_candidates_{sfx}")(bvh._h, p(pts), len(pts), p(off), p(small), 8, C.byref(total))
        assert st == capi.ERR_CAPACITY
        check_fetch(off, off_ok.astype(np.uint64), cand_ok, total)
    finally:
        bvh.free()
