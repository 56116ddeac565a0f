"""bvhgpu_triangle_pairs_* / bvhgpu_triangle_pairs_trees_* (Bvh.triangle_pairs, triangle_pairs_with and their _dev forms) against the
exact model of tests/tritri.py, byte for byte: offsets and hits, f32 and f64, both skip_shared values.  Scenes: overlapping, nested
and vertex-touching icospheres, tori, the configs[1] cubes (coincident faces: the exact coplanar path), Sponza, the adversarial
families, small-grid soups; every build mode; refit / update / remove / add; the identities between the forms; launch and capacity
edges, refusals, two contexts, sticky builds and the _dev forms on a side stream."""
import ctypes as C

import numpy as np
import pytest

from bvh_b200 import scenes
from bvh_b200.dtypes import BY_PREC
from oracle import oracle as O
from tests import adversarial as A, crossings as X, overlapref as R, tritri as T

pytestmark = pytest.mark.gpu
FT = {"f32": np.float32, "f64": np.float64}


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A_

    return A_


def _aabbs(prec, mn, mx):
    a = np.zeros(len(mn), dtype=BY_PREC[prec]["aabb"])
    a["min"], a["max"] = mn, mx
    return a


def _tree(api, tris, prec, mode=0, ctx=None, boxes=None):
    F = FT[prec]
    tris = np.ascontiguousarray(tris, dtype=F).reshape(-1, 3, 3)
    mn, mx = T.tri_boxes(tris, F) if boxes is None else boxes
    b = api.Bvh.build(_aabbs(prec, mn, mx), prec=prec, mode=mode, ctx=ctx)
    if len(tris):
        b.set_triangles(tris)
    return b


def _leaf(bvh):
    from bvh_b200 import capi

    n = bvh.num_shapes
    nodes = np.zeros(max(2 * n - 1, 0), dtype=bvh._d["node"])
    idx = np.zeros(n, dtype=np.uint32)
    capi.check(getattr(capi.lib(), f"bvhgpu_tree_nodes_{bvh._d['suffix']}")(bvh._h, nodes.ctypes.data_as(C.c_void_p), idx.ctypes.data_as(C.c_void_p)))
    return idx


def _dev_self(b, skip, n, cap):
    import torch

    d_off = torch.full((n + 1,), 7, dtype=torch.int32, device="cuda")
    d_hits = torch.full((max(cap, 1),), 7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    tot = b.triangle_pairs_dev(d_off.data_ptr(), d_hits.data_ptr(), cap, skip_shared=skip, want_total=True)
    return d_off.cpu().numpy().view(np.uint32), d_hits.cpu().numpy().view(np.uint32)[:tot]


def _dev_cross(a, b, n, cap):
    import torch

    d_off = torch.full((n + 1,), 7, dtype=torch.int32, device="cuda")
    d_hits = torch.full((max(cap, 1),), 7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    tot = a.triangle_pairs_with_dev(b, d_off.data_ptr(), d_hits.data_ptr(), cap, want_total=True)
    return d_off.cpu().numpy().view(np.uint32), d_hits.cpu().numpy().view(np.uint32)[:tot]


def check_self(b, tris, F, boxes=None, dev=True):
    """Both skip_shared values of the host form (and the _dev form) equal the model on the tree's current leaves."""
    mn, mx = T.tri_boxes(tris, F) if boxes is None else boxes
    leaf = _leaf(b)
    model = T.Model(tris, F)
    out = {}
    for skip in (True, False):
        ro, rh = T.self_rows(tris, mn, mx, leaf, F, skip, model)
        off, hits = b.triangle_pairs(skip_shared=skip)
        assert off.tobytes() == ro.tobytes() and hits.tobytes() == rh.tobytes(), skip
        if dev:
            do, dh = _dev_self(b, skip, len(tris), len(rh))
            assert do.tobytes() == ro.tobytes() and dh.tobytes() == rh.tobytes(), skip
        out[skip] = (off, hits)
    return out


def check_cross(a, b, tris_a, tris_b, F, boxes_a=None, boxes_b=None, dev=True):
    amn, amx = T.tri_boxes(tris_a, F) if boxes_a is None else boxes_a
    bmn, bmx = T.tri_boxes(tris_b, F) if boxes_b is None else boxes_b
    ro, rh = T.cross_tri_rows(tris_a, amn, amx, tris_b, bmn, bmx, _leaf(b), F)
    off, hits = a.triangle_pairs_with(b)
    assert off.tobytes() == ro.tobytes() and hits.tobytes() == rh.tobytes()
    if dev:
        do, dh = _dev_cross(a, b, len(amn), len(rh))
        assert do.tobytes() == ro.tobytes() and dh.tobytes() == rh.tobytes()
    return off, hits


def _soup(rng, n, F, extent=12, size=4):
    """n triangles on a grid of half-integers: corners at integer cells of [0, extent)^3, vertices up to size / 2 away.  Coplanar,
    touching and shared-vertex pairs are frequent; each triangle meets a few others."""
    c = rng.integers(0, extent, size=(n, 1, 3))
    return ((2 * c + rng.integers(0, size + 1, size=(n, 3, 3))) / 2).astype(F)


def _sphere(F, level=3, r=1.0, c=(0, 0, 0)):
    return (X.icosphere(level) * r + np.array(c)).astype(F)


@pytest.mark.parametrize("prec", FT)
def test_icospheres_overlapping_nested_and_touching(api, prec):
    F = FT[prec]
    s = _sphere(F)
    for other, want in ((_sphere(F, c=(0.9, 0.3, 0.1)), "some"), (_sphere(F, r=0.5), "none")):
        both = np.concatenate([s, other])
        b = _tree(api, both, prec)
        rows = check_self(b, both, F)
        ta, tb = _tree(api, s, prec), _tree(api, other, prec)
        off, hits = check_cross(ta, tb, s, other, F)
        assert (len(hits) > 0) == (want == "some")
        if want == "none":                                  # nested: the only pairs are the adjacent faces of one sphere
            assert len(rows[True][1]) == 0
        for t in (b, ta, tb):
            t.free()
    # touching at exactly one vertex: a sphere's vertex mirrored onto a second sphere's vertex
    v = s.reshape(-1, 3)[np.argmax(s.reshape(-1, 3)[:, 0])]          # the vertex of largest x
    mirror = (np.array([2 * v[0], 0, 0]) + s * np.array([-1, 1, 1])).astype(F)   # reflected across x = v.x: shares exactly v
    ta, tb = _tree(api, s, prec), _tree(api, mirror, prec)
    off, hits = check_cross(ta, tb, s, mirror, F)
    touching = {(int(a), int(b)) for a, b in R.pairs(off, hits)}
    around = np.nonzero(np.all(s == v, axis=2).any(axis=1))[0]
    assert len(touching) == len(around) ** 2 and {a for a, _ in touching} == set(around.tolist())
    for t in (ta, tb):
        t.free()


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("prec", FT)
def test_tori_every_build_mode(api, prec, mode):
    F = FT[prec]
    a = X.torus(F=F).astype(F)
    b = (X.torus(F=F) + np.array([0.9, 0.25, 0.125])).astype(F)
    both = np.concatenate([a, b])
    t = _tree(api, both, prec, mode=mode)
    rows = check_self(t, both, F, dev=mode == 0)
    assert len(rows[True][1]) > 0
    ta, tb = _tree(api, a, prec, mode=mode), _tree(api, b, prec, mode=mode)
    check_cross(ta, tb, a, b, F, dev=mode == 0)
    check_cross(tb, ta, b, a, F, dev=False)
    for x in (t, ta, tb):
        x.free()


@pytest.mark.parametrize("prec", FT)
def test_configs1_cubes_coplanar_path(api, prec):
    """The cube scene: each cube's faces share edges; against a copy moved by one cube along x, the copy's -x faces lie on the +x
    faces, which puts their pairs on the coplanar path."""
    F = FT[prec]
    tris = scenes.create_n_cubes_tris(1500, prec)
    boxes = (scenes.create_n_cubes_aabbs(1500, prec)["min"], scenes.create_n_cubes_aabbs(1500, prec)["max"])
    b = _tree(api, tris, prec, boxes=boxes)
    rows = check_self(b, tris, F, boxes=boxes)
    assert len(rows[False][1]) > len(rows[True][1])
    shift = np.array([1, 0, 0], dtype=F)                      # the copy's -x faces on the +x faces: coincident coplanar triangles
    shifted = (tris + shift).astype(F)
    sb = ((boxes[0] + shift).astype(F), (boxes[1] + shift).astype(F))
    c = _tree(api, shifted, prec, boxes=sb)
    off, hits = check_cross(b, c, tris, shifted, F, boxes_a=boxes, boxes_b=sb)
    assert len(hits) > 0
    b.free()
    c.free()


def _sponza(F):
    z = np.load(__import__("os").path.join(__import__("os").path.dirname(__file__), "golden", "sponza_tris.npz"))
    return z["vertices"][z["triangles"].astype(np.int64)].astype(F)


@pytest.mark.parametrize("prec", FT)
def test_sponza_rows(api, prec):
    """Sponza: a seeded sample of 5 000 rows, and with skip_shared every row the device reports non-empty, against the overlap rows
    filtered by the model (the overlap rows themselves are held to their brute force by the overlap tests)."""
    F = FT[prec]
    tris = _sponza(F)
    b = _tree(api, tris, prec)
    o_off, o_hits = b.overlap_pairs()
    model = T.Model(tris, F)
    rng = np.random.default_rng(7)
    for skip in (True, False):
        off, hits = b.triangle_pairs(skip_shared=skip)
        n = len(tris)
        rows = set(rng.choice(n, 5000, replace=False).tolist())
        if skip:                                            # without skip_shared nearly every row holds its neighbours: sampled only
            rows |= set(np.nonzero(np.diff(off.astype(np.int64)))[0].tolist())
        rows = np.array(sorted(rows))
        lo, hi = o_off[rows].astype(np.int64), o_off[rows + 1].astype(np.int64)
        s = np.repeat(rows, hi - lo)
        cand = np.concatenate([o_hits[a:e] for a, e in zip(lo, hi)]) if len(rows) else np.zeros(0, np.uint32)
        keep = model.keep(s, cand, skip)
        want_counts = np.bincount(np.searchsorted(rows, s[keep]), minlength=len(rows))
        assert np.array_equal(np.diff(off.astype(np.int64))[rows], want_counts)
        got = np.concatenate([hits[off[r]:off[r + 1]] for r in rows])
        assert got.tobytes() == cand[keep].astype(np.uint32).tobytes()
        if skip:
            assert len(hits) > 0
    b.free()


def _box_tris(mn, mx, F):
    """A triangle spanning three corners of every box: degenerate for point and flat boxes."""
    a = mn
    b = np.stack([mx[:, 0], mn[:, 1], mx[:, 2]], axis=1)
    c = np.stack([mn[:, 0], mx[:, 1], mx[:, 2]], axis=1)
    return np.stack([a, b, c], axis=1).astype(F)


@pytest.mark.parametrize("family", ["shared_edges", "degenerate", "large_coordinates", "mixed_scales", "overflow", "grid_soup"])
@pytest.mark.parametrize("prec", FT)
def test_adversarial_families(api, prec, family):
    F = FT[prec]
    if family in ("shared_edges", "degenerate"):
        tris = getattr(A, family)(F)[0].reshape(-1, 3, 3).astype(F)
    elif family == "grid_soup":
        rng = np.random.default_rng(21)
        tris = _soup(rng, 600, F, extent=6)
    else:
        mn, mx = getattr(A, family)(F, 3)[:2]
        tris = _box_tris(np.asarray(mn, dtype=F), np.asarray(mx, dtype=F), F)
    t = _tree(api, tris, prec)
    check_self(t, tris, F)
    half = len(tris) // 2
    ta, tb = _tree(api, tris[:half], prec), _tree(api, tris[half:], prec)
    check_cross(ta, tb, tris[:half], tris[half:], F)
    for x in (t, ta, tb):
        x.free()


@pytest.mark.parametrize("prec", FT)
def test_dynamic_calls_and_stale_triangles(api, prec):
    from bvh_b200 import capi

    F = FT[prec]
    rng = np.random.default_rng(31)
    tris = _soup(rng, 700, F)
    t = _tree(api, tris, prec)
    check_self(t, tris, F, dev=False)
    # refit to moved triangles, then set them: the moved scene
    moved = (tris + rng.integers(-2, 3, size=(len(tris), 1, 3)) / 2).astype(F)
    mn, mx = T.tri_boxes(moved, F)
    t.refit(_aabbs(prec, mn, mx))
    # stale triangles: the result is still the new overlap rows filtered by the old triangles
    leaf = _leaf(t)
    for skip in (True, False):
        ro, rh = T.self_rows(tris, mn, mx, leaf, F, skip)
        off, hits = t.triangle_pairs(skip_shared=skip)
        assert off.tobytes() == ro.tobytes() and hits.tobytes() == rh.tobytes()
    t.set_triangles(moved)
    check_self(t, moved, F, dev=False)
    # update_shapes with a rebuild
    changed = rng.choice(len(moved), 80, replace=False)
    moved[changed] = (moved[changed] + 3).astype(F)
    mn, mx = T.tri_boxes(moved, F)
    t.update_shapes(changed, _aabbs(prec, mn, mx), max_growth=1.5)
    t.set_triangles(moved)
    check_self(t, moved, F, dev=False)
    # remove_shapes: the triangles follow their shapes
    gone = rng.choice(len(moved), 90, replace=False)
    moves = t.remove_shapes(gone)
    after = moved.copy()
    for new_i, old_i in moves:
        after[new_i] = moved[old_i]
    moved = after[: len(after) - len(gone)].copy()
    check_self(t, moved, F, dev=False)
    # add_shapes drops the triangles: refused until set_triangles again
    extra = _soup(rng, 40, F)
    t.add_shapes(_aabbs(prec, *T.tri_boxes(extra, F)))
    with pytest.raises(capi.BvhGpuError) as e:
        t.triangle_pairs()
    assert e.value.status == capi.ERR_INVALID
    moved = np.concatenate([moved, extra])
    t.set_triangles(moved)
    check_self(t, moved, F)
    t.free()


@pytest.mark.parametrize("prec", FT)
def test_identities(api, prec):
    F = FT[prec]
    rng = np.random.default_rng(41)
    a_t = _soup(rng, 500, F, extent=8)
    b_t = (_soup(rng, 450, F, extent=8) + F(0.25)).astype(F)
    a, b = _tree(api, a_t, prec), _tree(api, b_t, prec)
    so, sh = a.triangle_pairs(skip_shared=False)
    mo, mh = check_cross(a, a, a_t, a_t, F)
    sym = {(s, t) for s, t in R.pairs(so, sh).tolist()} | {(t, s) for s, t in R.pairs(so, sh).tolist()}
    sym |= {(s, s) for s in range(len(a_t)) if T.classify(a_t[s], F)[0] != T.EXCLUDED}
    assert set(map(tuple, R.pairs(mo, mh).tolist())) == sym and len(mh) == len(sym)
    off, hits = check_cross(a, b, a_t, b_t, F)
    to, th = check_cross(b, a, b_t, a_t, F)
    assert set(map(tuple, R.pairs(off, hits).tolist())) == {(s, t) for t, s in R.pairs(to, th).tolist()}
    assert len(hits) > 0
    a.free()
    b.free()


@pytest.mark.parametrize("n", [255, 256, 257, 2047, 2048, 2049])
def test_launch_geometry(api, n):
    F = np.float32
    rng = np.random.default_rng(n)
    tris = _soup(rng, n, F, extent=int(2 * n ** (1 / 3)) + 2)
    t = _tree(api, tris, "f32")
    check_self(t, tris, F)
    u = _tree(api, tris[: n // 3], "f32")
    check_cross(t, u, tris, tris[: n // 3], F)
    t.free()
    u.free()


def _fn(bvh, trees=False, dev=False):
    from bvh_b200 import capi

    return getattr(capi.lib(), f"bvhgpu_triangle_pairs_{'trees_' if trees else ''}{'dev_' if dev else ''}{bvh._d['suffix']}")


@pytest.mark.parametrize("prec", FT)
def test_contract(api, prec):
    import torch

    from bvh_b200 import capi

    F = FT[prec]
    rng = np.random.default_rng(51)
    tris = _soup(rng, 800, F, extent=8)
    mn, mx = T.tri_boxes(tris, F)
    t = _tree(api, tris, prec)
    ro, rh = T.self_rows(tris, mn, mx, _leaf(t), F, True)
    tot = len(rh)
    assert tot > 100
    P = api._ptr
    # a short capacity: BVHGPU_ERR_CAPACITY with *total and the offsets, then the fetch of the retained list
    off = np.zeros(len(tris) + 1, dtype=np.uint32)
    hits = np.full(tot, 7, dtype=np.uint32)
    total = C.c_size_t(0)
    assert _fn(t)(t._h, 1, P(off), P(hits), tot - 1, C.byref(total)) == capi.ERR_CAPACITY
    assert total.value == tot and off.tobytes() == ro.tobytes() and (hits == 7).all()
    capi.check(getattr(capi.lib(), f"bvhgpu_traverse_fetch_{t._d['suffix']}")(t._h, P(hits), tot))
    assert hits.tobytes() == rh.tobytes()
    o2, h2 = t.triangle_pairs(cap=tot // 3)
    assert o2.tobytes() == ro.tobytes() and h2.tobytes() == rh.tobytes()
    # refusals write nothing: null pointers, missing triangles, two contexts
    ctx2 = api.Context(0)
    u = _tree(api, tris[:300], prec, ctx=ctx2)
    bare = api.Bvh.build(_aabbs(prec, mn, mx), prec=prec)
    for args, trees in (((None, 1), False), ((t._h, 1, None), False), ((bare._h, 1), False), ((None, t._h), True), ((t._h, None), True),
                        ((t._h, u._h), True), ((t._h, bare._h), True), ((bare._h, t._h), True)):
        off = np.full(len(tris) + 1, 7, dtype=np.uint32)
        hits = np.full(tot, 7, dtype=np.uint32)
        po = None if len(args) == 3 else P(off)
        assert _fn(t, trees)(*args[:2], po, P(hits), tot, C.byref(total)) == capi.ERR_INVALID
        assert (off == 7).all() and (hits == 7).all()
    d_off = torch.full((len(tris) + 1,), 7, dtype=torch.int32, device="cuda")
    d_hits = torch.full((tot,), 7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    assert _fn(t, dev=True)(bare._h, 1, C.c_void_p(d_off.data_ptr()), C.c_void_p(d_hits.data_ptr()), tot, None) == capi.ERR_INVALID
    assert _fn(t, True, True)(t._h, u._h, C.c_void_p(d_off.data_ptr()), C.c_void_p(d_hits.data_ptr()), tot, None) == capi.ERR_INVALID
    torch.cuda.synchronize()
    assert (d_off == 7).all() and (d_hits == 7).all()
    # another class or precision is refused before any C call
    with pytest.raises(ValueError):
        t.triangle_pairs_with(_tree(api, tris[:10], "f64" if prec == "f32" else "f32"))
    with pytest.raises(TypeError):
        t.triangle_pairs_with(object())
    # the dev form without a total: complete offsets, a prefix of length cap, nothing behind it
    cap = tot // 2
    t.triangle_pairs_dev(d_off.data_ptr(), d_hits.data_ptr(), cap)
    t.ctx.synchronize()
    assert d_off.cpu().numpy().view(np.uint32).tobytes() == ro.tobytes()
    h = d_hits.cpu().numpy().view(np.uint32)
    assert h[:cap].tobytes() == rh[:cap].tobytes() and (h[cap:] == 7).all()
    with pytest.raises(capi.BvhGpuError) as e:
        t.triangle_pairs_dev(d_off.data_ptr(), d_hits.data_ptr(), cap, want_total=True)
    assert e.value.status == capi.ERR_CAPACITY
    u.free()
    bare.free()
    ctx2.close()
    # n in {0, 1, 2}: self n < 2 gives zeros; cross n_a = 0 gives [0], n_b = 0 zeros
    for n in (0, 1, 2):
        x = _tree(api, tris[:n], prec)
        check_self(x, tris[:n], F)
        for m in (0, 1, 2):
            y = _tree(api, tris[3:3 + m], prec)
            off, hits = check_cross(x, y, tris[:n], tris[3:3 + m], F)
            if m == 0:
                assert off.tolist() == [0] * (n + 1)
            y.free()
        x.free()
    t.free()


def test_failed_build_is_sticky(api):
    import torch

    from bvh_b200 import capi

    shapes, tris = O.create_n_cubes(100, want_tris=True)
    good = api.Bvh.build(shapes)
    good.set_triangles(tris)
    bad_shapes = shapes.copy()
    bad_shapes["min"][33][1] = np.nan
    d = torch.from_numpy(bad_shapes.view(np.uint8).reshape(-1)).cuda()
    torch.cuda.synchronize()
    bad = api.Bvh.build_dev(d.data_ptr(), len(shapes))
    for x, y in ((bad, good), (good, bad), (bad, bad)):
        with pytest.raises(capi.BvhGpuError) as e:
            x.triangle_pairs_with(y)
        assert e.value.status == capi.ERR_NAN                    # before the missing triangles of `bad`
    with pytest.raises(capi.BvhGpuError) as e:
        bad.triangle_pairs()
    assert e.value.status == capi.ERR_NAN
    good.triangle_pairs()
    bad.free()
    good.free()


@pytest.mark.parametrize("prec", FT)
def test_dev_forms_on_a_side_stream(api, prec):
    import torch

    F = FT[prec]
    tris = X.torus(nu=160, nv=80, F=F).astype(F)
    other = (tris + np.array([0.7, 0.3, 0.05])).astype(F)
    a, b = _tree(api, tris, prec), _tree(api, other, prec)
    so, sh = a.triangle_pairs(skip_shared=False)
    co, ch = a.triangle_pairs_with(b)
    assert len(ch) > 100
    dev = torch.device("cuda", 0)
    side = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(side):
        d = [torch.full((len(tris) + 1,), 7, dtype=torch.int32, device=dev), torch.full((len(sh) + 1,), 7, dtype=torch.int32, device=dev),
             torch.full((len(tris) + 1,), 7, dtype=torch.int32, device=dev), torch.full((len(ch) + 1,), 7, dtype=torch.int32, device=dev)]
        a.ctx.set_stream(side.cuda_stream)
        try:
            a.triangle_pairs_dev(d[0].data_ptr(), d[1].data_ptr(), len(sh), skip_shared=False)
            a.triangle_pairs_with_dev(b, d[2].data_ptr(), d[3].data_ptr(), len(ch))
        finally:
            a.ctx.set_stream(None)
        side.synchronize()
    assert d[0].cpu().numpy().view(np.uint32).tobytes() == so.tobytes()
    assert d[1].cpu().numpy().view(np.uint32)[:len(sh)].tobytes() == sh.tobytes()
    assert d[2].cpu().numpy().view(np.uint32).tobytes() == co.tobytes()
    assert d[3].cpu().numpy().view(np.uint32)[:len(ch)].tobytes() == ch.tobytes()
    a.free()
    b.free()
