"""Polygons of 2-D trees on the device (bvhgpu_tree_set_segments_*x2, bvhgpu_contains_points_*x2, bvhgpu_knn_segments_*x2,
bvhgpu_signed_distance_*x2) held byte for byte to the model of tests/polygons.py (itself pinned by tests/test_polygons_cpu.py):
class and winding under both fill rules, knn rows (shape, distance, closest point) with and without radii, and the signed distance,
in f32 and f64:
- hand cases (squares of both orientations, a hole, a pentagram, points on vertices and edges and one ulp off, collinear vertices,
  cancelling edges, zero-length and NaN segments, the f64 range), a Koch snowflake, a map of star polygons with holes, and the
  adversarial box families of tests/adversarial.py made into segments;
- every build mode, and "no split wins" trees (overflow-scale boxes) whose empty child boxes the walk must enter;
- refit with stale segments (the result over the segments the walk reaches), update_shapes, remove_shapes (the segments follow their
  shapes), add_shapes (refused until set_segments);
- identities: reversed segments negate every winding, the union of two sets adds windings, |signed distance| is knn at k = 1;
- launch edges around 128 and a large batch, refusals with guarded outputs, two contexts, n in {0, 1, 2}, an empty tree, a side stream."""
import numpy as np
import pytest

from tests import adversarial as ADV
from tests import polygons as P

pytestmark = pytest.mark.gpu
U32_MAX = 0xFFFFFFFF
FT = {"f32": np.float32, "f64": np.float64}
RULES = {"even_odd": P.EVEN_ODD, "nonzero": P.NONZERO}


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A_

    return A_


def _aabbs(api, prec, mn, mx):
    a = np.zeros(len(mn), dtype=api.BY_PREC_2D[prec]["aabb"])
    a["min"], a["max"] = mn, mx
    return a


def _tree(api, segs, prec, mode=0, ctx=None, boxes=None):
    mn, mx = P.seg_boxes(segs) if boxes is None else boxes
    bvh = api.Bvh2.build(_aabbs(api, prec, mn, mx), prec=prec, ctx=ctx, mode=mode)
    bvh.set_segments(segs)
    return bvh


def _limits(F, n, rng, scale):
    r = (rng.uniform(0, 1, n) * scale).astype(F)
    r[::11] = F(0)
    r[1::11] = F(-0.0)
    r[2::11] = F(-1)
    r[3::11] = F(np.nan)
    r[4::11] = F(np.inf)
    return r


def check_contains(bvh, segs, pts, F):
    for name, rule in RULES.items():
        cls, w = bvh.contains(pts, name, winding=True)
        mc, mw = P.classes(segs, pts, F, rule)
        assert np.array_equal(cls, mc), name
        assert np.array_equal(w, mw), name
        assert np.array_equal(bvh.contains(pts, name), cls)


def check_knn(bvh, segs, pts, F, rng, ks=(1, 4, 5, 9), scale=1.0):
    mn, mx = P.seg_boxes(segs)
    assert all(P.bounded(p, segs, mn, mx).all() for p in pts if np.isfinite(p).all())
    for md in (None, _limits(F, len(pts), rng, scale)):
        bs, bd, bq = P.brute(segs, pts, max(ks), md)
        for k in ks:
            s, d, q = bvh.knn_segments(pts, k, md, closest=True)
            assert np.array_equal(s, bs[:, :k]), (k, md is None)
            assert d.tobytes() == np.ascontiguousarray(bd[:, :k]).tobytes(), (k, md is None)
            assert q.tobytes() == np.ascontiguousarray(bq[:, :k]).tobytes(), (k, md is None)
            s2, d2 = bvh.knn_segments(pts, k, md)
            assert np.array_equal(s2, s) and d2.tobytes() == d.tobytes()


def check_signed(bvh, segs, pts, F):
    for name, rule in RULES.items():
        s, d, q = bvh.signed_distance(pts, name, closest=True)
        ms, md, mq = P.signed(segs, pts, rule)
        assert np.array_equal(s, ms) and d.tobytes() == md.tobytes() and q.tobytes() == mq.tobytes(), name
        ks, kd = bvh.knn_segments(pts, 1)
        assert np.array_equal(ks[:, 0], s) and np.abs(d).tobytes() == kd[:, 0].tobytes()


def check_all(bvh, segs, pts, F, rng, scale=1.0, ks=(1, 4, 5, 9)):
    check_contains(bvh, segs, pts, F)
    check_knn(bvh, segs, pts, F, rng, ks, scale)
    check_signed(bvh, segs, pts, F)


def _square(x0, y0, x1, y1, ccw=True):
    v = np.array([[x0, y0], [x1, y0], [x1, y1], [x0, y1]], dtype=np.float64)
    return P.loop(v if ccw else v[::-1])


def _probe_points(segs, F, rng, m, pad=0.25):
    """Uniform points over the scene's bounds, the segments' end points and midpoints, and end points moved one ulp each way."""
    fin = segs[np.isfinite(segs).all(1)].astype(np.float64)
    lo, hi = fin.reshape(-1, 2).min(0), fin.reshape(-1, 2).max(0)
    ext = hi - lo
    u = rng.uniform(lo - pad * ext, hi + pad * ext, (m, 2))
    ends = fin[:, :2][rng.choice(len(fin), min(len(fin), m // 4), replace=False)]
    mids = (fin[:, :2] + fin[:, 2:]) / 2
    mids = mids[rng.choice(len(fin), min(len(fin), m // 8), replace=False)]
    e = ends.astype(F)
    moved = np.concatenate([np.nextafter(e, F(np.inf)), np.nextafter(e, F(-np.inf))])
    return np.concatenate([u.astype(F), e, mids.astype(F), moved]).astype(F)


# ---- hand cases ----
@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_hand_cases(api, prec):
    F = FT[prec]
    rng = np.random.default_rng(1)
    t = np.pi / 2 + np.arange(5) * 4 * np.pi / 5
    scenes = {
        "ccw": _square(0, 0, 1, 1),
        "cw": _square(0, 0, 1, 1, ccw=False),
        "hole": np.vstack([_square(0, 0, 4, 4), _square(1, 1, 3, 3, ccw=False)]),
        "pentagram": P.loop(np.stack([np.cos(t), np.sin(t)], axis=1)),
        "collinear": P.loop(np.array([[0, 0], [0.25, 0], [0.5, 0], [1, 0], [1, 1], [0, 1]], dtype=np.float64)),
        "cancel": np.vstack([_square(0, 0, 1, 1), _square(1, 0, 2, 1)]),
        "degenerate": np.vstack([_square(0, 0, 1, 1), [[0.5, 0.5, 0.5, 0.5], [0.2, 0.2, 0.2, 0.2]]]),
    }
    grid = np.stack(np.meshgrid(np.arange(-4, 21) / 4, np.arange(-4, 21) / 4), axis=-1).reshape(-1, 2).astype(F)
    for name, segs in scenes.items():
        segs = segs.astype(F)
        pts = np.concatenate([grid, _probe_points(segs, F, rng, 200), np.array([[np.nan, 0.5], [0.5, np.inf]], dtype=F)])
        bvh = _tree(api, segs, prec)
        check_all(bvh, segs, pts, F, rng, scale=2.0)
        bvh.free()
    # the pentagram's centre winds twice
    bvh = _tree(api, scenes["pentagram"].astype(F), prec)
    cls_eo, w = bvh.contains(np.zeros((1, 2), dtype=F), "even_odd", winding=True)
    assert w[0] == 2 and cls_eo[0] == P.OUTSIDE and bvh.contains(np.zeros((1, 2), dtype=F), "nonzero")[0] == P.INSIDE
    bvh.free()
    # NaN segments: boxes from the finite end point, excluded everywhere; knn keys of NaN segments never qualify
    segs = np.vstack([_square(0, 0, 1, 1), [[np.nan, 0.5, 0.5, 0.5], [0.25, np.inf, 0.25, 0.5]]]).astype(F)
    mn, mx = P.seg_boxes(segs)
    mn, mx = np.where(np.isfinite(mn), mn, 0), np.where(np.isfinite(mx), mx, 1)
    bvh = _tree(api, segs, prec, boxes=(mn.astype(F), mx.astype(F)))
    pts = _probe_points(segs, F, rng, 300)
    check_contains(bvh, segs, pts, F)
    check_signed(bvh, segs, pts, F)
    bvh.free()


def test_f64_range(api):
    F = np.float64
    lo, hi = 2.0 ** -300, 2.0 ** 300
    s = hi / 2
    segs = np.vstack([_square(-s, -s, s, s), _square(0, 0, 1, 1), [[1.0, -1.0, 2.0 ** 301, 1.0], [2.0 ** -301, -1.0, 0.5, 1.0]]]).astype(F)
    pts = np.array([[np.nextafter(lo, 0), 0.5], [lo, 0.5], [0.5, 0.5], [1.0, 0.5], [0.25, 0.0], [hi * 0.75, 0.0], [np.nextafter(hi, np.inf), 0],
                    [-lo, 3.0], [-2.0 ** -301, 3.0], [5e-324, 0.5], [0.0, 0.0], [-0.0, 0.5]], dtype=F)
    bvh = _tree(api, segs, "f64")
    check_contains(bvh, segs, pts, F)
    cls = bvh.contains(pts)
    assert (cls == P.UNDECIDED).any() and (cls == P.BOUNDARY).any()
    check_signed(bvh, segs, pts, F)
    bvh.free()


# ---- scenes ----
@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_koch_every_build_mode(api, prec, mode):
    F = FT[prec]
    rng = np.random.default_rng(2 + mode)
    segs = P.koch(5 if mode else 6, F)
    pts = _probe_points(segs, F, rng, 3000)
    bvh = _tree(api, segs, prec, mode=mode)
    check_contains(bvh, segs, pts, F)
    check_knn(bvh, segs, pts[:600], F, rng, ks=(1, 8, 9))
    check_signed(bvh, segs, pts[:600], F)
    bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_star_map(api, prec):
    F = FT[prec]
    rng = np.random.default_rng(4)
    segs = P.star_map(100, 8, F)                                     # 3 200 segments, 100 stars with holes of opposite orientation
    pts = _probe_points(segs, F, rng, 6000, pad=0.05)
    bvh = _tree(api, segs, prec)
    check_contains(bvh, segs, pts, F)
    cls, w = bvh.contains(pts, "nonzero", winding=True)
    assert set(np.unique(w)) >= {0, 1} and (cls == P.BOUNDARY).any()
    check_knn(bvh, segs, pts[:500], F, rng, ks=(1, 8))
    check_signed(bvh, segs, pts[:800], F)
    bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("family", sorted(ADV.BOX_FAMILIES))
def test_adversarial_families_as_segments(api, prec, family):
    """Every box of a family becomes its diagonal (even shapes) or anti-diagonal (odd), so the box is exactly the segment's."""
    F = FT[prec]
    rng = np.random.default_rng(5)
    mn, mx, p = ADV.BOX_FAMILIES[family](F, 2)
    segs = np.hstack([mn, mx]).astype(F)
    odd = np.arange(len(segs)) % 2 == 1
    segs[odd] = np.stack([mn[odd, 0], mx[odd, 1], mx[odd, 0], mn[odd, 1]], axis=1)
    pts = np.concatenate([p, _probe_points(segs, F, rng, 200)]).astype(F)
    bvh = _tree(api, segs, prec)
    scale = float(np.nanmax(np.abs(segs[np.isfinite(segs)])))
    check_all(bvh, segs, pts, F, rng, scale=scale, ks=(1, 4, 9))
    bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_no_split_wins_tree_enters_empty_boxes(api, prec):
    F = FT[prec]
    rng = np.random.default_rng(6)
    mn, mx, _ = ADV.overflow(F, 2, n=300)
    segs = np.hstack([mn, mx]).astype(F)
    bvh = _tree(api, segs, prec)
    nodes, _ = bvh.nodes_and_index()
    inner = nodes["child_l"] != U32_MAX
    empty = ((nodes["l_aabb"]["min"] > nodes["l_aabb"]["max"]).any(1) | (nodes["r_aabb"]["min"] > nodes["r_aabb"]["max"]).any(1)) & inner
    assert empty.any()                                                # the walk has empty child boxes to enter
    pts = _probe_points(segs, F, rng, 400)
    check_contains(bvh, segs, pts, F)
    cls, w = bvh.contains(pts, winding=True)
    if F == np.float32:
        assert (w != 0).any()
    else:
        assert (cls == P.UNDECIDED).any()                            # f64 surface areas overflow only beyond the exact range 2^300
    check_signed(bvh, segs, pts, F)
    bvh.free()


# ---- dynamic calls ----
@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_dynamic_calls(api, prec):
    from bvh_b200 import capi

    F = FT[prec]
    rng = np.random.default_rng(7)
    segs = P.star_map(16, 6, F)
    pts = _probe_points(segs, F, rng, 1500, pad=0.05)
    bvh = _tree(api, segs, prec)
    # refit with larger boxes: still exact
    mn, mx = P.seg_boxes(segs)
    bvh.refit(_aabbs(api, prec, mn - F(0.5), mx + F(0.5)))
    check_contains(bvh, segs, pts, F)
    # refit with boxes moved away from their segments: the result is the contract over the segments the walk reaches (boxes that meet
    # [px, +inf] x [py, py])
    shift = np.where(np.arange(len(segs)) % 3 == 0, 2.0, 0.0).astype(F)
    smn, smx = mn + shift[:, None], mx + shift[:, None]
    bvh.refit(_aabbs(api, prec, smn, smx))
    sub = pts[:300]
    for name, rule in RULES.items():
        cls, w = bvh.contains(sub, name, winding=True)
        for i, p in enumerate(sub):
            reach = (smx[:, 0] >= p[0]) & (smn[:, 1] <= p[1]) & (smx[:, 1] >= p[1])
            mc, mw = P.classes(segs[reach], p[None], F, rule)
            assert cls[i] == mc[0] and w[i] == mw[0], (name, i)
    # update_shapes: new segments and boxes for some shapes
    moved = segs.copy()
    ch = rng.choice(len(segs), 40, replace=False)
    moved[ch] = (segs[ch] + F(0.75)).astype(F)
    mmn, mmx = P.seg_boxes(moved)
    bvh.refit(_aabbs(api, prec, mn, mx))
    bvh.update_shapes(ch, _aabbs(api, prec, mmn, mmx))
    bvh.set_segments(moved)
    check_all(bvh, moved, pts[:400], F, rng, scale=3.0, ks=(1, 5))
    # remove_shapes: the segments follow their shapes
    gone = rng.choice(len(moved), 50, replace=False)
    moves = bvh.remove_shapes(gone)
    after = moved.copy()
    for new_i, old_i in moves:
        after[new_i] = moved[old_i]
    after = after[: len(moved) - len(gone)]
    check_all(bvh, after, pts[:400], F, rng, scale=3.0, ks=(1, 5))
    # add_shapes drops them: every segment call refuses until set_segments
    extra = _square(40, 40, 41, 41).astype(F)
    emn, emx = P.seg_boxes(extra)
    bvh.add_shapes(_aabbs(api, prec, emn, emx))
    for call in (lambda: bvh.contains(pts), lambda: bvh.knn_segments(pts, 2), lambda: bvh.signed_distance(pts)):
        with pytest.raises(capi.BvhGpuError) as e:
            call()
        assert e.value.status == capi.ERR_INVALID
    full = np.vstack([after, extra]).astype(F)
    bvh.set_segments(full)
    check_all(bvh, full, np.concatenate([pts[:300], np.array([[40.5, 40.5]], dtype=F)]), F, rng, scale=3.0, ks=(1, 5))
    # removing everything leaves an empty tree: class 0, rows of padding
    bvh.remove_shapes(np.arange(len(full)))
    cls, w = bvh.contains(pts[:10], winding=True)
    assert (cls == 0).all() and (w == 0).all()
    s, d = bvh.knn_segments(pts[:10], 3)
    assert (s == U32_MAX).all() and np.isposinf(d).all()
    bvh.free()


# ---- identities ----
@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_identities(api, prec):
    F = FT[prec]
    rng = np.random.default_rng(8)
    a = P.star_map(9, 7, F, seed=1)
    b = (P.koch(4, F) * F(6)).astype(F)
    pts = _probe_points(np.vstack([a, b]), F, rng, 3000, pad=0.05)
    ta, tb = _tree(api, a, prec), _tree(api, b, prec)
    tr = _tree(api, a[:, [2, 3, 0, 1]].copy(), prec)
    tu = _tree(api, np.vstack([a, b]), prec)
    ca, wa = ta.contains(pts, "nonzero", winding=True)
    cb, wb = tb.contains(pts, "nonzero", winding=True)
    cr, wr = tr.contains(pts, "nonzero", winding=True)
    cu, wu = tu.contains(pts, "nonzero", winding=True)
    assert np.array_equal(wr, -wa) and np.array_equal(cr, ca)
    nb = (ca != P.BOUNDARY) & (cb != P.BOUNDARY)
    assert np.array_equal(wu[nb], (wa + wb)[nb])
    assert ((cu == P.BOUNDARY) == ((ca == P.BOUNDARY) | (cb == P.BOUNDARY))).all()
    for t in (ta, tu):
        s, d = t.signed_distance(pts, "even_odd")
        ks, kd = t.knn_segments(pts, 1)
        assert np.array_equal(ks[:, 0], s) and np.abs(d).tobytes() == kd[:, 0].tobytes()
        assert (d < 0).any() and (d > 0).any()
    for t in (ta, tb, tr, tu):
        t.free()


# ---- launch edges and the contract ----
@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_launch_edges(api, prec):
    F = FT[prec]
    rng = np.random.default_rng(9)
    segs = P.star_map(4, 5, F)
    bvh = _tree(api, segs, prec)
    big = _probe_points(segs, F, rng, 140_000)
    for n in (1, 2, 31, 32, 33, 127, 128, 129, 255, 256, 257, 1023, 1024, 1025, len(big)):
        pts = big[:n]
        cls, w = bvh.contains(pts, "nonzero", winding=True)
        mc, mw = P.classes(segs, pts, F, P.NONZERO)
        assert np.array_equal(cls, mc) and np.array_equal(w, mw), n
        if n <= 1025:
            s, d, q = bvh.knn_segments(pts, 3, closest=True)
            bs, bd, bq = P.brute(segs, pts, 3)
            assert np.array_equal(s, bs) and d.tobytes() == bd.tobytes() and q.tobytes() == bq.tobytes(), n
    s, d = bvh.signed_distance(big, "nonzero")
    ks, kd = bvh.knn_segments(big, 1)
    assert np.array_equal(ks[:, 0], s) and np.abs(d).tobytes() == kd[:, 0].tobytes()
    assert (np.signbit(d) == ((cls == P.INSIDE) & (s != U32_MAX))).all()     # inside at a rounded distance 0 gives -0
    bvh.free()


def test_refusals_leave_outputs_untouched(api):
    from bvh_b200 import capi

    F = np.float32
    segs = _square(0, 0, 1, 1).astype(F)
    pts = np.full((8, 2), 0.5, dtype=F)
    bvh = _tree(api, segs, "f32")
    L = capi.lib()
    ptr = api._ptr

    def guards():
        return (np.full(8, 7, dtype=np.uint8), np.full(8, 7, dtype=np.int32), np.full((8, 70), 7, dtype=np.uint32),
                np.full((8, 70), 7, dtype=F), np.full((8, 70, 2), 7, dtype=F))

    def untouched(g):
        return all((a == 7).all() for a in g)

    for rule, tree, pp, pc, n in ((2, bvh._h, pts, True, 8), (-1, bvh._h, pts, True, 8), (0, None, pts, True, 8), (0, bvh._h, None, True, 8),
                                  (0, bvh._h, pts, False, 8), (0, bvh._h, pts, True, 2 ** 31)):
        g = guards()
        st = L.bvhgpu_contains_points_f32x2(tree, ptr(pp), n, rule, ptr(g[0]) if pc else None, ptr(g[1]))
        assert st == capi.ERR_INVALID and untouched(g), (rule, tree is None, pp is None, pc, n)
        g = guards()
        st = L.bvhgpu_signed_distance_f32x2(tree, ptr(pp), n, rule, ptr(g[2]) if pc else None, ptr(g[3]), ptr(g[4]))
        assert st == capi.ERR_INVALID and untouched(g), (rule, tree is None, pp is None, pc, n)
    for k, tree, pp, n in ((0, bvh._h, pts, 8), (65, bvh._h, pts, 8), (4, None, pts, 8), (4, bvh._h, None, 8), (4, bvh._h, pts, 2 ** 31)):
        g = guards()
        st = L.bvhgpu_knn_segments_f32x2(tree, ptr(pp), n, k, None, ptr(g[2]), ptr(g[3]), ptr(g[4]))
        assert st == capi.ERR_INVALID and untouched(g), (k, tree is None, pp is None, n)
    assert L.bvhgpu_tree_set_segments_f32x2(bvh._h, ptr(segs), 3) == capi.ERR_INVALID       # n != shape count
    assert L.bvhgpu_tree_set_segments_f32x2(bvh._h, None, 4) == capi.ERR_INVALID
    bvh.free()
    plain = api.Bvh2.build(_aabbs(api, "f32", *P.seg_boxes(segs)))                          # no segments set
    g = guards()
    assert L.bvhgpu_contains_points_f32x2(plain._h, ptr(pts), 8, 0, ptr(g[0]), ptr(g[1])) == capi.ERR_INVALID and untouched(g)
    assert L.bvhgpu_knn_segments_f32x2(plain._h, ptr(pts), 8, 2, None, ptr(g[2]), ptr(g[3]), None) == capi.ERR_INVALID and untouched(g)
    assert L.bvhgpu_signed_distance_f32x2(plain._h, ptr(pts), 8, 0, ptr(g[2]), ptr(g[3]), None) == capi.ERR_INVALID and untouched(g)
    plain.free()
    with pytest.raises(TypeError):
        api.Bvh4.from_segments(np.zeros((1, 2, 2)))


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_housekeeping(api, prec):
    import torch

    F = FT[prec]
    rng = np.random.default_rng(10)
    sq = _square(0, 0, 1, 1).astype(F)
    pts = _probe_points(sq, F, rng, 200)
    for n in (0, 1, 2):                                              # tiny trees (n = 0: an empty tree)
        segs = sq[:n]
        bvh = api.Bvh2.build(_aabbs(api, prec, *P.seg_boxes(segs)) if n else np.zeros(0, dtype=api.BY_PREC_2D[prec]["aabb"]), prec=prec)
        bvh.set_segments(segs.reshape(-1, 4))
        check_contains(bvh, segs.reshape(-1, 4), pts, F)
        s, d, q = bvh.knn_segments(pts, 3, closest=True)
        bs, bd, bq = P.brute(segs.reshape(-1, 4), pts, 3)
        assert np.array_equal(s, bs) and d.tobytes() == bd.tobytes() and q.tobytes() == bq.tobytes()
        for m in (0, 1, 2):                                          # batches of 0, 1 and 2 points
            assert len(bvh.contains(pts[:m])) == m and bvh.knn_segments(pts[:m], 2)[0].shape == (m, 2)
        bvh.free()
    # two contexts, and calls after set_stream on a side stream
    ctx2 = api.Context(0)
    segs = P.star_map(4, 5, F)
    t1, t2 = _tree(api, segs, prec), _tree(api, segs, prec, ctx=ctx2)
    pts = _probe_points(segs, F, rng, 2000)
    c1, w1 = t1.contains(pts, winding=True)
    side = torch.cuda.Stream()
    ctx2.set_stream(side.cuda_stream)
    try:
        c2, w2 = t2.contains(pts, winding=True)
        s2, d2 = t2.signed_distance(pts)
        k2 = t2.knn_segments(pts, 4, closest=True)
    finally:
        ctx2.set_stream(None)
    assert np.array_equal(c1, c2) and np.array_equal(w1, w2)
    s1, d1 = t1.signed_distance(pts)
    k1 = t1.knn_segments(pts, 4, closest=True)
    assert np.array_equal(s1, s2) and d1.tobytes() == d2.tobytes()
    assert all(a.tobytes() == b.tobytes() for a, b in zip(k1, k2))
    t1.free(); t2.free()
    ctx2.close()
