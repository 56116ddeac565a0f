"""Aabb / Point / Ball queries and nearest_to on 2-D and 4-D trees (bvhgpu_query_* / bvhgpu_nearest_* / bvhgpu_nearest_candidates_*
with the x2 and x4 suffixes):
- D = 4 against the dimension-generic restatement (tests/dimref.py, pinned to the C++ oracle at D = 3 by test_dim_queries_cpu.py)
  run over the device's own nodes and flat array: CSR hit lists equal in order, nearest shapes equal, distances bit-identical;
- D = 4 lift identity: a 3-D scene through the 3-D entry points and its lift w = [c, c] through the 4-D ones agree bit for bit;
- D = 2 against the C++ oracle on the device's nodes and flat array lifted to z = [0, 0], and against the restatement in 2-D;
- at 200 k shapes and 20 k queries, against a vectorised numpy brute force;
- the contract: bad arguments, short capacities, the device-pointer form on a non-default stream, and Bvh2.nearest_to."""
import ctypes as C

import numpy as np
import pytest

from tests import dimref

pytestmark = pytest.mark.gpu
U32_MAX = 0xFFFFFFFF
FT = {"f32": np.float32, "f64": np.float64}
KINDS = (dimref.AABB, dimref.POINT, dimref.BALL)


@pytest.fixture(scope="module")
def A():
    from bvh_b200 import api

    return api


def _table(D):
    from bvh_b200.dtypes import BY_PREC, BY_PREC_2D, BY_PREC_4D

    return {2: BY_PREC_2D, 3: BY_PREC, 4: BY_PREC_4D}[D]


def _shapes(mn, mx, prec):
    a = np.zeros(len(mn), dtype=_table(mn.shape[1])[prec]["aabb"])
    a["min"], a["max"] = mn, mx
    return a


def _bits(a):
    return np.ascontiguousarray(a).tobytes()


def _cls(A, D):
    return {2: A.Bvh2, 3: A.Bvh, 4: A.Bvh4}[D]


def _check_against_restatement(A, bvh, tree, mn, mx, F, rng, m=120):
    """Every kind in both modes, nearest in both modes and nearest_candidates, against dimref.Tree `tree`."""
    from bvh_b200 import capi

    for kind in KINDS:
        q = dimref.queries(kind, mn, mx, m, F, rng)
        for mode in (capi.TRAVERSE_BVH, capi.TRAVERSE_FLAT):
            off, hits = bvh.query_batch(kind, q, mode=mode)
            assert len(off) == m + 1 and off[-1] == len(hits)
            for i in range(m):
                want = tree.query_flat(kind, q[i]) if mode == capi.TRAVERSE_FLAT else tree.query_bvh(kind, q[i])
                assert hits[off[i]:off[i + 1]].tolist() == want, (kind, mode, i)
    p = dimref.points(mn, mx, m, F, rng)
    for mode in (capi.TRAVERSE_BVH, capi.TRAVERSE_FLAT):
        s, d = bvh.nearest_to_batch(p, mode=mode)
        for i in range(m):
            ws, wd = tree.nearest_flat(p[i]) if mode == capi.TRAVERSE_FLAT else tree.nearest_bvh(p[i])
            if ws == U32_MAX:
                assert s[i] == U32_MAX and d[i] == 0
            else:
                assert s[i] == ws and _bits(d[i]) == _bits(wd), (mode, i)
    off, cand = bvh.nearest_candidates(p)
    s, _ = bvh.nearest_to_batch(p)
    for i in range(m):
        lst = cand[off[i]:off[i + 1]].tolist()
        assert (s[i] in lst) if s[i] != U32_MAX else not lst, i


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("scene,n", [("random", 600), ("coincident", 300), ("axis", 300), ("peel", 300), ("overflow", 400),
                                     ("random", 0), ("random", 1)])
def test_dim4_against_restatement(A, scene, n, prec):
    F = FT[prec]
    rng = np.random.default_rng(n + len(scene))
    mn, mx = dimref.scene(scene, n, 4, F, rng, axis=2)
    shapes = _shapes(mn, mx, prec)
    bvh = A.Bvh4.build(shapes, prec=prec)
    nodes, _ = bvh.nodes_and_index()
    flat = bvh.flatten()
    if scene == "overflow" and prec == "f32":
        assert np.any(nodes["l_aabb"]["min"][:, 0] == np.inf)          # empty child boxes on the device too
    _check_against_restatement(A, bvh, dimref.Tree(nodes, shapes, flat), mn, mx, F, rng)
    bvh.free()


def _lift(a, c, F):
    return np.concatenate([a, np.full(a.shape[:-1] + (1,), c, dtype=F)], axis=-1)


def _lift_rec(kind, q, D, c, F):
    col = np.full((len(q), 1), c, dtype=F)
    if kind == dimref.AABB:
        return np.ascontiguousarray(np.concatenate([q[:, :D], col, q[:, D:], col], axis=1))
    return np.ascontiguousarray(np.concatenate([q[:, :D], col, q[:, D:]], axis=1))


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_dim4_lift_identity(A, prec):
    """The 3-D entry points (pinned to the C++ oracle by the existing suite) and the 4-D ones on the w-lift agree bit for bit."""
    from bvh_b200 import capi

    F = FT[prec]
    rng = np.random.default_rng(3)
    c = F(2.5)
    mn, mx = dimref.scene("random", 3000, 3, F, rng)
    b3 = A.Bvh.build(_shapes(mn, mx, prec), prec=prec)
    b4 = A.Bvh4.build(_shapes(_lift(mn, c, F), _lift(mx, c, F), prec), prec=prec)
    for kind in KINDS:
        q = dimref.queries(kind, mn, mx, 2000, F, rng)
        for mode in (capi.TRAVERSE_BVH, capi.TRAVERSE_FLAT):
            o3, h3 = b3.query_batch(kind, q, mode=mode)
            o4, h4 = b4.query_batch(kind, _lift_rec(kind, q, 3, c, F), mode=mode)
            assert np.array_equal(o3, o4) and np.array_equal(h3, h4), (kind, mode)
    p = dimref.points(mn, mx, 2000, F, rng)
    p4 = _lift_rec(dimref.POINT, p, 3, c, F)
    for mode in (capi.TRAVERSE_BVH, capi.TRAVERSE_FLAT):
        s3, d3 = b3.nearest_to_batch(p, mode=mode)
        s4, d4 = b4.nearest_to_batch(p4, mode=mode)
        assert np.array_equal(s3, s4) and _bits(d3) == _bits(d4), mode
    o3, c3 = b3.nearest_candidates(p)
    o4, c4 = b4.nearest_candidates(p4)
    assert np.array_equal(o3, o4) and np.array_equal(c3, c4)
    b3.free(); b4.free()


def _lift_tree_to_3d(nodes2, flat2, shapes2, prec):
    """A 2-D tree in the 3-D C-ABI layout with z = [0, 0] everywhere (the embedding's node / flat / shape boxes)."""
    from oracle import oracle as O

    d = O._DT[prec]
    nodes = np.zeros(len(nodes2), dtype=d["node"])
    for f in ("parent", "child_l", "child_r", "shape"):
        nodes[f] = nodes2[f]
    for side in ("l_aabb", "r_aabb"):
        for e in ("min", "max"):
            nodes[side][e][:, :2] = nodes2[side][e]
    flat = np.zeros(len(flat2), dtype=d["flat"])
    for f in ("entry_index", "exit_index", "shape_index"):
        flat[f] = flat2[f]
    for e in ("min", "max"):
        flat["aabb"][e][:, :2] = flat2["aabb"][e]
    shapes = np.zeros(len(shapes2), dtype=d["aabb"])
    for e in ("min", "max"):
        shapes[e][:, :2] = shapes2[e]
    return nodes, flat, shapes


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("scene,n", [("random", 800), ("coincident", 300), ("axis", 300), ("peel", 300), ("overflow", 400),
                                     ("random", 0), ("random", 1)])
def test_dim2_against_oracle_and_restatement(A, scene, n, prec):
    from bvh_b200 import capi
    from oracle import oracle as O

    F = FT[prec]
    rng = np.random.default_rng(7 * n + len(scene))
    mn, mx = dimref.scene(scene, n, 2, F, rng, axis=1)
    shapes = _shapes(mn, mx, prec)
    bvh = A.Bvh2.build(shapes, prec=prec)
    nodes2, _ = bvh.nodes_and_index()
    flat2 = bvh.flatten()
    nodes3, flat3, shapes3 = _lift_tree_to_3d(nodes2, flat2, shapes, prec)
    for kind in KINDS:
        q = dimref.queries(kind, mn, mx, 300, F, rng)
        q3 = _lift_rec(kind, q, 2, F(0), F)
        for mode in (capi.TRAVERSE_BVH, capi.TRAVERSE_FLAT):
            off, hits = bvh.query_batch(kind, q, mode=mode)
            wo, wh = O.query(kind, q3, nodes3, shapes3, flat=flat3 if mode == capi.TRAVERSE_FLAT else None, prec=prec)
            assert np.array_equal(off.astype(np.uint64), wo) and np.array_equal(hits, wh), (kind, mode)
    p = dimref.points(mn, mx, 300, F, rng)
    p3 = _lift_rec(dimref.POINT, p, 2, F(0), F)
    for mode in (capi.TRAVERSE_BVH, capi.TRAVERSE_FLAT):
        s, d = bvh.nearest_to_batch(p, mode=mode)
        flat_mode = mode == capi.TRAVERSE_FLAT
        ws, wd = O.nearest_to(flat3 if flat_mode else nodes3, shapes3, p3, prec=prec, flat=flat_mode)
        assert np.array_equal(s, ws), mode
        if n:
            assert _bits(d) == _bits(wd), mode
        else:
            assert np.all(s == U32_MAX) and np.all(d == 0)
    _check_against_restatement(A, bvh, dimref.Tree(nodes2, shapes, flat2), mn, mx, F, rng, m=80)
    bvh.free()


# ---- scale: vectorised brute force, every sum left to right in T -------------------------------------------------------------
def _brute_hits(kind, rec, mn, mx):
    """(len(rec), n) hit matrix of the restated predicates."""
    D = mn.shape[1]
    with np.errstate(all="ignore"):
        if kind == dimref.AABB:
            qmn, qmx = rec[:, None, :D], rec[:, None, D:]
            return ~np.any((qmx < mn[None]) | (mx[None] < qmn), axis=2)
        if kind == dimref.POINT:
            p = rec[:, None, :]
            return np.all(p >= mn[None], axis=2) & np.all(p <= mx[None], axis=2)
        c, r = rec[:, :D], rec[:, D]
        d2 = np.zeros((len(rec), len(mn)), dtype=mn.dtype)
        for k in range(D):
            x = np.where(c[:, None, k] < mn[None, :, k], mn[None, :, k], c[:, None, k])
            x = np.where(x > mx[None, :, k], mx[None, :, k], x)
            d = x - c[:, None, k]
            d2 = d2 + d * d
        return d2 <= (r * r)[:, None]


def _brute_min_d2(p, mn, mx):
    F = mn.dtype.type
    with np.errstate(all="ignore"):
        acc = None
        for k in range(mn.shape[1]):
            hs = (mx[:, k] - mn[:, k]) * F(0.5)
            c = mn[:, k] + hs
            q = np.abs(p[:, None, k] - c[None]) - hs[None]
            o = np.where(q > F(0), q, F(0))
            acc = o * o if acc is None else acc + o * o
    return acc


@pytest.mark.parametrize("D", [2, 4])
def test_scale_against_brute_force(A, D):
    from bvh_b200 import capi

    F, prec, n, m, checked = np.float32, "f32", 200_000, 20_000, 256
    rng = np.random.default_rng(D)
    mn = rng.uniform(-1000, 1000, (n, D)).astype(F)
    mx = (mn + rng.uniform(0, 6, (n, D))).astype(F)
    bvh = _cls(A, D).build(_shapes(mn, mx, prec), prec=prec)
    sub = rng.choice(m, checked, replace=False)
    for kind in KINDS:
        q = dimref.queries(kind, mn, mx, m, F, rng)
        if kind == dimref.AABB:                                # tens of hits per query, not thousands
            q[:, D:] = q[:, :D] + (q[:, D:] - q[:, :D]) / F(100)
        if kind == dimref.BALL:
            q[:, D] = q[:, D] / F(20)
        off, hits = bvh.query_batch(kind, q, mode=capi.TRAVERSE_BVH)
        off_f, hits_f = bvh.query_batch(kind, q, mode=capi.TRAVERSE_FLAT)
        assert np.array_equal(off, off_f) and np.array_equal(hits, hits_f)   # tight tree: the two semantics agree
        for c0 in range(0, checked, 32):
            rows = sub[c0:c0 + 32]
            hm = _brute_hits(kind, q[rows], mn, mx)
            for j, i in enumerate(rows):
                assert set(hits[off[i]:off[i + 1]].tolist()) == set(np.flatnonzero(hm[j]).tolist()), (kind, i)
                assert off[i + 1] - off[i] == int(hm[j].sum())
    p = dimref.points(mn, mx, m, F, rng)
    s, d = bvh.nearest_to_batch(p)
    s_f, d_f = bvh.nearest_to_batch(p, mode=capi.TRAVERSE_FLAT)
    off, cand = bvh.nearest_candidates(p)
    for c0 in range(0, checked, 32):
        rows = sub[c0:c0 + 32]
        d2 = _brute_min_d2(p[rows], mn, mx)
        for j, i in enumerate(rows):
            best = d2[j].min()
            for ss, dd in ((s, d), (s_f, d_f)):
                assert d2[j][ss[i]] == best and _bits(dd[i]) == _bits(np.sqrt(best)), i
            assert int(np.argmin(d2[j])) in cand[off[i]:off[i + 1]].tolist(), i
    bvh.free()


# ---- contract ---------------------------------------------------------------------------------------------------------------
def _fn(name, d):
    from bvh_b200 import capi

    return getattr(capi.lib(), f"bvhgpu_{name}_{d['suffix']}")


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("D", [2, 4])
def test_contract(A, D, prec):
    from bvh_b200 import capi

    F = FT[prec]
    d = _table(D)[prec]
    rng = np.random.default_rng(21)
    mn, mx = dimref.scene("random", 500, D, F, rng)
    bvh = _cls(A, D).build(_shapes(mn, mx, prec), prec=prec)
    q = dimref.queries(dimref.AABB, mn, mx, 64, F, rng, nan=False)
    q[:, D:] = q[:, :D] + F(40)                                 # wide boxes: many hits
    off = np.full(65, 7, dtype=np.uint32)
    hits = np.full(4, 7, dtype=np.uint32)
    total = C.c_size_t(99)
    query, nearest, cand = _fn("query", d), _fn("nearest", d), _fn("nearest_candidates", d)
    # bad kind / mode / null pointers / too many: BVHGPU_ERR_INVALID, nothing written
    bad = [query(bvh._h, 0, k, _p(q), 64, _p(off), _p(hits), 4, C.byref(total)) for k in (0, 4, -1)]
    bad.append(query(bvh._h, 2, dimref.AABB, _p(q), 64, _p(off), _p(hits), 4, C.byref(total)))
    bad.append(query(bvh._h, 0, dimref.AABB, None, 64, _p(off), _p(hits), 4, C.byref(total)))
    bad.append(query(bvh._h, 0, dimref.AABB, _p(q), 64, None, _p(hits), 4, C.byref(total)))
    bad.append(query(None, 0, dimref.AABB, _p(q), 64, _p(off), _p(hits), 4, C.byref(total)))
    bad.append(query(bvh._h, 0, dimref.AABB, _p(q), 2 ** 31, _p(off), _p(hits), 4, C.byref(total)))
    sh = np.full(64, 7, dtype=np.uint32)
    dist = np.full(64, 7, dtype=F)
    pts = np.ascontiguousarray(q[:, :D])
    bad.append(nearest(bvh._h, 2, _p(pts), 64, _p(sh), _p(dist)))
    bad.append(nearest(bvh._h, 0, None, 64, _p(sh), _p(dist)))
    bad.append(nearest(bvh._h, 0, _p(pts), 64, None, _p(dist)))
    bad.append(nearest(bvh._h, 0, _p(pts), 2 ** 31, _p(sh), _p(dist)))
    bad.append(cand(bvh._h, None, 64, _p(off), _p(hits), 4, C.byref(total)))
    bad.append(cand(bvh._h, _p(pts), 2 ** 31, _p(off), _p(hits), 4, C.byref(total)))
    assert bad == [capi.ERR_INVALID] * len(bad)
    assert np.all(off == 7) and np.all(hits == 7) and total.value == 99 and np.all(sh == 7) and np.all(dist == 7)
    # a short cap: valid offsets and *total, BVHGPU_ERR_CAPACITY; then cap = *total succeeds with the same CSR
    for mode in (capi.TRAVERSE_BVH, capi.TRAVERSE_FLAT):
        want_off, want_hits = bvh.query_batch(dimref.AABB, q, mode=mode)
        assert len(want_hits) > 4
        st = query(bvh._h, mode, dimref.AABB, _p(q), 64, _p(off), _p(hits), 4, C.byref(total))
        assert st == capi.ERR_CAPACITY and total.value == len(want_hits) and np.array_equal(off, want_off)
        full = np.zeros(total.value, dtype=np.uint32)
        assert query(bvh._h, mode, dimref.AABB, _p(q), 64, _p(off), _p(full), total.value, C.byref(total)) == capi.OK
        assert np.array_equal(off, want_off) and np.array_equal(full, want_hits)
    want_off, want_c = bvh.nearest_candidates(pts)
    st = cand(bvh._h, _p(pts), 64, _p(off), _p(hits), 0, C.byref(total))
    if len(want_c) > 0:
        assert st == capi.ERR_CAPACITY and total.value == len(want_c) and np.array_equal(off, want_off)
    # an empty tree: zero offsets; nearest = BVHGPU_INVALID_INDEX and distance 0
    e = _cls(A, D).build(_shapes(mn[:0], mx[:0], prec), prec=prec)
    for kind in KINDS:
        o, h = e.query_batch(kind, dimref.queries(kind, mn, mx, 10, F, rng))
        assert np.all(o == 0) and len(h) == 0
    s, dd = e.nearest_to_batch(pts)
    assert np.all(s == U32_MAX) and np.all(dd == 0)
    o, c = e.nearest_candidates(pts)
    assert np.all(o == 0) and len(c) == 0
    assert e.nearest_to(pts[0], [], lambda s_, p_: 0.0) is None
    e.free(); bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_query_dev_on_a_side_stream(A, prec):
    import torch
    from bvh_b200 import capi

    F = FT[prec]
    rng = np.random.default_rng(4)
    mn, mx = dimref.scene("random", 4000, 4, F, rng)
    bvh = A.Bvh4.build(_shapes(mn, mx, prec), prec=prec)
    for kind in KINDS:
        q = dimref.queries(kind, mn, mx, 1000, F, rng)
        d_q = torch.from_numpy(q).cuda()
        for mode in (capi.TRAVERSE_BVH, capi.TRAVERSE_FLAT):
            want_off, want_hits = bvh.query_batch(kind, q, mode=mode)
            tot = len(want_hits)
            d_off = torch.zeros(len(q) + 1, dtype=torch.int32, device="cuda")
            d_hits = torch.zeros(max(tot, 1), dtype=torch.int32, device="cuda")
            assert bvh.query_dev(kind, d_q.data_ptr(), len(q), d_off.data_ptr(), d_hits.data_ptr(), tot, mode=mode, want_total=True) == tot
            assert np.array_equal(d_off.cpu().numpy().view(np.uint32), want_off)
            assert np.array_equal(d_hits[:tot].cpu().numpy().view(np.uint32), want_hits)
            s = torch.cuda.Stream()
            bvh.ctx.set_stream(s.cuda_stream)
            try:
                d_off.zero_(); d_hits.zero_()
                torch.cuda.synchronize()
                short = tot // 2
                bvh.query_dev(kind, d_q.data_ptr(), len(q), d_off.data_ptr(), d_hits.data_ptr(), short, mode=mode, want_total=False)
                s.synchronize()
            finally:
                bvh.ctx.set_stream(None)
            assert np.array_equal(d_off.cpu().numpy().view(np.uint32), want_off)     # offsets always complete
            got = d_hits.cpu().numpy().view(np.uint32)
            assert np.array_equal(got[:short], want_hits[:short]) and np.all(got[short:] == 0)   # a prefix
    bvh.free()


@pytest.mark.parametrize("D", [2, 4])
def test_nearest_to_with_sphere_shapes(A, D):
    """Bvh2 / Bvh4.nearest_to with the shape's own distance: spheres inside their AABBs, brute-force nearest picked."""
    rng = np.random.default_rng(D + 40)
    n = 3000
    ctr = rng.uniform(-50, 50, (n, D))
    rad = rng.uniform(0.1, 3, n)
    spheres = [(ctr[i], rad[i]) for i in range(n)]
    bvh = _cls(A, D).build(_shapes((ctr - rad[:, None]).astype(np.float64), (ctr + rad[:, None]).astype(np.float64), "f64"), prec="f64")

    def dist2(s, p):
        return max(float(np.linalg.norm(np.asarray(p) - s[0])) - s[1], 0.0) ** 2

    for p in rng.uniform(-60, 60, (40, D)):
        shape, dist = bvh.nearest_to(p, spheres, dist2)
        want = min(dist2(s, p) for s in spheres)
        assert dist2(shape, p) == want and dist == np.sqrt(want)
    bvh.free()


@pytest.mark.parametrize("D", [2, 3, 4])
def test_a_total_past_the_first_buffer_fits_cap(A, D):
    """A host CSR call whose total passes the tree's first retained hit buffer (max(per_item * n, 1024) on a fresh tree) but fits the
    caller's cap: the fill runs again into the grown buffer and returns the CSR of a call whose first buffer fits, for queries and
    self-overlap.  In 3-D a short cap leaves the full list for bvhgpu_traverse_fetch_*."""
    from bvh_b200 import capi

    F, prec, n, m = np.float32, "f32", 300, 8
    rng = np.random.default_rng(40 + D)
    mn = rng.uniform(0, 4, (n, D)).astype(F)
    mx = (mn + rng.uniform(1, 3, (n, D))).astype(F)
    d = _table(D)[prec]
    q = np.concatenate([np.full((m, D), -1, F), np.full((m, D), 10, F)], axis=1)   # every query meets every box: n hits each
    query = _fn("query", d)
    total = C.c_size_t(0)
    for short in (False, True):
        bvh = _cls(A, D).build(_shapes(mn, mx, prec), prec=prec)
        off = np.zeros(m + 1, dtype=np.uint32)
        hits = np.zeros(m * n, dtype=np.uint32)
        cap = 10 if short else m * n                            # m n = 2400 > 1024 = the first buffer
        st = query(bvh._h, capi.TRAVERSE_BVH, dimref.AABB, _p(q), m, _p(off), _p(hits), cap, C.byref(total))
        assert total.value == m * n and st == (capi.ERR_CAPACITY if short else capi.OK), capi.lib().bvhgpu_last_error()
        if short and D == 3:
            capi.check(capi.lib().bvhgpu_traverse_fetch_f32x3(bvh._h, _p(hits), m * n))
        elif short:                                             # no retained list: the call again with cap = *total refills
            st = query(bvh._h, capi.TRAVERSE_BVH, dimref.AABB, _p(q), m, _p(off), _p(hits), m * n, C.byref(total))
            assert st == capi.OK and total.value == m * n, capi.lib().bvhgpu_last_error()
        want_off, want_hits = bvh.query_batch(dimref.AABB, q)      # the retained buffer holds the total now: no refill
        assert np.array_equal(off, want_off) and np.array_equal(hits, want_hits)
        assert all(sorted(hits[off[i]:off[i + 1]].tolist()) == list(range(n)) for i in range(m))
        if not short:
            fresh = _cls(A, D).build(_shapes(mn, mx, prec), prec=prec)
            o1, p1 = fresh.overlap_pairs(cap=n * n)                 # about n (n - 1) / 2 pairs > max(4 n, 1024)
            fresh.free()
            o2, p2 = bvh.overlap_pairs(cap=n * n)
            o3, p3 = bvh.overlap_pairs(cap=n * n)
            assert len(p1) > max(4 * n, 1024) and np.array_equal(o1, o3) and np.array_equal(p1, p3)
            assert np.array_equal(o2, o3) and np.array_equal(p2, p3)
            meet = np.all((mx[:, None, :] >= mn[None, :, :]) & (mx[None, :, :] >= mn[:, None, :]), axis=2)   # brute force
            want = sorted(zip(*np.nonzero(np.triu(meet, 1))))
            rows = np.repeat(np.arange(n), np.diff(o1.astype(np.int64)))
            got = sorted((min(a_, b_), max(a_, b_)) for a_, b_ in zip(rows.tolist(), p1.tolist()))
            assert got == [(int(a_), int(b_)) for a_, b_ in want]            # every intersecting pair, each once
        bvh.free()
