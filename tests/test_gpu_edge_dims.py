"""The walks added after the 3-D edge suite, on the edge inputs of tests/edge_dims.py in D = 2, 3 and 4, f32 and f64: "huge" (surface
areas overflow in f32 and f64: empty stored child boxes), "mixed" and "subnormal" scenes, the six ray families (axis and face rays
along every axis, origins on faces moving in and out, tiny and subnormal direction components on every axis), points on faces, with
+-0 components, at a few subnormal steps and with keys that overflow, radii whose r * r overflows, underflows or rounds up onto a key,
and limits at 0, -0, the smallest subnormal, +inf and each ray's own entry and exit.  Every comparison is bit for bit:
- traversal of 2-D and 4-D trees, BVH and FLAT, against dimorder's candidate walk (a leaf reached through its stored box; FLAT re-tests
  the shape's own box), the 4-D device form with a capacity retry; the 3-D traversal with compact (origin + direction) rays against the
  oracle, whose inverse is recomputed on the device;
- ordered traversal (both orders) and AABB-mode closest hit of 2-D and 4-D trees against dimorder;
- any hit and multi hit (k = 1, 3, 64) in AABB mode, D = 2, 3, 4, every limit family, every form (3-D: host, FULL and OD device rays;
  4-D: host and device), against tests/anyhit.py and tests/multihit.py;
- triangle mode of closest, any and multi hit in D = 3 on triangles inside the edge boxes, against the models and the oracle (the
  weaker guarantee only on the rows multihit.brute_triangles calls unbounded); hits only on the mixed scene, misses elsewhere;
- knn in D = 2, 3, 4 with and without radii against knnref's brute force, and knn_triangles in D = 3 on the bounded points;
- nearest_to (BVH and FLAT) of 2-D and 4-D trees against dimref; nearest_candidates in every D list for list against prunedmodel
  and its contract (prunedcheck); Aabb, Point and Ball queries in every D, BVH and FLAT, against dimref;
- the walks again after a refit and an update_shapes of each D's huge and subnormal trees (the 3-D traversal against the oracle)."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O
from tests import anyhit as H, dimorder, dimref, edge_dims as ED, knnref as K, knntri as KT, multihit as MH, prunedcheck as PC
from tests import prunedmodel as M
from tests.test_gpu_any_hit import _forms as any_forms
from tests.test_gpu_dim_ordered import _check as ordered_check
from tests.test_gpu_multi_hit import _aabbs, _cls, _forms as multi_forms, _nodes, _rays, _same

pytestmark = pytest.mark.gpu
U32_MAX = 0xFFFFFFFF
FT = ED.FT
UINT = {np.float32: np.uint32, np.float64: np.uint64}
CASES = [(kind, D, prec) for kind in ED.SCENE_KINDS for D in ED.DIMS for prec in ED.PRECS]
N_SHAPES, PER_FAMILY, N_POINTS = 160, 8, 80
KNN_KS = (1, 4, 5, 8, 9, 16, 17, 32, 33, 64)                # every K bucket of knn_walk, both sides of each edge


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A_

    return A_


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(UINT[a.dtype.type])


def _setup(api, kind, D, prec, n=N_SHAPES):
    mn, mx = ED.scene(kind, n, D, prec)
    o, d, inv, fam = ED.ray_batch(mn, mx, PER_FAMILY, prec)
    shapes = _aabbs(api, D, prec, mn, mx)
    return mn, mx, shapes, _rays(api, D, prec, o, d, inv), fam


def _check_traversal(api, bvh, D, shapes, rays, prec):
    """BVH and FLAT CSR against dimorder's candidates; the 4-D device form with a short capacity, then the exact one."""
    import torch

    from bvh_b200 import capi

    tree = dimorder.Tree(_nodes(bvh, D), shapes)
    o, inv = rays["origin"], rays["inv_direction"]
    want_b, want_f = [], []
    for i in range(len(rays)):
        ray = (list(o[i]), list(inv[i]))
        c = [s for s, _ in tree._candidates(ray)]
        want_b.append(c)
        want_f.append([s for s in c if dimorder.slice(ray, *tree.shapes[s]) is not None])
    for mode, want in ((capi.TRAVERSE_BVH, want_b), (capi.TRAVERSE_FLAT, want_f)):
        off, hits = bvh.traverse_batch(rays, mode=mode)
        for i in range(len(rays)):
            assert hits[off[i]:off[i + 1]].tolist() == want[i], (mode, i)
        if D == 4:
            d_rays = torch.from_numpy(rays.view(np.uint8).copy()).cuda()
            d_off = torch.full((len(rays) + 1,), 7, dtype=torch.int32, device="cuda")
            d_hits = torch.full((max(len(hits), 1),), 7, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            if len(hits) > 1:                                # a short capacity is refused with the total and complete offsets
                total = C.c_size_t(0)
                fn = getattr(capi.lib(), f"bvhgpu_traverse_dev_{bvh._d['suffix']}")
                st = fn(bvh._h, mode, C.c_void_p(d_rays.data_ptr()), len(rays), C.c_void_p(d_off.data_ptr()), C.c_void_p(d_hits.data_ptr()),
                        len(hits) // 3, C.byref(total))
                torch.cuda.synchronize()
                assert st == capi.ERR_CAPACITY and total.value == len(hits), (st, total.value, len(hits))
                assert np.array_equal(d_off.cpu().numpy().view(np.uint32), off)
                d_off.fill_(7)
            total = bvh.traverse_dev(d_rays.data_ptr(), len(rays), d_off.data_ptr(), d_hits.data_ptr(), len(hits), mode=mode, want_total=True)
            bvh.ctx.synchronize()                            # the call returns once the total is known; the fill may still run
            assert total == len(hits) and np.array_equal(d_off.cpu().numpy().view(np.uint32), off)
            assert np.array_equal(d_hits.cpu().numpy().view(np.uint32)[:len(hits)], hits)
    return sum(map(len, want_b))


def _check_hits(bvh, D, shapes, rays, prec):
    """any hit and multi hit, AABB mode, every limit family, every form, against the models; returns the filled multi-hit slots."""
    F = FT[prec]
    nodes = _nodes(bvh, D)
    o, inv = rays["origin"], rays["inv_direction"]
    lims, dstar = ED.limits(dimorder.Tree(nodes, shapes), o, inv, prec)
    filled = 0
    for name, tm in lims.items():
        want = H.aabb_batch(nodes, shapes, o, inv, tm)
        for f, got in enumerate(any_forms(bvh, D, rays, tm, prec)):
            assert np.array_equal(got, want), ("any", name, f)
        for k in (1, 3, 64) if name in ("null", "exact", "exit", "subnormal") else (3,):
            w = MH.aabb_batch(nodes, shapes, o, inv, k, tm)
            zeros = np.zeros((len(rays), k, 2), dtype=F)
            for f, got in enumerate(multi_forms(bvh, D, rays, k, tm, prec)):
                assert _same(got, w, zeros), ("multi", name, k, f)
            filled += int((w[0] != U32_MAX).sum())
    return filled


def _check_knn(bvh, mn, mx, prec, seed=0):
    pts, _ = ED.points(mn, mx, N_POINTS, prec, seed)
    r, _ = ED.radii(mn, mx, pts, prec, seed)
    filled = 0
    for md in (None, r):
        bs, bd = K.brute(mn, mx, pts, 64, md)
        for k in KNN_KS:
            s, d = bvh.knn(pts, k, md)
            assert np.array_equal(s, bs[:, :k]), (k, md is None)
            assert d.tobytes() == np.ascontiguousarray(bd[:, :k]).tobytes(), (k, md is None)
        filled += int((bs != U32_MAX).sum())
    return pts, filled


def _check_nearest(bvh, D, mn, mx, shapes, pts, prec):
    """nearest_to (BVH and FLAT) against dimref; nearest_candidates list for list against prunedmodel.Tree.candidates, and the
    contract of prunedcheck.check_candidates (every shape at the minimal exact distance, nearest_to's and the brute force's shape).
    On huge and subnormal scenes every list holds every shape (the bound overflows, resp. every square underflows to 0), so there the
    comparison checks completeness and order; on mixed scenes the bound prunes."""
    from bvh_b200 import capi

    F = mn.dtype.type
    nodes = _nodes(bvh, D)
    if D != 3:
        t = dimref.Tree(nodes, shapes, bvh.flatten())
        for mode, fn in ((capi.TRAVERSE_BVH, t.nearest_bvh), (capi.TRAVERSE_FLAT, t.nearest_flat)):
            s, d = bvh.nearest_to_batch(pts, mode=mode)
            for i, p in enumerate(pts):
                ws, wd = fn(list(p))
                assert s[i] == ws and _bits(d[i:i + 1])[0] == _bits(np.array([wd], dtype=F))[0], (mode, i)
    pts = pts[:40]
    off, cand = bvh.nearest_candidates(pts)
    lists = [cand[off[i]:off[i + 1]].tolist() for i in range(len(pts))]
    tree = M.Tree(nodes, shapes)
    for i, p in enumerate(pts):
        assert lists[i] == tree.candidates(list(p)), i
    PC.check_candidates(lists, nodes, shapes, pts, prec)
    return sum(len(lst) < len(mn) for lst in lists)


def _check_queries(bvh, D, mn, mx, shapes, prec):
    """Aabb, Point and Ball queries, BVH and FLAT, against dimref.Tree.query_bvh / query_flat on the device's own nodes."""
    from bvh_b200 import capi

    F = mn.dtype.type
    nodes = _nodes(bvh, D)
    flat = bvh.flatten().nodes if D == 3 else bvh.flatten()
    t = dimref.Tree(nodes, shapes, flat)
    total = 0
    for qk in (dimref.AABB, dimref.POINT, dimref.BALL):
        q = ED.queries(qk, mn, mx, N_POINTS, prec)
        for mode, fn in ((capi.TRAVERSE_BVH, t.query_bvh), (capi.TRAVERSE_FLAT, t.query_flat)):
            off, hits = bvh.query_batch(qk, q, mode=mode)
            for i in range(len(q)):
                assert hits[off[i]:off[i + 1]].tolist() == fn(qk, [F(v) for v in q[i]]), (qk, mode, i)
            total += len(hits)
    return total


@pytest.mark.parametrize("kind,D,prec", CASES)
def test_walks_equal_the_models(api, kind, D, prec):
    mn, mx, shapes, rays, fam = _setup(api, kind, D, prec)
    bvh = _cls(api, D).build(shapes, prec=prec)
    try:
        if D != 3:
            assert _check_traversal(api, bvh, D, shapes, rays, prec) > 0
            ordered_check(bvh, shapes, rays, rays["origin"], rays["inv_direction"], prec, tight=False)
        else:
            ref = O.traverse(bvh.nodes, shapes, rays, O.MODE_RECURSIVE, prec)
            for compact in (False, True):                    # compact: the device divides 1 / direction itself
                off, hits = bvh.traverse_batch(rays, compact=compact)
                assert np.array_equal(off.astype(np.uint64), ref.offsets) and np.array_equal(hits, ref.hits), compact
        assert _check_hits(bvh, D, shapes, rays, prec) > 0
        pts, filled = _check_knn(bvh, mn, mx, prec)
        assert filled > 0
        pruned = _check_nearest(bvh, D, mn, mx, shapes, pts, prec)
        if kind == "mixed":
            assert pruned > 0                                # the bound prunes below the no-split top
        assert _check_queries(bvh, D, mn, mx, shapes, prec) > 0
    finally:
        bvh.free()


@pytest.mark.parametrize("kind,D", [(k, D) for k in ("huge", "subnormal") for D in ED.DIMS])
@pytest.mark.parametrize("prec", ED.PRECS)
def test_walks_after_refit_and_update(api, kind, D, prec):
    """The caches follow the boxes: a refit that shrinks every box to its lower half, then an update_shapes that moves a third of the
    shapes onto other shapes' boxes, each followed by the walks."""
    F = FT[prec]
    mn, mx, shapes, rays, _ = _setup(api, kind, D, prec)
    bvh = _cls(api, D).build(shapes, prec=prec)
    try:
        shapes["max"] = (shapes["min"] * F(0.5) + shapes["max"] * F(0.5)).astype(F)
        bvh.refit(shapes)
        for step in range(2):
            m2, x2 = np.ascontiguousarray(shapes["min"]), np.ascontiguousarray(shapes["max"])
            if D != 3:
                _check_traversal(api, bvh, D, shapes, rays, prec)
                ordered_check(bvh, shapes, rays, rays["origin"], rays["inv_direction"], prec, tight=False)
            else:
                ref = O.traverse(bvh.nodes, shapes, rays, O.MODE_RECURSIVE, prec)
                for compact in (False, True):
                    off, hits = bvh.traverse_batch(rays, compact=compact)
                    assert np.array_equal(off.astype(np.uint64), ref.offsets) and np.array_equal(hits, ref.hits), (step, compact)
            assert _check_hits(bvh, D, shapes, rays, prec) > 0
            _check_knn(bvh, m2, x2, prec, seed=1 + step)
            if step == 0:
                rng = np.random.default_rng(5)
                changed = rng.choice(len(shapes), len(shapes) // 3, replace=False)
                src = rng.integers(0, len(shapes), len(changed))
                shapes["min"][changed], shapes["max"][changed] = shapes["min"][src], shapes["max"][src]
                bvh.update_shapes(changed, shapes, max_growth=1.5)
    finally:
        bvh.free()


@pytest.mark.parametrize("kind", ED.SCENE_KINDS)
@pytest.mark.parametrize("prec", ED.PRECS)
def test_triangle_modes_equal_the_models(api, kind, prec):
    """Closest, any and multi hit in triangle mode on triangles inside the edge boxes, against the models and closest hit against the
    oracle's loop (prunedcheck.check_closest); knn_triangles on the points whose triangles are all bounded (the others are outside the
    exact guarantee), with radii on the triangle keys.  Triangle mode hits only on the unit-scale half of the mixed scene: at huge
    scale the cross products overflow and at subnormal scale det < eps, so there it is exercised through misses, as in the reference."""
    F = FT[prec]
    mn, mx = ED.scene(kind, N_SHAPES, 3, prec)
    tris = ED.triangles(mn, mx, prec)
    shapes = O.tri_aabbs(tris, prec)
    o, d, inv, _ = ED.ray_batch(shapes["min"], shapes["max"], PER_FAMILY, prec)
    rays = _rays(api, 3, prec, o, d, inv)
    bvh = api.Bvh.build(shapes, prec=prec)
    try:
        bvh.set_triangles(tris)
        nodes = bvh.nodes
        cs, cd, cuv = bvh.closest_hit(rays, triangles=True)
        ws, wd, wuv = O.closest_hit(nodes, shapes, rays, tris, prec)                # the reference's loop over Bvh::traverse
        PC.check_closest(cs, cd, cuv, ws, wd, tris, shapes, rays, prec)
        w = MH.triangles(nodes, shapes, tris, rays, 1, None)
        assert np.array_equal(cs, w[0][:, 0]) and np.array_equal(_bits(cd), _bits(w[1][:, 0])) and np.array_equal(_bits(cuv), _bits(w[2][:, 0]))
        lims = H.tmax_families(cd, F, np.random.default_rng(6))
        lims["subnormal"] = np.full(len(rays), np.finfo(F).smallest_subnormal, dtype=F)
        for name, tm in lims.items():
            want = H.triangles(nodes, shapes, tris, rays, tm)
            for f, got in enumerate(any_forms(bvh, 3, rays, tm, prec, triangles=True)):
                assert np.array_equal(got, want), ("any", name, f)
            for k in (1, 3, 64) if name in ("null", "exact") else (3,):
                w = MH.triangles(nodes, shapes, tris, rays, k, tm)
                for f, got in enumerate(multi_forms(bvh, 3, rays, k, tm, prec, triangles=True)):
                    assert _same(got, w, w[2]), ("multi", name, k, f)
                bs, bd, buv, bounded = MH.brute_triangles(nodes, shapes, tris, rays, k, tm)
                assert np.array_equal(w[0][bounded], bs[bounded]) and np.array_equal(_bits(w[1][bounded]), _bits(bd[bounded])), (name, k)
        if kind == "mixed":
            assert np.any(cs != U32_MAX)
        else:                                                               # subnormal: det < eps; huge: the cross products
            assert np.all(cs == U32_MAX)                                    # overflow; a miss in the reference too
        pts, _ = ED.points(mn, mx, N_POINTS, prec)
        t3 = tris.reshape(-1, 3, 3)
        ok = np.array([KT.bounded(p, t3, shapes["min"], shapes["max"]).all() for p in pts])
        assert ok.sum() > len(pts) // 2
        pts = pts[ok]
        r, _ = ED.radii(mn, mx, pts, prec, key_fn=lambda p: KT.keys(p, t3))   # roundup / exact radii on triangle keys
        for md in (None, r):
            bs, bd, bq = KT.brute(t3, pts, 64, md)
            for k in KNN_KS:
                s, dd, q = bvh.knn_triangles(pts, k, md, closest=True)
                assert np.array_equal(s, bs[:, :k]) and dd.tobytes() == np.ascontiguousarray(bd[:, :k]).tobytes(), (k, md is None)
                assert q.tobytes() == np.ascontiguousarray(bq[:, :k]).tobytes(), (k, md is None)
    finally:
        bvh.free()
