"""The distance-pruned walks on adversarial geometry (tests/adversarial.py), on the device:
- triangle-mode closest_hit equals the restatement of tests/prunedmodel.py bit for bit, in the host form and the device-pointer
  form with both ray layouts, and meets the contract of tests/prunedcheck.py against the reference's unpruned loop;
- AABB-mode closest_hit, traverse_ordered, nearest_to and nearest_triangles (BVH and FLAT) remain replays of the oracle on the same
  scenes, bit for bit;
- nearest_candidates in D = 2, 3 and 4 equals the restatement list for list and meets its contract.
Run on an H100:  python -m pytest tests/test_gpu_pruned_walks.py -m gpu"""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O
from tests import adversarial as A, prunedcheck as PC, prunedmodel as M

pytestmark = pytest.mark.gpu
FT = {"f32": np.float32, "f64": np.float64}


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A_

    return A_


def _scene(family, prec):
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


def _closest_dev(bvh, rays, layout, prec):
    """bvhgpu_closest_hit_dev_* in triangle mode on device copies of the rays (FULL: the Ray structs, OD: origin + direction)."""
    import torch

    from bvh_b200 import capi

    F = FT[prec]
    n = len(rays)
    src = rays if layout == capi.RAYS_FULL else np.ascontiguousarray(np.concatenate([rays["origin"], rays["direction"]], axis=1))
    d_rays = torch.from_numpy(np.frombuffer(src.tobytes(), dtype=np.uint8).copy()).cuda()
    sh = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    dist = torch.zeros(n, dtype=torch.float32 if prec == "f32" else torch.float64, device="cuda")
    uv = torch.zeros(2 * n, dtype=dist.dtype, device="cuda")
    torch.cuda.synchronize()
    sfx = "f32x3" if prec == "f32" else "f64x3"
    capi.check(getattr(capi.lib(), f"bvhgpu_closest_hit_dev_{sfx}")(bvh._h, C.c_void_p(d_rays.data_ptr()), layout, n, 1, C.c_void_p(sh.data_ptr()),
                                                                      C.c_void_p(dist.data_ptr()), C.c_void_p(uv.data_ptr())))
    bvh.ctx.synchronize()
    return sh.cpu().numpy().view(np.uint32), dist.cpu().numpy().astype(F), uv.cpu().numpy().reshape(n, 2)


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("family", ["grazing", "shared", "degenerate", "offset_lo", "offset_hi"])
def test_closest_triangles_equal_the_model(api, family, prec):
    from bvh_b200 import capi

    tris, rays = _scene(family, prec)
    shapes = O.tri_aabbs(tris, prec)
    bvh = api.Bvh.build(shapes, prec=prec)
    try:
        nodes = bvh.nodes
        bvh.set_triangles(tris)
        ms, md, muv = M.closest_triangles(nodes, shapes, tris, rays)
        ws, wd, _ = O.closest_hit(nodes, shapes, rays, tris, prec)
        results = [bvh.closest_hit(rays, triangles=True)] + [_closest_dev(bvh, rays, lay, prec) for lay in (capi.RAYS_FULL, capi.RAYS_OD)]
        for gs, gd, guv in results:
            assert gs.tobytes() == ms.tobytes() and gd.tobytes() == md.tobytes() and guv.tobytes() == muv.tobytes()
        ndiff = PC.check_closest(ms, md, muv, ws, wd, tris, shapes, rays, prec)
        if family == "grazing" and prec == "f32":
            assert ndiff >= 20                         # the case the family exists for reaches the device
        assert (ws != O.U32_MAX).sum() > 0
    finally:
        bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("family", ["grazing", "shared", "degenerate", "offset_hi"])
def test_replayed_walks_on_adversarial_scenes(api, family, prec):
    """AABB-mode closest_hit, traverse_ordered, nearest_to and nearest_triangles stay replays of the oracle on these scenes."""
    from bvh_b200 import capi

    tris, rays = _scene(family, prec)
    shapes = O.tri_aabbs(tris, prec)
    bvh = api.Bvh.build(shapes, prec=prec)
    try:
        nodes = bvh.nodes
        bvh.set_triangles(tris)
        ws, wd, _ = O.closest_hit(nodes, shapes, rays, prec=prec)
        gs, gd, _ = bvh.closest_hit(rays)
        assert gs.tobytes() == ws.tobytes() and gd.tobytes() == wd.tobytes()
        off, hits, dists = bvh.traverse_ordered(rays, True)
        r = O.traverse(nodes, shapes, rays, O.MODE_RECURSIVE, prec)
        for i in range(len(rays)):
            mine, want = hits[off[i]:off[i + 1]], r.hits[r.offsets[i]:r.offsets[i + 1]]
            assert sorted(mine.tolist()) == sorted(want.tolist()), i
            dd = dists[off[i]:off[i + 1]]
            assert np.all(dd[1:] >= dd[:-1])
            if len(mine):
                assert mine[0] == gs[i] and dd[0] == gd[i]
        pts = np.concatenate([rays["origin"], tris.reshape(-1, 3)[::3]])
        flat = O.flatten(nodes, prec)
        for mode, tree, is_flat in ((capi.TRAVERSE_BVH, nodes, False), (capi.TRAVERSE_FLAT, flat, True)):
            s, d = bvh.nearest_to_batch(pts, mode)
            es, ed = O.nearest_to(tree, shapes, pts, prec, flat=is_flat)
            assert s.tobytes() == es.tobytes() and d.tobytes() == ed.tobytes(), mode
            s, d = bvh.nearest_triangles_batch(pts, mode)
            es, ed = O.nearest_to(tree, shapes, pts, prec, flat=is_flat, kind=O.DIST_TRIANGLE, tris=tris)
            assert s.tobytes() == es.tobytes() and d.tobytes() == ed.tobytes(), mode
    finally:
        bvh.free()


def _shapes(mn, mx, prec):
    from bvh_b200.dtypes import BY_PREC, BY_PREC_2D, BY_PREC_4D

    a = np.zeros(len(mn), dtype={2: BY_PREC_2D, 3: BY_PREC, 4: BY_PREC_4D}[mn.shape[1]][prec]["aabb"])
    a["min"], a["max"] = mn, mx
    return a


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("D", [2, 3, 4])
@pytest.mark.parametrize("family", sorted(A.BOX_FAMILIES))
def test_nearest_candidates_equal_the_model(api, family, D, prec):
    F = FT[prec]
    mn, mx, pts = A.BOX_FAMILIES[family](F, D)
    shapes = _shapes(mn, mx, prec)
    cls = {2: api.Bvh2, 3: api.Bvh, 4: api.Bvh4}[D]
    bvh = cls.build(shapes, prec=prec)
    try:
        nodes = bvh.nodes if D == 3 else bvh.nodes_and_index()[0]
        off, cand = bvh.nearest_candidates(pts)
        lists = [cand[off[i]:off[i + 1]].tolist() for i in range(len(pts))]
        tree = M.Tree(nodes, shapes)
        for i, p in enumerate(pts):
            assert lists[i] == tree.candidates(list(p)), i
        PC.check_candidates(lists, nodes, shapes, pts, prec)
        if family == "overflow":
            assert all(sorted(lst) == list(range(len(mn))) for lst in lists)
    finally:
        bvh.free()
