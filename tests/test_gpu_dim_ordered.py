"""Distance-ordered traversal and AABB-mode closest hit on 2-D and 4-D trees (bvhgpu_traverse_ordered_* / bvhgpu_closest_hit_* with the
x2 and x4 suffixes, bvhgpu_closest_hit_dev_*x4), f32 and f64:
- against the dimension-generic restatement (tests/dimorder.py, pinned to the C++ oracle at D = 3 by test_dim_ordered_cpu.py) run over
  the device's own nodes: ordered hit lists and distance bits, offsets equal to traverse_batch(..., TRAVERSE_BVH), closest shape and
  entry distance bits;
- closest = the head of ordered ascending on tight trees; f32 overflow-scale trees list leaves under empty boxes at 0 / +inf while
  closest still keys on the shapes' own boxes;
- at 200 k shapes and 20 k rays, closest against a brute force over every shape (ties: leaf preorder);
- the contract: n = 0 and n = 1, a short capacity, refusals, determinism, the device-pointer form on a side stream, and results
  that follow update_shapes / add_shapes / remove_shapes."""
import ctypes as C

import numpy as np
import pytest

from tests import dimorder, dimref

pytestmark = pytest.mark.gpu
U32_MAX = 0xFFFFFFFF
FT = {"f32": np.float32, "f64": np.float64}
UINT = {"f32": np.uint32, "f64": np.uint64}
CASES = [(D, p) for D in (2, 4) for p in ("f32", "f64")]


@pytest.fixture(scope="module")
def A():
    from bvh_b200 import api

    return api


def _cls(A, D):
    return {2: A.Bvh2, 4: A.Bvh4}[D]


def _aabbs(A, D, prec, mn, mx):
    a = np.zeros(len(mn), dtype=_cls(A, D)._TABLE[prec]["aabb"])
    a["min"], a["max"] = mn, mx
    return a


def _rays(A, D, prec, o, d, inv):
    r = np.zeros(len(o), dtype=_cls(A, D)._TABLE[prec]["ray"])
    r["origin"], r["direction"], r["inv_direction"] = o, d, inv
    return r


def _check(bvh, shapes, rays, o, inv, prec, tight=True):
    """ordered (both orders) and closest against the restatement on the device's own nodes; returns the ascending CSR."""
    from bvh_b200 import capi

    F, U = FT[prec], UINT[prec]
    nodes, _ = bvh.nodes_and_index()
    tree = dimorder.Tree(nodes, shapes)
    toff, _ = bvh.traverse_batch(rays, mode=capi.TRAVERSE_BVH)
    out = {}
    for ascending in (True, False):
        off, hits, dists = bvh.traverse_ordered(rays, ascending)
        assert np.array_equal(off, toff), ascending
        for i in range(len(rays)):
            want = tree.ordered((list(o[i]), list(inv[i])), ascending)
            got_h = hits[off[i]:off[i + 1]].tolist()
            assert got_h == [s for s, _ in want], (ascending, i)
            assert dists[off[i]:off[i + 1]].view(U).tolist() == np.array([d for _, d in want], dtype=F).view(U).tolist(), (ascending, i)
        out[ascending] = (off, hits, dists)
    cs, cd = bvh.closest_hit(rays)
    for i in range(len(rays)):
        s, d = tree.closest((list(o[i]), list(inv[i])))
        assert cs[i] == s and cd[i:i + 1].view(U)[0] == np.array([np.inf if d is None else d], dtype=F).view(U)[0], i
    off, hits, dists = out[True]
    empty = off[:-1] == off[1:]
    assert np.all(cs[empty] == U32_MAX) and np.all(np.isinf(cd[empty]))
    if tight:                                                   # closest = the head of ordered ascending
        head = ~empty
        assert np.array_equal(cs[head], hits[off[:-1][head]])
        assert np.array_equal(cd[head].view(U), dists[off[:-1][head]].view(U))
    return out, cs, cd


@pytest.mark.parametrize("scene", ["random", "coincident", "axis", "overflow"])
@pytest.mark.parametrize("D,prec", CASES)
def test_ordered_and_closest_equal_the_restatement(A, D, prec, scene):
    F = FT[prec]
    rng = np.random.default_rng(40 + D)
    mn, mx = dimref.scene(scene, 400, D, F, rng)
    o, d, inv = dimorder.rays(mn, mx, 300, F, rng)
    bvh = _cls(A, D).build(_aabbs(A, D, prec, mn, mx), prec=prec)
    nodes, _ = bvh.nodes_and_index()
    inner = nodes["child_l"] != U32_MAX                          # leaves always hold empty child boxes
    overflow = bool(np.any(nodes["l_aabb"]["min"][inner, 0] == np.inf))
    if scene == "overflow" and prec == "f32":
        assert overflow                                         # "no split wins": empty stored boxes
    out, cs, cd = _check(bvh, _aabbs(A, D, prec, mn, mx), _rays(A, D, prec, o, d, inv), o, inv, prec, tight=not overflow)
    if overflow:
        off, hits, dists = out[True]
        assert np.any(dists == 0)
        offd, hitsd, distsd = out[False]
        assert np.any(np.isinf(distsd))                         # exit +inf of an empty box
        assert np.sum(cs != U32_MAX) < len(hits)               # closest keys the shapes' own boxes, not the listed leaves
    elif scene != "coincident":                                 # point boxes: a rounded aim rarely hits them
        assert np.sum(cs != U32_MAX) > 0
    bvh.free()


@pytest.mark.parametrize("D,prec", CASES)
def test_closest_against_brute_force_at_scale(A, D, prec):
    """200 k shapes, 20 k rays: the minimum entry over every shape whose own box the ray enters, ties to the lower leaf preorder
    position (node_index), computed on the device with torch elementwise ops (each one rounds once, as the slab test does)."""
    import torch

    F = FT[prec]
    rng = np.random.default_rng(7 + D)
    n, m = 200_000, 20_000
    mn = rng.uniform(-1000, 1000, (n, D)).astype(F)
    mx = (mn + rng.uniform(0, 6, (n, D))).astype(F)
    o, d, inv = dimorder.rays(mn, mx, m, F, rng)
    bvh = _cls(A, D).build(_aabbs(A, D, prec, mn, mx), prec=prec)
    cs, cd = bvh.closest_hit(_rays(A, D, prec, o, d, inv))
    _, node_index = bvh.nodes_and_index()
    dev = torch.device("cuda", 0)
    tmn, tmx = torch.from_numpy(mn).to(dev), torch.from_numpy(mx).to(dev)
    rank = torch.from_numpy(node_index.astype(np.int64)).to(dev)
    ws, wd = np.full(m, U32_MAX, dtype=np.uint32), np.full(m, np.inf, dtype=F)
    for a in range(0, m, 256):
        to, ti = torch.from_numpy(o[a:a + 256]).to(dev)[:, None, :], torch.from_numpy(inv[a:a + 256]).to(dev)[:, None, :]
        l, r = (tmn[None] - to) * ti, (tmx[None] - to) * ti
        nan = torch.isnan(l).any(-1) | torch.isnan(r).any(-1)
        tmin, tmax = torch.minimum(l, r).amax(-1), torch.maximum(l, r).amin(-1)
        entry = torch.where(tmin > 0, tmin, torch.zeros_like(tmin))
        hit = ~nan & ~(entry > tmax)
        key = torch.where(hit, entry, torch.full_like(entry, float("inf")))
        best = key.amin(-1, keepdim=True)
        cand = hit & (key == best)
        pos = torch.where(cand, rank[None], torch.full_like(rank[None], 1 << 40)).argmin(-1)
        anyhit = cand.any(-1)
        ws[a:a + 256] = np.where(anyhit.cpu().numpy(), pos.cpu().numpy(), U32_MAX).astype(np.uint32)
        wd[a:a + 256] = np.where(anyhit.cpu().numpy(), best[:, 0].cpu().numpy(), np.inf).astype(F)
    assert np.sum(ws != U32_MAX) > m // 10
    assert np.array_equal(cs, ws)
    assert np.array_equal(cd.view(UINT[prec]), wd.view(UINT[prec]))
    bvh.free()


@pytest.mark.parametrize("D,prec", CASES)
def test_contract(A, D, prec):
    from bvh_b200 import capi

    F = FT[prec]
    L = capi.lib()
    rng = np.random.default_rng(90 + D)
    cls = _cls(A, D)
    suf = cls._TABLE[prec]["suffix"]
    mn, mx = dimref.scene("random", 600, D, F, rng)
    o, d, inv = dimorder.rays(mn, mx, 200, F, rng)
    rays = _rays(A, D, prec, o, d, inv)
    # n = 0: all-zero offsets, no hit
    b0 = cls.build(_aabbs(A, D, prec, mn[:0], mx[:0]), prec=prec)
    off, hits, dists = b0.traverse_ordered(rays)
    assert not off.any() and len(hits) == 0 and len(dists) == 0
    s, dd = b0.closest_hit(rays)
    assert np.all(s == U32_MAX) and np.all(np.isinf(dd))
    b0.free()
    # n = 1: the root leaf is decided by the shape's own box
    b1 = cls.build(_aabbs(A, D, prec, mn[:1], mx[:1]), prec=prec)
    _check(b1, _aabbs(A, D, prec, mn[:1], mx[:1]), rays, o, inv, prec)
    b1.free()
    bvh = cls.build(_aabbs(A, D, prec, mn, mx), prec=prec)
    full = bvh.traverse_ordered(rays)
    assert len(full[1]) > 4
    # short cap: BVHGPU_ERR_CAPACITY with valid offsets and total, then the full result
    n = len(rays)
    off = np.zeros(n + 1, dtype=np.uint32)
    hits = np.zeros(3, dtype=np.uint32)
    dists = np.zeros(3, dtype=F)
    total = C.c_size_t(0)
    fn = getattr(L, f"bvhgpu_traverse_ordered_{suf}")
    st = fn(bvh._h, rays.ctypes.data, n, 1, off.ctypes.data, hits.ctypes.data, dists.ctypes.data, 3, C.byref(total))
    assert st == capi.ERR_CAPACITY and total.value == len(full[1]) and np.array_equal(off, full[0])
    hits = np.zeros(total.value, dtype=np.uint32)
    dists = np.zeros(total.value, dtype=F)
    assert fn(bvh._h, rays.ctypes.data, n, 1, off.ctypes.data, hits.ctypes.data, dists.ctypes.data, total.value, C.byref(total)) == capi.OK
    assert np.array_equal(hits, full[1]) and dists.tobytes() == full[2].tobytes()
    # refusals write nothing
    off = np.full(n + 1, 7, dtype=np.uint32)
    shape_out = np.full(n, 7, dtype=np.uint32)
    dist_out = np.full(n, 7, dtype=F)
    assert fn(bvh._h, None, n, 1, off.ctypes.data, hits.ctypes.data, dists.ctypes.data, len(hits), C.byref(total)) == capi.ERR_INVALID
    assert fn(bvh._h, rays.ctypes.data, n, 1, off.ctypes.data, None, dists.ctypes.data, len(hits), C.byref(total)) == capi.ERR_INVALID
    assert fn(bvh._h, rays.ctypes.data, 1 << 31, 1, off.ctypes.data, hits.ctypes.data, dists.ctypes.data, len(hits), C.byref(total)) == capi.ERR_INVALID
    assert fn(None, rays.ctypes.data, n, 1, off.ctypes.data, hits.ctypes.data, dists.ctypes.data, len(hits), C.byref(total)) == capi.ERR_INVALID
    ch = getattr(L, f"bvhgpu_closest_hit_{suf}")
    assert ch(bvh._h, rays.ctypes.data, n, None, dist_out.ctypes.data) == capi.ERR_INVALID
    assert ch(bvh._h, rays.ctypes.data, 1 << 31, shape_out.ctypes.data, dist_out.ctypes.data) == capi.ERR_INVALID
    assert np.all(off == 7) and np.all(shape_out == 7) and np.all(dist_out == 7)
    # two calls, byte-identical results
    again = bvh.traverse_ordered(rays)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(full, again))
    c1, c2 = bvh.closest_hit(rays), bvh.closest_hit(rays)
    assert c1[0].tobytes() == c2[0].tobytes() and c1[1].tobytes() == c2[1].tobytes()
    bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_closest_hit_dev_on_a_side_stream_equals_the_host_form(A, prec):
    import torch

    F = FT[prec]
    rng = np.random.default_rng(5)
    mn, mx = dimref.scene("random", 3000, 4, F, rng)
    o, d, inv = dimorder.rays(mn, mx, 5000, F, rng)
    rays = _rays(A, 4, prec, o, d, inv)
    bvh = A.Bvh4.build(_aabbs(A, 4, prec, mn, mx), prec=prec)
    hs, hd = bvh.closest_hit(rays)
    dev = torch.device("cuda", 0)
    side = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(side):
        d_rays = torch.from_numpy(rays.view(np.uint8)).to(dev, non_blocking=False)
        d_s = torch.full((len(rays),), -1, dtype=torch.int32, device=dev)
        d_d = torch.zeros(len(rays), dtype=torch.float32 if prec == "f32" else torch.float64, device=dev)
        bvh.ctx.set_stream(side.cuda_stream)
        try:
            bvh.closest_hit_dev(d_rays.data_ptr(), len(rays), d_s.data_ptr(), d_d.data_ptr())
        finally:
            bvh.ctx.set_stream(None)
        side.synchronize()
    assert np.array_equal(d_s.cpu().numpy().view(np.uint32), hs)
    assert d_d.cpu().numpy().tobytes() == hd.tobytes()
    from bvh_b200 import capi

    fn = getattr(capi.lib(), f"bvhgpu_closest_hit_dev_{bvh._d['suffix']}")
    assert fn(bvh._h, None, 4, d_s.data_ptr(), d_d.data_ptr()) == capi.ERR_INVALID
    bvh.free()


@pytest.mark.parametrize("D,prec", CASES)
def test_results_follow_update_add_and_remove(A, D, prec):
    F = FT[prec]
    rng = np.random.default_rng(60 + D)
    mn, mx = dimref.scene("random", 500, D, F, rng)
    o, d, inv = dimorder.rays(mn, mx, 150, F, rng)
    rays = _rays(A, D, prec, o, d, inv)
    aabbs = _aabbs(A, D, prec, mn, mx)
    bvh = _cls(A, D).build(aabbs, prec=prec)
    _check(bvh, aabbs, rays, o, inv, prec)                      # builds the traversal records before the tree changes
    changed = rng.choice(len(aabbs), 60, replace=False)
    shift = rng.uniform(-20, 20, (60, D)).astype(F)
    aabbs["min"][changed] = (aabbs["min"][changed] + shift).astype(F)
    aabbs["max"][changed] = (aabbs["max"][changed] + shift).astype(F)
    bvh.update_shapes(changed, aabbs, max_growth=1.5)
    _check(bvh, aabbs, rays, o, inv, prec)
    nmn, nmx = dimref.scene("random", 40, D, F, rng)
    new = _aabbs(A, D, prec, nmn, nmx)
    bvh.add_shapes(new)
    aabbs = np.concatenate([aabbs, new])
    _check(bvh, aabbs, rays, o, inv, prec)
    gone = rng.choice(len(aabbs), 70, replace=False)
    moves = bvh.remove_shapes(gone)
    keep = np.ones(len(aabbs), dtype=bool)
    keep[gone] = False
    after = aabbs.copy()
    for new_i, old_i in moves:
        after[new_i] = aabbs[old_i]
    after = after[: len(aabbs) - len(gone)]
    assert bvh.n == len(after)
    _check(bvh, after, rays, o, inv, prec)
    bvh.free()
