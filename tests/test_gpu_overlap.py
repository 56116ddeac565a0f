"""The self-overlap pairs on the device (bvhgpu_overlap_pairs_* / bvhgpu_overlap_pairs_dev_*).  Every comparison is exact: offsets
and hits equal byte for byte.
- against the brute force of tests/overlapref.py in D = 2, 3, 4 and f32 / f64, on every dimref scene, every adversarial box family
  (the overflow family's trees really store empty child boxes) and the edge_dims huge / mixed / subnormal scenes, for every build
  mode the dimension accepts;
- the current boxes after refit, update_shapes (loose boxes and rebuilds), add_shapes and remove_shapes;
- at scale: the 120 k boxes of BASELINE.json configs[1] and the Sponza triangle boxes against a chunked torch brute force;
- identities: 2-D rows equal the 3-D rows of the lifted scene, 4-D rows with a constant fourth axis equal the 3-D rows, and on tight
  trees the symmetric closure equals query_batch(QUERY_AABB, own boxes) minus the shape itself;
- the contract: n = 0 and 1, a short capacity (then the retry, and the fetch in 3-D), the dev form's prefix without a total, refusals
  with the output buffers untouched, the sticky failed build, the dev form on a torch side stream, and one total above 2^32 - 1."""
import ctypes as C

import numpy as np
import pytest

from bvh_b200 import scenes
from oracle import oracle as O
from tests import adversarial as A, dimref, edge_dims, overlapref as R

pytestmark = pytest.mark.gpu
U32_MAX = 0xFFFFFFFF
FT = {"f32": np.float32, "f64": np.float64}
CASES = [(D, p) for D in (2, 3, 4) for p in ("f32", "f64")]
MODES = {2: (0, 1, 2), 3: (0, 1, 2), 4: (0,)}                     # SAH, LBVH, LBVH + treelet


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A_

    return A_


def _cls(api, D):
    return {2: api.Bvh2, 3: api.Bvh, 4: api.Bvh4}[D]


def _aabbs(api, D, prec, mn, mx):
    from bvh_b200.dtypes import BY_PREC

    t = BY_PREC[prec] if D == 3 else _cls(api, D)._TABLE[prec]
    a = np.zeros(len(mn), dtype=t["aabb"])
    a["min"], a["max"] = mn, mx
    return a


def _build(api, D, prec, mn, mx, mode=0):
    return _cls(api, D).build(_aabbs(api, D, prec, mn, mx), prec=prec, mode=mode)


def _nodes_and_index(bvh, D):
    """The tree's current nodes and leaf node indices, read fresh."""
    from bvh_b200 import capi

    if D != 3:
        return bvh.nodes_and_index()
    n = bvh.num_shapes
    nodes = np.zeros(max(2 * n - 1, 0), dtype=bvh._d["node"])
    idx = np.zeros(n, dtype=np.uint32)
    capi.check(getattr(capi.lib(), f"bvhgpu_tree_nodes_{bvh._d['suffix']}")(bvh._h, bvh_ptr(nodes), bvh_ptr(idx)))
    return nodes, idx


def bvh_ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _check(bvh, D, mn, mx):
    """bvh.overlap_pairs equals the model on the tree's current leaves; returns the number of pairs."""
    _, leaf = _nodes_and_index(bvh, D)
    off, hits = bvh.overlap_pairs()
    ro, rh = R.rows(np.ascontiguousarray(mn), np.ascontiguousarray(mx), leaf)
    assert off.tobytes() == ro.tobytes()
    assert hits.tobytes() == rh.tobytes()
    return len(hits)


@pytest.mark.parametrize("scene", dimref.SCENES)
@pytest.mark.parametrize("D,prec", CASES)
def test_dimref_scenes_every_build_mode(api, D, prec, scene):
    F = FT[prec]
    rng = np.random.default_rng(20 * D + (prec == "f64") + 100 * dimref.SCENES.index(scene))
    mn, mx = dimref.scene(scene, 300, D, F, rng)
    for mode in MODES[D]:
        bvh = _build(api, D, prec, mn, mx, mode)
        npairs = _check(bvh, D, mn, mx)
        if scene == "coincident":
            assert npairs == 300 * 299 // 2
        bvh.free()


@pytest.mark.parametrize("family", sorted(A.BOX_FAMILIES))
@pytest.mark.parametrize("D,prec", CASES)
def test_adversarial_box_families(api, D, prec, family):
    mn, mx, _ = A.BOX_FAMILIES[family](FT[prec], D)
    for mode in MODES[D]:
        bvh = _build(api, D, prec, mn, mx, mode)
        if family == "overflow" and mode == 0:
            nodes, _ = _nodes_and_index(bvh, D)
            assert edge_dims.empty_child_boxes(nodes) > 0             # "no split wins" nodes: the walk must enter their empty boxes
        _check(bvh, D, mn, mx)
        bvh.free()


@pytest.mark.parametrize("kind", edge_dims.SCENE_KINDS)
@pytest.mark.parametrize("D,prec", CASES)
def test_edge_dims_scenes(api, D, prec, kind):
    mn, mx = edge_dims.scene(kind, 240, D, prec)
    for mode in MODES[D]:
        bvh = _build(api, D, prec, mn, mx, mode)
        _check(bvh, D, mn, mx)
        bvh.free()


@pytest.mark.parametrize("D,prec", CASES)
def test_current_boxes_after_refit_update_add_and_remove(api, D, prec):
    F = FT[prec]
    rng = np.random.default_rng(60 + D)
    mn, mx = dimref.scene("random", 400, D, F, rng)
    mx = (mn + (mx - mn) * 6).astype(F)                        # boxes large enough to overlap in D = 4 too
    aabbs = _aabbs(api, D, prec, mn, mx)
    bvh = _cls(api, D).build(aabbs, prec=prec)

    def check(a):
        return _check(bvh, D, a["min"], a["max"])

    assert check(aabbs) > 0
    shift = rng.uniform(-3, 3, (len(aabbs), D)).astype(F)
    aabbs["min"], aabbs["max"] = (aabbs["min"] + shift).astype(F), (aabbs["max"] + shift).astype(F)
    bvh.refit(aabbs)
    check(aabbs)
    for growth in (0.0, 1.5):                                  # loose boxes (refit of the changed paths only), then rebuilds
        changed = rng.choice(len(aabbs), 60, replace=False)
        shift = rng.uniform(-40, 40, (60, D)).astype(F)
        aabbs["min"][changed] = (aabbs["min"][changed] + shift).astype(F)
        aabbs["max"][changed] = (aabbs["max"][changed] + shift).astype(F)
        bvh.update_shapes(changed, aabbs, max_growth=growth)
        check(aabbs)
    nmn, nmx = dimref.scene("random", 40, D, F, rng)
    new = _aabbs(api, D, prec, nmn, nmx)
    bvh.add_shapes(new)
    aabbs = np.concatenate([aabbs, new])
    check(aabbs)
    gone = rng.choice(len(aabbs), 70, replace=False)
    moves = bvh.remove_shapes(gone)
    after = aabbs.copy()
    for new_i, old_i in moves:
        after[new_i] = aabbs[old_i]
    check(after[: len(aabbs) - len(gone)])
    bvh.free()


def _torch_rows(mn, mx, leaf, chunk=512):
    """The model on the device with torch, in the same comparison order: boxes in leaf order, row i against the columns j > i."""
    import torch

    dev = torch.device("cuda", 0)
    n = len(mn)
    perm = np.argsort(leaf, kind="stable")
    pmn, pmx = torch.from_numpy(np.ascontiguousarray(mn[perm])).to(dev), torch.from_numpy(np.ascontiguousarray(mx[perm])).to(dev)
    col = torch.arange(n, device=dev)
    ii, jj = [], []
    for a in range(0, n, chunk):
        b = min(a + chunk, n)
        ok = ~((pmx[a:b, None, :] < pmn[None]) | (pmx[None] < pmn[a:b, None, :]))
        m = ok.all(dim=2) & (col[None, :] > torch.arange(a, b, device=dev)[:, None])
        i, j = torch.nonzero(m, as_tuple=True)
        ii.append((i + a).cpu().numpy())
        jj.append(j.cpu().numpy())
    i, j = np.concatenate(ii), np.concatenate(jj)
    s, t = perm[i], perm[j]
    o = np.argsort(s, kind="stable")                                   # rows by shape, partners still in leaf order
    offsets = np.zeros(n + 1, dtype=np.uint32)
    np.cumsum(np.bincount(s, minlength=n), out=offsets[1:])
    return offsets, t[o].astype(np.uint32)


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_configs1_and_sponza_at_scale(api, prec):
    from tests import scenes as S

    for aabbs in (scenes.create_n_cubes_aabbs(10_000, prec).reshape(-1), S.sponza(prec)):
        bvh = api.Bvh.build(aabbs, prec=prec)
        _, leaf = _nodes_and_index(bvh, 3)
        off, hits = bvh.overlap_pairs()
        ro, rh = _torch_rows(np.ascontiguousarray(aabbs["min"]), np.ascontiguousarray(aabbs["max"]), leaf)
        assert len(rh) > len(aabbs)
        got = set(map(tuple, np.sort(R.pairs(off, hits), axis=1).tolist()))
        want = set(map(tuple, np.sort(R.pairs(ro, rh), axis=1).tolist()))
        assert got == want and len(got) == len(hits)
        assert off.tobytes() == ro.tobytes() and hits.tobytes() == rh.tobytes()
        bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_lifts_and_the_query_identity(api, prec):
    from bvh_b200 import capi

    F = FT[prec]
    rng = np.random.default_rng(70)
    mn2, mx2 = dimref.scene("random", 600, 2, F, rng)
    z = lambda a, v: np.concatenate([a, np.full((len(a), 1), v, dtype=F)], axis=1).astype(F)   # noqa: E731
    b2, b3 = _build(api, 2, prec, mn2, mx2), _build(api, 3, prec, z(mn2, 0), z(mx2, 0))
    b4 = _build(api, 4, prec, z(z(mn2, 0), 3.5), z(z(mx2, 0), 3.5))
    o2, h2 = b2.overlap_pairs()
    o3, h3 = b3.overlap_pairs()
    o4, h4 = b4.overlap_pairs()
    assert len(h3) > 0
    assert o2.tobytes() == o3.tobytes() and h2.tobytes() == h3.tobytes()
    assert o4.tobytes() == o3.tobytes() and h4.tobytes() == h3.tobytes()
    # tight trees: the symmetric closure is the Aabb query with every shape's own box, minus the shape itself
    for D, b, mn, mx in ((2, b2, mn2, mx2), (3, b3, z(mn2, 0), z(mx2, 0)), (4, b4, z(z(mn2, 0), 3.5), z(z(mx2, 0), 3.5))):
        nodes, _ = _nodes_and_index(b, D)
        assert edge_dims.empty_child_boxes(nodes) == 0
        off, hits = b.overlap_pairs()
        qo, qh = b.query_batch(capi.QUERY_AABB, np.concatenate([mn, mx], axis=1))
        cl = R.closure(off, hits, len(mn))
        for s in range(len(mn)):
            assert cl[s] == sorted(int(t) for t in qh[qo[s]:qo[s + 1]] if t != s), (D, s)
    for b in (b2, b3, b4):
        b.free()


def _fn(bvh, dev=False):
    from bvh_b200 import capi

    return getattr(capi.lib(), f"bvhgpu_overlap_pairs_{'dev_' if dev else ''}{bvh._d['suffix']}")


@pytest.mark.parametrize("D,prec", CASES)
def test_contract(api, D, prec):
    import torch

    from bvh_b200 import capi

    F = FT[prec]
    rng = np.random.default_rng(40 + D)
    mn, mx = dimref.scene("random", 500, D, F, rng)
    mx = (mn + (mx - mn) * 10).astype(F)                       # boxes large enough to overlap in D = 4 too
    bvh = _build(api, D, prec, mn, mx)
    _, leaf = _nodes_and_index(bvh, D)
    ro, rh = R.rows(mn, mx, leaf)
    tot = len(rh)
    assert tot > 100
    P = api._ptr
    # a short capacity: BVHGPU_ERR_CAPACITY, *total and the offsets right, then the fetch (3-D) or the retry (2-D, 4-D)
    off = np.zeros(len(mn) + 1, dtype=np.uint32)
    hits = np.full(tot, 7, dtype=np.uint32)
    total = C.c_size_t(0)
    assert _fn(bvh)(bvh._h, P(off), P(hits), tot - 1, C.byref(total)) == capi.ERR_CAPACITY
    assert total.value == tot and off.tobytes() == ro.tobytes() and (hits == 7).all()
    if D == 3:
        capi.check(getattr(capi.lib(), f"bvhgpu_traverse_fetch_{bvh._d['suffix']}")(bvh._h, P(hits), tot))
    else:
        assert _fn(bvh)(bvh._h, P(off), P(hits), tot, C.byref(total)) == capi.OK
    assert hits.tobytes() == rh.tobytes() and off.tobytes() == ro.tobytes()
    # refusals: a null tree or offsets pointer writes nothing
    for tree, po in ((None, True), (bvh._h, False)):
        off = np.full(len(mn) + 1, 7, dtype=np.uint32)
        hits = np.full(tot, 7, dtype=np.uint32)
        assert _fn(bvh)(tree, P(off) if po else None, P(hits), tot, C.byref(total)) == capi.ERR_INVALID
        assert (off == 7).all() and (hits == 7).all()
    if D != 2:
        dev = torch.device("cuda", 0)
        d_off = torch.full((len(mn) + 1,), 7, dtype=torch.int32, device=dev)
        d_hits = torch.full((tot,), 7, dtype=torch.int32, device=dev)
        for tree, po in ((None, True), (bvh._h, False)):
            st = _fn(bvh, True)(tree, C.c_void_p(d_off.data_ptr()) if po else None, C.c_void_p(d_hits.data_ptr()), tot, None)
            assert st == capi.ERR_INVALID
        torch.cuda.synchronize()
        assert (d_off == 7).all() and (d_hits == 7).all()
        # the dev form without a total: complete offsets, a prefix of length cap, nothing behind it
        cap = tot // 2
        bvh.overlap_pairs_dev(d_off.data_ptr(), d_hits.data_ptr(), cap)
        bvh.ctx.synchronize()
        assert d_off.cpu().numpy().view(np.uint32).tobytes() == ro.tobytes()
        h = d_hits.cpu().numpy().view(np.uint32)
        assert h[:cap].tobytes() == rh[:cap].tobytes() and (h[cap:] == 7).all()
        with pytest.raises(capi.BvhGpuError) as e:
            bvh.overlap_pairs_dev(d_off.data_ptr(), d_hits.data_ptr(), cap, want_total=True)
        assert e.value.status == capi.ERR_CAPACITY
        assert bvh.overlap_pairs_dev(d_off.data_ptr(), d_hits.data_ptr(), tot, want_total=True) == tot
        assert d_hits.cpu().numpy().view(np.uint32).tobytes() == rh.tobytes()
    bvh.free()
    for n in (0, 1):                                               # all-zero offsets
        b = _build(api, D, prec, mn[:n], mx[:n])
        off, hits = b.overlap_pairs()
        assert off.tolist() == [0] * (n + 1) and len(hits) == 0
        if D != 2:
            d_off = torch.full((n + 1,), 7, dtype=torch.int32, device="cuda")
            assert b.overlap_pairs_dev(d_off.data_ptr(), 0, 0, want_total=True) == 0
            assert (d_off == 0).all()
        b.free()


def test_failed_build_is_sticky(api):
    import torch

    from bvh_b200 import capi

    shapes, _ = O.create_n_cubes(100, want_tris=True)
    shapes = shapes.copy()
    shapes["min"][33][1] = np.nan
    d = torch.from_numpy(shapes.view(np.uint8).reshape(-1)).cuda()
    torch.cuda.synchronize()
    bvh = api.Bvh.build_dev(d.data_ptr(), len(shapes))
    d_off = torch.zeros(len(shapes) + 1, dtype=torch.int32, device="cuda")
    d_hits = torch.zeros(4096, dtype=torch.int32, device="cuda")
    for _ in range(2):
        with pytest.raises(capi.BvhGpuError) as e:
            bvh.overlap_pairs()
        assert e.value.status == capi.ERR_NAN
        with pytest.raises(capi.BvhGpuError) as e:
            bvh.overlap_pairs_dev(d_off.data_ptr(), d_hits.data_ptr(), 4096, want_total=True)
        assert e.value.status == capi.ERR_NAN
    bvh.free()


@pytest.mark.parametrize("D,prec", [(3, "f32"), (3, "f64"), (4, "f32"), (4, "f64")])
def test_dev_form_on_a_side_stream_equals_the_host_form(api, D, prec):
    import torch

    F = FT[prec]
    rng = np.random.default_rng(5 + D)
    mn, mx = dimref.scene("random", 20_000, D, F, rng)
    mx = (mn + (mx - mn) * 4).astype(F)
    bvh = _build(api, D, prec, mn, mx)
    ho, hh = bvh.overlap_pairs()
    assert len(hh) > 1000
    dev = torch.device("cuda", 0)
    side = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(side):
        d_off = torch.full((len(mn) + 1,), 7, dtype=torch.int32, device=dev)
        d_hits = torch.full((len(hh),), 7, dtype=torch.int32, device=dev)
        bvh.ctx.set_stream(side.cuda_stream)
        try:
            bvh.overlap_pairs_dev(d_off.data_ptr(), d_hits.data_ptr(), len(hh))
        finally:
            bvh.ctx.set_stream(None)
        side.synchronize()
    assert d_off.cpu().numpy().view(np.uint32).tobytes() == ho.tobytes()
    assert d_hits.cpu().numpy().view(np.uint32).tobytes() == hh.tobytes()
    bvh.free()


def test_a_total_above_u32_saturates_the_offsets(api):
    """92 683 identical boxes: n (n - 1) / 2 = 4 295 022 903 pairs, one more than fits the u32 offsets.  The dev form returns
    BVHGPU_ERR_CAPACITY with that total; offsets saturate at 0xFFFFFFFF from the first row whose start does not fit."""
    import torch

    from bvh_b200 import capi

    n = 92_683
    mn = np.zeros((n, 3), dtype=np.float32)
    bvh = _build(api, 3, "f32", mn, mn + 1)
    _, leaf = _nodes_and_index(bvh, 3)
    d_off = torch.zeros(n + 1, dtype=torch.int32, device="cuda")
    d_hits = torch.zeros(1024, dtype=torch.int32, device="cuda")
    total = C.c_size_t(0)
    st = _fn(bvh, True)(bvh._h, C.c_void_p(d_off.data_ptr()), C.c_void_p(d_hits.data_ptr()), 1024, C.byref(total))
    assert st == capi.ERR_CAPACITY and total.value == n * (n - 1) // 2 == 4_295_022_903
    rank = np.empty(n, dtype=np.int64)
    rank[np.argsort(leaf, kind="stable")] = np.arange(n)
    start = rank * (n - 1) - rank * (rank - 1) // 2                   # pairs in the rows of the earlier leaves
    want = np.append(np.minimum(start, U32_MAX), U32_MAX).astype(np.uint32)
    assert d_off.cpu().numpy().view(np.uint32).tobytes() == want.tobytes()
    order = np.argsort(leaf, kind="stable")                           # hits[0 ..) = the row of the first leaf: every other shape
    assert d_hits.cpu().numpy().view(np.uint32).tolist() == order[1:1025].tolist()
    bvh.free()
