"""The overlap pairs between two trees on the device (bvhgpu_overlap_trees_* / bvhgpu_overlap_trees_dev_*).  Every comparison is
exact: offsets and hits equal byte for byte.
- against the brute force of tests/crossref.py in D = 2, 3, 4 and f32 / f64: pairs of dimref scenes with every build mode of the
  dimension on each side, every adversarial box family as B with a perturbed copy as A (the overflow family's B really stores empty
  child boxes, and the Aabb query of A's boxes on B misses pairs there), and the edge_dims huge / mixed / subnormal scenes;
- both trees through refit, update_shapes (loose boxes and rebuilds), add_shapes and remove_shapes, interleaved;
- identities: a is b, the transpose, the Aabb query of A's boxes on tight trees, 2-D rows = 3-D rows of the lifted scenes, 4-D rows
  with a constant fourth axis = 3-D rows;
- at scale: the 120 k boxes of BASELINE.json configs[1] and the Sponza triangle boxes against translated copies, against a chunked
  torch brute force;
- launch geometry: n_a on both sides of 256 and of CSR_SCAN_TILE (2048);
- the contract: n_a, n_b in {0, 1}, a short capacity (then the retry, and the fetch on A in 3-D), the dev form's prefix without a
  total, refusals with the output buffers untouched (null a, b or offsets, trees of two contexts), the sticky failed build of A and
  of B, the dev form on a torch side stream, and one total above 2^32 - 1."""
import ctypes as C

import numpy as np
import pytest

from bvh_b200 import scenes
from oracle import oracle as O
from tests import adversarial as A, dimref, edge_dims, overlapref as R
from tests.crossref import cross_rows

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


def _build(api, D, prec, mn, mx, mode=0, ctx=None):
    return _cls(api, D).build(_aabbs(api, D, prec, mn, mx), prec=prec, mode=mode, ctx=ctx)


def _leaf(bvh, D):
    """The tree's current leaf node index of every shape, read fresh."""
    from bvh_b200 import capi

    if D != 3:
        return bvh.nodes_and_index()[1]
    n = bvh.num_shapes
    nodes = np.zeros(max(2 * n - 1, 0), dtype=bvh._d["node"])
    idx = np.zeros(n, dtype=np.uint32)
    capi.check(getattr(capi.lib(), f"bvhgpu_tree_nodes_{bvh._d['suffix']}")(bvh._h, nodes.ctypes.data_as(C.c_void_p), idx.ctypes.data_as(C.c_void_p)))
    return idx


def _nodes(bvh, D):
    if D != 3:
        return bvh.nodes_and_index()[0]
    return bvh.nodes


def _check(a, b, D, amn, amx, bmn, bmx):
    """a.overlap_pairs_with(b) equals the model on B's current leaves; returns the CSR."""
    off, hits = a.overlap_pairs_with(b)
    ro, rh = cross_rows(np.ascontiguousarray(amn), np.ascontiguousarray(amx), np.ascontiguousarray(bmn), np.ascontiguousarray(bmx), _leaf(b, D))
    assert off.tobytes() == ro.tobytes()
    assert hits.tobytes() == rh.tobytes()
    return off, hits


def _perturbed(mn, mx, F, rng):
    """A copy of the boxes, each moved by up to half its extent per axis (infinite extents stay put)."""
    with np.errstate(over="ignore", invalid="ignore"):
        d = rng.uniform(-0.5, 0.5, mn.shape) * (mx.astype(np.float64) - mn)
        d = np.where(np.isfinite(d), d, 0.0)
        return (mn + d).astype(F), (mx + d).astype(F)


@pytest.mark.parametrize("scene_b", dimref.SCENES)
@pytest.mark.parametrize("D,prec", CASES)
def test_dimref_scene_pairs_every_build_mode(api, D, prec, scene_b):
    F = FT[prec]
    i = dimref.SCENES.index(scene_b)
    scene_a = dimref.SCENES[(i + 1) % len(dimref.SCENES)]
    amn, amx = dimref.scene(scene_a, 260, D, F, np.random.default_rng(30 * D + (prec == "f64") + 7 * i))
    bmn, bmx = dimref.scene(scene_b, 300, D, F, np.random.default_rng(31 * D + (prec == "f64") + 11 * i))
    if scene_a == "random":
        amx = (amn + (amx - amn) * 8).astype(F)                 # large enough to meet the axis and peel scenes
    As = [_build(api, D, prec, amn, amx, m) for m in MODES[D]]
    Bs = [_build(api, D, prec, bmn, bmx, m) for m in MODES[D]]
    for a in As:
        for b in Bs:
            _check(a, b, D, amn, amx, bmn, bmx)
    for t in As + Bs:
        t.free()


@pytest.mark.parametrize("family", sorted(A.BOX_FAMILIES))
@pytest.mark.parametrize("D,prec", CASES)
def test_adversarial_box_families(api, D, prec, family):
    from bvh_b200 import capi

    F = FT[prec]
    bmn, bmx, _ = A.BOX_FAMILIES[family](F, D)
    amn, amx = _perturbed(bmn, bmx, F, np.random.default_rng(D))
    a = _build(api, D, prec, amn, amx)
    for mode in MODES[D]:
        b = _build(api, D, prec, bmn, bmx, mode)
        off, hits = _check(a, b, D, amn, amx, bmn, bmx)
        assert len(hits) >= len(amn)                          # every box meets its own perturbed copy
        qo, qh = b.query_batch(capi.QUERY_AABB, np.concatenate([amn, amx], axis=1))
        got, q = set(map(tuple, R.pairs(off, hits).tolist())), set(map(tuple, R.pairs(qo, qh).tolist()))
        if family == "overflow" and mode == 0:
            assert edge_dims.empty_child_boxes(_nodes(b, D)) > 0   # "no split wins" nodes: the walk must enter their empty boxes
            assert q < got                                       # the query prunes those boxes and misses pairs
        else:
            assert q <= got
        b.free()
    a.free()


@pytest.mark.parametrize("kind", edge_dims.SCENE_KINDS)
@pytest.mark.parametrize("D,prec", CASES)
def test_edge_dims_scenes(api, D, prec, kind):
    F = FT[prec]
    bmn, bmx = edge_dims.scene(kind, 240, D, prec)
    amn, amx = _perturbed(bmn, bmx, F, np.random.default_rng(3 + D))
    amn, amx = np.concatenate([amn[::2], bmn[1::3]]), np.concatenate([amx[::2], bmx[1::3]])   # moved and identical boxes
    for ma in MODES[D]:
        a = _build(api, D, prec, amn, amx, ma)
        for mb in MODES[D]:
            b = _build(api, D, prec, bmn, bmx, mb)
            _check(a, b, D, amn, amx, bmn, bmx)
            b.free()
        a.free()


@pytest.mark.parametrize("D,prec", CASES)
def test_both_trees_through_refit_update_add_and_remove(api, D, prec):
    F = FT[prec]
    rng = np.random.default_rng(80 + D)
    trees, boxes = [], []
    for n in (400, 330):
        mn, mx = dimref.scene("random", n, D, F, rng)
        mx = (mn + (mx - mn) * 6).astype(F)
        boxes.append(_aabbs(api, D, prec, mn, mx))
        trees.append(_cls(api, D).build(boxes[-1], prec=prec))

    def check():
        _check(trees[0], trees[1], D, boxes[0]["min"], boxes[0]["max"], boxes[1]["min"], boxes[1]["max"])
        _check(trees[1], trees[0], D, boxes[1]["min"], boxes[1]["max"], boxes[0]["min"], boxes[0]["max"])

    check()
    for side in (0, 1):                                         # refit
        shift = rng.uniform(-3, 3, (len(boxes[side]), D)).astype(F)
        boxes[side]["min"], boxes[side]["max"] = (boxes[side]["min"] + shift).astype(F), (boxes[side]["max"] + shift).astype(F)
        trees[side].refit(boxes[side])
        check()
    for side, growth in ((1, 0.0), (0, 1.5), (0, 0.0), (1, 1.5)):   # loose boxes (refit of the changed paths only), then rebuilds
        changed = rng.choice(len(boxes[side]), 50, replace=False)
        shift = rng.uniform(-40, 40, (50, D)).astype(F)
        boxes[side]["min"][changed] = (boxes[side]["min"][changed] + shift).astype(F)
        boxes[side]["max"][changed] = (boxes[side]["max"][changed] + shift).astype(F)
        trees[side].update_shapes(changed, boxes[side], max_growth=growth)
        check()
    for side in (1, 0):                                         # add_shapes, then remove_shapes on the other side
        nmn, nmx = dimref.scene("random", 40, D, F, rng)
        new = _aabbs(api, D, prec, nmn, (nmn + (nmx - nmn) * 6).astype(F))
        trees[side].add_shapes(new)
        boxes[side] = np.concatenate([boxes[side], new])
        check()
        other = 1 - side
        gone = rng.choice(len(boxes[other]), 60, replace=False)
        moves = trees[other].remove_shapes(gone)
        after = boxes[other].copy()
        for new_i, old_i in moves:
            after[new_i] = boxes[other][old_i]
        boxes[other] = after[: len(after) - len(gone)].copy()
        check()
    for t in trees:
        t.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_identities(api, prec):
    from bvh_b200 import capi

    F = FT[prec]
    rng = np.random.default_rng(90)
    amn2, amx2 = dimref.scene("random", 500, 2, F, rng)
    bmn2, bmx2 = dimref.scene("random", 450, 2, F, rng)
    z = lambda a, v: np.concatenate([a, np.full((len(a), 1), v, dtype=F)], axis=1).astype(F)   # noqa: E731
    scenes_ = {2: (amn2, amx2, bmn2, bmx2), 3: (z(amn2, 0), z(amx2, 0), z(bmn2, 0), z(bmx2, 0)),
               4: (z(z(amn2, 0), 3.5), z(z(amx2, 0), 3.5), z(z(bmn2, 0), 3.5), z(z(bmx2, 0), 3.5))}
    rows = {}
    for D, (amn, amx, bmn, bmx) in scenes_.items():
        a, b = _build(api, D, prec, amn, amx), _build(api, D, prec, bmn, bmx)
        assert edge_dims.empty_child_boxes(_nodes(b, D)) == 0
        off, hits = _check(a, b, D, amn, amx, bmn, bmx)
        assert len(hits) > 0
        rows[D] = (off.tobytes(), hits.tobytes())
        # tight trees: row a is the Aabb query of a's box on B, BVH mode
        qo, qh = b.query_batch(capi.QUERY_AABB, np.concatenate([amn, amx], axis=1))
        assert qo.tobytes() == off.tobytes() and qh.tobytes() == hits.tobytes()
        # transpose: the pairs of (B, A) reversed
        to, th = _check(b, a, D, bmn, bmx, amn, amx)
        assert set(map(tuple, R.pairs(off, hits).tolist())) == {(s, t) for t, s in R.pairs(to, th).tolist()}
        # a is b: the self-overlap rows both ways, plus (s, s) for every box that meets itself
        so, sh = a.overlap_pairs()
        mo, mh = _check(a, a, D, amn, amx, amn, amx)
        sym = {(s, t) for s, t in R.pairs(so, sh).tolist()} | {(t, s) for s, t in R.pairs(so, sh).tolist()}
        sym |= {(s, s) for s in range(len(amn))}
        assert set(map(tuple, R.pairs(mo, mh).tolist())) == sym and len(mh) == len(sym)
        a.free()
        b.free()
    assert rows[2] == rows[3] == rows[4]                         # 2-D = lifted 3-D = 3-D with a constant fourth axis


def _torch_cross_rows(amn, amx, bmn, bmx, leaf_b, chunk=512):
    """The model on the device with torch: B's boxes in leaf order, a chunk of A's rows at a time."""
    import torch

    dev = torch.device("cuda", 0)
    order = np.argsort(leaf_b, kind="stable")
    pmn, pmx = torch.from_numpy(np.ascontiguousarray(bmn[order])).to(dev), torch.from_numpy(np.ascontiguousarray(bmx[order])).to(dev)
    tmn, tmx = torch.from_numpy(np.ascontiguousarray(amn)).to(dev), torch.from_numpy(np.ascontiguousarray(amx)).to(dev)
    n = len(amn)
    counts, cols = np.zeros(n, dtype=np.int64), []
    for s in range(0, n, chunk):
        e = min(s + chunk, n)
        ok = ~((tmx[s:e, None, :] < pmn[None]) | (pmx[None] < tmn[s:e, None, :]))
        r, c = torch.nonzero(ok.all(dim=2), as_tuple=True)          # row-major: rows in order, partners in leaf order
        counts[s:e] = torch.bincount(r, minlength=e - s).cpu().numpy()
        cols.append(c.cpu().numpy())
    offsets = np.zeros(n + 1, dtype=np.uint32)
    np.cumsum(counts, out=offsets[1:])
    return offsets, order[np.concatenate(cols)].astype(np.uint32)


def _shifted(aabbs, shift):
    out = aabbs.copy()
    F = out["min"].dtype.type
    out["min"], out["max"] = (aabbs["min"] + F(shift)).astype(F), (aabbs["max"] + F(shift)).astype(F)
    return out


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_configs1_and_sponza_at_scale(api, prec):
    from tests import scenes as S

    sp = S.sponza(prec)
    ext = (sp["max"].max(axis=0).astype(np.float64) - sp["min"].min(axis=0)) * 1e-3
    for aabbs, shift in ((scenes.create_n_cubes_aabbs(10_000, prec).reshape(-1), 0.5), (sp, ext)):
        other = _shifted(aabbs, shift)
        a, b = api.Bvh.build(aabbs, prec=prec), api.Bvh.build(other, prec=prec)
        off, hits = a.overlap_pairs_with(b)
        ro, rh = _torch_cross_rows(aabbs["min"], aabbs["max"], other["min"], other["max"], _leaf(b, 3))
        assert len(rh) > len(aabbs)
        assert off.tobytes() == ro.tobytes() and hits.tobytes() == rh.tobytes()
        a.free()
        b.free()


@pytest.mark.parametrize("n_a", [255, 256, 257, 2047, 2048, 2049])
@pytest.mark.parametrize("D", [2, 3, 4])
def test_launch_geometry(api, D, n_a):
    import torch

    F = np.float32
    rng = np.random.default_rng(n_a + D)
    amn, amx = dimref.scene("random", n_a, D, F, rng)
    bmn, bmx = dimref.scene("random", 700, D, F, rng)
    amx = (amn + (amx - amn) * 8).astype(F)
    a, b = _build(api, D, "f32", amn, amx), _build(api, D, "f32", bmn, bmx)
    off, hits = _check(a, b, D, amn, amx, bmn, bmx)
    if D != 2:
        d_off = torch.full((n_a + 1,), 7, dtype=torch.int32, device="cuda")
        d_hits = torch.full((len(hits) + 16,), 7, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        assert a.overlap_pairs_with_dev(b, d_off.data_ptr(), d_hits.data_ptr(), len(hits) + 16, want_total=True) == len(hits)
        assert d_off.cpu().numpy().view(np.uint32).tobytes() == off.tobytes()
        h = d_hits.cpu().numpy().view(np.uint32)
        assert h[:len(hits)].tobytes() == hits.tobytes() and (h[len(hits):] == 7).all()
    a.free()
    b.free()


def _fn(bvh, dev=False):
    from bvh_b200 import capi

    return getattr(capi.lib(), f"bvhgpu_overlap_trees_{'dev_' if dev else ''}{bvh._d['suffix']}")


@pytest.mark.parametrize("D,prec", CASES)
def test_contract(api, D, prec):
    import torch

    from bvh_b200 import capi

    F = FT[prec]
    rng = np.random.default_rng(40 + D)
    amn, amx = dimref.scene("random", 500, D, F, rng)
    bmn, bmx = dimref.scene("random", 420, D, F, rng)
    amx, bmx = (amn + (amx - amn) * 10).astype(F), (bmn + (bmx - bmn) * 6).astype(F)   # boxes large enough to overlap in D = 4 too
    a, b = _build(api, D, prec, amn, amx), _build(api, D, prec, bmn, bmx)
    ro, rh = cross_rows(amn, amx, bmn, bmx, _leaf(b, D))
    tot = len(rh)
    assert tot > 100
    P = api._ptr
    # a short capacity: BVHGPU_ERR_CAPACITY, *total and the offsets right, then the fetch on A (3-D) or the retry (2-D, 4-D)
    off = np.zeros(len(amn) + 1, dtype=np.uint32)
    hits = np.full(tot, 7, dtype=np.uint32)
    total = C.c_size_t(0)
    assert _fn(a)(a._h, b._h, P(off), P(hits), tot - 1, C.byref(total)) == capi.ERR_CAPACITY
    assert total.value == tot and off.tobytes() == ro.tobytes() and (hits == 7).all()
    if D == 3:
        capi.check(getattr(capi.lib(), f"bvhgpu_traverse_fetch_{a._d['suffix']}")(a._h, P(hits), tot))
    else:
        assert _fn(a)(a._h, b._h, P(off), P(hits), tot, C.byref(total)) == capi.OK
    assert hits.tobytes() == rh.tobytes() and off.tobytes() == ro.tobytes()
    o2, h2 = a.overlap_pairs_with(b, cap=tot // 3)              # the wrappers complete a short capacity
    assert o2.tobytes() == ro.tobytes() and h2.tobytes() == rh.tobytes()
    # refusals: a null tree or offsets pointer, or trees of two contexts, write nothing
    ctx2 = api.Context(0)
    b2 = _build(api, D, prec, bmn, bmx, ctx=ctx2)
    for ta, tb, po in ((None, b._h, True), (a._h, None, True), (a._h, b._h, False), (a._h, b2._h, True), (b2._h, a._h, True)):
        off = np.full(len(amn) + 1, 7, dtype=np.uint32)
        hits = np.full(tot, 7, dtype=np.uint32)
        assert _fn(a)(ta, tb, P(off) if po else None, P(hits), tot, C.byref(total)) == capi.ERR_INVALID
        assert (off == 7).all() and (hits == 7).all()
    # a tree of another dimension or precision is refused before any C call
    Dx = 2 if D != 2 else 3
    xmn, xmx = dimref.scene("random", 20, Dx, F, rng)
    wrong = [_build(api, Dx, prec, xmn, xmx), _build(api, D, "f64" if prec == "f32" else "f32", bmn, bmx)]
    with pytest.raises(TypeError):
        a.overlap_pairs_with(wrong[0])
    with pytest.raises(ValueError):
        a.overlap_pairs_with(wrong[1])
    for t in wrong:
        t.free()
    if D != 2:
        dev = torch.device("cuda", 0)
        d_off = torch.full((len(amn) + 1,), 7, dtype=torch.int32, device=dev)
        d_hits = torch.full((tot,), 7, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        for ta, tb, po in ((None, b._h, True), (a._h, None, True), (a._h, b._h, False), (a._h, b2._h, True)):
            st = _fn(a, True)(ta, tb, C.c_void_p(d_off.data_ptr()) if po else None, C.c_void_p(d_hits.data_ptr()), tot, None)
            assert st == capi.ERR_INVALID
        torch.cuda.synchronize()
        assert (d_off == 7).all() and (d_hits == 7).all()
        # the dev form without a total: complete offsets, a prefix of length cap, nothing behind it
        cap = tot // 2
        a.overlap_pairs_with_dev(b, d_off.data_ptr(), d_hits.data_ptr(), cap)
        a.ctx.synchronize()
        assert d_off.cpu().numpy().view(np.uint32).tobytes() == ro.tobytes()
        h = d_hits.cpu().numpy().view(np.uint32)
        assert h[:cap].tobytes() == rh[:cap].tobytes() and (h[cap:] == 7).all()
        with pytest.raises(capi.BvhGpuError) as e:
            a.overlap_pairs_with_dev(b, d_off.data_ptr(), d_hits.data_ptr(), cap, want_total=True)
        assert e.value.status == capi.ERR_CAPACITY
        assert a.overlap_pairs_with_dev(b, d_off.data_ptr(), d_hits.data_ptr(), tot, want_total=True) == tot
        assert d_hits.cpu().numpy().view(np.uint32).tobytes() == rh.tobytes()
    b2.free()
    ctx2.close()
    # n_a, n_b in {0, 1}: n_b = 0 gives all-zero offsets, n_b = 1 is decided by the single box
    for na in (0, 1, len(amn)):
        for nb in (0, 1):
            ta, tb = _build(api, D, prec, amn[:na], amx[:na]), _build(api, D, prec, amn[3:3 + nb], amx[3:3 + nb])
            off, hits = _check(ta, tb, D, amn[:na], amx[:na], amn[3:3 + nb], amx[3:3 + nb])
            if nb == 0:
                assert off.tolist() == [0] * (na + 1)
            if nb == 1 and na > 3:
                assert hits[off[3]:off[4]].tolist() == [0]
            if D != 2:
                d_off = torch.full((na + 1,), 7, dtype=torch.int32, device="cuda")
                d_hits = torch.full((max(len(hits), 1),), 7, dtype=torch.int32, device="cuda")
                torch.cuda.synchronize()
                assert ta.overlap_pairs_with_dev(tb, d_off.data_ptr(), d_hits.data_ptr(), len(hits), want_total=True) == len(hits)
                assert d_off.cpu().numpy().view(np.uint32).tobytes() == off.tobytes()
                assert d_hits.cpu().numpy().view(np.uint32)[:len(hits)].tobytes() == hits.tobytes()
            ta.free()
            tb.free()
    a.free()
    b.free()


def test_failed_build_is_sticky_on_either_side(api):
    import torch

    from bvh_b200 import capi

    shapes, _ = O.create_n_cubes(100, want_tris=True)
    good = api.Bvh.build(shapes)
    shapes = shapes.copy()
    shapes["min"][33][1] = np.nan
    d = torch.from_numpy(shapes.view(np.uint8).reshape(-1)).cuda()
    torch.cuda.synchronize()
    bad = api.Bvh.build_dev(d.data_ptr(), len(shapes))
    d_off = torch.zeros(len(shapes) + 1, dtype=torch.int32, device="cuda")
    d_hits = torch.zeros(1 << 16, dtype=torch.int32, device="cuda")
    for x, y in ((bad, good), (good, bad), (bad, bad)):
        for _ in range(2):
            with pytest.raises(capi.BvhGpuError) as e:
                x.overlap_pairs_with(y)
            assert e.value.status == capi.ERR_NAN
            with pytest.raises(capi.BvhGpuError) as e:
                x.overlap_pairs_with_dev(y, d_off.data_ptr(), d_hits.data_ptr(), 1 << 16, want_total=True)
            assert e.value.status == capi.ERR_NAN
    good.overlap_pairs_with(good)                                 # the good tree is unaffected
    bad.free()
    good.free()


@pytest.mark.parametrize("D,prec", [(3, "f32"), (3, "f64"), (4, "f32"), (4, "f64")])
def test_dev_form_on_a_side_stream_equals_the_host_form(api, D, prec):
    import torch

    F = FT[prec]
    rng = np.random.default_rng(5 + D)
    amn, amx = dimref.scene("random", 20_000, D, F, rng)
    bmn, bmx = dimref.scene("random", 15_000, D, F, rng)
    amx, bmx = (amn + (amx - amn) * 4).astype(F), (bmn + (bmx - bmn) * 4).astype(F)
    a, b = _build(api, D, prec, amn, amx), _build(api, D, prec, bmn, bmx)
    ho, hh = a.overlap_pairs_with(b)
    assert len(hh) > 1000
    dev = torch.device("cuda", 0)
    side = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(side):
        d_off = torch.full((len(amn) + 1,), 7, dtype=torch.int32, device=dev)
        d_hits = torch.full((len(hh),), 7, dtype=torch.int32, device=dev)
        a.ctx.set_stream(side.cuda_stream)
        try:
            a.overlap_pairs_with_dev(b, d_off.data_ptr(), d_hits.data_ptr(), len(hh))
        finally:
            a.ctx.set_stream(None)
        side.synchronize()
    assert d_off.cpu().numpy().view(np.uint32).tobytes() == ho.tobytes()
    assert d_hits.cpu().numpy().view(np.uint32).tobytes() == hh.tobytes()
    a.free()
    b.free()


def test_a_total_above_u32_saturates_the_offsets(api):
    """65 536 identical boxes in A and 65 537 in B: 4 295 032 832 pairs, more than the u32 offsets hold.  The dev form's count
    (cap = 0, no hits) returns BVHGPU_ERR_CAPACITY with that total; row s starts at s * 65 537, saturated at 0xFFFFFFFF."""
    import torch

    from bvh_b200 import capi

    na, nb = 65_536, 65_537
    mn = np.zeros((nb, 3), dtype=np.float32)
    a, b = _build(api, 3, "f32", mn[:na], mn[:na] + 1), _build(api, 3, "f32", mn, mn + 1)
    d_off = torch.zeros(na + 1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    total = C.c_size_t(0)
    st = _fn(a, True)(a._h, b._h, C.c_void_p(d_off.data_ptr()), None, 0, C.byref(total))
    assert st == capi.ERR_CAPACITY and total.value == na * nb == 4_295_032_832
    want = np.minimum(np.arange(na + 1, dtype=np.int64) * nb, U32_MAX)
    want[-1] = U32_MAX
    assert d_off.cpu().numpy().view(np.uint32).tobytes() == want.astype(np.uint32).tobytes()
    a.free()
    b.free()
