"""The fused multi-GPU traversal step (bvhgpu_traverse_sharded_dev_f32x3 / _f64x3) at 1 to 8 ranks, run in one process on one GPU by
tests/shardref.VirtualShards: every rank's global offsets and hit lists after every step == the oracle's CSR of the concatenated
batch (O.traverse, MODE_RECURSIVE for BVH, MODE_FLAT for FLAT), with new rays every step, all-miss steps, steps where one rank has
all the hits, a straggling rank, each count width at its thresholds (the staging read back byte for byte), shard sizes and offsets at
the tile and quad edges, hit pieces shorter than a quad, a capacity below the total, and the argument checks that must fail before
anything is enqueued.  Every buffer carries a canary guard that must survive every step.
Run on an H100:  python -m pytest tests/test_gpu_sharded.py -m gpu"""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O
from tests import shardref as S
from tests.edge_inputs import edge_ray_batch, edge_scene

pytestmark = pytest.mark.gpu
BVH, FLAT = 0, 1
FULL, OD = 0, 1


@pytest.fixture(scope="module")
def capi():
    from bvh_b200 import capi as c

    return c


def _check_step(vs, want, what):
    """Every rank's global CSR == want, every guard intact, and the step's mailbox words in every rank's mailbox."""
    vs.synchronize()
    off_w, hits_w = S.global_csr(want.offsets, want.hits)
    totals = [int(want.offsets[b] - want.offsets[a]) for a, b in zip(S.rays_before(vs.sizes)[:-1], S.rays_before(vs.sizes)[1:])]
    for r in range(vs.W):
        off, hits = vs.fetch(r)
        assert np.array_equal(off, off_w), f"{what}: offsets of rank {r}/{vs.W}, first bad ray {np.flatnonzero(off != off_w)[:5]}"
        assert np.array_equal(hits, hits_w), f"{what}: hits of rank {r}/{vs.W}, first bad slot {np.flatnonzero(hits != hits_w)[:5]}"
        box = vs.mailbox(r)
        for word, v in S.mailbox_words(vs.seq, totals).items():
            assert int(box[word]) == v, f"{what}: mailbox word {word} of rank {r}"
    assert vs.guards_intact(), what


# ---- the matrix: world sizes x precision x mode x ray layout, several steps each ---------------------------------------------
@pytest.mark.parametrize("layout", [FULL, OD], ids=["full", "od"])
@pytest.mark.parametrize("mode", [BVH, FLAT], ids=["bvh", "flat"])
@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("W", [1, 2, 3, 5, 8])
def test_steps_match_the_oracle(capi, W, prec, mode, layout):
    """Five steps with new rays each (both staging halves and both mailbox parities reused with new data), one step in which every
    ray misses, one in which only one rank has hits; a rank held back before three of the steps.  On the "no split wins" scene, where
    BVH and FLAT semantics differ."""
    shapes = edge_scene("huge", 1500, prec)
    nodes = O.build(shapes, prec).nodes
    flat = O.flatten(nodes, prec)
    oracle = (lambda rays: O.traverse(nodes, shapes, rays, O.MODE_RECURSIVE, prec, threads=8)) if mode == BVH else \
             (lambda rays: O.traverse(flat, shapes, rays, O.MODE_FLAT, prec, threads=8))
    batches = [edge_ray_batch(shapes, 350, prec, seed)[0] for seed in range(5)]
    ng = len(batches[0])
    sizes = S.uneven(ng, W)
    if W > 1:
        assert any(int(b) % 4 for b in S.rays_before(sizes)[1:-1])
    rb = S.rays_before(sizes)
    batches.append(S.miss_rays(shapes, ng, prec, 7))
    lone = W // 2                                       # only this rank's rays hit
    one = S.miss_rays(shapes, ng, prec, 8)
    one[rb[lone]: rb[lone + 1]] = batches[0][rb[lone]: rb[lone + 1]]
    batches.append(one)
    wants = [oracle(b) for b in batches]
    if mode == FLAT:
        other = O.traverse(nodes, shapes, batches[0], O.MODE_RECURSIVE, prec, threads=8)
        assert not np.array_equal(other.offsets, wants[0].offsets)     # the two modes really differ on this scene
    assert len(wants[5].hits) == 0
    per_rank = np.diff(wants[6].offsets.astype(np.int64)[rb])
    assert per_rank[lone] > 0 and per_rank.sum() == per_rank[lone]
    assert len({len(w.hits) for w in wants[:5]}) > 1                   # new data every step, not the same totals
    cap = max(len(w.hits) for w in wants) + 64
    vs = S.VirtualShards(shapes, sizes, cap, prec, layout, mode)
    try:
        vs.warm_up(vs.upload(batches[0]))
        for k, (rays, want) in enumerate(zip(batches, wants)):
            d_rays = vs.upload(rays)
            vs.step(d_rays, straggler=(k % W) if k in (1, 3, 6) else None)
            _check_step(vs, want, f"W={W} {prec} mode {mode} layout {layout} step {k + 1}")
        for r in range(W):                                             # the trace ring: one record per step, at its seq
            tr = vs.trace(r)
            assert sorted(tr) == list(range(1, vs.seq + 1)) and all(tr[s] == s for s in tr)
    finally:
        vs.close()


# ---- count widths at their thresholds -------------------------------------------------------------------------------------------


@pytest.mark.parametrize("n", [255, 256, 65535, 65536])
def test_count_widths_at_their_thresholds(capi, n):
    """A pile of n boxes around the origin: rays through the origin hit exactly n, the rest 0, so the largest count of a tile sits
    exactly on a width threshold.  Three ranks (4099, 2049, 1 rays: 3 + 2 + 1 tiles), widths mixed within rank 0 (a tile without
    origin rays keeps width 1), two steps with the origin rays in other places.  The last step's staging half of every rank ==
    tests/shardref's image byte for byte (counts in the tile's width, tile table), and the CSR == the oracle."""
    shapes = S.pile(n)
    nodes = O.build(shapes).nodes
    sizes = [4099, 2049, 1]
    ng = sum(sizes)
    steps = [[5, 4096 + 1, 4099 + 2048, ng - 1], [0, 2047, 4098, 4099 + 100, ng - 1]]
    vs = S.VirtualShards(shapes, sizes, n * 6 + 64, "f32", FULL, BVH)
    try:
        for k, through in enumerate(steps):
            rays = S.pile_rays(ng, through, seed=k)
            want = O.traverse(nodes, shapes, rays, O.MODE_RECURSIVE, threads=8)
            counts = np.diff(want.offsets.astype(np.int64))
            assert sorted(set(counts.tolist())) == [0, n] and np.array_equal(np.flatnonzero(counts), sorted(through))
            d_rays = vs.upload(rays)
            if k == 0:
                vs.warm_up(d_rays)
            vs.step(d_rays)
            _check_step(vs, want, f"pile {n} step {k + 1}")
        widths = [w for *_x, w, _o in S.tiles(sizes, counts)]
        assert widths[1] == 1 and S.width(n) in widths
        img, written = S.staging_image(sizes, counts)
        for r in range(vs.W):
            got = vs.staging(r)[: len(img)]
            bad = np.flatnonzero((got != img) & written)
            assert len(bad) == 0, f"rank {r}: staging differs at bytes {bad[:8]}"
    finally:
        vs.close()


# ---- shard sizes and offsets at the tile and quad edges, short hit pieces --------------------------------------------------


EDGE_SPLITS = [[1], [7], [2047], [2048], [2049], [4099],
               [4099, 1, 2049, 7, 2048, 2047],
               [7, 2047, 1, 4099, 2049, 2048],
               [2049, 2049, 2049],
               [1, 1, 1, 1, 1, 1, 1, 4099],
               [4099, 1, 1, 1, 1, 1, 1, 1],
               [3, 2046, 5, 2050, 6, 2047, 9, 2]]


@pytest.mark.parametrize("sizes", EDGE_SPLITS, ids=lambda s: "-".join(map(str, s)))
def test_shard_edges_and_short_pieces(capi, sizes):
    shapes = S.line_scene()
    nodes = O.build(shapes).nodes
    starts = S.rays_before(sizes)[1:-1]
    if len(sizes) > 1:
        assert any(int(s) % 4 for s in starts)
    batches = [S.line_rays(sizes, seed) for seed in range(3)]
    wants = [O.traverse(nodes, shapes, b, O.MODE_RECURSIVE, threads=8) for b in batches]
    assert all(np.max(np.diff(w.offsets.astype(np.int64))) == 1 for w in wants)
    vs = S.VirtualShards(shapes, sizes, max(len(w.hits) for w in wants) + 8, "f32", FULL, BVH)
    try:
        for k, (rays, want) in enumerate(zip(batches, wants)):
            d_rays = vs.upload(rays)
            if k == 0:
                vs.warm_up(d_rays)
            vs.step(d_rays, straggler=len(sizes) - 1 if k == 1 and len(sizes) > 1 else None)
            _check_step(vs, want, f"sizes {sizes} step {k + 1}")
    finally:
        vs.close()


# ---- capacity below the total ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("short", [1, 5, "half"])
def test_capacity_below_the_total(capi, short):
    """cap < total: the hits [0, cap) of every rank == the oracle's prefix, nothing lands at or past cap (the guard behind the
    buffer), the offsets are still exact, and the fetch raises ERR_CAPACITY."""
    sizes = [2049, 3, 4099]
    shapes = S.line_scene()
    rays = S.line_rays(sizes, 11)
    want = O.traverse(O.build(shapes).nodes, shapes, rays, O.MODE_RECURSIVE, threads=8)
    total = len(want.hits)
    cap = total // 2 + 3 if short == "half" else total - short
    vs = S.VirtualShards(shapes, sizes, cap, "f32", FULL, BVH)
    try:
        d_rays = vs.upload(rays)
        vs.warm_up(d_rays)
        for _ in range(2):
            vs.step(d_rays)
            vs.synchronize()
            off_w, hits_w = S.global_csr(want.offsets, want.hits)
            for r in range(vs.W):
                assert np.array_equal(vs.offsets(r), off_w)
                assert np.array_equal(vs.hits(r), hits_w[:cap])
                with pytest.raises(capi.BvhGpuError) as e:
                    vs.fetch(r)
                assert e.value.status == capi.ERR_CAPACITY
            assert vs.guards_intact()
    finally:
        vs.close()


# ---- argument checks before any launch -------------------------------------------------------------------------------------
def _bad_shards(capi, good, nrays):
    def mod(**kw):
        s = capi.Shard.from_buffer_copy(good)
        for k, v in kw.items():
            if isinstance(v, tuple):
                getattr(s, k)[v[0]] = v[1]
            else:
                setattr(s, k, v)
        return s
    return {"seq 0": mod(seq=0), "ray_layout 2": mod(ray_layout=2), "ray_layout -1": mod(ray_layout=-1),
            "world 0": mod(world=0), "world 9": mod(world=9), "rank = world": mod(rank=good.world), "rank -1": mod(rank=-1),
            "null offsets": mod(offsets=None), "null peer counts": mod(peer_counts=(1, None)), "null peer hits": mod(peer_hits=(1, None)),
            "null peer mailbox": mod(peer_mailbox=(0, None)), "null own counts": mod(peer_counts=(good.rank, None)),
            "shard_rays[rank] != nrays": mod(shard_rays=(good.rank, nrays + 1)), "empty peer shard": mod(shard_rays=(1, 0)),
            "2^31 rays": mod(shard_rays=(1, 0x7FFFFFFF))}


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_bad_shards_fail_before_any_launch(capi, prec):
    """Every malformed shard returns ERR_INVALID and enqueues nothing (ctx.launch_count() unchanged), on a tree whose traversal
    records are not built yet as well as on a warmed one; a good step afterwards is still exact."""
    shapes = S.line_scene(prec=prec)
    sizes = [300, 301]
    rays = S.line_rays(sizes, 3, prec)
    want = O.traverse(O.build(shapes, prec).nodes, shapes, rays, O.MODE_RECURSIVE, prec, threads=8)
    vs = S.VirtualShards(shapes, sizes, len(want.hits) + 8, prec, FULL, BVH)
    try:
        d_rays = vs.upload(rays)
        for warmed in (False, True):
            if warmed:
                vs.warm_up(d_rays)
            for r in range(vs.W):
                good = vs.shards[r]
                good.seq = vs.seq + 1
                for name, bad in _bad_shards(capi, good, sizes[r]).items():
                    before = vs.ctxs[r].launch_count()
                    st = vs.fn(vs.bvhs[r]._h, BVH, C.c_void_p(d_rays[r].data_ptr()), sizes[r], C.byref(bad))
                    assert st == capi.ERR_INVALID, (name, st)
                    assert vs.ctxs[r].launch_count() == before, name
        vs.synchronize()
        vs.step(d_rays)
        _check_step(vs, want, "after the refused calls")
    finally:
        vs.close()
