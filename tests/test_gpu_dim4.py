"""Bvh<T,4> on the device (dim4.cu): build, nodes, flatten and both traversals against the 4-D restatement in tests/pyref.py node for
node, the large-range builder against the bit-exact 3-D builder through a constant fourth axis, large traversals against brute force,
and the behaviour of the entry points."""
import ctypes as C

import numpy as np
import pytest

from tests import pyref

pytestmark = pytest.mark.gpu
U32_MAX = 0xFFFFFFFF


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A

    return A


def _F(prec):
    return np.float32 if prec == "f32" else np.float64


def _scene4(kind, n, prec, rng):
    from bvh_b200.dtypes import BY_PREC_4D

    F = _F(prec)
    a = np.zeros(n, dtype=BY_PREC_4D[prec]["aabb"])
    if kind == "random":
        mn = rng.uniform(-100, 100, (n, 4))
        a["min"], a["max"] = mn, mn + rng.uniform(0, 8, (n, 4)) ** 2 / 8
    elif kind == "coincident":                               # zero centroid extent: the halving branch all the way down
        a["min"], a["max"] = [1, 2, 3, 4], [1, 2, 3, 4]
    elif kind.startswith("axis"):                            # all centres on one axis
        k = int(kind[-1])
        c = np.zeros((n, 4)); c[:, k] = rng.uniform(-50, 50, n)
        a["min"], a["max"] = c - 0.5, c + 0.5
    elif kind == "peel":                                     # geometric centroids: large ranges split a few shapes off per level
        c = np.zeros((n, 4)); c[:, 0] = 1.12 ** np.arange(n); c[:, 1:] = rng.uniform(-1, 1, (n, 3))
        a["min"], a["max"] = c, c
    elif kind == "overflow":                                 # f32 surface areas overflow: empty child boxes
        c = rng.uniform(-3e19, 3e19, (n, 4))
        a["min"], a["max"] = c - 1e18, c + 1e18
    return a


def _as_pyref(a, F):
    return [{"min": [F(v) for v in r["min"]], "max": [F(v) for v in r["max"]]} for r in a]


def _rays4(a, m, prec, rng, axis_aligned=True):
    from bvh_b200.dtypes import BY_PREC_4D

    F = _F(prec)
    n = len(a)
    org = rng.uniform(-120, 120, (m, 4)); tgt = rng.uniform(-100, 100, (m, 4))
    if n:
        lo, hi = a["min"].min(axis=0).astype(np.float64), a["max"].max(axis=0).astype(np.float64)
        ok = np.all(np.isfinite(lo)) and np.all(hi - lo < 1e30)
        if ok:
            span = np.maximum(hi - lo, 1.0)
            org = lo - 0.2 * span + rng.uniform(0, 1.4, (m, 4)) * span
            tgt = lo + rng.uniform(0, 1, (m, 4)) * span
    dirs = tgt - org
    if axis_aligned and n:
        for i in range(min(64, m)):                          # along each of the 4 axes, starting on box faces (0 * inf = NaN rule)
            dirs[i] = 0.0
            dirs[i, i % 4] = 1.0 if (i // 4) % 2 else -1.0
            if i % 8 < 4:
                org[i] = a["min"][rng.integers(0, n)]
    rays = np.zeros(m, dtype=BY_PREC_4D[prec]["ray"])
    prs = [pyref.ray_new(F, org[i], dirs[i]) for i in range(m)]
    for i, (o, d, inv) in enumerate(prs):
        rays["origin"][i], rays["direction"][i], rays["inv_direction"][i] = o, d, inv
    return rays, prs


def _check_against_pyref(api, a, prec, rng, m=200):
    F = _F(prec)
    pa = _as_pyref(a, F)
    want_nodes, want_index = pyref.build(pa, F)
    bvh = api.Bvh4.build(a, prec=prec)
    nodes, index = bvh.nodes_and_index()
    assert list(index) == list(want_index)
    for i, w in enumerate(want_nodes):
        if w[0] == "leaf":
            assert (nodes["parent"][i], nodes["child_l"][i], nodes["child_r"][i], nodes["shape"][i]) == (w[1], U32_MAX, U32_MAX, w[2]), i
            assert np.all(nodes["l_aabb"]["min"][i] == np.inf) and np.all(nodes["r_aabb"]["max"][i] == -np.inf)
        else:
            assert (nodes["parent"][i], nodes["child_l"][i], nodes["child_r"][i]) == (w[1], w[2], w[3]), i
            for side, box in (("l_aabb", w[4]), ("r_aabb", w[5])):
                assert np.array_equal(nodes[side]["min"][i], np.array(box[0], dtype=F)), (i, side)
                assert np.array_equal(nodes[side]["max"][i], np.array(box[1], dtype=F)), (i, side)
    flat = bvh.flatten()
    wflat = pyref.flatten(want_nodes)
    assert len(flat) == len(wflat)
    for i, (box, entry, exit_, shape) in enumerate(wflat):
        assert (flat["entry_index"][i], flat["exit_index"][i], flat["shape_index"][i]) == (entry, exit_, shape), i
        if box is not None:
            assert np.array_equal(flat["aabb"]["min"][i], np.array(box[0], dtype=F)) and np.array_equal(flat["aabb"]["max"][i], np.array(box[1], dtype=F))
        else:
            assert np.all(flat["aabb"]["min"][i] == np.inf) and np.all(flat["aabb"]["max"][i] == -np.inf)
    from bvh_b200 import capi

    rays, prs = _rays4(a, m, prec, rng)
    off, hits = bvh.traverse_batch(rays, mode=capi.TRAVERSE_BVH)
    off2, hits2 = bvh.traverse_batch(rays, mode=capi.TRAVERSE_FLAT)
    for i in range(m):
        ray = (prs[i][0], prs[i][2])
        want = pyref.traverse_recursive(want_nodes, pa, ray, F)
        assert hits[off[i]:off[i + 1]].tolist() == want, i
        # FLAT visits the same records and re-tests the shape's AABB at every reached leaf (flat_bvh.rs:396-431)
        want_flat = [s for s in want if pyref.hit(F, ray, pa[s]["min"], pa[s]["max"])]
        assert hits2[off2[i]:off2[i + 1]].tolist() == want_flat, i
    bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("kind,n", [("random", 0), ("random", 1), ("random", 2), ("random", 33), ("random", 700), ("coincident", 300),
                                    ("axis0", 200), ("axis1", 200), ("axis2", 200), ("axis3", 200), ("peel", 300), ("overflow", 400),
                                    ("random", 257), ("random", 513), ("random", 16385), ("coincident", 5000)])
def test_four_dimensional_bvh_matches_the_4d_restatement(api, kind, n, prec):
    rng = np.random.default_rng(n * 11 + len(kind))
    a = _scene4(kind, n, prec, rng)
    _check_against_pyref(api, a, prec, rng)


def _lift(a3, prec, c=1.5):
    from bvh_b200.dtypes import BY_PREC_4D

    a4 = np.zeros(len(a3), dtype=BY_PREC_4D[prec]["aabb"])
    a4["min"][:, :3], a4["max"][:, :3] = a3["min"], a3["max"]
    a4["min"][:, 3], a4["max"][:, 3] = c, c
    return a4


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("scene", ["cubes", "random_1m"])
def test_large_4d_builds_equal_the_3d_builder_through_a_constant_fourth_axis(api, scene, prec):
    """w = [c, c] never changes the tree (test_dim4_cpu.py), so the 4-D builder's large-range path must reproduce the bit-exact 3-D
    builder node for node: create_n_cubes(10 000) (120 000 triangles) and 1.2 M random boxes."""
    from bvh_b200 import scenes
    from bvh_b200.dtypes import BY_PREC

    F = _F(prec)
    if scene == "cubes":
        a3 = scenes.create_n_cubes_aabbs(10000, prec)
    else:
        rng = np.random.default_rng(12)
        a3 = np.zeros(1_200_000, dtype=BY_PREC[prec]["aabb"])
        mn = rng.uniform(-1000, 1000, (len(a3), 3))
        a3["min"], a3["max"] = mn, mn + rng.uniform(0, 3, (len(a3), 3))
    b3 = api.Bvh.build(a3, prec=prec)
    n3, i3 = b3.nodes, b3.node_index
    b4 = api.Bvh4.build(_lift(a3, prec), prec=prec)
    n4, i4 = b4.nodes_and_index()
    assert np.array_equal(i4, i3)
    for f in ("parent", "child_l", "child_r", "shape"):
        assert np.array_equal(n4[f], n3[f]), f
    for side in ("l_aabb", "r_aabb"):
        for mm in ("min", "max"):
            assert np.array_equal(n4[side][mm][:, :3], n3[side][mm]), (side, mm)
    leaf = n3["child_l"] == U32_MAX
    for side in ("l_aabb", "r_aabb"):
        assert np.all(n4[side]["min"][leaf, 3] == np.inf) and np.all(n4[side]["max"][leaf, 3] == -np.inf)
        assert np.all(n4[side]["min"][~leaf, 3] == F(1.5)) and np.all(n4[side]["max"][~leaf, 3] == F(1.5))
    b3.free(); b4.free()


def _random_rays_torch(m, prec, seed, lo=-1100.0, hi=1100.0):
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    dt = torch.float32 if prec == "f32" else torch.float64
    o = (torch.rand((m, 4), generator=g, device="cuda", dtype=torch.float64) * (hi - lo) + lo).to(dt)
    d = (torch.rand((m, 4), generator=g, device="cuda", dtype=torch.float64) * 2 - 1).to(dt)
    d = d / torch.sqrt((d * d).sum(dim=1, keepdim=True))
    inv = 1 / d
    return torch.cat([o, d, inv], dim=1).contiguous()          # bvh_ray4 layout: origin, direction, inv_direction


def test_large_traversal_equals_brute_force_in_dfs_order(api):
    """120 000 random 4-D boxes, 16 384 random rays, f32 and f64: every ray's hit list is the set of shape boxes it hits (brute force
    on the device, same T, separate sub and mul), sorted by node index -- the DFS order."""
    import torch
    from bvh_b200 import capi
    from bvh_b200.dtypes import BY_PREC_4D

    for prec in ("f32", "f64"):
        dt = torch.float32 if prec == "f32" else torch.float64
        rng = np.random.default_rng(120)
        n = 120_000
        a = np.zeros(n, dtype=BY_PREC_4D[prec]["aabb"])
        mn = rng.uniform(-1000, 1000, (n, 4))
        a["min"], a["max"] = mn, mn + rng.uniform(0, 60, (n, 4))
        bvh = api.Bvh4.build(a, prec=prec)
        _, node_index = bvh.nodes_and_index()
        m = 16384
        rays = _random_rays_torch(m, prec, 7)
        host_rays = rays.cpu().numpy().view(BY_PREC_4D[prec]["ray"]).reshape(-1)
        bmin = torch.from_numpy(np.ascontiguousarray(a["min"])).to("cuda", dt)
        bmax = torch.from_numpy(np.ascontiguousarray(a["max"])).to("cuda", dt)
        ni = torch.from_numpy(node_index.astype(np.int64)).cuda()
        for mode in (capi.TRAVERSE_BVH, capi.TRAVERSE_FLAT):
            off, hits = bvh.traverse_batch(host_rays, mode=mode)
            off_t, hits_t = torch.from_numpy(off.astype(np.int64)).cuda(), torch.from_numpy(hits.astype(np.int64)).cuda()
            for r0 in range(0, m, 64):
                o, inv = rays[r0:r0 + 64, None, 0:4], rays[r0:r0 + 64, None, 8:12]
                l = torch.mul(torch.sub(bmin[None], o), inv)
                r = torch.mul(torch.sub(bmax[None], o), inv)
                nan = torch.isnan(l).any(dim=2) | torch.isnan(r).any(dim=2)
                tmin = torch.minimum(l, r).amax(dim=2)
                tmax = torch.maximum(l, r).amin(dim=2)
                hit = ~nan & (tmax >= torch.clamp(tmin, min=0))
                ray_i, shape = hit.nonzero(as_tuple=True)
                order = torch.argsort((ray_i + r0) * (1 << 32) + ni[shape])
                want = shape[order]
                got = hits_t[off_t[r0]:off_t[min(r0 + 64, m)]]
                assert torch.equal(got, want), (prec, mode, r0)
                cnt = torch.bincount(ray_i, minlength=min(64, m - r0))
                assert torch.equal(off_t[r0 + 1:r0 + 65] - off_t[r0:r0 + 64], cnt), (prec, mode, r0)
        bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_capacity_retry_and_device_pointers(api, prec):
    import torch
    from bvh_b200 import capi
    from bvh_b200.dtypes import BY_PREC_4D

    rng = np.random.default_rng(5)
    a = _scene4("random", 3000, prec, rng)
    bvh = api.Bvh4.build(a, prec=prec)
    rays, _ = _rays4(a, 2000, prec, rng)
    off, hits = bvh.traverse_batch(rays)                       # retries with cap = *total when the first guess is short
    assert len(hits) == off[-1] and len(hits) > 0
    fn = getattr(capi.lib(), f"bvhgpu_traverse_{BY_PREC_4D[prec]['suffix']}")
    off2 = np.zeros(len(rays) + 1, dtype=np.uint32)
    small = np.zeros(7, dtype=np.uint32)
    total = C.c_size_t(0)
    st = fn(bvh._h, capi.TRAVERSE_BVH, rays.ctypes.data_as(C.c_void_p), len(rays), off2.ctypes.data_as(C.c_void_p),
            small.ctypes.data_as(C.c_void_p), 7, C.byref(total))
    assert st == capi.ERR_CAPACITY and total.value == len(hits) and np.array_equal(off2, off)
    hits_full = np.zeros(total.value, dtype=np.uint32)
    st = fn(bvh._h, capi.TRAVERSE_BVH, rays.ctypes.data_as(C.c_void_p), len(rays), off2.ctypes.data_as(C.c_void_p),
            hits_full.ctypes.data_as(C.c_void_p), total.value, C.byref(total))
    assert st == capi.OK and np.array_equal(hits_full, hits)
    # device pointers: the same CSR; with want_total = False the call does not wait for the stream
    ctx = bvh.ctx
    d_rays = torch.from_numpy(rays.view(np.uint8).copy()).cuda()
    d_off = torch.zeros(len(rays) + 1, dtype=torch.int32, device="cuda")
    d_hits = torch.zeros(len(hits), dtype=torch.int32, device="cuda")
    for mode in (capi.TRAVERSE_BVH, capi.TRAVERSE_FLAT):
        want_off, want_hits = bvh.traverse_batch(rays, mode=mode)
        tot = bvh.traverse_dev(d_rays.data_ptr(), len(rays), d_off.data_ptr(), d_hits.data_ptr(), len(hits), mode=mode, want_total=True)
        assert tot == len(want_hits)
        assert np.array_equal(d_off.cpu().numpy().view(np.uint32), want_off) and np.array_equal(d_hits[:tot].cpu().numpy().view(np.uint32), want_hits)
    s = torch.cuda.Stream()
    ctx.set_stream(s.cuda_stream)
    try:
        d_off.zero_(); d_hits.zero_()
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(200_000_000)                     # keeps the stream busy for ~0.1 s
        bvh.traverse_dev(d_rays.data_ptr(), len(rays), d_off.data_ptr(), d_hits.data_ptr(), 5, want_total=False)
        assert not s.query()                                   # returned while the stream was still running
        s.synchronize()
    finally:
        ctx.set_stream(None)
    assert np.array_equal(d_off.cpu().numpy().view(np.uint32), off)
    assert np.array_equal(d_hits[:5].cpu().numpy().view(np.uint32), hits[:5]) and int(d_hits[5:].abs().sum()) == 0   # beyond cap: dropped
    bvh.free()


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_bad_input_small_trees_and_determinism(api, prec):
    from bvh_b200 import capi
    from bvh_b200.dtypes import BY_PREC_4D

    d = BY_PREC_4D[prec]
    rng = np.random.default_rng(9)
    a = _scene4("random", 5000, prec, rng)
    bad = a.copy()
    bad["max"][4321, 3] = np.nan
    with pytest.raises(capi.BvhGpuError) as e:
        api.Bvh4.build(bad, prec=prec)
    assert e.value.status == capi.ERR_NAN
    for mode in (capi.BUILD_LBVH, capi.BUILD_LBVH_TREELET):
        with pytest.raises(capi.BvhGpuError) as e:
            api.Bvh4.build(a, prec=prec, mode=mode)
        assert e.value.status == capi.ERR_UNSUPPORTED and "EXACT_SAH" in str(e.value)
    h = C.c_void_p()
    assert getattr(capi.lib(), f"bvhgpu_build_{d['suffix']}")(api.Context.default()._h, None, 3, 0, C.byref(h)) == capi.ERR_INVALID
    # n = 0: empty tree, no flat nodes, no hits; n = 1: a root leaf whose box is tested (bvh_node.rs:314)
    empty = api.Bvh4.build(a[:0], prec=prec)
    assert getattr(capi.lib(), f"bvhgpu_tree_num_shapes_{d['suffix']}")(empty._h) == 0
    assert len(empty.flatten()) == 0
    rays, _ = _rays4(a, 100, prec, rng)
    off, hits = empty.traverse_batch(rays)
    assert not off.any() and len(hits) == 0
    one = api.Bvh4.build(a[:1], prec=prec)
    nodes, idx = one.nodes_and_index()
    assert (nodes["parent"][0], nodes["child_l"][0], nodes["child_r"][0], nodes["shape"][0]) == (0, U32_MAX, U32_MAX, 0) and idx[0] == 0
    fl = one.flatten()
    assert len(fl) == 1 and (fl["entry_index"][0], fl["exit_index"][0], fl["shape_index"][0]) == (U32_MAX, 1, 0)
    F = _F(prec)
    pa = _as_pyref(a[:1], F)
    rays1, prs1 = _rays4(a[:1], 100, prec, np.random.default_rng(9))
    off, hits = one.traverse_batch(rays1)
    for i in range(100):
        assert hits[off[i]:off[i + 1]].tolist() == pyref.traverse_recursive([("leaf", 0, 0)], pa, (prs1[i][0], prs1[i][2]), F)
    empty.free(); one.free()
    # two builds of the same input are byte-identical
    big = _scene4("random", 50_000, prec, rng)
    n1, i1 = api.Bvh4.build(big, prec=prec).nodes_and_index()
    n2, i2 = api.Bvh4.build(big, prec=prec).nodes_and_index()
    assert n1.tobytes() == n2.tobytes() and np.array_equal(i1, i2)


def test_device_memory_returns_to_its_level(api):
    import torch

    rng = np.random.default_rng(3)
    a = _scene4("random", 20_000, "f32", rng)
    rays, _ = _rays4(a, 4096, "f32", rng)

    def rnd():
        b = api.Bvh4.build(a, prec="f32")
        b.flatten()
        b.traverse_batch(rays)
        b.free()

    rnd()
    api.Context.default().synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(20):
        rnd()
    api.Context.default().synchronize()
    assert free0 - torch.cuda.mem_get_info()[0] < 16 << 20
