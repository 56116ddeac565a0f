#!/usr/bin/env python
"""Small workload touching every kernel family once (builders in all strategy combinations, flatten, traversal, queries,
refit / optimize), meant to be run under `compute-sanitizer --tool memcheck|racecheck|initcheck`."""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bvh_b200 import api, capi, scenes
ctx = api.Context.default()
rng = np.random.default_rng(0)
for prec, ncubes in (("f32", 60), ("f32", 700), ("f64", 300)):
    a = scenes.create_n_cubes_aabbs(ncubes, prec)
    for small, sub, gang in ((-1, -1, -1), (0, 0, 0), (1, 0, 1), (0, 1, 1)):
        ctx.set_option("build_small", small); ctx.set_option("build_subtree", sub); ctx.set_option("build_gang", gang)
        for mode in (capi.BUILD_EXACT_SAH, capi.BUILD_LBVH, capi.BUILD_LBVH_TREELET):
            b = api.Bvh.build(a, prec=prec, mode=mode)
            b.flatten()
            b.free()
    ctx.set_option("build_small", -1); ctx.set_option("build_subtree", -1); ctx.set_option("build_gang", -1)
    b = api.Bvh.build(a, prec=prec)
    o, d = scenes.ray_endpoints(4096, prec=prec)
    rays = api.Ray.new(o, d, prec=prec)
    for mode in (capi.TRAVERSE_BVH, capi.TRAVERSE_FLAT):
        off, hits = b.traverse_batch(rays, mode=mode)
    pts = rng.uniform(-120000, 120000, (512, 3))
    for mode in (capi.TRAVERSE_BVH, capi.TRAVERSE_FLAT):
        ns, nd = b.nearest_to_batch(pts, mode=mode)
    coff, cand = b.nearest_candidates(pts)
    qoff, qh = b.query_batch(capi.QUERY_BALL, np.concatenate([pts[:64], np.full((64, 1), 5000.0)], axis=1))
    m = a.copy()
    mv = rng.choice(len(a), len(a) // 10, replace=False)
    dl = rng.uniform(-10, 10, (len(mv), 3)).astype(a["min"].dtype)
    m["min"][mv] += dl; m["max"][mv] += dl
    b.refit(m)
    m["min"][mv] += dl; m["max"][mv] += dl
    print(prec, ncubes, "optimize rebuilt", b.optimize(m, 1.5), "hits", len(hits), "candidates", len(cand))
    # round 2: compact ray layout, update_shapes (incremental), closest hit (both modes), ordered traversal, triangle nearest_to
    off2, hits2 = b.traverse_batch(rays, compact=True)
    mv2 = rng.choice(len(a), max(1, len(a) // 50), replace=False)
    m["min"][mv2] += 3; m["max"][mv2] += 3
    print("  update rebuilt", b.update_shapes(mv2, m, 1.5), b.update_shapes(mv2, m, 0.0))
    from oracle import oracle as O
    _, tris = O.create_n_cubes(ncubes, prec=prec, want_tris=True)
    b.set_triangles(tris)
    cs, cd, _ = b.closest_hit(rays, triangles=True)
    cs2, cd2, _ = b.closest_hit(rays, triangles=False)
    ts_, td_ = b.nearest_triangles_batch(pts[:256])
    b.traverse_ordered(rays[:512], True)
    # any hit: both modes, host form with and without limits, device form with both ray layouts
    ah_t, ah_a = b.any_hit(rays, cd, triangles=True), b.any_hit(rays, cd2 * 2)
    b.any_hit(rays)
    import ctypes as C, torch
    sfx = "f32x3" if prec == "f32" else "f64x3"
    tdt = torch.float32 if prec == "f32" else torch.float64
    d_tm = torch.from_numpy(np.ascontiguousarray(cd)).to("cuda:0"); d_sh = torch.empty(len(rays), dtype=torch.int32, device="cuda:0")
    for lay, src in ((capi.RAYS_FULL, rays), (capi.RAYS_OD, np.ascontiguousarray(np.concatenate([rays["origin"], rays["direction"]], axis=1)))):
        d_r = torch.from_numpy(np.frombuffer(src.tobytes(), dtype=np.uint8).copy()).to("cuda:0"); torch.cuda.synchronize()
        for tri in (0, 1):
            capi.check(getattr(capi.lib(), f"bvhgpu_any_hit_dev_{sfx}")(b._h, C.c_void_p(d_r.data_ptr()), lay, len(rays), C.c_void_p(d_tm.data_ptr()), tri,
                                                                         C.c_void_p(d_sh.data_ptr())))
        ctx.synchronize()
    print("  any hit", int((ah_t != 0xFFFFFFFF).sum()), int((ah_a != 0xFFFFFFFF).sum()))
    # multi hit: both modes, every K bucket, with and without limits, host form with uv and the device form with OD rays
    for k in (1, 5, 9, 17, 33):
        b.multi_hit(rays, k, cd, triangles=True, uv=True); b.multi_hit(rays, k, triangles=False)
    d_ms = torch.empty(len(rays) * 7, dtype=torch.int32, device="cuda:0"); d_md = torch.empty(len(rays) * 7, dtype=tdt, device="cuda:0")
    b.multi_hit_dev(d_r.data_ptr(), len(rays), 7, d_tm.data_ptr(), d_ms.data_ptr(), d_md.data_ptr(), triangles=True, layout=capi.RAYS_OD)
    ctx.synchronize()
    # crossing counts (with and without limits, OD rays on the device), point-in-mesh under both rules, signed distance with closest points
    b.count_hits(rays); b.count_hits(rays, cd)
    b.count_hits_dev(d_r.data_ptr(), len(rays), d_tm.data_ptr(), d_ms.data_ptr(), d_ms.data_ptr() + 4 * len(rays), layout=capi.RAYS_OD)
    cpts = np.concatenate([pts[:200], scenes.create_n_cubes_tris(ncubes, prec).reshape(-1, 12, 9)[:, :, :3].mean(axis=1)[:200]])
    b.contains(cpts, "even_odd"); b.contains(cpts, "nonzero"); b.signed_distance(cpts, closest=True)
    d_cp = torch.from_numpy(np.ascontiguousarray(cpts, dtype=a["min"].dtype)).to("cuda:0")
    b.signed_distance_dev(d_cp.data_ptr(), len(cpts), d_ms.data_ptr(), d_md.data_ptr(), 0, rule="nonzero")
    ctx.synchronize()
    b.free()
# D = 2
from bvh_b200.dtypes import BY_PREC_2D
for prec in ("f32", "f64"):
    a2 = np.zeros(500, dtype=BY_PREC_2D[prec]["aabb"]); mn = rng.uniform(-100, 100, (500, 2)); a2["min"] = mn; a2["max"] = mn + rng.uniform(0, 5, (500, 2))
    b2 = api.Bvh2.build(a2, prec=prec)
    b2.nodes_and_index(); b2.flatten()
    r2 = np.zeros(300, dtype=BY_PREC_2D[prec]["ray"])
    o2 = rng.uniform(-120, 120, (300, 2)); d2 = rng.normal(0, 1, (300, 2)); d2 /= np.linalg.norm(d2, axis=1, keepdims=True)
    r2["origin"], r2["direction"], r2["inv_direction"] = o2, d2, 1.0 / d2
    for mode in (capi.TRAVERSE_BVH, capi.TRAVERSE_FLAT):
        b2.traverse_batch(r2, mode=mode)
    b2.traverse_ordered(r2, True); b2.traverse_ordered(r2, False); _, c2 = b2.closest_hit(r2)
    b2.any_hit(r2); b2.any_hit(r2, np.nextafter(c2, np.inf))
    b2.multi_hit(r2, 3); b2.multi_hit(r2, 40, np.nextafter(c2, np.inf))
    b2.free()
# 4-D ordered traversal, closest hit and any hit (host and device-pointer forms)
from bvh_b200.dtypes import BY_PREC_4D
for prec in ("f32", "f64"):
    a4 = np.zeros(500, dtype=BY_PREC_4D[prec]["aabb"]); mn = rng.uniform(-100, 100, (500, 4)); a4["min"] = mn; a4["max"] = mn + rng.uniform(0, 5, (500, 4))
    b4 = api.Bvh4.build(a4, prec=prec)
    r4 = np.zeros(300, dtype=BY_PREC_4D[prec]["ray"])
    o4 = rng.uniform(-120, 120, (300, 4)); d4 = rng.normal(0, 1, (300, 4)); d4 /= np.linalg.norm(d4, axis=1, keepdims=True)
    r4["origin"], r4["direction"], r4["inv_direction"] = o4, d4, 1.0 / d4
    b4.traverse_ordered(r4, True); b4.traverse_ordered(r4, False); s4, _ = b4.closest_hit(r4)
    import torch
    dr = torch.from_numpy(r4.view(np.uint8)).to("cuda:0"); ds = torch.empty(300, dtype=torch.int32, device="cuda:0")
    dd = torch.empty(300, dtype=torch.float32 if prec == "f32" else torch.float64, device="cuda:0")
    torch.cuda.synchronize()
    b4.closest_hit_dev(dr.data_ptr(), 300, ds.data_ptr(), dd.data_ptr()); ctx.synchronize()
    b4.any_hit(r4); b4.any_hit(r4, np.full(300, 50.0))
    b4.any_hit_dev(dr.data_ptr(), 300, dd.data_ptr(), ds.data_ptr()); b4.any_hit_dev(dr.data_ptr(), 300, 0, ds.data_ptr()); ctx.synchronize()
    b4.multi_hit(r4, 3); b4.multi_hit(r4, 40, np.full(300, 50.0)); b4.multi_hit_dev(dr.data_ptr(), 300, 1, 0, ds.data_ptr(), dd.data_ptr()); ctx.synchronize()
    b4.free()
# self-overlap pairs: host and device forms in D = 2, 3, 4, a short capacity (fetch / retry), an overflow-scale scene
for prec in ("f32", "f64"):
    import torch
    for D, cls in ((2, api.Bvh2), (3, api.Bvh), (4, api.Bvh4)):
        lo = rng.uniform(-50, 50, (800, D))
        bo = np.zeros(len(lo), dtype=(cls._TABLE[prec] if D != 3 else api.BY_PREC[prec])["aabb"])
        bo["min"], bo["max"] = lo, lo + rng.uniform(0, 6, (len(lo), D))
        bt = cls.build(bo, prec=prec)
        po, ph = bt.overlap_pairs()
        bt.overlap_pairs(cap=len(ph) // 2)
        if D != 2:
            d_o = torch.zeros(len(lo) + 1, dtype=torch.int32, device="cuda:0"); d_h = torch.zeros(len(ph), dtype=torch.int32, device="cuda:0")
            bt.overlap_pairs_dev(d_o.data_ptr(), d_h.data_ptr(), len(ph) // 3); bt.overlap_pairs_dev(d_o.data_ptr(), d_h.data_ptr(), len(ph), True)
        bo["min"], bo["max"] = lo * 1e30, lo * 1e30 + 1e29
        bt.free()
        bt = cls.build(bo, prec=prec)
        bt.overlap_pairs()
        print("  overlap", prec, D, len(ph))
        bt.free()
# overlap pairs between two trees: host and device forms in D = 2, 3, 4, a short capacity (fetch / retry), a == b, an overflow-scale B
for prec in ("f32", "f64"):
    import torch
    for D, cls in ((2, api.Bvh2), (3, api.Bvh), (4, api.Bvh4)):
        dt = (cls._TABLE[prec] if D != 3 else api.BY_PREC[prec])["aabb"]
        boxes = []
        for n in (700, 500):
            lo = rng.uniform(-50, 50, (n, D))
            bo = np.zeros(n, dtype=dt)
            bo["min"], bo["max"] = lo, lo + rng.uniform(0, 6, (n, D))
            boxes.append(bo)
        ta, tb = cls.build(boxes[0], prec=prec), cls.build(boxes[1], prec=prec)
        po, ph = ta.overlap_pairs_with(tb)
        ta.overlap_pairs_with(tb, cap=len(ph) // 2)
        ta.overlap_pairs_with(ta)
        if D != 2:
            d_o = torch.zeros(len(boxes[0]) + 1, dtype=torch.int32, device="cuda:0"); d_h = torch.zeros(len(ph), dtype=torch.int32, device="cuda:0")
            ta.overlap_pairs_with_dev(tb, d_o.data_ptr(), d_h.data_ptr(), len(ph) // 3); ta.overlap_pairs_with_dev(tb, d_o.data_ptr(), d_h.data_ptr(), len(ph), True)
        tb.free()
        boxes[1]["min"], boxes[1]["max"] = boxes[1]["min"] * 1e30, boxes[1]["min"] * 1e30 + 1e29
        tb = cls.build(boxes[1], prec=prec)
        ta.overlap_pairs_with(tb)
        print("  overlap_trees", prec, D, len(ph))
        ta.free()
        tb.free()
# triangle pairs (3-D): self (both skip_shared values) and between trees, host and device forms, a short capacity (fetch), a == b,
# refused without triangles; a soup on a half-integer grid puts pairs on the exact coplanar path
for prec in ("f32", "f64"):
    import torch
    F = api.BY_PREC[prec]["scalar"]
    tris = []
    for n in (600, 450):
        c = rng.integers(0, 10, size=(n, 1, 3))
        tris.append(((2 * c + rng.integers(0, 5, size=(n, 3, 3))) / 2).astype(F))
    ts = []
    for t in tris:
        bo = np.zeros(len(t), dtype=api.BY_PREC[prec]["aabb"])
        bo["min"], bo["max"] = t.min(axis=1), t.max(axis=1)
        ts.append(api.Bvh.build(bo, prec=prec))
    try:
        ts[0].triangle_pairs()
    except capi.BvhGpuError:
        pass
    for b, t in zip(ts, tris):
        b.set_triangles(t)
    po, ph = ts[0].triangle_pairs(skip_shared=False)
    ts[0].triangle_pairs(skip_shared=True)
    ts[0].triangle_pairs(skip_shared=False, cap=len(ph) // 2)
    qo, qh = ts[0].triangle_pairs_with(ts[1])
    ts[0].triangle_pairs_with(ts[0])
    d_o = torch.zeros(len(tris[0]) + 1, dtype=torch.int32, device="cuda:0"); d_h = torch.zeros(max(len(ph), len(qh), 1), dtype=torch.int32, device="cuda:0")
    ts[0].triangle_pairs_dev(d_o.data_ptr(), d_h.data_ptr(), len(ph) // 3, skip_shared=False)
    ts[0].triangle_pairs_with_dev(ts[1], d_o.data_ptr(), d_h.data_ptr(), len(qh), True)
    print("  triangle_pairs", prec, len(ph), len(qh))
    for b in ts:
        b.free()
# host path on a batch large enough to be chunked (under the sanitizer the library takes the copy-then-walk form; forced streaming too)
a = scenes.create_n_cubes_aabbs(300)
b = api.Bvh.build(a)
o, d = scenes.ray_endpoints(300_000)
rays = api.Ray.new(o, d)
for opt in (-1, 1):
    ctx.set_option("traverse_stream", opt)
    b.traverse_batch(rays, compact=True)
ctx.set_option("traverse_stream", -1)
# the sharded step with one rank (every exchange kernel; gloo only swaps the handles)
import torch.distributed as dist, torch
os.environ.setdefault("MASTER_ADDR", "127.0.0.1"); os.environ.setdefault("MASTER_PORT", "29671")
dist.init_process_group("gloo", rank=0, world_size=1)
from bvh_b200.dist import ShardedTraversal
d_rays = torch.from_numpy(rays.view(np.uint8).reshape(-1)).to("cuda:0")
sh = ShardedTraversal(b, len(rays), 4 * len(rays))
for _ in range(3):
    sh.step(d_rays.data_ptr(), len(rays))
goff, ghits = sh.fetch()
print("  sharded hits", len(ghits))
sh.close()
dist.destroy_process_group()
b.free()
print("sanitize targets done")
