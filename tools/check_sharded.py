#!/usr/bin/env python
"""torchrun --nproc-per-node N tools/check_sharded.py : fused P2P sharded traversal == NCCL all-gather path == oracle.
Case 1: sparse cube scene, uneven shards, counts fit one byte.  Case 2: a pile of boxes around the origin: the first rays hit all
of them (> 65 535 hits per ray -> 4-byte counts on the rank that owns them, 1-byte counts elsewhere), also in the compact ray layout.
With >= 2 ranks also the cases of tests/shardref.py over real CUDA IPC: f64 FLAT steps on the "no split wins" scene with new rays
every step (uneven shards, compact layout), and piles at the 2- and 4-byte width thresholds; these print "fused==oracle" only."""
import os, sys, numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
dev = torch.device("cuda", local); torch.cuda.set_device(dev)
dist.init_process_group("nccl", device_id=dev)
from bvh_b200 import api, capi, scenes
from bvh_b200.dist import ShardedTraversal, allgather_csr, shard_range
from oracle import oracle as O
ctx = api.Context(local)
stream = torch.cuda.Stream(dev); torch.cuda.set_stream(stream); ctx.set_stream(stream.cuda_stream)
all_ok = True

def run_case(tag, shapes, allrays, cap, layout):
    global all_ok
    N = len(allrays)
    lo, hi = shard_range(N, rank, world)
    rays = allrays[lo:hi]
    if layout == capi.RAYS_OD:
        od = np.empty((hi - lo, 6), dtype=np.float32); od[:, :3], od[:, 3:] = rays["origin"], rays["direction"]
        d_in = torch.from_numpy(od.reshape(-1)).to(dev)
    else:
        d_in = torch.from_numpy(rays.view(np.uint8).reshape(-1)).to(dev)
    d_rays = torch.from_numpy(rays.view(np.uint8).reshape(-1)).to(dev)
    bvh = api.Bvh.build(shapes, ctx=ctx)
    sh = ShardedTraversal(bvh, hi - lo, cap, ray_layout=layout)
    for it in range(3):                      # several steps: mailbox parity, buffer reuse
        sh.step(d_in.data_ptr(), hi - lo)
    off, hits = sh.fetch()
    d_off = torch.empty(hi - lo + 1, dtype=torch.int32, device=dev); d_hits = torch.empty(cap, dtype=torch.int32, device=dev)
    bvh.traverse_dev(d_rays.data_ptr(), hi - lo, d_off.data_ptr(), d_hits.data_ptr(), cap)
    g_off, g_hits = allgather_csr(d_off, d_hits)
    ok_nccl = np.array_equal(g_off.cpu().numpy().astype(np.uint32), off) and np.array_equal(g_hits.cpu().numpy().view(np.uint32), hits)
    res = O.build(shapes)
    r = O.traverse(res.nodes, shapes, allrays, O.MODE_RECURSIVE, threads=8)
    ok_oracle = np.array_equal(off.astype(np.uint64), r.offsets) and np.array_equal(hits, r.hits)
    print(f"[{tag}] rank {rank}/{world}: fused==nccl {ok_nccl}  fused==oracle {ok_oracle}  total hits {len(hits)}", flush=True)
    all_ok = all_ok and ok_nccl and ok_oracle
    sh.close()
    bvh.free()

# case 1
shapes = scenes.create_n_cubes_aabbs(2000)
oo, dd = scenes.ray_endpoints(200_003, 0)
run_case("cubes", shapes, O.ray_new(oo, dd), 4 * 200_003, capi.RAYS_FULL)
# case 2
n = 70_000
rng = np.random.default_rng(5)
half = rng.uniform(1.0, 2.0, (n, 3))
pile = O.make_aabbs(-half, half)
m = 6_001
origins = rng.uniform(-50, 50, (m, 3)); dirs = rng.uniform(-1, 1, (m, 3))
origins[:24] = rng.uniform(-20, 20, (24, 3)); dirs[:24] = -origins[:24]           # the first 24 rays go through the origin: n hits each
run_case("pile", pile, O.ray_new(origins, dirs), 24 * n + 400_000, capi.RAYS_OD)


def run_steps(tag, shapes, batches, prec, mode, layout):
    """Several steps with new rays each over S.uneven shards: this rank's copy of the global CSR == the oracle after every step."""
    global all_ok
    N = len(batches[0])
    sizes = S.uneven(N, world)
    rb = S.rays_before(sizes)
    wants = [S.oracle_csr(shapes, b, mode, prec) for b in batches]
    bvh = api.Bvh.build(shapes, prec=prec, ctx=ctx)
    sh = ShardedTraversal(bvh, sizes[rank], max(len(w.hits) for w in wants) + 64, ray_layout=layout)
    for k, (rays, want) in enumerate(zip(batches, wants)):
        part = rays[rb[rank]: rb[rank + 1]]
        host = S.od_layout(part) if layout == capi.RAYS_OD else part
        d_in = torch.from_numpy(np.ascontiguousarray(host).view(np.uint8).reshape(-1)).to(dev)
        torch.cuda.synchronize(dev)
        sh.step(d_in.data_ptr(), sizes[rank], mode)
        off, hits = sh.fetch()
        off_w, hits_w = S.global_csr(want.offsets, want.hits)
        ok = np.array_equal(off, off_w) and np.array_equal(hits, hits_w)
        print(f"[{tag}] rank {rank}/{world} step {k + 1}: fused==oracle {ok}  total hits {len(hits)}", flush=True)
        all_ok = all_ok and ok
    sh.close()
    bvh.free()


if world > 1:                    # the cases of the in-process suite need its helpers (tests/); one rank runs the two cases above only
    from tests import shardref as S
    from tests.edge_inputs import edge_ray_batch, edge_scene
    huge = edge_scene("huge", 1500, "f64")
    batches = [edge_ray_batch(huge, 350, "f64", seed)[0] for seed in range(5)] + [S.miss_rays(huge, 2100, "f64", 7)]
    run_steps("f64 flat", huge, batches, "f64", capi.TRAVERSE_FLAT, capi.RAYS_OD)
    for n in (256, 65536):
        steps = [[5, 2048 + 9, 6148], [0, 4099, 6000]]
        run_steps(f"pile {n}", S.pile(n), [S.pile_rays(6149, t, seed=k) for k, t in enumerate(steps)], "f32", capi.TRAVERSE_BVH, capi.RAYS_FULL)
dist.destroy_process_group()
sys.exit(0 if all_ok else 1)
