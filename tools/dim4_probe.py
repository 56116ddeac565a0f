#!/usr/bin/env python
"""D = 4 timings (DESIGN.md section 5): the exact 4-D build of 120 k and 1.2 M shapes (f32 and f64) next to the 3-D exact build of the
same scenes with w = [1.5, 1.5] dropped, and the device-resident 4-D traversal of 1 M random rays over a 120 k-shape random 4-D scene
next to the 3-D plain persistent walk (traverse_top = 0) on config 2 (create_n_cubes(10 000), 1 M create_ray rays).  CUDA events on
the context's stream, median of 5 after one warm-up call.  Visits per ray of the 4-D walk are counted on a 256-ray sample from the
node array (a record is visited when its parent was entered).  Prints one JSON line with the card name and its power limit.

    python tools/dim4_probe.py
"""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bvh_b200 import api, capi, scenes  # noqa: E402
from bvh_b200.dtypes import BY_PREC, BY_PREC_4D  # noqa: E402


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:                                                # read-only query
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    return name, power


def timed(fn, stream, reps=5):
    import torch

    fn()                                                # warm-up
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        out.append(a.elapsed_time(b))
    return round(float(np.median(out)), 3)


def lift(a3, prec):
    a4 = np.zeros(len(a3), dtype=BY_PREC_4D[prec]["aabb"])
    a4["min"][:, :3], a4["max"][:, :3] = a3["min"], a3["max"]
    a4["min"][:, 3], a4["max"][:, 3] = 1.5, 1.5
    return a4


def builds(ctx, stream):
    L = capi.lib()
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    rows = []
    for prec in ("f32", "f64"):
        rng = np.random.default_rng(12)
        big = np.zeros(1_200_000, dtype=BY_PREC[prec]["aabb"])
        mn = rng.uniform(-1000, 1000, (len(big), 3))
        big["min"], big["max"] = mn, mn + rng.uniform(0, 3, (len(big), 3))
        for name, a3 in (("cubes_120k", scenes.create_n_cubes_aabbs(10000, prec)), ("random_1.2M", big)):
            a4 = lift(a3, prec)
            row = {"scene": name, "prec": prec, "n": len(a3)}
            for dim, arr, suf in ((3, a3, BY_PREC[prec]["suffix"]), (4, a4, BY_PREC_4D[prec]["suffix"])):
                h = C.c_void_p()

                def run():
                    capi.check(getattr(L, f"bvhgpu_build_{suf}")(ctx._h, p(arr), len(arr), capi.BUILD_EXACT_SAH, C.byref(h)))
                    getattr(L, f"bvhgpu_tree_free_{suf}")(h)
                row[f"build{dim}d_ms"] = timed(run, stream)
            row["ratio_4d_over_3d"] = round(row["build4d_ms"] / row["build3d_ms"], 2)
            rows.append(row)
    return rows


def visits_per_ray(nodes, rays, prec, sample=256):
    import torch

    dt = torch.float32 if prec == "f32" else torch.float64
    nn = len(nodes)
    parent = nodes["parent"].astype(np.int64)
    depth = np.zeros(nn, dtype=np.int64)
    for i in range(1, nn):                              # preorder: parents come first
        depth[i] = depth[parent[i]] + 1
    is_left = np.zeros(nn, dtype=bool)
    is_left[1:] = nodes["child_l"][parent[1:]] == np.arange(1, nn)
    box_min = np.where(is_left[:, None], nodes["l_aabb"]["min"][parent], nodes["r_aabb"]["min"][parent])
    box_max = np.where(is_left[:, None], nodes["l_aabb"]["max"][parent], nodes["r_aabb"]["max"][parent])
    bmin, bmax = torch.from_numpy(box_min[1:]).to("cuda", dt), torch.from_numpy(box_max[1:]).to("cuda", dt)
    par = torch.from_numpy(parent).cuda()
    levels = [torch.from_numpy(np.flatnonzero(depth == d)).cuda() for d in range(1, int(depth.max()) + 1)]
    total = 0
    for r0 in range(0, sample, 16):
        o, inv = rays[r0:r0 + 16, None, 0:4], rays[r0:r0 + 16, None, 8:12]
        l, r = (bmin[None] - o) * inv, (bmax[None] - o) * inv
        nan = torch.isnan(l).any(dim=2) | torch.isnan(r).any(dim=2)
        hit = ~nan & (torch.minimum(l, r).amax(dim=2).clamp(min=0) <= torch.maximum(l, r).amin(dim=2))
        hit = torch.cat([torch.ones_like(hit[:, :1]), hit], dim=1)
        entered = torch.zeros_like(hit)
        entered[:, 0] = True
        for idx in levels:
            entered[:, idx] = hit[:, idx] & entered[:, par[idx]]
        total += int(entered[:, par[1:]].sum())
    return total / sample


def traversals(ctx, stream):
    import torch

    out = {}
    # 4-D: 120 k random boxes, 1 M random rays, device pointers, no host synchronisation inside the timed call
    for prec in ("f32", "f64"):
        dt = torch.float32 if prec == "f32" else torch.float64
        rng = np.random.default_rng(120)
        a = np.zeros(120_000, dtype=BY_PREC_4D[prec]["aabb"])
        mn = rng.uniform(-1000, 1000, (len(a), 4))
        a["min"], a["max"] = mn, mn + rng.uniform(0, 60, (len(a), 4))
        bvh = api.Bvh4.build(a, prec=prec, ctx=ctx)
        g = torch.Generator(device="cuda").manual_seed(7)
        m = 1 << 20
        o = (torch.rand((m, 4), generator=g, device="cuda", dtype=torch.float64) * 2200 - 1100).to(dt)
        d = (torch.rand((m, 4), generator=g, device="cuda", dtype=torch.float64) * 2 - 1).to(dt)
        d = d / torch.sqrt((d * d).sum(dim=1, keepdim=True))
        rays = torch.cat([o, d, 1 / d], dim=1).contiguous()
        offs = torch.zeros(m + 1, dtype=torch.int32, device="cuda")
        total = bvh.traverse_dev(rays.data_ptr(), m, offs.data_ptr(), 0, 0, want_total=True)
        hits = torch.zeros(max(total, 1), dtype=torch.int32, device="cuda")
        run = lambda: bvh.traverse_dev(rays.data_ptr(), m, offs.data_ptr(), hits.data_ptr(), total)
        ms = timed(run, stream)
        nodes, _ = bvh.nodes_and_index()
        out[f"traverse4d_{prec}"] = {"n": len(a), "rays": m, "hits": total, "ms": ms, "mrays_per_s": round(m / ms / 1e3, 1),
                                     "visits_per_ray_sampled": round(visits_per_ray(nodes, rays, prec), 1)}
        bvh.free()
    # 3-D reference point: config 2, plain persistent walk (no shared-memory top of the tree)
    a3 = scenes.create_n_cubes_aabbs(10000, "f32")
    bvh3 = api.Bvh.build(a3, prec="f32", ctx=ctx)
    org, dirs = scenes.ray_endpoints(1_000_000, prec="f32")
    r3 = torch.from_numpy(api.Ray.new(org, dirs, "f32", ctx=ctx).view(np.uint8)).cuda()
    m = 1_000_000
    offs = torch.zeros(m + 1, dtype=torch.int32, device="cuda")
    ctx.set_option("traverse_top", 0)
    try:
        total = bvh3.traverse_dev(r3.data_ptr(), m, offs.data_ptr(), 0, 0, want_total=True)
        hits = torch.zeros(max(total, 1), dtype=torch.int32, device="cuda")
        ms = timed(lambda: bvh3.traverse_dev(r3.data_ptr(), m, offs.data_ptr(), hits.data_ptr(), total), stream)
    finally:
        ctx.set_option("traverse_top", -1)
    out["traverse3d_f32_config2_plain"] = {"rays": m, "hits": total, "ms": ms, "mrays_per_s": round(m / ms / 1e3, 1)}
    bvh3.free()
    return out


def main():
    import torch

    ctx = api.Context(0)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    name, power = card()
    res = {"card": name, "power_limit": power, "what": "CUDA events on the context's stream, median of 5 after one warm-up call"}
    res["builds"] = builds(ctx, stream)
    res.update(traversals(ctx, stream))
    ctx.set_stream(None)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
