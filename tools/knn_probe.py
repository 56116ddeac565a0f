#!/usr/bin/env python
"""k nearest shapes against the one-result nearest_to (DESIGN.md section 5): the 120 k triangle boxes of BASELINE.json configs[1]
(scenes.create_n_cubes_aabbs(10 000)) and 1 M points of the scene generator's seed chain (the origins of scenes.ray_endpoints),
f32 and f64, k in {1, 8, 32, 64}, without a limit and with a radius of 2 000 (a few shapes qualify for most points).
- knn: bvhgpu_knn_dev_* on device pointers, CUDA events on the context's stream, median of 5 after one warm-up call;
- kernel times of knn_kernel and of nearest_kernel (bvhgpu_nearest_*, BVH mode, the same points) from torch.profiler's CUDA activities,
  in a profiled run of their own.
Prints one JSON line with the card name and its power limit, read in the same call.

    python tools/knn_probe.py
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bvh_b200 import api, scenes  # noqa: E402
from tools.dim_query_probe import card, timed  # noqa: E402

N_POINTS = 1_000_000
RADIUS = 2000.0


def kernel_ms(fn, name):
    """Mean device time per launch of the kernels whose name contains `name`, over 3 calls of fn, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
    tot, cnt = 0.0, 0
    for e in prof.key_averages():
        if name in e.key:
            tot += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
            cnt += e.count
    return round(tot / max(cnt, 1) / 1e3, 3)


def run(prec, ctx, stream, dev):
    import torch

    F = np.float32 if prec == "f32" else np.float64
    dt = torch.float32 if prec == "f32" else torch.float64
    aabbs = scenes.create_n_cubes_aabbs(10_000, prec)
    pts, _ = scenes.ray_endpoints(N_POINTS, prec=prec)
    b = api.Bvh.build(aabbs, prec=prec, ctx=ctx)
    d_p = torch.from_numpy(pts).to(dev)
    d_r = torch.full((N_POINTS,), RADIUS, dtype=dt, device=dev)
    out = {"shapes": len(aabbs), "points": N_POINTS}
    _, nd = b.nearest_to_batch(pts)
    out["nearest_kernel_ms"] = kernel_ms(lambda: b.nearest_to_batch(pts), "nearest_kernel")
    for k in (1, 8, 32, 64):
        d_s = torch.empty(N_POINTS * k, dtype=torch.int32, device=dev)
        d_d = torch.empty(N_POINTS * k, dtype=dt, device=dev)
        for lim, tag in ((None, "none"), (d_r, "radius")):
            def call():
                b.knn_dev(d_p.data_ptr(), N_POINTS, k, lim.data_ptr() if lim is not None else 0, d_s.data_ptr(), d_d.data_ptr())

            row = {"event_ms": round(timed(call, stream, reps=5), 3), "kernel_ms": kernel_ms(call, "knn_kernel")}
            call()
            stream.synchronize()
            found = (d_s.view(N_POINTS, k) != -1).sum(1).float()
            row["mean_found"] = round(float(found.mean()), 2)
            if k == 1 and lim is None:                          # knn(k = 1) and nearest_to agree on the distance on this scene
                row["k1_dist_equals_nearest"] = bool(np.array_equal(d_d.cpu().numpy(), nd))
            out[f"k{k}_{tag}"] = row
    b.free()
    return out


def main():
    import torch

    name, power = card()
    dev = torch.device("cuda", 0)
    ctx = api.Context.default()
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    res = {"card": name, "power_limit": power}
    with torch.cuda.stream(stream):
        for prec in ("f32", "f64"):
            res[prec] = run(prec, ctx, stream, dev)
    ctx.set_stream(None)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
