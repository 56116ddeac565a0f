#!/usr/bin/env python
"""Throughput of the 2-D and 4-D distance-ordered traversal and closest hit (DESIGN.md section 5): 1 M random shapes and 1 M rays
aimed at them, f32 and f64, in D = 2 and D = 4.  Ordered ascending and descending and closest_hit through the host-pointer entry
points (host rays in, host results out, transfers included), closest_hit_dev (D = 4) from device pointers, and traverse_batch
(BVH semantics) on the same rays for comparison.  CUDA events on the context's stream, median of 3 after one warm-up call.  Prints
one JSON line with the card name and its power limit, read in the same call.

    python tools/dim_ordered_probe.py
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bvh_b200 import api, capi  # noqa: E402
from tools.dim_query_probe import card, timed  # noqa: E402

N = 1 << 20
M = 1 << 20


def scene(D, F, rng):
    mn = rng.uniform(-1000, 1000, (N, D))
    mx = mn + rng.uniform(0, 4, (N, D))
    o = rng.uniform(-1100, 1100, (M, D))
    t = rng.integers(0, N, M)
    d = 0.5 * (mn[t] + mx[t]) - o
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return mn.astype(F), mx.astype(F), o.astype(F), d.astype(F)


def row(ms, extra=None):
    r = {"ms": round(ms, 3), "mrays_per_s": round(M / ms / 1e3, 1)}
    r.update(extra or {})
    return r


def probe(D, prec, ctx, stream):
    import torch

    F = np.float32 if prec == "f32" else np.float64
    cls = api.Bvh2 if D == 2 else api.Bvh4
    t = cls._TABLE[prec]
    mn, mx, o, d = scene(D, F, np.random.default_rng(D))
    a = np.zeros(N, dtype=t["aabb"]); a["min"], a["max"] = mn, mx
    rays = np.zeros(M, dtype=t["ray"])
    with np.errstate(divide="ignore"):
        rays["origin"], rays["direction"], rays["inv_direction"] = o, d, (F(1) / d).astype(F)
    b = cls.build(a, prec=prec, ctx=ctx)
    out = {}
    off, hits = b.traverse_batch(rays, mode=capi.TRAVERSE_BVH)
    out["traverse_batch"] = row(timed(lambda: b.traverse_batch(rays, mode=capi.TRAVERSE_BVH), stream), {"hits": int(off[-1])})
    out["ordered_asc"] = row(timed(lambda: b.traverse_ordered(rays, True), stream))
    out["ordered_desc"] = row(timed(lambda: b.traverse_ordered(rays, False), stream))
    s, _ = b.closest_hit(rays)
    out["closest_host"] = row(timed(lambda: b.closest_hit(rays), stream), {"hit_rays": int((s != 0xFFFFFFFF).sum())})
    if D == 4:
        dev = torch.device("cuda", 0)
        dr = torch.from_numpy(rays.view(np.uint8)).to(dev)
        ds = torch.empty(M, dtype=torch.int32, device=dev)
        dd = torch.empty(M, dtype=torch.float32 if prec == "f32" else torch.float64, device=dev)
        out["closest_dev"] = row(timed(lambda: b.closest_hit_dev(dr.data_ptr(), M, ds.data_ptr(), dd.data_ptr()), stream))
    b.free()
    return out


def main():
    import torch

    name, power = card()
    ctx = api.Context.default()
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    res = {"card": name, "power_limit": power, "shapes": N, "rays": M}
    with torch.cuda.stream(stream):
        for D in (2, 4):
            for prec in ("f32", "f64"):
                res[f"{D}d_{prec}"] = probe(D, prec, ctx, stream)
    ctx.set_stream(None)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
