#!/usr/bin/env python
"""Churn cost of the 2-D and 4-D bvhgpu_remove_shapes_* / bvhgpu_add_shapes_*: per call, remove 1 % and add 1 % of the shapes (host
inputs pre-gathered, host clock around the synchronous C call, after one warm-up round), against a full exact build of the same n
timed the same way, and the SAH cost after the churn rounds relative to a fresh build over the same shapes.  Three trees of 1.2 M
random boxes: 4-D f32, 4-D f64 and 2-D f32.  Prints one JSON line with the card name and its power limit.

    python tools/dim_churn_probe.py [--rounds 10] [--small]      (--small: 120 k shapes, for a quick look)
"""
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bvh_b200 import api, capi  # noqa: E402
from tools.churn_probe import card  # noqa: E402


def boxes(cls, prec, n, rng):
    D = cls._DIM
    a = np.zeros(n, dtype=cls._TABLE[prec]["aabb"])
    mn = rng.uniform(-1000, 1000, (n, D))
    a["min"], a["max"] = mn, mn + rng.uniform(0, 3, (n, D))
    return a


def sah_cost(nodes):
    """Sum over non-root nodes of SA(box in the parent) / SA(root box), in double (tests/dimcheck.py)."""
    i = np.flatnonzero(nodes["child_l"] != 0xFFFFFFFF)
    tot = 0.0
    for side in ("l_aabb", "r_aabb"):
        s = nodes[side]["max"][i].astype(np.float64) - nodes[side]["min"][i].astype(np.float64)
        tot += float((2.0 * (s * s).sum(axis=1)).sum())
    rs = np.maximum(nodes["l_aabb"]["max"][0], nodes["r_aabb"]["max"][0]).astype(np.float64) - \
        np.minimum(nodes["l_aabb"]["min"][0], nodes["r_aabb"]["min"][0]).astype(np.float64)
    return tot / (2.0 * float((rs * rs).sum()))


def probe(cls, prec, n, rounds, rng, ctx):
    L = capi.lib()
    suf = cls._TABLE[prec]["suffix"]
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    shapes = boxes(cls, prec, n, rng)
    k = n // 100
    h = C.c_void_p()
    build_ms = []
    for _ in range(3):                                  # full exact build of the same n (upload included, as the churn calls upload theirs)
        ctx.synchronize()
        t0 = time.perf_counter()
        capi.check(getattr(L, f"bvhgpu_build_{suf}")(ctx._h, p(shapes), n, capi.BUILD_EXACT_SAH, C.byref(h)))
        ctx.synchronize()
        build_ms.append((time.perf_counter() - t0) * 1e3)
        getattr(L, f"bvhgpu_tree_free_{suf}")(h)
    bvh = cls.build(shapes, prec=prec, ctx=ctx)
    cur = shapes.copy()
    rm_ms, add_ms, rebuilt = [], [], []
    rb = C.c_size_t(0)
    for r in range(rounds + 1):                         # round 0 is the warm-up
        idx = rng.choice(len(cur), k, replace=False).astype(np.uint32)
        new = cur[idx].copy()
        dl = rng.uniform(-20.0, 20.0, (k, cls._DIM))
        new["min"] += dl; new["max"] += dl
        ctx.synchronize()
        t0 = time.perf_counter()
        capi.check(getattr(L, f"bvhgpu_remove_shapes_{suf}")(bvh._h, p(idx), k))
        ctx.synchronize()
        t1 = time.perf_counter()
        capi.check(getattr(L, f"bvhgpu_add_shapes_{suf}")(bvh._h, p(new), k, C.c_double(1.5), C.byref(rb)))
        ctx.synchronize()
        t2 = time.perf_counter()
        mv = api.swap_moves(len(cur), idx)
        cur[mv[:, 0]] = cur[mv[:, 1]]
        cur = np.concatenate([cur[: len(cur) - k], new])
        if r:
            rm_ms.append((t1 - t0) * 1e3); add_ms.append((t2 - t1) * 1e3); rebuilt.append(int(rb.value))
    bvh._sync_n()
    sah = sah_cost(bvh.nodes_and_index()[0])
    fresh = cls.build(cur, prec=prec, ctx=ctx)
    sah_fresh = sah_cost(fresh.nodes_and_index()[0])
    bvh.free(); fresh.free()
    med = lambda v: float(np.median(v))
    return {"n": n, "k": k, "D": cls._DIM, "prec": prec, "remove_ms_median": round(med(rm_ms), 3), "add_ms_median": round(med(add_ms), 3),
            "build_ms_median": round(med(build_ms), 3), "remove_ms": [round(t, 3) for t in rm_ms], "add_ms": [round(t, 3) for t in add_ms],
            "build_ms": [round(t, 3) for t in build_ms], "add_rebuilt_shapes": rebuilt,
            "sah_after_rounds": sah, "sah_fresh_build": sah_fresh, "sah_ratio": sah / sah_fresh}


def main():
    rounds = int(sys.argv[sys.argv.index("--rounds") + 1]) if "--rounds" in sys.argv else 10
    n = 120_000 if "--small" in sys.argv else 1_200_000
    ctx = api.Context(0)
    rng = np.random.default_rng(21)
    name, power = card()
    out = {"card": name, "power_limit": power, "rounds": rounds, "what": "host clock around the synchronous C call, inputs pre-gathered, median after one warm-up round"}
    for key, cls, prec in (("4d_f32", api.Bvh4, "f32"), ("4d_f64", api.Bvh4, "f64"), ("2d_f32", api.Bvh2, "f32")):
        out[key] = probe(cls, prec, n, rounds, rng, ctx)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
