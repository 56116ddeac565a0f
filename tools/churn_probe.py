#!/usr/bin/env python
"""Churn cost of bvhgpu_remove_shapes_* / bvhgpu_add_shapes_*: per call, remove 1 % and add 1 % of the shapes (host inputs pre-gathered,
host clock around the synchronous C call, after one warm-up round), against a full exact build of the same n timed the same way, and the
SAH cost after 10 churn rounds relative to a fresh build over the same shapes.  Two trees: 10 M f64 shapes (the config 5 scene of
scenes.create_n_cubes_aabbs) and 1.2 M f32 shapes.  Prints one JSON line with the card name and its power limit.

    python tools/churn_probe.py [--rounds 10] [--small]      (--small: 1 M f64 / 120 k f32, for a quick look)
"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bvh_b200 import api, capi, scenes  # noqa: E402


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:                                                # read-only query
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    return name, power


def probe(shapes, prec, rounds, rng, ctx):
    L = capi.lib()
    suf = {"f32": "f32x3", "f64": "f64x3"}[prec]
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    n = len(shapes)
    k = n // 100
    h = C.c_void_p()
    build_ms = []
    for _ in range(3):                                  # full exact build of the same n (upload included, as the churn calls upload theirs)
        t0 = time.perf_counter()
        capi.check(getattr(L, f"bvhgpu_build_{suf}")(ctx._h, p(shapes), n, capi.BUILD_EXACT_SAH, C.byref(h)))
        build_ms.append((time.perf_counter() - t0) * 1e3)
        getattr(L, f"bvhgpu_tree_free_{suf}")(h)
    bvh = api.Bvh.build(shapes, prec=prec, ctx=ctx)
    cur = shapes.copy()
    rm_ms, add_ms, rebuilt = [], [], []
    rb = C.c_size_t(0)
    for r in range(rounds + 1):                         # round 0 is the warm-up
        idx = rng.choice(len(cur), k, replace=False).astype(np.uint32)
        new = cur[idx].copy()
        dl = rng.uniform(-20.0, 20.0, (k, 3))
        new["min"] += dl; new["max"] += dl
        ctx.synchronize()
        t0 = time.perf_counter()
        capi.check(getattr(L, f"bvhgpu_remove_shapes_{suf}")(bvh._h, p(idx), k))
        t1 = time.perf_counter()
        capi.check(getattr(L, f"bvhgpu_add_shapes_{suf}")(bvh._h, p(new), k, C.c_double(1.5), C.byref(rb)))
        t2 = time.perf_counter()
        mv = api.swap_moves(len(cur), idx)
        cur[mv[:, 0]] = cur[mv[:, 1]]
        cur = np.concatenate([cur[: len(cur) - k], new])
        if r:
            rm_ms.append((t1 - t0) * 1e3); add_ms.append((t2 - t1) * 1e3); rebuilt.append(int(rb.value))
    bvh._nodes = None
    sah = bvh.sah_cost()[0]
    fresh = api.Bvh.build(cur, prec=prec, ctx=ctx)
    sah_fresh = fresh.sah_cost()[0]
    bvh.free(); fresh.free()
    med = lambda v: float(np.median(v))
    return {"n": n, "k": k, "prec": prec, "remove_ms_median": round(med(rm_ms), 3), "add_ms_median": round(med(add_ms), 3),
            "build_ms_median": round(med(build_ms), 3), "remove_ms": [round(t, 3) for t in rm_ms], "add_ms": [round(t, 3) for t in add_ms],
            "build_ms": [round(t, 3) for t in build_ms], "add_rebuilt_shapes": rebuilt,
            "sah_after_rounds": sah, "sah_fresh_build": sah_fresh, "sah_ratio": sah / sah_fresh}


def main():
    rounds = int(sys.argv[sys.argv.index("--rounds") + 1]) if "--rounds" in sys.argv else 10
    small = "--small" in sys.argv
    ctx = api.Context(0)
    rng = np.random.default_rng(21)
    name, power = card()
    out = {"card": name, "power_limit": power, "rounds": rounds, "what": "host clock around the synchronous C call, inputs pre-gathered, median after one warm-up round"}
    n64, n32 = (1_000_000, 120_000) if small else (10_000_000, 1_200_000)
    a64 = scenes.create_n_cubes_aabbs((n64 + 11) // 12, "f64")[:n64]
    out["f64"] = probe(a64, "f64", rounds, rng, ctx)
    del a64
    a32 = scenes.create_n_cubes_aabbs((n32 + 11) // 12, "f32")[:n32]
    out["f32"] = probe(a32, "f32", rounds, rng, ctx)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
