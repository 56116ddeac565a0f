#!/usr/bin/env python
"""Host-pointer CSR calls around the retained hit buffer, f32, CUDA events on the context's stream:
- d3_query_*: 3-D Aabb / Point / Ball queries, 1 M random shapes, 1 M queries, BVH mode, through bvhgpu_query_f32x3 (host records in,
  host CSR out, transfers included); median of 3 after one warm-up call, so the retained buffer already holds the total;
- d3_overflow / d4_overflow: a query batch whose total passes the first retained buffer (max(16 n, 1024) hits) of a fresh tree, the
  tree rebuilt before every call and only the call timed; median of 3.  The call is made as Bvh.query_batch makes it: a cap of
  max(16 n, 1024), then bvhgpu_traverse_fetch_* (3-D) or a second call with cap = total (4-D);
- d4_overflow steady_ms: the same batch again on the same tree (the retained buffer holds the total), median of 3 after a warm-up.
Prints one JSON line with the card name and its power limit, read in the same call.

    python tools/csr_host_probe.py [--lib path/to/libbvh_b200.so]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bvh_b200 import api, capi  # noqa: E402
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


def event_ms(fn, stream):
    import torch

    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    fn()
    b.record(stream)
    b.synchronize()
    return a.elapsed_time(b)


def steady(fn, stream, reps=3):
    fn()                                                # warm-up
    return round(float(np.median([event_ms(fn, stream) for _ in range(reps)])), 3)


def scene(D, n, size, seed):
    table = (BY_PREC if D == 3 else BY_PREC_4D)["f32"]
    rng = np.random.default_rng(seed)
    a = np.zeros(n, dtype=table["aabb"])
    mn = rng.uniform(-1000, 1000, (n, D))
    a["min"], a["max"] = mn, mn + rng.uniform(0, size, (n, D))
    return a, rng


def overflow(D, ctx, stream, reps=3):
    """n = 256 k shapes, m = 64 k Aabb queries of about 40 hits each: the total passes 16 m."""
    n, m = 1 << 18, 1 << 16
    a, rng = scene(D, n, 60.0 if D == 4 else 12.0, 10 + D)
    cls = api.Bvh if D == 3 else api.Bvh4
    p = rng.uniform(-1000, 1000, (m, D)).astype(np.float32)
    q = np.ascontiguousarray(np.concatenate([p, p + np.float32(200.0 if D == 4 else 100.0)], axis=1))
    times, hits = [], 0
    for _ in range(reps + 1):
        bvh = cls.build(a, prec="f32", ctx=ctx)
        out = {}
        t = event_ms(lambda: out.setdefault("r", bvh.query_batch(capi.QUERY_AABB, q)), stream)
        hits = int(out["r"][0][-1])
        times.append(t)
        if _ == reps and D == 4:
            st = steady(lambda: bvh.query_batch(capi.QUERY_AABB, q), stream)
        bvh.free()
    res = {"shapes": n, "queries": m, "hits": hits, "first_buffer": 16 * m, "ms": round(float(np.median(times[1:])), 3)}
    if D == 4:
        res["steady_ms"] = st
    return res


def d3_queries(ctx, stream):
    n = m = 1 << 20
    a, rng = scene(3, n, 12.0, 3)
    bvh = api.Bvh.build(a, prec="f32", ctx=ctx)
    p = rng.uniform(-1000, 1000, (m, 3)).astype(np.float32)
    recs = {
        capi.QUERY_AABB: ("aabb", np.concatenate([p, p + rng.uniform(0, 12.0, (m, 3)).astype(np.float32)], axis=1)),
        capi.QUERY_POINT: ("point", p),
        capi.QUERY_BALL: ("ball", np.concatenate([p, rng.uniform(0, 6.0, (m, 1)).astype(np.float32)], axis=1)),
    }
    out = {}
    for kind, (name, q) in recs.items():
        q = np.ascontiguousarray(q)
        off, _ = bvh.query_batch(kind, q)
        out[f"d3_query_{name}"] = {"ms": steady(lambda: bvh.query_batch(kind, q), stream), "hits": int(off[-1])}
    bvh.free()
    return out


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="the libbvh_b200.so to load (default: the package's)")
    args = ap.parse_args()
    if args.lib:
        capi.SO_PATH = os.path.abspath(args.lib)
    ctx = api.Context(0)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    name, power = card()
    res = {"card": name, "power_limit": power, "lib": capi.SO_PATH}
    try:
        res.update(d3_queries(ctx, stream))
        res["d3_overflow"] = overflow(3, ctx, stream)
        res["d4_overflow"] = overflow(4, ctx, stream)
    finally:
        ctx.set_stream(None)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
