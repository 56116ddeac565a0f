#!/usr/bin/env python
"""Throughput of the 2-D and 4-D queries and nearest_to (DESIGN.md section 5): 1 M random f32 shapes, 1 M queries of each kind
(Aabb, Point, Ball), nearest_to and nearest_candidates, BVH and FLAT mode, through the host-pointer entry points (host records in,
host CSR out, transfers included) and, for D = 4, the device-pointer query form.  CUDA events on the context's stream, median of 3
after one warm-up call.  Prints one JSON line with the card name and its power limit, read in the same call.

    python tools/dim_query_probe.py
"""
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bvh_b200 import api, capi  # noqa: E402
from bvh_b200.dtypes import BY_PREC_2D, BY_PREC_4D  # noqa: E402

N = 1 << 20
M = 1 << 20


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:                                                # read-only query
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    return name, power


def timed(fn, stream, reps=3):
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
    return float(np.median(out))


def row(ms, extra=None):
    r = {"ms": round(ms, 3), "mq_per_s": round(M / ms / 1e3, 1)}
    r.update(extra or {})
    return r


def probe(D, ctx, stream):
    import torch

    table = {2: BY_PREC_2D, 4: BY_PREC_4D}[D]["f32"]
    size = 3.0 if D == 2 else 60.0                      # about one shape per point query in either dimension
    rng = np.random.default_rng(D)
    a = np.zeros(N, dtype=table["aabb"])
    mn = rng.uniform(-1000, 1000, (N, D))
    a["min"], a["max"] = mn, mn + rng.uniform(0, size, (N, D))
    bvh = (api.Bvh2 if D == 2 else api.Bvh4).build(a, prec="f32", ctx=ctx)
    p = rng.uniform(-1000, 1000, (M, D)).astype(np.float32)
    recs = {
        "aabb": np.concatenate([p, p + rng.uniform(0, size, (M, D)).astype(np.float32)], axis=1),
        "point": p,
        "ball": np.concatenate([p, rng.uniform(0, size / 2, (M, 1)).astype(np.float32)], axis=1),
    }
    kinds = {"aabb": capi.QUERY_AABB, "point": capi.QUERY_POINT, "ball": capi.QUERY_BALL}
    out = {"shapes": N, "queries": M}
    for name, q in recs.items():
        q = np.ascontiguousarray(q)
        for mode_name, mode in (("bvh", capi.TRAVERSE_BVH), ("flat", capi.TRAVERSE_FLAT)):
            off, _ = bvh.query_batch(kinds[name], q, mode=mode)
            out[f"query_{name}_{mode_name}"] = row(timed(lambda: bvh.query_batch(kinds[name], q, mode=mode), stream), {"hits": int(off[-1])})
            if D == 4:
                dq = torch.from_numpy(q).cuda()
                doff = torch.zeros(M + 1, dtype=torch.int32, device="cuda")
                dh = torch.zeros(max(int(off[-1]), 1), dtype=torch.int32, device="cuda")
                run = lambda: bvh.query_dev(kinds[name], dq.data_ptr(), M, doff.data_ptr(), dh.data_ptr(), int(off[-1]), mode=mode)
                out[f"query_dev_{name}_{mode_name}"] = row(timed(run, stream))
    for mode_name, mode in (("bvh", capi.TRAVERSE_BVH), ("flat", capi.TRAVERSE_FLAT)):
        out[f"nearest_{mode_name}"] = row(timed(lambda: bvh.nearest_to_batch(p, mode=mode), stream))
    off, _ = bvh.nearest_candidates(p)
    out["nearest_candidates"] = row(timed(lambda: bvh.nearest_candidates(p), stream), {"candidates": int(off[-1])})
    bvh.free()
    return out


def main():
    import torch

    ctx = api.Context(0)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    name, power = card()
    res = {"card": name, "power_limit": power, "what": "CUDA events on the context's stream, median of 3 after one warm-up call; "
           "host forms include the host <-> device copies; mq_per_s = million queries per second"}
    try:
        res["d2_f32"] = probe(2, ctx, stream)
        res["d4_f32"] = probe(4, ctx, stream)
    finally:
        ctx.set_stream(None)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
