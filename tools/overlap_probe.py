#!/usr/bin/env python
"""Self-overlap pairs against the query workaround (DESIGN.md section 5), device-pointer forms on the same tree, CUDA events on the
context's stream, median of 5 after one warm-up call:
- overlap_pairs_dev: the walk from every shape's own leaf onwards, each pair once;
- the workaround: every shape's own box uploaded as a BVHGPU_QUERY_AABB query and run through query_dev (BVH mode), which lists
  every pair twice and every shape with itself.  Only the query is timed: dropping the self hits and one copy of every pair would
  come on top.
Scenes: the 120 k triangle boxes of BASELINE.json configs[1] (scenes.create_n_cubes_aabbs(10 000)) and the 66 450 Sponza triangle
boxes (tests/golden/sponza_tris.npz), f32 and f64.  Prints one JSON line with the card name and its power limit, read in the same
call.

    python tools/overlap_probe.py
"""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bvh_b200 import api, capi, scenes  # noqa: E402
from bvh_b200.dtypes import BY_PREC  # noqa: E402
from tools.dim_query_probe import card  # noqa: E402


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
    return float(np.median(out))


def sponza(prec):
    z = np.load(os.path.join(ROOT, "tests", "golden", "sponza_tris.npz"))
    tris = z["vertices"][z["triangles"].astype(np.int64)]
    a = np.zeros(len(tris), dtype=BY_PREC[prec]["aabb"])
    a["min"], a["max"] = tris.min(axis=1), tris.max(axis=1)
    return a


def one(name, aabbs, prec, ctx, stream):
    import torch

    dev = torch.device("cuda", 0)
    b = api.Bvh.build(aabbs, prec=prec, ctx=ctx)
    n = len(aabbs)
    L = capi.lib()
    sfx = b._d["suffix"]
    d_off = torch.zeros(n + 1, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    tot = C.c_size_t(0)
    st = getattr(L, f"bvhgpu_overlap_pairs_dev_{sfx}")(b._h, C.c_void_p(d_off.data_ptr()), None, 0, C.byref(tot))
    assert st in (capi.OK, capi.ERR_CAPACITY)
    pairs = tot.value
    d_hits = torch.zeros(max(pairs, 1), dtype=torch.int32, device=dev)
    q = np.concatenate([np.asarray(aabbs["min"]), np.asarray(aabbs["max"])], axis=1).astype(BY_PREC[prec]["scalar"])
    d_q = torch.from_numpy(np.ascontiguousarray(q)).to(dev)
    d_qoff = torch.zeros(n + 1, dtype=torch.int32, device=dev)
    capi.check(getattr(L, f"bvhgpu_query_dev_{sfx}")(b._h, capi.TRAVERSE_BVH, capi.QUERY_AABB, C.c_void_p(d_q.data_ptr()), n,
                                                     C.c_void_p(d_qoff.data_ptr()), None, 0, C.byref(tot)))
    qhits = tot.value
    d_qh = torch.zeros(qhits, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()                            # the buffers above were filled on torch's stream

    def overlap():
        capi.check(getattr(L, f"bvhgpu_overlap_pairs_dev_{sfx}")(b._h, C.c_void_p(d_off.data_ptr()), C.c_void_p(d_hits.data_ptr()), pairs, None))

    def query():
        capi.check(getattr(L, f"bvhgpu_query_dev_{sfx}")(b._h, capi.TRAVERSE_BVH, capi.QUERY_AABB, C.c_void_p(d_q.data_ptr()), n,
                                                         C.c_void_p(d_qoff.data_ptr()), C.c_void_p(d_qh.data_ptr()), qhits, None))

    t_o, t_q = timed(overlap, stream), timed(query, stream)
    b.free()
    return {"scene": name, "prec": prec, "shapes": n, "pairs": pairs, "query_hits": qhits, "twice_plus_self": qhits == 2 * pairs + n, "overlap_ms": round(t_o, 3),
            "query_ms": round(t_q, 3), "speedup": round(t_q / t_o, 2)}


def main():
    import torch

    name, power = card()
    ctx = api.Context.default()
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    rows = []
    try:
        for prec in ("f32", "f64"):
            rows.append(one("configs1_cubes", scenes.create_n_cubes_aabbs(10_000, prec).reshape(-1), prec, ctx, stream))
            rows.append(one("sponza", sponza(prec), prec, ctx, stream))
    finally:
        ctx.set_stream(None)
    print(json.dumps({"card": name, "power_limit": power, "rows": rows}))


if __name__ == "__main__":
    main()
