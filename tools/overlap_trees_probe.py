#!/usr/bin/env python
"""Overlap pairs between two trees against the query workaround (DESIGN.md section 5), device-pointer forms, CUDA events on the
context's stream, median of 5 after one warm-up call:
- overlap_trees_dev(A, B): A's shapes in A's leaf order, each walking B's records;
- the workaround: A's boxes, already on the device, run as BVHGPU_QUERY_AABB queries through query_dev on B (BVH mode), in A's
  shape numbering.  Only the query is timed.
Scenes: the 120 k triangle boxes of BASELINE.json configs[1] (scenes.create_n_cubes_aabbs(10 000)) against a copy translated by
half a cube width, and the 66 450 Sponza triangle boxes (tests/golden/sponza_tris.npz) against a copy translated by 1e-3 of the
scene's extent, f32 and f64; A in its natural numbering and with its shapes randomly permuted.  Prints one JSON line with the card
name and its power limit, read in the same call.

    python tools/overlap_trees_probe.py
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
from tools.overlap_probe import sponza, timed  # noqa: E402


def shifted(aabbs, shift):
    out = aabbs.copy()
    F = out["min"].dtype.type
    out["min"], out["max"] = (aabbs["min"] + F(shift)).astype(F), (aabbs["max"] + F(shift)).astype(F)
    return out


def scene_pairs(prec):
    """(name, A's boxes, B's boxes) in A's natural numbering."""
    cubes = scenes.create_n_cubes_aabbs(10_000, prec).reshape(-1)
    sp = sponza(prec)
    ext = (sp["max"].max(axis=0).astype(np.float64) - sp["min"].min(axis=0)) * 1e-3
    return [("configs1_cubes", cubes, shifted(cubes, 0.5)), ("sponza", sp, shifted(sp, ext))]


def one(name, a_boxes, b_boxes, prec, ctx, stream):
    import torch

    dev = torch.device("cuda", 0)
    a = api.Bvh.build(a_boxes, prec=prec, ctx=ctx)
    b = api.Bvh.build(b_boxes, prec=prec, ctx=ctx)
    n = len(a_boxes)
    L = capi.lib()
    sfx = a._d["suffix"]
    d_off = torch.zeros(n + 1, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    tot = C.c_size_t(0)
    st = getattr(L, f"bvhgpu_overlap_trees_dev_{sfx}")(a._h, b._h, C.c_void_p(d_off.data_ptr()), None, 0, C.byref(tot))
    assert st in (capi.OK, capi.ERR_CAPACITY)
    pairs = tot.value
    d_hits = torch.zeros(max(pairs, 1), dtype=torch.int32, device=dev)
    q = np.concatenate([np.asarray(a_boxes["min"]), np.asarray(a_boxes["max"])], axis=1).astype(BY_PREC[prec]["scalar"])
    d_q = torch.from_numpy(np.ascontiguousarray(q)).to(dev)
    d_qoff = torch.zeros(n + 1, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    capi.check(getattr(L, f"bvhgpu_query_dev_{sfx}")(b._h, capi.TRAVERSE_BVH, capi.QUERY_AABB, C.c_void_p(d_q.data_ptr()), n,
                                                     C.c_void_p(d_qoff.data_ptr()), None, 0, C.byref(tot)))
    qhits = tot.value
    d_qh = torch.zeros(max(qhits, 1), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()                            # the buffers above were filled on torch's stream

    def overlap():
        capi.check(getattr(L, f"bvhgpu_overlap_trees_dev_{sfx}")(a._h, b._h, C.c_void_p(d_off.data_ptr()), C.c_void_p(d_hits.data_ptr()), pairs, None))

    def query():
        capi.check(getattr(L, f"bvhgpu_query_dev_{sfx}")(b._h, capi.TRAVERSE_BVH, capi.QUERY_AABB, C.c_void_p(d_q.data_ptr()), n,
                                                         C.c_void_p(d_qoff.data_ptr()), C.c_void_p(d_qh.data_ptr()), qhits, None))

    t_o, t_q = timed(overlap, stream), timed(query, stream)
    same = bool(torch.equal(d_off, d_qoff) and torch.equal(d_hits[:pairs], d_qh[:qhits]))
    a.free()
    b.free()
    return {"scene": name, "prec": prec, "shapes_a": n, "shapes_b": len(b_boxes), "pairs": pairs, "query_hits": qhits, "same_csr": same,
            "overlap_ms": round(t_o, 3), "query_ms": round(t_q, 3), "speedup": round(t_q / t_o, 2)}


def main():
    import torch

    name, power = card()
    ctx = api.Context.default()
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    rows = []
    try:
        for prec in ("f32", "f64"):
            for scene, a_boxes, b_boxes in scene_pairs(prec):
                rows.append(one(scene, a_boxes, b_boxes, prec, ctx, stream))
                perm = np.random.default_rng(1).permutation(len(a_boxes))
                rows.append(one(scene + "_permuted", a_boxes[perm], b_boxes, prec, ctx, stream))
    finally:
        ctx.set_stream(None)
    print(json.dumps({"card": name, "power_limit": power, "rows": rows}))


if __name__ == "__main__":
    main()
