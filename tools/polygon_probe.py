#!/usr/bin/env python
"""Polygons of 2-D trees (DESIGN.md section 5): exact point-in-polygon, k nearest segments and signed distance against the
floating-point workaround.  Host-pointer calls (the only form 2-D trees have), CUDA events on the context's stream around each call,
median of 3 after one warm-up call; a time includes the pageable copies of the points and the results.
- Scenes: a Koch snowflake of level 7 (49 152 segments) and a "map" of 16 384 star polygons of 16 spikes, each with a star hole of the
  opposite orientation (1 048 576 segments), f32 (and the snowflake in f64).
- Points: 1 M and 16 M uniform over the scene's bounds.
- Calls: contains_points (even-odd), knn_segments at k = 1 and k = 8, signed_distance.
- The workaround on a subset of points: the Aabb query [px, +inf] x [py, py] per point (query_batch, the candidate CSR copied back),
  then a floating-point crossing test on the host in the tree's precision (numpy); the host part is timed with a host clock.  The
  points whose parity differs from the exact class (boundary points left out) are counted.
One JSON line per row and a final line with the card name and its power limit, read in the same call.

    python tools/polygon_probe.py [--quick]
"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bvh_b200 import api, capi  # noqa: E402
from bvh_b200.dtypes import BY_PREC_2D  # noqa: E402
from tests import polygons as P  # noqa: E402
from tools.dim_query_probe import card  # noqa: E402


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


def tree(segs, prec, ctx):
    mn, mx = P.seg_boxes(segs)
    a = np.zeros(len(segs), dtype=BY_PREC_2D[prec]["aabb"])
    a["min"], a["max"] = mn, mx
    b = api.Bvh2.build(a, prec=prec, ctx=ctx)
    b.set_segments(segs)
    return b


def workaround(bvh, segs, pts):
    """(query ms (device CSR + copy back, events), host crossing-test ms, even-odd parity per point)."""
    F = segs.dtype.type
    q = np.stack([pts[:, 0], pts[:, 1], np.full(len(pts), np.inf, dtype=F), pts[:, 1]], axis=1).astype(F)
    t0 = time.perf_counter()
    off, hits = bvh.query_batch(capi.QUERY_AABB, q)
    t1 = time.perf_counter()
    row = np.repeat(np.arange(len(pts)), np.diff(off.astype(np.int64)))
    s = segs[hits.astype(np.int64)]
    px, py = pts[row, 0], pts[row, 1]
    ax, ay, bx, by = s[:, 0], s[:, 1], s[:, 2], s[:, 3]
    with np.errstate(all="ignore"):
        cross = ((ay > py) != (by > py)) & (px < (bx - ax) * (py - ay) / (by - ay) + ax)
    parity = np.zeros(len(pts), dtype=np.int64)
    np.add.at(parity, row[cross], 1)
    t2 = time.perf_counter()
    return (t1 - t0) * 1e3, (t2 - t1) * 1e3, parity & 1, len(hits)


def main(quick=False):
    import torch

    ctx = api.Context(0)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    rng = np.random.default_rng(0)
    n_stars = 256 if quick else 16384
    scenes = [("koch7", P.koch(4 if quick else 7, np.float64), ["f32", "f64"]),
              ("map", P.star_map(n_stars, 16, np.float64, seed=1), ["f32"])]
    sizes = [1 << 16] if quick else [1 << 20, 1 << 24]
    rows = []
    for name, segs64, precs in scenes:
        for prec in precs:
            F = BY_PREC_2D[prec]["scalar"]
            segs = segs64.astype(F)
            bvh = tree(segs, prec, ctx)
            lo, hi = segs.reshape(-1, 2).min(0).astype(np.float64), segs.reshape(-1, 2).max(0).astype(np.float64)
            for n in sizes:
                pts = rng.uniform(lo, hi, (n, 2)).astype(F)
                r = {"scene": name, "segments": len(segs), "prec": prec, "points": n}
                r["contains_ms"] = round(timed(lambda: bvh.contains(pts, "even_odd"), stream), 3)
                r["knn1_ms"] = round(timed(lambda: bvh.knn_segments(pts, 1), stream), 3)
                r["knn8_ms"] = round(timed(lambda: bvh.knn_segments(pts, 8), stream), 3)
                r["signed_ms"] = round(timed(lambda: bvh.signed_distance(pts, "even_odd"), stream), 3)
                r["contains_mpts_per_s"] = round(n / r["contains_ms"] / 1e3, 1)
                cls = bvh.contains(pts, "even_odd")
                r["inside"] = int((cls == P.INSIDE).sum())
                r["boundary"] = int((cls == P.BOUNDARY).sum())
                if n == sizes[0]:
                    sub = pts[: min(n, 1 << 18)]
                    bvh.query_batch(capi.QUERY_AABB, np.zeros((1, 4), dtype=F))          # warm-up
                    q_ms, host_ms, parity, cand = workaround(bvh, segs, sub)
                    exact = cls[: len(sub)]
                    keep = exact != P.BOUNDARY
                    r.update({"workaround_points": len(sub), "workaround_candidates": cand, "workaround_query_ms": round(q_ms, 3),
                              "workaround_host_ms": round(host_ms, 3),
                              "workaround_disagree": int((parity[keep] != (exact[keep] == P.INSIDE)).sum()),
                              "exact_contains_ms_same_points": round(timed(lambda: bvh.contains(sub, "even_odd"), stream), 3)})
                print(json.dumps(r), flush=True)
                rows.append(r)
            bvh.free()
    ctx.set_stream(None)
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power}), flush=True)
    return rows


if __name__ == "__main__":
    main(quick="--quick" in sys.argv)
