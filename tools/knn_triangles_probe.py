#!/usr/bin/env python
"""k nearest triangles against the one-result nearest_triangles and the box kNN (DESIGN.md section 5).  Two scenes: Sponza
(tests/golden/sponza_tris.npz, 66 450 triangles) and the 120 k triangles of BASELINE.json configs[1] (scenes.create_n_cubes_tris(10 000)).
1 M points per scene: half surface samples plus noise of 1 % of the scene's extent, half uniform in its bounding box.  f32 and f64,
k in {1, 8, 32, 64}, without a limit and with a radius of 1 % of the extent.
- knn_triangles: bvhgpu_knn_triangles_dev_* on device pointers with closest points, CUDA events on the context's stream, median of 5
  after one warm-up call;
- kernel times of knn_tri_kernel, of nearest_kernel in triangle mode (bvhgpu_nearest_triangles_*, BVH mode) and of knn_kernel (the box
  kNN) on the same points, from torch.profiler's CUDA activities, in profiled runs of their own.
Prints one JSON line with the card name and its power limit, read in the same call.

    python tools/knn_triangles_probe.py
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bvh_b200 import api, scenes  # noqa: E402
from tools.dim_query_probe import card, timed  # noqa: E402
from tools.knn_probe import kernel_ms  # noqa: E402

N_POINTS = 1_000_000


def scene_tris(name, prec):
    F = np.float32 if prec == "f32" else np.float64
    if name == "sponza":
        z = np.load(os.path.join(ROOT, "tests", "golden", "sponza_tris.npz"))
        return z["vertices"][z["triangles"].astype(np.int64)].astype(F)
    return scenes.create_n_cubes_tris(10_000, prec)


def points(tris, rng):
    F = tris.dtype.type
    t = tris.astype(np.float64)
    lo, hi = t.reshape(-1, 3).min(0), t.reshape(-1, 3).max(0)
    ext = float((hi - lo).max())
    h = N_POINTS // 2
    i = rng.integers(0, len(t), h)
    w = rng.dirichlet(np.ones(3), h)
    surf = np.einsum("mj,mjk->mk", w, t[i]) + rng.normal(size=(h, 3)) * 0.01 * ext
    uni = rng.uniform(lo, hi, (N_POINTS - h, 3))
    return np.ascontiguousarray(np.concatenate([surf, uni]).astype(F)), ext


def run(name, prec, ctx, stream, dev):
    import torch

    dt = torch.float32 if prec == "f32" else torch.float64
    tris = scene_tris(name, prec)
    pts, ext = points(tris, np.random.default_rng(1))
    b = api.Bvh.build(scenes_aabbs(tris, prec), prec=prec, ctx=ctx)
    b.set_triangles(tris)
    d_p = torch.from_numpy(pts).to(dev)
    radius = 0.01 * ext
    d_r = torch.full((N_POINTS,), radius, dtype=dt, device=dev)
    out = {"triangles": len(tris), "points": N_POINTS, "radius": radius}
    _, nd = b.nearest_triangles_batch(pts)
    out["nearest_triangles_kernel_ms"] = kernel_ms(lambda: b.nearest_triangles_batch(pts), "nearest_kernel")
    for k in (1, 8, 32, 64):
        d_s = torch.empty(N_POINTS * k, dtype=torch.int32, device=dev)
        d_d = torch.empty(N_POINTS * k, dtype=dt, device=dev)
        d_q = torch.empty(N_POINTS * k * 3, dtype=dt, device=dev)
        for lim, tag in ((None, "none"), (d_r, "radius")):
            r_ptr = lim.data_ptr() if lim is not None else 0

            def call():
                b.knn_triangles_dev(d_p.data_ptr(), N_POINTS, k, r_ptr, d_s.data_ptr(), d_d.data_ptr(), d_q.data_ptr())

            def box():
                b.knn_dev(d_p.data_ptr(), N_POINTS, k, r_ptr, d_s.data_ptr(), d_d.data_ptr())

            row = {"event_ms": round(timed(call, stream, reps=5), 3), "kernel_ms": kernel_ms(call, "knn_tri_kernel"),
                   "box_knn_kernel_ms": kernel_ms(box, "knn_kernel")}
            call()
            stream.synchronize()
            found = (d_s.view(N_POINTS, k) != -1).sum(1).float()
            row["mean_found"] = round(float(found.mean()), 2)
            if k == 1 and lim is None:
                row["k1_dist_equals_nearest_triangles"] = float(np.mean(d_d.cpu().numpy() == nd))
            out[f"k{k}_{tag}"] = row
    b.free()
    return out


def scenes_aabbs(tris, prec):
    """The triangles' own boxes (vertex min / max), as Triangle::new builds them."""
    from bvh_b200.dtypes import BY_PREC

    a = np.zeros(len(tris), dtype=BY_PREC[prec]["aabb"])
    a["min"], a["max"] = tris.min(axis=1), tris.max(axis=1)
    return a


def main():
    import torch

    name, power = card()
    dev = torch.device("cuda", 0)
    ctx = api.Context.default()
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    res = {"card": name, "power_limit": power}
    with torch.cuda.stream(stream):
        for scene in ("sponza", "cubes"):
            for prec in ("f32", "f64"):
                res[f"{scene}_{prec}"] = run(scene, prec, ctx, stream, dev)
    ctx.set_stream(None)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
