#!/usr/bin/env python
"""Multi hit against closest hit on the same rays (DESIGN.md section 5).  Two scenes: the 120 k triangles of BASELINE.json configs[1]
(scenes.create_n_cubes_tris(10 000)) with 1 M rays of the create_ray chain (scenes.ray_endpoints), and Sponza (tests/golden/sponza_tris.npz,
66 450 triangles) with the 1024 x 1024 primary rays of scenes.pinhole_rays.  f32 and f64, triangle and AABB mode, k in {1, 4, 16, 64},
no limit: bvhgpu_multi_hit_dev_* and bvhgpu_closest_hit_dev_* on device pointers (FULL rays, uv written), CUDA events on the context's
stream, median of 5 after one warm-up call.  Prints one JSON line with the card name and its power limit, read in the same call.

    python tools/multi_hit_probe.py
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
from tools.dim_query_probe import card, timed  # noqa: E402


def scene(name, prec):
    F = np.float32 if prec == "f32" else np.float64
    if name == "sponza":
        z = np.load(os.path.join(ROOT, "tests", "golden", "sponza_tris.npz"))
        tris = z["vertices"][z["triangles"].astype(np.int64)].astype(F)
        o, d = scenes.pinhole_rays(1024, 1024, prec)
    else:
        tris = scenes.create_n_cubes_tris(10_000, prec)
        o, d = scenes.ray_endpoints(1_000_000, prec=prec)
    return tris, o, d


def run(name, prec, ctx, stream, dev):
    import torch

    dt = torch.float32 if prec == "f32" else torch.float64
    suf = BY_PREC[prec]["suffix"]
    L = capi.lib()
    tris, o, d = scene(name, prec)
    a = np.zeros(len(tris), dtype=BY_PREC[prec]["aabb"])
    a["min"], a["max"] = tris.min(axis=1), tris.max(axis=1)
    b = api.Bvh.build(a, prec=prec, ctx=ctx)
    b.set_triangles(tris.reshape(-1, 9))
    rays = api.Ray.new(o, d, prec=prec, ctx=ctx)
    n = len(rays)
    d_r = torch.from_numpy(rays.view(np.uint8).reshape(-1)).to(dev)
    out = {"triangles": len(tris), "rays": n}
    for tri, mode in ((1, "triangles"), (0, "aabb")):
        d_s = torch.empty(n, dtype=torch.int32, device=dev)
        d_d = torch.empty(n, dtype=dt, device=dev)
        d_uv = torch.empty(2 * n, dtype=dt, device=dev)
        closest = getattr(L, f"bvhgpu_closest_hit_dev_{suf}")
        t_cl = timed(lambda: capi.check(closest(b._h, C.c_void_p(d_r.data_ptr()), capi.RAYS_FULL, n, tri, C.c_void_p(d_s.data_ptr()),
                                                C.c_void_p(d_d.data_ptr()), C.c_void_p(d_uv.data_ptr()))), stream, reps=5)
        row = {"closest_hit_ms": round(t_cl, 3), "hit_fraction": round(float((d_s != -1).float().mean()), 4)}
        del d_s, d_d, d_uv
        for k in (1, 4, 16, 64):
            m_s = torch.empty(n * k, dtype=torch.int32, device=dev)
            m_d = torch.empty(n * k, dtype=dt, device=dev)
            m_uv = torch.empty(2 * n * k, dtype=dt, device=dev)
            t = timed(lambda: b.multi_hit_dev(d_r.data_ptr(), n, k, 0, m_s.data_ptr(), m_d.data_ptr(), m_uv.data_ptr(), triangles=bool(tri)),
                      stream, reps=5)
            found = (m_s.view(n, k) != -1).sum(1).float()
            row[f"k{k}"] = {"ms": round(t, 3), "ratio_to_closest_hit": round(t / t_cl, 3), "mean_found": round(float(found.mean()), 3)}
            del m_s, m_d, m_uv
        out[mode] = row
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
        for sc in ("cubes", "sponza"):
            for prec in ("f32", "f64"):
                res[f"{sc}_{prec}"] = run(sc, prec, ctx, stream, dev)
    ctx.set_stream(None)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
