#!/usr/bin/env python
"""Any hit against closest hit + threshold (DESIGN.md section 5), device-pointer forms, CUDA events on the context's stream, median
of 7 after one warm-up call:
- Sponza (tests/golden/sponza_tris.npz, f32): the 2048 x 2048 primary rays of scenes.pinhole_rays (BASELINE.json configs[2]'s camera)
  find their hit points with triangle-mode closest_hit_dev; from every hit point a shadow ray goes to a point light in the atrium
  (the centre of the scene's bounding box), tmax = the distance to the light.  any_hit_dev (triangle and AABB mode) against
  closest_hit_dev followed by `dist < tmax` on the same shadow rays, with the occluded fraction and how often the two answers agree;
- the 4-D scene of tools/dim_ordered_probe.py (1 M shapes, 1 M rays aimed at box centres), tmax = the distance to the aimed centre.
Prints one JSON line with the card name and its power limit, read in the same call.

    python tools/any_hit_probe.py
"""
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bvh_b200 import api, capi, scenes  # noqa: E402
from bvh_b200.dtypes import BY_PREC  # noqa: E402
from tools.dim_ordered_probe import scene as scene4  # noqa: E402
from tools.dim_query_probe import card, timed  # noqa: E402

INVALID = -1                                             # BVHGPU_INVALID_INDEX seen through int32


def sponza(ctx, stream, dev):
    import torch

    z = np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "sponza_tris.npz"))
    tris = z["vertices"][z["triangles"].astype(np.int64)].astype(np.float32)
    sp = np.zeros(len(tris), dtype=BY_PREC["f32"]["aabb"])
    sp["min"], sp["max"] = tris.min(axis=1), tris.max(axis=1)
    b = api.Bvh.build(sp, ctx=ctx)
    b.set_triangles(tris.reshape(-1, 9))
    L = capi.lib()
    o, d = scenes.pinhole_rays(2048, 2048)
    prim = api.Ray.new(o, d, ctx=ctx)
    n = len(prim)
    d_prim = torch.from_numpy(prim.view(np.uint8).reshape(-1)).to(dev)
    d_s = torch.empty(n, dtype=torch.int32, device=dev)
    d_d = torch.empty(n, dtype=torch.float32, device=dev)
    capi.check(L.bvhgpu_closest_hit_dev_f32x3(b._h, C.c_void_p(d_prim.data_ptr()), capi.RAYS_FULL, n, 1, C.c_void_p(d_s.data_ptr()),
                                              C.c_void_p(d_d.data_ptr()), None))
    ctx.synchronize()
    s, t = d_s.cpu().numpy(), d_d.cpu().numpy()
    hit = s != INVALID
    light = (0.5 * (sp["min"].min(axis=0).astype(np.float64) + sp["max"].max(axis=0))).astype(np.float32)
    p = o[hit].astype(np.float64) + (t[hit, None].astype(np.float64) - 1e-3) * (prim["direction"][hit].astype(np.float64))   # just in front of the surface
    to_light = light.astype(np.float64) - p
    tmax = np.linalg.norm(to_light, axis=1).astype(np.float32)
    shadow = api.Ray.new(p.astype(np.float32), to_light.astype(np.float32), ctx=ctx)
    m = len(shadow)
    d_sh = torch.from_numpy(shadow.view(np.uint8).reshape(-1)).to(dev)
    d_tm = torch.from_numpy(tmax).to(dev)
    d_any = torch.empty(m, dtype=torch.int32, device=dev)
    d_cs = torch.empty(m, dtype=torch.int32, device=dev)
    d_cd = torch.empty(m, dtype=torch.float32, device=dev)
    out = {"primary_rays": n, "shadow_rays": m, "light": light.tolist()}
    for tri, name in ((1, "triangles"), (0, "aabb")):
        def any_hit():
            capi.check(L.bvhgpu_any_hit_dev_f32x3(b._h, C.c_void_p(d_sh.data_ptr()), capi.RAYS_FULL, m, C.c_void_p(d_tm.data_ptr()), tri,
                                                  C.c_void_p(d_any.data_ptr())))

        def closest_threshold():
            capi.check(L.bvhgpu_closest_hit_dev_f32x3(b._h, C.c_void_p(d_sh.data_ptr()), capi.RAYS_FULL, m, tri, C.c_void_p(d_cs.data_ptr()),
                                                      C.c_void_p(d_cd.data_ptr()), None))
            closest_threshold.occluded = d_cd < d_tm

        t_any = timed(any_hit, stream, reps=7)
        t_cl = timed(closest_threshold, stream, reps=7)
        occ_any = (d_any != INVALID).cpu().numpy()
        occ_cl = closest_threshold.occluded.cpu().numpy()
        out[name] = {"any_hit_ms": round(t_any, 3), "closest_plus_threshold_ms": round(t_cl, 3),
                     "occluded_fraction": round(float(occ_any.mean()), 4), "agree_fraction": float((occ_any == occ_cl).mean())}
    b.free()
    return out


def four_d(ctx, stream, dev, prec):
    import torch

    F = np.float32 if prec == "f32" else np.float64
    t = api.Bvh4._TABLE[prec]
    rng = np.random.default_rng(4)
    mn, mx, o, d = scene4(4, F, rng)
    a = np.zeros(len(mn), dtype=t["aabb"])
    a["min"], a["max"] = mn, mx
    rays = np.zeros(len(o), dtype=t["ray"])
    with np.errstate(divide="ignore"):
        rays["origin"], rays["direction"], rays["inv_direction"] = o, d, (F(1) / d).astype(F)
    rng = np.random.default_rng(4)                    # scene4's own draws, again, for the aimed centres
    _mn = rng.uniform(-1000, 1000, (len(mn), 4))
    _mx = _mn + rng.uniform(0, 4, (len(mn), 4))
    _o = rng.uniform(-1100, 1100, (len(o), 4))
    tgt = rng.integers(0, len(mn), len(o))
    tmax = np.linalg.norm(0.5 * (_mn[tgt] + _mx[tgt]) - _o, axis=1).astype(F)
    b = api.Bvh4.build(a, prec=prec, ctx=ctx)
    m = len(rays)
    dt = torch.float32 if prec == "f32" else torch.float64
    d_r = torch.from_numpy(rays.view(np.uint8)).to(dev)
    d_tm = torch.from_numpy(tmax).to(dev)
    d_any = torch.empty(m, dtype=torch.int32, device=dev)
    d_cs = torch.empty(m, dtype=torch.int32, device=dev)
    d_cd = torch.empty(m, dtype=dt, device=dev)

    def closest_threshold():
        b.closest_hit_dev(d_r.data_ptr(), m, d_cs.data_ptr(), d_cd.data_ptr())
        closest_threshold.occluded = d_cd < d_tm

    t_any = timed(lambda: b.any_hit_dev(d_r.data_ptr(), m, d_tm.data_ptr(), d_any.data_ptr()), stream, reps=7)
    t_cl = timed(closest_threshold, stream, reps=7)
    occ_any = (d_any != INVALID).cpu().numpy()
    occ_cl = closest_threshold.occluded.cpu().numpy()
    b.free()
    return {"shapes": len(mn), "rays": m, "any_hit_ms": round(t_any, 3), "closest_plus_threshold_ms": round(t_cl, 3),
            "occluded_fraction": round(float(occ_any.mean()), 4), "agree_fraction": float((occ_any == occ_cl).mean())}


def main():
    import torch

    name, power = card()
    dev = torch.device("cuda", 0)
    ctx = api.Context.default()
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    res = {"card": name, "power_limit": power}
    with torch.cuda.stream(stream):
        res["sponza_f32"] = sponza(ctx, stream, dev)
        for prec in ("f32", "f64"):
            res[f"4d_{prec}"] = four_d(ctx, stream, dev, prec)
    ctx.set_stream(None)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
