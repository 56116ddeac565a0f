#!/usr/bin/env python
"""Crossing counts, point-in-mesh and signed distance against the workaround a caller had before them (DESIGN.md section 4.21).
Scenes: the 120 k triangles of BASELINE.json configs[1] (scenes.create_n_cubes_tris(10 000)) with 2^20 rays of the create_ray chain and
2^18 points around random cubes; Sponza (tests/golden/sponza_tris.npz) with its 512 x 512 primary rays (scenes.pinhole_rays) and 2^18
points in its bounding box.  f32 and f64, device pointers, CUDA events on the context's stream, median of 5 after one warm-up call:
    count_hits_dev        against traverse_dev (BVH semantics, capacity sized by one untimed call) + Moeller-Trumbore in both windings
                          over every candidate in torch + a segmented sum (index_add_)
    contains_dev          against the same workaround on the 3 n rays of the points (built by bvhgpu_rays_new_dev_*) + the vote
    signed_distance_dev   against knn_triangles_dev (k = 1) + the contains workaround + the sign
Prints one JSON line with the card name and its power limit, read in the same call, and whether the workaround's counts equal
count_hits' (torch evaluates one operation per kernel, so without FMA contraction).

    python tools/crossings_probe.py
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bvh_b200 import api, scenes  # noqa: E402
from bvh_b200.dtypes import BY_PREC  # noqa: E402
from tools.dim_query_probe import card, timed  # noqa: E402

DIRS = np.array([[0.7548776662466927, 0.5698402909980532, 0.3247179572447460], [-0.5698402909980532, 0.3247179572447460, 0.7548776662466927],
                 [0.3247179572447460, -0.7548776662466927, 0.5698402909980532]])     # BVHGPU_CONTAINS_DIRECTIONS


def scene(name, prec, rng):
    F = np.float32 if prec == "f32" else np.float64
    if name == "sponza":
        z = np.load(os.path.join(ROOT, "tests", "golden", "sponza_tris.npz"))
        tris = z["vertices"][z["triangles"].astype(np.int64)].astype(F)
        o, d = scenes.pinhole_rays(512, 512, prec)
        lo, hi = tris.reshape(-1, 3).min(axis=0), tris.reshape(-1, 3).max(axis=0)
        pts = rng.uniform(lo, hi, (1 << 18, 3))
    else:
        tris = scenes.create_n_cubes_tris(10_000, prec)
        o, d = scenes.ray_endpoints(1 << 20, prec=prec)
        c = tris.reshape(-1, 12, 3, 3).mean(axis=(1, 2))
        pts = c[rng.integers(0, len(c), 1 << 18)] + rng.uniform(-1, 1, (1 << 18, 3))
    return tris, o, d, pts.astype(F)


def _mt(o, d, a, b, c, eps):
    """Ray::intersects_triangle hit mask in torch, one operation per kernel."""
    import torch

    def cross(x, y):
        return torch.stack([x[:, 1] * y[:, 2] - x[:, 2] * y[:, 1], x[:, 2] * y[:, 0] - x[:, 0] * y[:, 2], x[:, 0] * y[:, 1] - x[:, 1] * y[:, 0]], 1)

    def dot(x, y):
        return (x[:, 0] * y[:, 0] + x[:, 1] * y[:, 1]) + x[:, 2] * y[:, 2]

    ab, ac = b - a, c - a
    uvec = cross(d, ac)
    det = dot(ab, uvec)
    inv_det = 1.0 / det
    ao = o - a
    u = dot(ao, uvec) * inv_det
    vvec = cross(ao, ab)
    v = dot(d, vvec) * inv_det
    dist = dot(ac, vvec) * inv_det
    return (det >= eps) & (u >= 0) & (u <= 1) & (v >= 0) & (u + v <= 1) & (dist > eps)


class Workaround:
    """traverse_dev into a CSR sized once, then both windings over every candidate and a segmented sum."""

    def __init__(self, bvh, d_rays, n, tris_t, dev):
        import torch

        self.bvh, self.d_rays, self.n, self.tris, self.dev = bvh, d_rays, n, tris_t, dev
        self.off = torch.empty(n + 1, dtype=torch.int32, device=dev)
        self.total = bvh.traverse_dev(d_rays.data_ptr(), n, self.off.data_ptr(), 0, 0, want_total=True)
        self.hits = torch.empty(max(self.total, 1), dtype=torch.int32, device=dev)
        self.eps = float(np.finfo(np.float32 if tris_t.dtype == torch.float32 else np.float64).eps)

    def __call__(self):
        import torch

        self.bvh.traverse_dev(self.d_rays.data_ptr(), self.n, self.off.data_ptr(), self.hits.data_ptr(), self.total)
        rays = self.d_rays.view(self.tris.dtype).view(self.n, 9)
        counts = torch.diff(self.off.long())
        r = torch.repeat_interleave(torch.arange(self.n, device=self.dev), counts, output_size=self.total)
        t = self.tris[self.hits[: self.total].long()]
        o, d = rays[r, 0:3], rays[r, 3:6]
        front = torch.zeros(self.n, dtype=torch.int32, device=self.dev).index_add_(0, r, _mt(o, d, t[:, 0:3], t[:, 3:6], t[:, 6:9], self.eps).int())
        back = torch.zeros(self.n, dtype=torch.int32, device=self.dev).index_add_(0, r, _mt(o, d, t[:, 0:3], t[:, 6:9], t[:, 3:6], self.eps).int())
        return front, back


def run(name, prec, ctx, stream, dev):
    import torch

    dt = torch.float32 if prec == "f32" else torch.float64
    rng = np.random.default_rng(7)
    tris, o, d, pts = scene(name, prec, rng)
    a = np.zeros(len(tris), dtype=BY_PREC[prec]["aabb"])
    a["min"], a["max"] = tris.min(axis=1), tris.max(axis=1)
    b = api.Bvh.build(a, prec=prec, ctx=ctx)
    b.set_triangles(tris.reshape(-1, 9))
    tris_t = torch.from_numpy(np.ascontiguousarray(tris.reshape(-1, 9))).to(dev)
    rays = api.Ray.new(o, d, prec=prec, ctx=ctx)
    n, m = len(rays), len(pts)
    d_r = torch.from_numpy(rays.view(np.uint8).reshape(-1).copy()).to(dev)
    d_p = torch.from_numpy(pts).to(dev)
    prays = api.Ray.new(np.repeat(pts, 3, axis=0), np.tile(DIRS, (m, 1)), prec=prec, ctx=ctx)
    d_pr = torch.from_numpy(prays.view(np.uint8).reshape(-1).copy()).to(dev)
    f = torch.empty(3 * max(n, m), dtype=torch.int32, device=dev)
    k = torch.empty(3 * max(n, m), dtype=torch.int32, device=dev)
    ins = torch.empty(m, dtype=torch.uint8, device=dev)
    s = torch.empty(m, dtype=torch.int32, device=dev)
    dist = torch.empty(m, dtype=dt, device=dev)
    out = {"triangles": len(tris), "rays": n, "points": m}

    t_new = timed(lambda: b.count_hits_dev(d_r.data_ptr(), n, 0, f.data_ptr(), k.data_ptr()), stream, reps=5)
    wa = Workaround(b, d_r, n, tris_t, dev)
    t_wa = timed(wa, stream, reps=5)
    wf, wb = wa()
    same = bool(torch.equal(wf, f[:n]) and torch.equal(wb, k[:n]))
    out["count_hits"] = {"ms": round(t_new, 3), "workaround_ms": round(t_wa, 3), "speedup": round(t_wa / t_new, 2), "candidates": wa.total,
                         "crossings": int(f[:n].sum() + k[:n].sum()), "workaround_equal": same}
    del wa

    t_in = timed(lambda: b.contains_dev(d_p.data_ptr(), m, ins.data_ptr()), stream, reps=5)
    wp = Workaround(b, d_pr, 3 * m, tris_t, dev)

    def contains_wa():
        pf, pb = wp()
        return (((pf + pb) & 1).view(m, 3).sum(1) >= 2).to(torch.uint8)

    t_inw = timed(contains_wa, stream, reps=5)
    same_in = bool(torch.equal(contains_wa(), ins))
    out["contains"] = {"ms": round(t_in, 3), "workaround_ms": round(t_inw, 3), "speedup": round(t_inw / t_in, 2), "inside": int(ins.sum()),
                       "candidates": wp.total, "workaround_equal": same_in}

    t_sd = timed(lambda: b.signed_distance_dev(d_p.data_ptr(), m, s.data_ptr(), dist.data_ptr()), stream, reps=5)
    ws, wd = torch.empty_like(s), torch.empty_like(dist)

    def signed_wa():
        b.knn_triangles_dev(d_p.data_ptr(), m, 1, 0, ws.data_ptr(), wd.data_ptr())
        inside = contains_wa().bool() & (ws != -1)
        return torch.where(inside, -wd, wd)

    t_sdw = timed(signed_wa, stream, reps=5)
    out["signed_distance"] = {"ms": round(t_sd, 3), "workaround_ms": round(t_sdw, 3), "speedup": round(t_sdw / t_sd, 2)}
    del wp
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
