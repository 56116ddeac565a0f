#!/usr/bin/env python
"""Triangle pairs against the floating-point workaround (DESIGN.md section 5), device-pointer forms, CUDA events on the context's
stream, median of 5 after one warm-up call:
- triangle_pairs_dev (self, skip_shared = 0) and triangle_pairs_with_dev (against a translated copy): the overlap walk with the exact
  predicate at the leaves;
- the workaround: overlap_pairs_dev / overlap_pairs_with_dev, then a gather of both triangles of every candidate pair and a vectorised
  Moeller triangle-triangle test in torch, in the tree's precision (interval test on the planes' line, 2-D edge and containment tests
  for coplanar pairs).
Also printed per row: the candidate (box) pairs, the pairs past the plane filter (neither triangle's plane separates the other by
Shewchuk's orient3d bound, no shared vertex: the pairs that reach the full predicate), and the pairs on which the workaround's answer
differs from the exact one.  Scenes: the 120 k cube triangles of BASELINE.json configs[1] and the 66 450 Sponza triangles, f32 and
f64; the copy is shifted by 0.5 (cubes) or 1e-3 of the extent (Sponza).  One JSON line with the card name and its power limit, read in
the same call.

    python tools/triangle_pairs_probe.py
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
from tools.overlap_probe import timed  # noqa: E402


def sponza_tris(prec):
    z = np.load(os.path.join(ROOT, "tests", "golden", "sponza_tris.npz"))
    return z["vertices"][z["triangles"].astype(np.int64)].astype(BY_PREC[prec]["scalar"])


def tree(tris, prec, ctx):
    a = np.zeros(len(tris), dtype=BY_PREC[prec]["aabb"])
    a["min"], a["max"] = tris.min(axis=1), tris.max(axis=1)
    b = api.Bvh.build(a, prec=prec, ctx=ctx)
    b.set_triangles(tris)
    return b


def _cross(a, b):
    import torch

    return torch.cross(a, b, dim=-1)


def _orient2(a, b, c):
    return (a[..., 0] - c[..., 0]) * (b[..., 1] - c[..., 1]) - (a[..., 1] - c[..., 1]) * (b[..., 0] - c[..., 0])


def _coplanar(P, Q, n):
    """Moeller's coplanar branch: project along the largest normal component, then edge-edge crossings and vertex containment."""
    import torch

    ax = torch.argmax(n.abs(), dim=-1)
    keep = torch.tensor([[1, 2], [0, 2], [0, 1]], device=P.device)[ax]             # (m, 2)
    p = torch.gather(P, 2, keep[:, None, :].expand(-1, 3, -1))
    q = torch.gather(Q, 2, keep[:, None, :].expand(-1, 3, -1))
    hit = torch.zeros(len(P), dtype=torch.bool, device=P.device)
    for i in range(3):
        a, b = p[:, i], p[:, (i + 1) % 3]
        for j in range(3):
            c, d = q[:, j], q[:, (j + 1) % 3]
            d1, d2, d3, d4 = _orient2(c, d, a), _orient2(c, d, b), _orient2(a, b, c), _orient2(a, b, d)
            hit |= (d1 * d2 <= 0) & (d3 * d4 <= 0) & ~((d1 == 0) & (d2 == 0))
    for x, y in ((p, q), (q, p)):
        s = [_orient2(y[:, k], y[:, (k + 1) % 3], x[:, 0]) for k in range(3)]
        hit |= ((s[0] >= 0) & (s[1] >= 0) & (s[2] >= 0)) | ((s[0] <= 0) & (s[1] <= 0) & (s[2] <= 0))
    return hit


def _interval(v, d):
    """Moeller's compute_intervals: the segment of the triangle on the planes' line, projected values v (m, 3), distances d (m, 3)."""
    import torch

    d0, d1, d2 = d.unbind(-1)
    iso = torch.where(d0 * d1 > 0, 2, torch.where(d0 * d2 > 0, 1, torch.where((d1 * d2 > 0) | (d0 != 0), 0, torch.where(d1 != 0, 1, 2))))
    j, k = (iso + 1) % 3, (iso + 2) % 3
    g = lambda t, i: torch.gather(t, 1, i[:, None])[:, 0]      # noqa: E731
    vi, vj, vk, di, dj, dk = g(v, iso), g(v, j), g(v, k), g(d, iso), g(d, j), g(d, k)
    t1 = vj + (vi - vj) * dj / (dj - di)
    t2 = vk + (vi - vk) * dk / (dk - di)
    return torch.minimum(t1, t2), torch.maximum(t1, t2)


def moeller(P, Q):
    """Moeller's triangle-triangle test (no epsilon) over (m, 3, 3) tensors: True where it reports an intersection."""
    import torch

    n1 = _cross(P[:, 1] - P[:, 0], P[:, 2] - P[:, 0])
    dq = ((Q - P[:, :1]) * n1[:, None]).sum(-1)
    n2 = _cross(Q[:, 1] - Q[:, 0], Q[:, 2] - Q[:, 0])
    dp = ((P - Q[:, :1]) * n2[:, None]).sum(-1)
    sep = ((dq > 0).all(1) | (dq < 0).all(1) | (dp > 0).all(1) | (dp < 0).all(1))
    cop = (dq == 0).all(1)
    dline = _cross(n1, n2)
    ax = torch.argmax(dline.abs(), dim=-1)
    vp = torch.gather(P, 2, ax[:, None, None].expand(-1, 3, 1))[..., 0]
    vq = torch.gather(Q, 2, ax[:, None, None].expand(-1, 3, 1))[..., 0]
    a0, a1 = _interval(vp, dp)
    b0, b1 = _interval(vq, dq)
    line = ~((a1 < b0) | (b1 < a0))
    return ~sep & torch.where(cop, _coplanar(P, Q, n1), line)


def _rows(d_off, n, total):
    import torch

    counts = (d_off[1:n + 1] - d_off[:n]).long()
    return torch.repeat_interleave(torch.arange(n, device=d_off.device), counts, output_size=total)


def plane_filter_survivors(PA, PB, s, t):
    """Candidate pairs without a shared vertex that no plane separates by the orient3d filter (the pairs reaching the predicate)."""
    from tests import tritri as T

    P, Q = PA[s].astype(np.float64), PB[t].astype(np.float64)
    shared = np.any(np.all(P[:, :, None, :] == Q[:, None, :, :], axis=-1), axis=(1, 2))
    sep = T._separated(P, Q) | T._separated(Q, P)
    return int(np.count_nonzero(~shared & ~sep))


def one(name, tris, shift, prec, ctx, stream):
    import torch

    dev = torch.device("cuda", 0)
    L = capi.lib()
    other = (tris + np.asarray(shift, dtype=tris.dtype)).astype(tris.dtype)
    a, b = tree(tris, prec, ctx), tree(other, prec, ctx)
    sfx = a._d["suffix"]
    n = len(tris)
    d_ta = torch.from_numpy(np.ascontiguousarray(tris)).to(dev)
    d_tb = torch.from_numpy(np.ascontiguousarray(other)).to(dev)
    out = []
    for form, cand_fn, exact_fn, args_c, args_e, tb in (
            ("self", "overlap_pairs_dev", "triangle_pairs_dev", (a._h,), (a._h, 0), d_ta),
            ("trees", "overlap_trees_dev", "triangle_pairs_trees_dev", (a._h, b._h), (a._h, b._h), d_tb)):
        fc, fe = getattr(L, f"bvhgpu_{cand_fn}_{sfx}"), getattr(L, f"bvhgpu_{exact_fn}_{sfx}")
        tot = C.c_size_t(0)
        d_off = torch.zeros(n + 1, dtype=torch.int32, device=dev)
        e_off = torch.zeros(n + 1, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        assert fc(*args_c, C.c_void_p(d_off.data_ptr()), None, 0, C.byref(tot)) in (capi.OK, capi.ERR_CAPACITY)
        cand = tot.value
        assert fe(*args_e, C.c_void_p(e_off.data_ptr()), None, 0, C.byref(tot)) in (capi.OK, capi.ERR_CAPACITY)
        exact = tot.value
        d_hits = torch.zeros(max(cand, 1), dtype=torch.int32, device=dev)
        e_hits = torch.zeros(max(exact, 1), dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        res = {}

        def run_exact():
            capi.check(fe(*args_e, C.c_void_p(e_off.data_ptr()), C.c_void_p(e_hits.data_ptr()), exact, None))

        def run_workaround():
            capi.check(fc(*args_c, C.c_void_p(d_off.data_ptr()), C.c_void_p(d_hits.data_ptr()), cand, None))
            with torch.cuda.stream(stream):
                s = _rows(d_off, n, cand)
                res["mask"] = moeller(d_ta[s], tb[d_hits[:cand].long()])

        t_e, t_w = timed(run_exact, stream), timed(run_workaround, stream)
        stream.synchronize()
        s = _rows(d_off, n, cand).cpu().numpy()
        t = d_hits[:cand].cpu().numpy().astype(np.int64)
        es = _rows(e_off, n, exact).cpu().numpy()
        et = e_hits[:exact].cpu().numpy().astype(np.int64)
        want = np.isin(s * (1 << 32) + t, es * (1 << 32) + et)
        wrong = int(np.count_nonzero(res["mask"].cpu().numpy() != want))
        out.append({"scene": name, "prec": prec, "form": form, "triangles": n, "candidates": cand, "pairs": exact,
                    "past_plane_filter": plane_filter_survivors(tris, tris if form == "self" else other, s, t),
                    "exact_ms": round(t_e, 3), "workaround_ms": round(t_w, 3), "workaround_wrong": wrong})
    a.free()
    b.free()
    return out


def main():
    import torch

    name, power = card()
    ctx = api.Context.default()
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    rows = []
    try:
        for prec in ("f32", "f64"):
            rows += one("configs1_cubes", scenes.create_n_cubes_tris(10_000, prec), 0.5, prec, ctx, stream)
            sp = sponza_tris(prec)
            ext = (sp.reshape(-1, 3).max(axis=0).astype(np.float64) - sp.reshape(-1, 3).min(axis=0)) * 1e-3
            rows += one("sponza", sp, ext, prec, ctx, stream)
    finally:
        ctx.set_stream(None)
    print(json.dumps({"card": name, "power_limit": power, "rows": rows}))


if __name__ == "__main__":
    main()
