"""tests/crossings.py -- restatement of the crossing counts, the point-in-mesh vote and the signed distance (crossings_kernel and
apply_sign_kernel, closest.cu), vectorised with numpy.float32 / numpy.float64 arrays: one rounding per operation, no FMA, so every
value is the device's bit for bit.  TEST INFRASTRUCTURE: pinned to the C++ oracle by tests/test_crossings_cpu.py and compared with the
device by tests/test_gpu_crossings.py.

    mt(o, d, a, b, c)            Ray::intersects_triangle (Moeller-Trumbore with back-face culling), the distance or +inf;
                                 mt(o, d, a, c, b) is the back-face test, the same function
    counts_csr                   (front, back) of the loop over a candidate CSR (Bvh::traverse's set), with an optional limit
    bounded_rows                 per ray: every triangle the loop counts is bounded (stored box entered at <= fl(d * (1 + 2^-16)))
    counts_brute                 (front, back) over every triangle
    directions / point_rays      BVHGPU_CONTAINS_DIRECTIONS of the header, Ray::new(p, D_j) as bvhgpu_rays_new_dev_* computes it
    vote                         inside per point from the (3 n,) counts of its three rays, EVEN_ODD or NONZERO
    signed                       the sign composition over a knn_triangles(k = 1) row"""
import os
import re

import numpy as np

U32_MAX = 0xFFFFFFFF
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EVEN_ODD, NONZERO = 0, 1


def _eps(F):
    return F(np.finfo(F).eps)


def _cross(a, b):
    return (a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
            a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0])


def _dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def mt(o, d, a, b, c):
    """Ray::intersects_triangle over arrays (m, 3) of one float type: the distance (m,), +inf for a miss or a back face.  Every check of
    the reference is evaluated; a miss at an earlier one can never be undone by a later one, so the result is the sequential one."""
    F = o.dtype.type
    eps = _eps(F)
    with np.errstate(all="ignore"):
        ab, ac = b - a, c - a
        uvec = np.stack(_cross(d, ac), axis=-1)
        det = _dot([ab[..., k] for k in range(3)], [uvec[..., k] for k in range(3)])
        miss = det < eps
        inv_det = F(1) / det
        ao = o - a
        u = _dot([ao[..., k] for k in range(3)], [uvec[..., k] for k in range(3)]) * inv_det
        miss |= ~((u >= F(0)) & (u <= F(1)))
        vvec = _cross(ao, ab)
        v = _dot([d[..., k] for k in range(3)], vvec) * inv_det
        miss |= (v < F(0)) | (u + v > F(1))
        dist = _dot([ac[..., k] for k in range(3)], vvec) * inv_det
        miss |= ~(dist > eps)
    return np.where(miss, F(np.inf), dist).astype(F)


def _rows(offsets):
    off = np.asarray(offsets, dtype=np.int64)
    return np.repeat(np.arange(len(off) - 1), np.diff(off))


def _windings(rays, tris, r, s):
    o, d = rays["origin"][r], rays["direction"][r]
    t = tris[s]
    return mt(o, d, t[:, 0], t[:, 1], t[:, 2]), mt(o, d, t[:, 0], t[:, 2], t[:, 1])


def _limit(tmax, F, m):
    return np.full(m, np.inf, dtype=F) if tmax is None else np.broadcast_to(np.asarray(tmax, dtype=F), (m,))


def counts_csr(rays, tris, offsets, hits, tmax=None):
    """(front, back) u32 of the loop over the CSR (offsets, hits) of candidate shapes: d < tmax[r] (+inf without a limit)."""
    F = rays["origin"].dtype.type
    tris = np.ascontiguousarray(tris, dtype=F).reshape(-1, 3, 3)
    r = _rows(offsets)
    s = np.asarray(hits, dtype=np.int64)
    lim = _limit(tmax, F, len(rays))
    df, db = _windings(rays, tris, r, s)
    m = len(rays)
    return (np.bincount(r[df < lim[r]], minlength=m).astype(np.uint32), np.bincount(r[db < lim[r]], minlength=m).astype(np.uint32))


def slab(o, inv, mn, mx):
    """Ray::intersection_slice_for_aabb as slab_slice evaluates it, over arrays: (hit, entry clamped at 0)."""
    F = o.dtype.type
    with np.errstate(all="ignore"):
        l, rr = (mn - o) * inv, (mx - o) * inv
    nan = np.isnan(l).any(axis=-1) | np.isnan(rr).any(axis=-1)
    lo, hi = np.minimum(l, rr), np.maximum(l, rr)
    tmin = np.maximum(np.maximum(lo[..., 0], lo[..., 1]), lo[..., 2])
    tmax = np.minimum(np.minimum(hi[..., 0], hi[..., 1]), hi[..., 2])
    entry = np.where(tmin > F(0), tmin, F(0)).astype(F)
    return ~nan & ~(entry > tmax), entry


def stored_boxes(nodes, shapes):
    """(min, max) (n, 3) of the box the walk tests last before each shape's leaf: its parent's child box, the own box at a root leaf."""
    n = len(shapes)
    mn, mx = shapes["min"].copy(), shapes["max"].copy()
    if n < 2:
        return mn, mx
    inner = nodes["child_l"] != U32_MAX
    for side, key in (("child_l", "l_aabb"), ("child_r", "r_aabb")):
        c = nodes[side][inner].astype(np.int64)
        leaf = nodes["child_l"][c] == U32_MAX
        s = nodes["shape"][c[leaf]].astype(np.int64)
        mn[s], mx[s] = nodes[key]["min"][inner][leaf], nodes[key]["max"][inner][leaf]
    return mn, mx


def bounded_rows(rays, tris, nodes, shapes, offsets, hits, tmax):
    """Per ray: every (triangle, winding) the loop over the CSR counts under the limit is bounded: the box its parent stores for it
    passes the slab test with entry <= fl(d * (1 + 2^-16))."""
    F = rays["origin"].dtype.type
    tris = np.ascontiguousarray(tris, dtype=F).reshape(-1, 3, 3)
    r = _rows(offsets)
    s = np.asarray(hits, dtype=np.int64)
    lim = _limit(tmax, F, len(rays))
    smn, smx = stored_boxes(nodes, shapes)
    hit, e = slab(rays["origin"][r], rays["inv_direction"][r], smn[s], smx[s])
    margin = F(1) + F(1.0 / 65536.0)
    ok = np.ones(len(rays), dtype=bool)
    for d in _windings(rays, tris, r, s):
        with np.errstate(all="ignore"):
            bad = (d < lim[r]) & ~(hit & (e <= d * margin))
        ok[r[bad]] = False
    return ok


def counts_brute(rays, tris, tmax=None, chunk=1 << 22):
    """(front, back) over every triangle, chunked over (ray, triangle) pairs."""
    F = rays["origin"].dtype.type
    tris = np.ascontiguousarray(tris, dtype=F).reshape(-1, 3, 3)
    m, n = len(rays), len(tris)
    lim = _limit(tmax, F, m)
    front, back = np.zeros(m, dtype=np.uint32), np.zeros(m, dtype=np.uint32)
    step = max(1, chunk // max(n, 1))
    for r0 in range(0, m, step):
        r = np.repeat(np.arange(r0, min(m, r0 + step)), n)
        s = np.tile(np.arange(n), min(m, r0 + step) - r0)
        df, db = _windings(rays, tris, r, s)
        front[r0:r0 + step] += np.bincount(r[df < lim[r]] - r0, minlength=min(m, r0 + step) - r0).astype(np.uint32)
        back[r0:r0 + step] += np.bincount(r[db < lim[r]] - r0, minlength=min(m, r0 + step) - r0).astype(np.uint32)
    return front, back


def directions():
    """BVHGPU_CONTAINS_DIRECTIONS of include/bvh_b200.h as (3, 3) float64 literals."""
    text = open(os.path.join(ROOT, "include", "bvh_b200.h")).read()
    body = re.search(r"#define BVHGPU_CONTAINS_DIRECTIONS((?:.*\\\n)*.*)", text).group(1)
    vals = [float(x) for x in re.findall(r"-?\d+\.\d+(?:[eE][-+]?\d+)?", body)]
    assert len(vals) == 9, vals
    return np.array(vals).reshape(3, 3)


def point_rays(points, F):
    """The 3 n rays of contains, point-major (ray 3 i + j = Ray::new(p_i, D_j)), as the Ray record of F with the arithmetic of
    rays_new_kernel: nrm = sqrt((dx dx + dy dy) + dz dz), d = D / nrm, inv = 1 / d."""
    from bvh_b200.dtypes import BY_PREC

    p = np.ascontiguousarray(points, dtype=F).reshape(-1, 3)
    D = directions().astype(F)
    nrm = np.sqrt((D[:, 0] * D[:, 0] + D[:, 1] * D[:, 1]) + D[:, 2] * D[:, 2])
    d = (D / nrm[:, None]).astype(F)
    rays = np.zeros(3 * len(p), dtype=BY_PREC["f32" if F == np.float32 else "f64"]["ray"])
    rays["origin"] = np.repeat(p, 3, axis=0)
    rays["direction"] = np.tile(d, (len(p), 1))
    rays["inv_direction"] = np.tile((F(1) / d).astype(F), (len(p), 1))
    return rays


def ray_votes(front, back, rule):
    """(3 n,) bool: each ray's vote."""
    f, b = np.asarray(front, dtype=np.int64), np.asarray(back, dtype=np.int64)
    return ((f + b) & 1) == 1 if rule == EVEN_ODD else b != f


def vote(front, back, rule):
    """(n,) bool: at least two of the three rays of each point vote inside."""
    return ray_votes(front, back, rule).reshape(-1, 3).sum(axis=1) >= 2


def signed(shape, dist, inside):
    """knn_triangles(k = 1) distances negated where inside and a triangle was found."""
    dist = np.array(dist, copy=True)
    flip = np.asarray(inside, dtype=bool) & (np.asarray(shape) != U32_MAX)
    dist[flip] = -dist[flip]
    return dist


# ---- analytic closed meshes, outward winding -----------------------------------------------------------------------------------------
def icosphere(level=2, F=np.float64):
    """Unit icosphere, (m, 3, 3), counter-clockwise seen from outside."""
    t = (1 + 5 ** 0.5) / 2
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t), (t, 0, -1), (t, 0, 1),
         (-t, 0, -1), (-t, 0, 1)]
    v = [np.array(x, dtype=np.float64) / np.linalg.norm(x) for x in v]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6), (7, 1, 8), (3, 9, 4),
         (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7), (9, 8, 1)]
    tris = np.array([[v[a], v[b], v[c]] for a, b, c in f])
    for _ in range(level):
        a, b, c = tris[:, 0], tris[:, 1], tris[:, 2]
        ab, bc, ca = [(x + y) / np.linalg.norm(x + y, axis=1, keepdims=True) for x, y in ((a, b), (b, c), (c, a))]
        tris = np.concatenate([np.stack(q, axis=1) for q in ((a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca))])
    return tris.astype(F)


def torus(R=1.0, r=0.4, nu=48, nv=24, F=np.float64):
    """Torus around z, (2 nu nv, 3, 3), counter-clockwise seen from outside."""
    u = np.arange(nu) * 2 * np.pi / nu
    v = np.arange(nv) * 2 * np.pi / nv

    def P(i, j):
        uu, vv = u[i % nu], v[j % nv]
        return np.array([(R + r * np.cos(vv)) * np.cos(uu), (R + r * np.cos(vv)) * np.sin(uu), r * np.sin(vv)])

    out = []
    for i in range(nu):
        for j in range(nv):
            a, b, c, d = P(i, j), P(i + 1, j), P(i + 1, j + 1), P(i, j + 1)
            out += [(a, b, c), (a, c, d)]
    return np.array(out).astype(F)


def outward(tris):
    """Fraction of triangles whose normal (b - a) x (c - a) points away from the origin (1.0 for the icosphere)."""
    t = np.asarray(tris, dtype=np.float64)
    n = np.cross(t[:, 1] - t[:, 0], t[:, 2] - t[:, 0])
    return float(np.mean(np.einsum("ij,ij->i", n, t.mean(axis=1)) > 0))
