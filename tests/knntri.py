"""tests/knntri.py -- models of the k-nearest-triangles query (bvhgpu_knn_triangles_*), numpy.float32 / numpy.float64, one rounding per
operation in the reference's order (elementwise numpy ops on T arrays round once in T; no FMA).

    closest     closest_point_triangle (testbase.rs:353-443) of one point against every triangle, vectorised over the triangles: the
                three repeated-vertex branches (closest_point_segment), then the seven Voronoi branches in the reference's order.
                Returns q (n, 3); key = dot(p - q, p - q) is Triangle::distance_squared.
    brute       the contract: s qualifies when key_s is not NaN and (no limit, or r >= 0 and key_s <= fl(r * r)); the row is the first k
                of a stable sort by (key_s, s), with fl(sqrt(key_s)) and q, then (U32_MAX, +inf, NaN x 3) padding.
    walk        knnref.Walk's restatement of knn_walk<3, T, K> with the triangle key at the leaves.
    bounded     per (point, triangle): not key_s < box_lower_d2(p, AABB_s) (queries.cuh's slacked bound of the triangle's own box); the
                walk can only lose a triangle where this is False.
"""
import numpy as np

from tests import knnref
from tests.prunedmodel import box_lower_d2 as box_lower_d2_scalar

U32_MAX = knnref.U32_MAX


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _segment(p, a, b):
    """closest_point_segment: a + clamp(dot(ab, ap) / dot(ab, ab), 0, 1) * ab."""
    F = a.dtype.type
    ab, ap = b - a, p - a
    s = _dot(ab, ap) / _dot(ab, ab)
    s = np.where(s < F(0), F(0), np.where(s > F(1), F(1), s)).astype(F)
    return a + s[:, None] * ab


def closest(p, tris):
    """q (n, 3) of closest_point_triangle(p, tri) for every triangle of tris (n, 3, 3); p is one point (3,) or one per triangle (n, 3)."""
    F = tris.dtype.type
    p = np.asarray(p, dtype=F)
    a, b, c = tris[:, 0], tris[:, 1], tris[:, 2]
    with np.errstate(all="ignore"):
        e_ab, e_bc, e_ac = (a == b).all(1), (b == c).all(1), (a == c).all(1)
        ab, ac, ap, bp, cp = b - a, c - a, p - a, p - b, p - c
        d1, d2, d3, d4, d5, d6 = _dot(ab, ap), _dot(ac, ap), _dot(ab, bp), _dot(ac, bp), _dot(ab, cp), _dot(ac, cp)
        vc, vb, va = d1 * d4 - d3 * d2, d5 * d2 - d1 * d6, d3 * d6 - d5 * d4
        v_ab = d1 / (d1 - d3)
        v_ac = d2 / (d2 - d6)
        x43, x56 = d4 - d3, d5 - d6
        v_bc = x43 / (x43 + x56)
        denom = F(1) / ((va + vb) + vc)
        v, w = vb * denom, vc * denom
        cands = [
            (e_ab & e_bc & e_ac, a),
            (e_ab, _segment(p, a, c)),
            (e_bc, _segment(p, a, b)),
            (e_ac, _segment(p, a, b)),
            ((d1 <= F(0)) & (d2 <= F(0)), a),
            ((d3 >= F(0)) & (d4 <= d3), b),
            ((d6 >= F(0)) & (d5 <= d6), c),
            ((vc <= F(0)) & (d1 >= F(0)) & (d3 <= F(0)), a + v_ab[:, None] * ab),
            ((vb <= F(0)) & (d2 >= F(0)) & (d6 <= F(0)), a + v_ac[:, None] * ac),
            ((va <= F(0)) & (x43 >= F(0)) & (x56 >= F(0)), b + v_bc[:, None] * (c - b)),
            (np.ones(len(a), dtype=bool), (a + v[:, None] * ab) + w[:, None] * ac),
        ]
        q = np.empty_like(a)
        done = np.zeros(len(a), dtype=bool)
        for cond, val in cands:
            take = cond & ~done
            q[take] = val[take]
            done |= take
    return q


def branch(p, tris):
    """Which branch of closest_point_triangle each triangle takes (0-3: repeated vertices, 4-6: vertex regions, 7-9: edges, 10: the
    interior) -- for the tests that check a family reaches what it claims."""
    F = tris.dtype.type
    p = np.asarray(p, dtype=F)
    a, b, c = tris[:, 0], tris[:, 1], tris[:, 2]
    with np.errstate(all="ignore"):
        e_ab, e_bc, e_ac = (a == b).all(1), (b == c).all(1), (a == c).all(1)
        ab, ac, ap, bp, cp = b - a, c - a, p - a, p - b, p - c
        d1, d2, d3, d4, d5, d6 = _dot(ab, ap), _dot(ac, ap), _dot(ab, bp), _dot(ac, bp), _dot(ab, cp), _dot(ac, cp)
        vc, vb, va = d1 * d4 - d3 * d2, d5 * d2 - d1 * d6, d3 * d6 - d5 * d4
        conds = [e_ab & e_bc & e_ac, e_ab, e_bc, e_ac, (d1 <= F(0)) & (d2 <= F(0)), (d3 >= F(0)) & (d4 <= d3), (d6 >= F(0)) & (d5 <= d6),
                 (vc <= F(0)) & (d1 >= F(0)) & (d3 <= F(0)), (vb <= F(0)) & (d2 >= F(0)) & (d6 <= F(0)),
                 (va <= F(0)) & (d4 - d3 >= F(0)) & (d5 - d6 >= F(0))]
    return np.select(conds, list(range(10)), 10)


def keys_and_closest(p, tris):
    """(key (n,), q (n, 3)): Triangle::distance_squared and its closest point for every triangle."""
    q = closest(p, tris)
    with np.errstate(all="ignore"):
        d = np.asarray(p, dtype=tris.dtype) - q
        return _dot(d, d), q


def keys(p, tris):
    return keys_and_closest(p, tris)[0]


def box_lower_d2(p, mn, mx):
    """queries.cuh's box_lower_d2 of one point (3,) -- or of one point per box (n, 3) -- against every box (n, 3), vectorised;
    prunedmodel.box_lower_d2 restated."""
    F = mn.dtype.type
    p = np.asarray(p, dtype=F)
    eps = F(np.finfo(F).eps)
    floor = F(2.0 ** -145) if F == np.float32 else F(2.0 ** -1070)
    d2 = np.zeros(len(mn), dtype=F)
    with np.errstate(all="ignore"):
        for k in range(3):
            a, b = mn[:, k] - p[..., k], p[..., k] - mx[:, k]
            d = np.where(a > b, a, b)
            m = np.broadcast_to(np.abs(p[..., k]), (len(mn),)).astype(F)
            nmn, ext = -mn[:, k], mx[:, k] - mn[:, k]
            m = np.where(nmn > m, nmn, m)
            m = np.where(mx[:, k] > m, mx[:, k], m)
            m = np.where(ext > m, ext, m)
            d = d - (m * (F(16) * eps) + floor)
            d = np.where(d > F(0), d, F(0)).astype(F)
            d2 = d2 + d * d
    return d2


def bounded(p, tris, mn, mx):
    """Per triangle: True unless key_s < box_lower_d2(p, own box) (a NaN key is bounded: it never qualifies)."""
    with np.errstate(all="ignore"):
        return ~(keys(p, tris) < box_lower_d2(p, mn, mx))


def qualifies(key, r):
    F = key.dtype.type
    with np.errstate(all="ignore"):
        if r is None:
            return ~np.isnan(key)
        r = F(r)
        if not r >= F(0):
            return np.zeros(len(key), dtype=bool)
        return key <= r * r


def brute(tris, pts, k, max_dist=None, only=None):
    """(shape (m, k) u32, dist (m, k) T, closest (m, k, 3) T) by the contract.  only(i, p) -> mask restricts the candidates (the
    bounded triangles, for the weaker guarantee)."""
    F = tris.dtype.type
    m = len(pts)
    out_s = np.full((m, k), U32_MAX, dtype=np.uint32)
    out_d = np.full((m, k), np.inf, dtype=F)
    out_q = np.full((m, k, 3), np.nan, dtype=F)
    for i in range(m):
        if len(tris) == 0:
            continue
        key, q = keys_and_closest(pts[i], tris)
        ok = qualifies(key, None if max_dist is None else max_dist[i])
        if only is not None:
            ok &= only(i, pts[i])
        idx = np.flatnonzero(ok)
        order = idx[np.argsort(key[idx], kind="stable")][:k]
        out_s[i, : len(order)] = order
        with np.errstate(all="ignore"):
            out_d[i, : len(order)] = np.sqrt(key[order])
        out_q[i, : len(order)] = q[order]
    return out_s, out_d, out_q


# ---- scenes ------------------------------------------------------------------------------------------------------------------------
def boxes(tris):
    """The triangles' own AABBs (Triangle::new grows an empty box by a, b, c: the vertex min / max), as (mn, mx)."""
    return tris.min(axis=1), tris.max(axis=1)


def near_points(tris, m, rng, spread=1.0):
    """m points near the triangles: a random vertex or the centroid of a random triangle plus a normal offset of `spread` times that
    triangle's extent (per-axis scales of 1e-6 .. 1 of it as well, so some points sit just outside a face), in T."""
    F = tris.dtype.type
    t = tris.astype(np.float64)
    i = rng.integers(0, len(t), m)
    w = rng.dirichlet(np.ones(3), m)
    w[: m // 3] = np.eye(3)[rng.integers(0, 3, m // 3)]
    base = np.einsum("mj,mjk->mk", w, t[i])
    ext = (t[i].max(1) - t[i].min(1)).max(1)
    ext = np.where(ext > 0, ext, np.abs(t[i]).max((1, 2)) * 1e-3 + 1e-300)
    off = rng.normal(size=(m, 3)) * (spread * ext * 10.0 ** rng.uniform(-6, 0, m))[:, None]
    with np.errstate(all="ignore"):
        return (base + off).astype(F)


def odd_points(F):
    """Points with NaN and infinite coordinates."""
    return np.array([[np.nan, 0, 0], [0, 0, np.inf], [-np.inf, 0, 0], [np.nan] * 3, [np.inf, -np.inf, 0]], dtype=F)


def soup(F, n, rng):
    """n random triangles of varied size in a 100-unit cube."""
    c = rng.uniform(-50, 50, (n, 1, 3))
    return (c + rng.normal(size=(n, 3, 3)) * 10.0 ** rng.uniform(-2, 1, (n, 1, 1))).astype(F)


def _slivers(F, rng, n=80):
    a = rng.uniform(-1, 1, (n, 3))
    d = rng.normal(size=(n, 3))
    L = 10.0 ** rng.uniform(-1, 2, n)[:, None]
    e = rng.normal(size=(n, 3)) * 10.0 ** rng.uniform(-7 if F == np.float32 else -15, -3, n)[:, None]
    c = a + d * L * rng.uniform(0, 1, (n, 1)) + e * L
    return np.stack([a, a + d * L, c], 1)


def _collinear(F, rng, n=80):
    """Exactly collinear: small integer vertices a, a + 2 d, a + d (every difference and dot product exact)."""
    a = rng.integers(-8, 8, (n, 3)).astype(float)
    d = rng.integers(-4, 5, (n, 3)).astype(float)
    d[(d == 0).all(1), 0] = 1
    perm = np.array([rng.permutation(3) for _ in range(n)])
    v = np.stack([a, a + 2 * d, a + d], 1)
    return v[np.arange(n)[:, None], perm]


def _near_collinear(F, rng, n=80):
    """Collinear up to one rounding: the middle vertex moved by one ulp on one axis."""
    v = _collinear(F, rng, n).astype(F) * F(1.0 / 3.0)
    j = rng.integers(0, 3, n)
    ax = rng.integers(0, 3, n)
    v[np.arange(n), j, ax] = np.nextafter(v[np.arange(n), j, ax], F(np.inf) * rng.choice([-1, 1], n).astype(F))
    return v


def _repeated(F, rng, n=80):
    """Repeated vertices: a == b, b == c, a == c, and all three, in turn (the closest_point_segment branches)."""
    v = soup(np.float64, n, rng)
    for i in range(n):
        kind = i % 4
        if kind == 0:
            v[i, 1] = v[i, 0]
        elif kind == 1:
            v[i, 2] = v[i, 1]
        elif kind == 2:
            v[i, 2] = v[i, 0]
        else:
            v[i, 1] = v[i, 2] = v[i, 0]
    return v


def _tiny_far(F, rng, n=80):
    """Triangles 1e-3 across at offsets of 1e5 (f32) / 1e13 (f64): coordinates carry a few significant bits of the shape."""
    off = 1e5 if F == np.float32 else 1e13
    return rng.choice([-1, 1], (n, 1, 3)) * off * rng.uniform(1, 2, (n, 1, 3)) + rng.normal(size=(n, 3, 3)) * 1e-3


def _subnormal(F, rng, n=80):
    """Subnormal extents: every coordinate a few dozen subnormal steps from 0."""
    tiny = float(np.finfo(F).smallest_subnormal)
    return rng.integers(-60, 60, (n, 3, 3)).astype(float) * tiny


def _overflow(F, rng, n=80):
    """Overflow-scale triangles: the dot products overflow to inf, keys become inf or NaN (inf - inf, 0 * inf)."""
    big = float(np.finfo(F).max) / 4
    return rng.uniform(-1, 1, (n, 3, 3)) * big


FAMILIES = {"slivers": _slivers, "collinear": _collinear, "near_collinear": _near_collinear, "repeated": _repeated, "tiny_far": _tiny_far,
            "subnormal": _subnormal, "overflow": _overflow}


def family(name, F, seed=0):
    """(tris (n, 3, 3) T, points (m, 3) T) of an adversarial family."""
    rng = np.random.default_rng(1000 + seed + sorted(FAMILIES).index(name))
    with np.errstate(all="ignore"):
        tris = np.asarray(FAMILIES[name](F, rng), dtype=np.float64).astype(F)
    spread = 1e-3 if name == "overflow" else 1.0
    pts = near_points(tris, 60, rng, spread)
    if name == "subnormal":
        pts = (rng.integers(-80, 80, (60, 3)).astype(float) * float(np.finfo(F).smallest_subnormal)).astype(F)
    return tris, pts


class Walk(knnref.Walk):
    """knn_walk over the node array with Triangle::distance_squared at the leaves.  knnref.Walk.row evaluates its leaf as
    dimref.min_distance_sq of self.shapes[s]; here the row is restated with the triangle key (precomputed per point: the leaf value
    is a function of (p, s) alone)."""

    def __init__(self, nodes, tris):
        mn, mx = tris.min(axis=1), tris.max(axis=1)
        super().__init__(nodes, mn, mx)
        self.tris = tris

    def row(self, p, k, r=None):
        F = self.F
        p = [F(x) for x in p]
        key_all = keys(np.array(p, dtype=F), self.tris) if len(self.tris) else np.zeros(0, dtype=F)
        inf = F(np.inf)
        lst = []
        visits = 0
        with np.errstate(all="ignore"):
            r2 = inf if r is None else F(r) * F(r)
        if self.cl and (r is None or F(r) >= F(0)):
            stack = [("node", 0)]
            while stack:
                item = stack.pop()
                if item[0] == "try":
                    t = lst[-1][0] if len(lst) == k else inf
                    if item[3] or (item[2] <= t and item[2] <= r2):
                        stack.append(("node", item[1]))
                    continue
                i = item[1]
                visits += 1
                if self.cl[i] == U32_MAX:
                    s = self.sh[i]
                    key = key_all[s]
                    if key <= r2 and (len(lst) < k or (key, s) < lst[-1]):
                        lst.append((key, s))
                        lst.sort()
                        del lst[k:]
                    continue
                lmn, lmx, rmn, rmx = self.box[i]
                dl, dr = box_lower_d2_scalar(p, lmn, lmx), box_lower_d2_scalar(p, rmn, rmx)
                el, er = any(a > b for a, b in zip(lmn, lmx)), any(a > b for a, b in zip(rmn, rmx))
                if dl > dr:
                    near, far = (self.cr[i], dr, er), (self.cl[i], dl, el)
                else:
                    near, far = (self.cl[i], dl, el), (self.cr[i], dr, er)
                stack.append(("try",) + far)
                stack.append(("try",) + near)
        s = np.full(k, U32_MAX, dtype=np.uint32)
        d = np.full(k, np.inf, dtype=F)
        for j, (key, sh) in enumerate(lst):
            s[j] = sh
            with np.errstate(all="ignore"):
                d[j] = np.sqrt(key)
        return s, d, visits
