"""tests/tritri.py -- an independent restatement of the triangle-pair contract (bvhgpu_triangle_pairs_*, include/bvh_b200.h) in exact
integer arithmetic (test infrastructure).

Every float is m * 2^e, so scaling a coordinate by 2^149 (f32) or 2^1074 (f64) gives an exact Python integer, and every orientation
sign is the sign of an integer polynomial.  meets(P, Q) follows the header's steps: excluded triangles (a non-finite coordinate, or
(b - a) x (c - a) = 0), f64 triangles with a nonzero coordinate outside [2^-300, 2^300] (unchecked: their pairs are kept), a shared
vertex (== on all three coordinates), then whether the closed triangles have a point in common: an edge of one meets the other.

The CSR model is the row model of tests/overlapref.py (self) or tests/crossref.py (two trees) filtered by meets.  A vectorised
double-precision filter (Shewchuk's orient3d bound; numpy rounds every operation and never contracts) decides the pairs that one
triangle's plane separates; every other pair goes to the integer path."""
import numpy as np

from tests import overlapref
from tests.crossref import cross_rows

U32_MAX = 0xFFFFFFFF
F64_LO, F64_HI = 2.0 ** -300, 2.0 ** 300
EXCLUDED, UNCHECKED, OK = 0, 1, 2


def _scale(F):
    return 149 if np.dtype(F) == np.float32 else 1074


def to_int(x, F):
    """The exact integer x * 2^149 (f32) or x * 2^1074 (f64) of a finite x."""
    n, d = float(x).as_integer_ratio()
    return n * ((1 << _scale(F)) // d)


# ---- exact signs on integer points ----
def _sgn(v):
    return (v > 0) - (v < 0)


def orient3(a, b, c, d):
    """Sign of det[a - d; b - d; c - d]."""
    ax, ay, az = a[0] - d[0], a[1] - d[1], a[2] - d[2]
    bx, by, bz = b[0] - d[0], b[1] - d[1], b[2] - d[2]
    cx, cy, cz = c[0] - d[0], c[1] - d[1], c[2] - d[2]
    return _sgn(ax * (by * cz - bz * cy) + ay * (bz * cx - bx * cz) + az * (bx * cy - by * cx))


def orient2(a, b, c, i, j):
    """Sign of (a - c) x (b - c) in the projection onto axes (i, j)."""
    return _sgn((a[i] - c[i]) * (b[j] - c[j]) - (a[j] - c[j]) * (b[i] - c[i]))


def projection(t):
    """(i, j, o): the first plane (x, y), (y, z), (z, x) where the triangle's projection has a nonzero signed area o; o = 0: degenerate."""
    for i, j in ((0, 1), (1, 2), (2, 0)):
        o = orient2(t[0], t[1], t[2], i, j)
        if o:
            return i, j, o
    return 0, 1, 0


def _in_tri2(p, t, pr):
    i, j, o = pr
    return all(orient2(t[k], t[(k + 1) % 3], p, i, j) != -o for k in range(3))


def _on_seg2(p, q, x, i, j):
    return min(p[i], q[i]) <= x[i] <= max(p[i], q[i]) and min(p[j], q[j]) <= x[j] <= max(p[j], q[j])


def _seg_seg2(p1, p2, q1, q2, i, j):
    d1, d2 = orient2(q1, q2, p1, i, j), orient2(q1, q2, p2, i, j)
    d3, d4 = orient2(p1, p2, q1, i, j), orient2(p1, p2, q2, i, j)
    if d1 * d2 < 0 and d3 * d4 < 0:
        return True
    return ((d1 == 0 and _on_seg2(q1, q2, p1, i, j)) or (d2 == 0 and _on_seg2(q1, q2, p2, i, j)) or
            (d3 == 0 and _on_seg2(p1, p2, q1, i, j)) or (d4 == 0 and _on_seg2(p1, p2, q2, i, j)))


def _seg_tri(u, v, t, pr):
    """The closed segment [u, v] meets the closed non-degenerate triangle t."""
    su, sv = orient3(t[0], t[1], t[2], u), orient3(t[0], t[1], t[2], v)
    if su == sv != 0:
        return False
    if su == 0 and sv == 0:
        i, j, _ = pr
        return (_in_tri2(u, t, pr) or _in_tri2(v, t, pr) or
                any(_seg_seg2(u, v, t[k], t[(k + 1) % 3], i, j) for k in range(3)))
    s = [orient3(u, v, t[k], t[(k + 1) % 3]) for k in range(3)]
    return min(s) >= 0 or max(s) <= 0


def tri_tri(p, q):
    """Two non-degenerate closed triangles of integer points have a point in common."""
    pp, qp = projection(p), projection(q)
    return (any(_seg_tri(p[k], p[(k + 1) % 3], q, qp) for k in range(3)) or
            any(_seg_tri(q[k], q[(k + 1) % 3], p, pp) for k in range(3)))


# ---- the steps of meets on float triangles ----
def classify(tri, F):
    """EXCLUDED, UNCHECKED (f64 out of range) or OK, and the integer points (None unless OK)."""
    t = np.asarray(tri, dtype=F).reshape(3, 3)
    if not np.all(np.isfinite(t)):
        return EXCLUDED, None
    if np.dtype(F) == np.float64:
        a = np.abs(t.astype(np.float64))
        if np.any((a != 0) & ((a < F64_LO) | (a > F64_HI))):
            return UNCHECKED, None
    pts = [tuple(to_int(x, F) for x in v) for v in t]
    return (OK, pts) if projection(pts)[2] else (EXCLUDED, None)


def shares_vertex(p, q):
    p, q = np.asarray(p).reshape(3, 3), np.asarray(q).reshape(3, 3)
    return bool(np.any(np.all(p[:, None, :] == q[None, :, :], axis=-1)))


def meets(p, q, F, skip_shared=False):
    """meets(P, Q) of the header for two triangles (3, 3) of precision F."""
    cp, ip = classify(p, F)
    cq, iq = classify(q, F)
    if EXCLUDED in (cp, cq):
        return False
    if UNCHECKED in (cp, cq):
        return True
    if shares_vertex(np.asarray(p, dtype=F), np.asarray(q, dtype=F)):
        return not skip_shared
    return tri_tri(ip, iq)


# ---- the vectorised plane filter ----
_O3 = (7.0 + 56.0 * 2.0 ** -53) * 2.0 ** -53


def orient3_filter(a, b, c, d):
    """Shewchuk's orient3d stage A over arrays (..., 3) of doubles: +1 / -1 where the bound decides the sign, 0 where it does not."""
    with np.errstate(all="ignore"):
        ad, bd, cd = a - d, b - d, c - d
        bdxcdy, cdxbdy = bd[..., 0] * cd[..., 1], cd[..., 0] * bd[..., 1]
        cdxady, adxcdy = cd[..., 0] * ad[..., 1], ad[..., 0] * cd[..., 1]
        adxbdy, bdxady = ad[..., 0] * bd[..., 1], bd[..., 0] * ad[..., 1]
        det = ad[..., 2] * (bdxcdy - cdxbdy) + bd[..., 2] * (cdxady - adxcdy) + cd[..., 2] * (adxbdy - bdxady)
        perm = ((np.abs(bdxcdy) + np.abs(cdxbdy)) * np.abs(ad[..., 2]) + (np.abs(cdxady) + np.abs(adxcdy)) * np.abs(bd[..., 2]) +
                (np.abs(adxbdy) + np.abs(bdxady)) * np.abs(cd[..., 2]))
        err = _O3 * perm
        return np.where(det > err, 1, np.where(-det > err, -1, 0))


def _separated(P, Q):
    """Pairs where every vertex of Q lies strictly on one side of P's plane (certainly, by the filter)."""
    s = np.stack([orient3_filter(P[:, 0], P[:, 1], P[:, 2], Q[:, k]) for k in range(3)], axis=1)
    return np.all(s > 0, axis=1) | np.all(s < 0, axis=1)


class Model:
    """meets over the triangles of one or two trees, with the per-triangle work done once."""

    def __init__(self, tris_a, F, tris_b=None):
        self.F = F
        self.a = np.asarray(tris_a, dtype=F).reshape(-1, 3, 3)
        self.b = self.a if tris_b is None else np.asarray(tris_b, dtype=F).reshape(-1, 3, 3)
        self.ca, self.ia = self._classes(self.a)
        self.cb, self.ib = (self.ca, self.ia) if tris_b is None else self._classes(self.b)
        self.exact_pairs = 0                                  # pairs the integer path decided in the last keep()

    def _classes(self, tris):
        cl, pts = np.zeros(len(tris), dtype=np.int8), [None] * len(tris)
        for i, t in enumerate(tris):
            cl[i], pts[i] = classify(t, self.F)
        return cl, pts

    def keep(self, s, t, skip_shared=False):
        """meets for the pairs (s[k] of A, t[k] of B), as a bool array."""
        s, t = np.asarray(s, dtype=np.int64), np.asarray(t, dtype=np.int64)
        ca, cb = self.ca[s], self.cb[t]
        out = np.zeros(len(s), dtype=bool)
        excl = (ca == EXCLUDED) | (cb == EXCLUDED)
        unch = ~excl & ((ca == UNCHECKED) | (cb == UNCHECKED))
        out[unch] = True
        rest = ~excl & ~unch
        P, Q = self.a[s].astype(np.float64), self.b[t].astype(np.float64)
        shared = np.any(np.all(P[:, :, None, :] == Q[:, None, :, :], axis=-1), axis=(1, 2))
        out[rest & shared] = not skip_shared
        rest &= ~shared
        idx = np.nonzero(rest)[0]
        if len(idx):
            sep = _separated(P[idx], Q[idx]) | _separated(Q[idx], P[idx])
            idx = idx[~sep]
        self.exact_pairs = len(idx)
        for k in idx:
            out[k] = tri_tri(self.ia[s[k]], self.ib[t[k]])
        return out


def _filter_csr(offsets, hits, keep):
    offsets = np.asarray(offsets, dtype=np.int64)
    rows = np.repeat(np.arange(len(offsets) - 1), np.diff(offsets))
    counts = np.bincount(rows[keep], minlength=len(offsets) - 1).astype(np.uint64)
    out = np.zeros(len(offsets), dtype=np.uint64)
    np.cumsum(counts, out=out[1:])
    return np.minimum(out, U32_MAX).astype(np.uint32), np.asarray(hits, dtype=np.uint32)[keep]


def self_rows(tris, mn, mx, leaf, F, skip_shared=True, model=None):
    """CSR (offsets u32[n + 1], hits u32) of bvhgpu_triangle_pairs_*: overlapref.rows filtered by meets."""
    off, hits = overlapref.rows(mn, mx, leaf)
    model = model or Model(tris, F)
    s = np.repeat(np.arange(len(off) - 1), np.diff(off.astype(np.int64)))
    return _filter_csr(off, hits, model.keep(s, hits, skip_shared))


def cross_tri_rows(tris_a, amn, amx, tris_b, bmn, bmx, leaf_b, F, model=None):
    """CSR of bvhgpu_triangle_pairs_trees_*: crossref.cross_rows filtered by meets (A's triangle against B's)."""
    off, hits = cross_rows(amn, amx, bmn, bmx, leaf_b)
    model = model or Model(tris_a, F, tris_b)
    s = np.repeat(np.arange(len(off) - 1), np.diff(off.astype(np.int64)))
    return _filter_csr(off, hits, model.keep(s, hits))


def tri_boxes(tris, F):
    """The triangles' own boxes (min, max) in precision F."""
    t = np.asarray(tris, dtype=F).reshape(-1, 3, 3)
    return t.min(axis=1), t.max(axis=1)
