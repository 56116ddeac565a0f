"""tests/polygons.py -- models of the polygon calls of 2-D trees (bvhgpu_contains_points_*x2, bvhgpu_knn_segments_*x2,
bvhgpu_signed_distance_*x2; include/bvh_b200.h, DESIGN.md 4.23) (test infrastructure).

    winding_exact   the contains contract for one point, in exact integer arithmetic: every finite float is m * 2^e, so scaling by 2^149
                    (f32) or 2^1074 (f64) gives an exact Python integer and orient2d is the sign of an integer polynomial.
    contains        the same contract vectorised over many points: the segments are binned by their y range against the points sorted
                    by y (only pairs with py in [min(ay, by), max(ay, by)] are formed), each sign is read from a double-precision
                    evaluation with Shewchuk's orient2d bound (numpy rounds every operation and never contracts), and the pairs the bound
                    leaves open go to the exact integer sign.  It must agree with winding_exact (tests/test_polygons_cpu.py).
    keys_and_closest / brute   the knn_segments key in T, operation for operation, and the brute-force rows of the contract.
    signed          the signed-distance contract from the two.
"""
import numpy as np

from tests.knntri import box_lower_d2, qualifies

U32_MAX = 0xFFFFFFFF
F64_LO, F64_HI = 2.0 ** -300, 2.0 ** 300
OUTSIDE, INSIDE, BOUNDARY, UNDECIDED = 0, 1, 2, 3
EVEN_ODD, NONZERO = 0, 1
_BOUND = (3.0 + 16.0 * 2.0 ** -53) * 2.0 ** -53


def _scale(F):
    return 149 if np.dtype(F) == np.float32 else 1074


def to_int(x, F):
    """The exact integer x * 2^149 (f32) or x * 2^1074 (f64) of a finite x."""
    n, d = float(x).as_integer_ratio()
    return n * ((1 << _scale(F)) // d)


def _sgn(v):
    return (v > 0) - (v < 0)


def orient2_int(a, b, c):
    """Sign of (a - c) x (b - c) on integer points."""
    return _sgn((a[0] - c[0]) * (b[1] - c[1]) - (a[1] - c[1]) * (b[0] - c[0]))


def in_range(x, F):
    """f64: zero or a magnitude in [2^-300, 2^300]; f32: always."""
    if np.dtype(F) == np.float32:
        return np.ones(np.shape(x), dtype=bool)
    a = np.abs(np.asarray(x, dtype=np.float64))
    return (a == 0) | ((a >= F64_LO) & (a <= F64_HI))


def classify(w, boundary, undecided, rule):
    inside = (w & 1) != 0 if rule == EVEN_ODD else w != 0
    return np.where(boundary, BOUNDARY, np.where(undecided, UNDECIDED, np.where(inside, INSIDE, OUTSIDE))).astype(np.uint8)


# ---- the contains contract, exact, one point ----
def winding_exact(segs, p, F):
    """(winding, boundary, undecided) of point p (2,) against segs (m, 4), every comparison and sign exact; None for a point that is not
    walked (non-finite: class 0; f64 out of range: class 3)."""
    px, py = float(p[0]), float(p[1])
    if not (np.isfinite(px) and np.isfinite(py)):
        return None
    if not (in_range(px, F) and in_range(py, F)):
        return None
    P = (to_int(px, F), to_int(py, F))
    w, boundary, undecided = 0, False, False
    for ax, ay, bx, by in np.asarray(segs, dtype=np.float64):
        if not all(np.isfinite(v) for v in (ax, ay, bx, by)) or (ax == bx and ay == by):
            continue
        if not (min(ay, by) <= py <= max(ay, by) and max(ax, bx) >= px):
            continue
        if not all(in_range(v, F) for v in (ax, ay, bx, by)):
            undecided = True
            continue
        o = orient2_int((to_int(ax, F), to_int(ay, F)), (to_int(bx, F), to_int(by, F)), P)
        if o == 0:
            boundary = boundary or (min(ax, bx) <= px <= max(ax, bx))
        elif o > 0 and ay <= py < by:
            w += 1
        elif o < 0 and by <= py < ay:
            w -= 1
    return w, boundary, undecided


def contains_exact(segs, pts, F, rule):
    """(class (n,), winding (n,)) by winding_exact; an empty tree (no segments) gives class 0 everywhere."""
    n = len(pts)
    cls, wind = np.zeros(n, dtype=np.uint8), np.zeros(n, dtype=np.int32)
    if len(segs) == 0:
        return cls, wind
    for i in range(n):
        r = winding_exact(segs, pts[i], F)
        if r is None:
            if np.isfinite(pts[i]).all():
                cls[i] = UNDECIDED
            continue
        w, b, u = r
        wind[i] = w
        cls[i] = classify(np.int32(w), b, u, rule)
    return cls, wind


# ---- the contains contract, vectorised ----
def _pairs(ylo, yhi, py_sorted, order, seg_idx, chunk=4_000_000):
    """Yields (segment index, point index) arrays of every pair with py in [ylo, yhi], in chunks."""
    lo = np.searchsorted(py_sorted, ylo, side="left")
    hi = np.searchsorted(py_sorted, yhi, side="right")
    cnt = np.maximum(hi - lo, 0)
    start = 0
    while start < len(cnt):
        csum = np.cumsum(cnt[start:])
        stop = start + max(int(np.searchsorted(csum, chunk, side="right")), 1)
        c = cnt[start:stop]
        tot = int(c.sum())
        if tot:
            s = np.repeat(np.arange(start, stop), c)
            first = np.repeat(np.cumsum(c) - c, c)
            pos = np.repeat(lo[start:stop], c) + (np.arange(tot) - first)
            yield seg_idx[s], order[pos]
        start = stop


def contains(segs, pts, F):
    """(winding (n,) i32, boundary (n,), undecided (n,), walked (n,)) for every point; walked = False for non-finite points and f64
    points out of range (winding 0).  Classes: classify(...) per rule, and UNDECIDED for finite points that were not walked."""
    segs = np.asarray(segs, dtype=F).reshape(-1, 4)
    pts = np.asarray(pts, dtype=F).reshape(-1, 2)
    n = len(pts)
    w = np.zeros(n, dtype=np.int64)
    boundary = np.zeros(n, dtype=bool)
    undecided = np.zeros(n, dtype=bool)
    P = pts.astype(np.float64)
    S = segs.astype(np.float64)
    walked = np.isfinite(P).all(1) & in_range(P[:, 0], F) & in_range(P[:, 1], F)
    if len(S) == 0 or not walked.any():
        return w.astype(np.int32), boundary, undecided, walked
    ax, ay, bx, by = S[:, 0], S[:, 1], S[:, 2], S[:, 3]
    ok = np.isfinite(S).all(1) & ~((ax == bx) & (ay == by))
    seg_idx = np.flatnonzero(ok)
    pidx = np.flatnonzero(walked)
    order = pidx[np.argsort(P[pidx, 1], kind="stable")]
    py_sorted = P[order, 1]
    ylo, yhi = np.minimum(ay, by)[seg_idx], np.maximum(ay, by)[seg_idx]
    seg_rng = in_range(S, F).all(1)
    for s, i in _pairs(ylo, yhi, py_sorted, order, seg_idx):
        px, py = P[i, 0], P[i, 1]
        rel = np.maximum(ax[s], bx[s]) >= px
        s, i, px, py = s[rel], i[rel], px[rel], py[rel]
        bad = ~seg_rng[s]
        np.logical_or.at(undecided, i[bad], True)
        s, i, px, py = s[~bad], i[~bad], px[~bad], py[~bad]
        with np.errstate(all="ignore"):
            l = (ax[s] - px) * (by[s] - py)
            r = (ay[s] - py) * (bx[s] - px)
            det = l - r
            err = _BOUND * (np.abs(l) + np.abs(r))
        o = np.where(det > err, 1, np.where(-det > err, -1, 0))
        for j in np.flatnonzero(~((det > err) | (-det > err))):
            a = (to_int(ax[s[j]], F), to_int(ay[s[j]], F))
            b = (to_int(bx[s[j]], F), to_int(by[s[j]], F))
            o[j] = orient2_int(a, b, (to_int(px[j], F), to_int(py[j], F)))
        on = (o == 0) & (np.minimum(ax[s], bx[s]) <= px)
        np.logical_or.at(boundary, i[on], True)
        up = (o > 0) & (ay[s] <= py) & (py < by[s])
        dn = (o < 0) & (by[s] <= py) & (py < ay[s])
        np.add.at(w, i, up.astype(np.int64) - dn.astype(np.int64))
    return w.astype(np.int32), boundary, undecided, walked


def classes(segs, pts, F, rule):
    """(class (n,) u8, winding (n,) i32) of bvhgpu_contains_points_*x2; an empty tree (no segments) gives class 0 everywhere."""
    if len(segs) == 0:
        n = len(np.asarray(pts).reshape(-1, 2))
        return np.zeros(n, dtype=np.uint8), np.zeros(n, dtype=np.int32)
    w, b, u, walked = contains(segs, pts, F)
    cls = classify(w, b, u, rule)
    finite = np.isfinite(np.asarray(pts, dtype=np.float64).reshape(-1, 2)).all(1)
    cls = np.where(walked, cls, np.where(finite, UNDECIDED, OUTSIDE)).astype(np.uint8)
    return cls, np.where(walked, w, 0).astype(np.int32)


# ---- k nearest segments ----
def keys_and_closest(p, segs):
    """(key (m,), q (m, 2)) of one point p (2,) against every segment of segs (m, 4), in T, the header's operation order."""
    F = segs.dtype.type
    px, py = F(p[0]), F(p[1])
    ax, ay, bx, by = segs[:, 0], segs[:, 1], segs[:, 2], segs[:, 3]
    with np.errstate(all="ignore"):
        ex, ey, wx, wy = bx - ax, by - ay, px - ax, py - ay
        num = wx * ex + wy * ey
        den = ex * ex + ey * ey
        t = num / den
        qx = np.where(num <= F(0), ax, np.where(num >= den, bx, ax + t * ex)).astype(F)
        qy = np.where(num <= F(0), ay, np.where(num >= den, by, ay + t * ey)).astype(F)
        dx, dy = px - qx, py - qy
        key = (dx * dx + dy * dy).astype(F)
    return key, np.stack([qx, qy], axis=1)


def brute(segs, pts, k, max_dist=None):
    """(shape (n, k) u32, dist (n, k) T, closest (n, k, 2) T) by the contract."""
    F = segs.dtype.type
    n = len(pts)
    out_s = np.full((n, k), U32_MAX, dtype=np.uint32)
    out_d = np.full((n, k), np.inf, dtype=F)
    out_q = np.full((n, k, 2), np.nan, dtype=F)
    for i in range(n):
        if len(segs) == 0:
            continue
        key, q = keys_and_closest(pts[i], segs)
        ok = qualifies(key, None if max_dist is None else max_dist[i])
        idx = np.flatnonzero(ok)
        order = idx[np.argsort(key[idx], kind="stable")][:k]
        out_s[i, : len(order)] = order
        with np.errstate(all="ignore"):
            out_d[i, : len(order)] = np.sqrt(key[order])
        out_q[i, : len(order)] = q[order]
    return out_s, out_d, out_q


def bounded(p, segs, mn, mx):
    """Per segment: not key_s < box_lower_d2(p, AABB_s) on the tree's embedding (z = 0 everywhere): the walk can lose a segment only
    where this is False."""
    F = segs.dtype.type
    key, _ = keys_and_closest(p, segs)
    z = np.zeros((len(segs), 1), dtype=F)
    lb = box_lower_d2(np.array([p[0], p[1], 0], dtype=F), np.hstack([mn, z]), np.hstack([mx, z]))
    with np.errstate(all="ignore"):
        return ~(key < lb)


def signed(segs, pts, rule):
    """(shape (n,), dist (n,), closest (n, 2)) of bvhgpu_signed_distance_*x2."""
    F = segs.dtype.type
    s, d, q = brute(segs, pts, 1)
    cls, _ = classes(segs, pts, F, rule)
    d = d[:, 0].copy()
    neg = (cls == INSIDE) & (s[:, 0] != U32_MAX)
    d[neg] = -d[neg]
    return s[:, 0], d, q[:, 0]


# ---- scenes ----
def loop(vertices):
    """Closed polyline (m, 2) -> segments (m, 4), vertex i to vertex i + 1."""
    v = np.asarray(vertices)
    return np.hstack([v, np.roll(v, -1, axis=0)])


def koch(level, F=np.float64):
    """Koch snowflake, counter-clockwise, 3 * 4^level segments."""
    poly = [np.array([0.0, 0.0]), np.array([1.0, 0.0]), np.array([0.5, np.sqrt(3) / 2])]     # counter-clockwise triangle
    for _ in range(level):
        nxt = []
        for i in range(len(poly)):
            a, b = poly[i], poly[(i + 1) % len(poly)]
            d = (b - a) / 3
            p1, p3 = a + d, a + 2 * d
            rot = np.array([d[0] * 0.5 + d[1] * np.sqrt(3) / 2, -d[0] * np.sqrt(3) / 2 + d[1] * 0.5])   # outward for a CCW loop
            nxt += [a, p1, p1 + rot, p3]
        poly = nxt
    return loop(np.array(poly)).astype(F)


def star(cx, cy, r_out, r_in, spikes, phase=0.0, ccw=True):
    """A star polygon as a loop, counter-clockwise (ccw) or clockwise."""
    t = phase + np.arange(2 * spikes) * np.pi / spikes
    r = np.where(np.arange(2 * spikes) % 2 == 0, r_out, r_in)
    v = np.stack([cx + r * np.cos(t), cy + r * np.sin(t)], axis=1)
    return loop(v if ccw else v[::-1])


def star_map(n_stars, spikes, F=np.float64, seed=0):
    """A "map": n_stars star polygons on a grid, each with a clockwise star hole inside (n_stars * 4 * spikes segments)."""
    rng = np.random.default_rng(seed)
    g = int(np.ceil(np.sqrt(n_stars)))
    out = []
    for k in range(n_stars):
        cx, cy = (k % g) * 3.0 + rng.uniform(-0.2, 0.2), (k // g) * 3.0 + rng.uniform(-0.2, 0.2)
        ph = rng.uniform(0, np.pi)
        out.append(star(cx, cy, 1.4, 0.8, spikes, ph, True))
        out.append(star(cx, cy, 0.6, 0.3, spikes, ph + 0.1, False))
    return np.vstack(out).astype(F)


def seg_boxes(segs):
    """The exact end-point boxes (mn, mx) of segments (m, 4) (NaN coordinates take the other end point's value)."""
    a, b = segs[:, 0:2], segs[:, 2:4]
    return np.fmin(a, b), np.fmax(a, b)
