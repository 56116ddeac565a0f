"""Adversarial scenes for the distance-pruned walks (triangle-mode closest_hit, nearest_candidates), generated from a seed.

Triangle families return (triangles (n, 9) in T, origins (m, 3), directions (m, 3)); box families return (mins (n, D), maxs (n, D),
points (m, D)).  Every family is deterministic; tests/test_pruned_walks_cpu.py checks that each one contains what it claims."""
import numpy as np

from oracle import oracle as O

MARGIN = 1.0 + 2.0 ** -16


def _prec(F):
    return "f32" if F == np.float32 else "f64"


def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def _front(tris, d):
    """Swap b and c where the triangle faces away from direction d (det <= 0 in f64), so that every triangle is a front face."""
    t = tris.astype(np.float64).reshape(-1, 3, 3)
    ab, ac = t[:, 1] - t[:, 0], t[:, 2] - t[:, 0]
    det = np.einsum("ij,ij->i", ab, np.cross(d, ac))
    out = tris.reshape(-1, 3, 3).copy()
    back = det < 0
    out[back, 1], out[back, 2] = tris.reshape(-1, 3, 3)[back, 2], tris.reshape(-1, 3, 3)[back, 1]
    return out.reshape(-1, 9)


def _mt(o, d, tri):
    """Ray::intersects_triangle vectorised in T (elementwise numpy, no FMA, the device's operation order): distances."""
    F = o.dtype.type
    eps = F(np.finfo(F).eps)
    t = tri.reshape(-1, 3, 3)
    a, b, c = t[:, 0], t[:, 1], t[:, 2]

    def cross(x, y):
        return np.stack([x[:, 1] * y[:, 2] - x[:, 2] * y[:, 1], x[:, 2] * y[:, 0] - x[:, 0] * y[:, 2], x[:, 0] * y[:, 1] - x[:, 1] * y[:, 0]], 1)

    def dot(x, y):
        return (x[:, 0] * y[:, 0] + x[:, 1] * y[:, 1]) + x[:, 2] * y[:, 2]

    with np.errstate(all="ignore"):
        ab, ac, ao = b - a, c - a, o - a
        uvec = cross(d, ac)
        det = dot(ab, uvec)
        inv = F(1) / det
        u = dot(ao, uvec) * inv
        vvec = cross(ao, ab)
        v = dot(d, vvec) * inv
        dist = dot(ac, vvec) * inv
    ok = (det >= eps) & (u >= 0) & (u <= 1) & (v >= 0) & (u + v <= 1) & (dist > eps)
    return np.where(ok, dist, F(np.inf))


def _slab(o, inv, mn, mx):
    F = o.dtype.type
    with np.errstate(all="ignore"):
        l, r = (mn - o) * inv, (mx - o) * inv
    tmin = np.minimum(l, r).max(axis=1)
    tmax = np.maximum(l, r).min(axis=1)
    e = np.where(tmin > 0, tmin, F(0))
    return np.where(np.isnan(l).any(1) | np.isnan(r).any(1) | (e > tmax), F(np.inf), e)


def grazing(F, seed=0, n_search=200_000, keep=48):
    """Grazing hits: tilt 1e-7 .. 1e-1 between the ray and triangle B, hits 5 .. 50 units away, origins spread over +-1000.  Of the
    searched triangles, the `keep` whose Moeller-Trumbore distance lies farthest in front of their own AABB's slab entry (beyond the
    2^-16 margin) are kept, each with a blocker A: a small front-facing triangle across the ray at a distance between B's computed
    distance and B's box entry; where B's distance is not beyond the margin (f64) B comes alone.  Returns the triangles, one ray
    per B, and the ratio entry / distance of each B."""
    rng = np.random.default_rng(seed)
    n = n_search
    o = rng.uniform(-1000, 1000, (n, 3))
    d = _unit(rng.normal(size=(n, 3)))
    w = _unit(np.cross(d, rng.normal(size=(n, 3))))
    e2 = np.cross(d, w)
    tilt = 10.0 ** rng.uniform(-7, -1, (n, 1))
    e1 = d * np.cos(tilt) + w * np.sin(tilt)
    h = o + rng.uniform(5, 50, (n, 1)) * d
    L, W, W2 = rng.uniform(0.5, 5, (n, 1)), rng.uniform(0.1, 2, (n, 1)), rng.uniform(0.1, 2, (n, 1))
    tri = np.concatenate([h - L * e1 - W * e2, h + L * e1 - W * e2, h + W2 * e2], axis=1)
    tri = _front(tri, d).astype(F)
    rays = O.ray_new(o, d, _prec(F))
    ro, rd, rinv = rays["origin"], rays["direction"], rays["inv_direction"]
    t = _mt(ro, rd, tri)
    tt = tri.reshape(-1, 3, 3)
    entry = _slab(ro, rinv, tt.min(axis=1), tt.max(axis=1))
    with np.errstate(all="ignore"):
        ratio = np.where(np.isfinite(t) & np.isfinite(entry) & (t > 0), entry.astype(np.float64) / t.astype(np.float64), 0.0)
    pick = np.argsort(-ratio)[:keep]
    out, org, dirs, ratios = [], [], [], []
    for i in pick:
        tb, eb = float(t[i]), float(entry[i])
        if ratio[i] > MARGIN * (1 + 1e-4):                  # f64 grazing errors stay far inside the margin: B alone
            ta = np.sqrt(tb * eb / MARGIN)                   # between tb and eb / (1 + 2^-16)
            ha = o[i] + ta * d[i]
            s = 1e-3 * ta
            a_tri = np.concatenate([ha - s * w[i] - s * e2[i], ha + s * w[i] - s * e2[i], ha + s * e2[i]])
            out.append(_front(a_tri[None], d[i][None])[0].astype(F))
        out.append(tri[i])
        org.append(o[i]); dirs.append(d[i]); ratios.append(ratio[i])
    return np.array(out, dtype=F).reshape(-1, 9), np.array(org, dtype=F), np.array(dirs, dtype=F), np.array(ratios)


def shared_edges(F, seed=1, grid=6):
    """A fan of triangles sharing edges and vertices on a tilted plane, rays aimed exactly at shared vertices and at points of
    shared edges (ties between neighbours: the lower index must win), plus rays through interiors."""
    rng = np.random.default_rng(seed)
    xs = np.arange(grid + 1, dtype=np.float64)
    P = np.stack(np.meshgrid(xs, xs, indexing="ij"), -1).reshape(-1, 2)
    V = np.concatenate([P, (0.25 * P[:, :1] + 0.125 * P[:, 1:])], axis=1).astype(F)      # exact in T: z = x/4 + y/8
    idx = lambda i, j: i * (grid + 1) + j
    tris = []
    for i in range(grid):
        for j in range(grid):
            a, b, c, dd = idx(i, j), idx(i + 1, j), idx(i + 1, j + 1), idx(i, j + 1)
            tris += [V[[a, b, c]].reshape(9), V[[a, c, dd]].reshape(9)]
    tris = np.array(tris, dtype=F)
    tgt = np.concatenate([V, (V[:-1] + V[1:]) / F(2), rng.uniform(0, grid, (60, 2)) @ np.array([[1, 0, 0.25], [0, 1, 0.125]])]).astype(np.float64)
    dirs = _unit(np.concatenate([rng.normal(size=(len(tgt), 2)) * 0.3, -np.ones((len(tgt), 1))], axis=1))
    org = tgt - 40.0 * dirs
    return _front(tris, -np.array([[0.0, 0.0, 1.0]])).astype(F), org.astype(F), dirs.astype(F)


def degenerate(F, seed=2):
    """Rays coplanar with a triangle (det = 0), back faces, slivers and zero-area triangles, origins on a triangle's plane and
    hits closer than eps."""
    rng = np.random.default_rng(seed)
    tris, org, dirs = [], [], []
    for k in range(24):
        c = np.array([k * 10.0, 0.0, 0.0])
        base = c + np.array([[0, 0, 0], [2, 0, 0], [0, 2, 0]], dtype=np.float64)
        tris.append(base.reshape(9))                                             # in z = 0, front face for -z rays
        org.append(c + [0.5, 0.5, 3.0]); dirs.append([0.0, 0.0, -1.0])           # plain hit
        org.append(c + [-1.0, 0.5, 0.0]); dirs.append([1.0, 0.0, 0.0])           # coplanar: det = 0
        org.append(c + [0.3, 0.3, 0.0]); dirs.append(_unit(rng.normal(size=3)))  # origin on the plane (t = 0)
        eps = float(np.finfo(F).eps)
        org.append(c + [0.4, 0.4, eps * rng.uniform(0.1, 4)]); dirs.append([0.0, 0.0, -1.0])   # hit closer than ~eps
        tris.append((base[[0, 2, 1]] + [0, 0, 5.0]).reshape(9))                   # back face above the first
        org.append(c + [0.5, 0.5, 8.0]); dirs.append([0.0, 0.0, -1.0])
        sl = c + np.array([[0, 0, -3], [2, 1e-6 * rng.uniform(), -3], [4, 2e-6 * rng.uniform(), -3]])
        tris.append(sl.reshape(9))                                                # sliver, nearly collinear
        tris.append(np.array([c + [1, 1, -4]] * 2 + [c + [1, 1.5, -4]]).reshape(9))   # zero area: a repeated vertex
        tris.append(np.array([c + [0, 0, -5], c + [1, 1, -5], c + [2, 2, -5]]).reshape(9))   # zero area: collinear
        org.append(c + [1.0, 1e-7, 2.0]); dirs.append(_unit(np.array([0.0, 0.0, -1.0]) + rng.normal(size=3) * 1e-3))
        org.append(c + [1.0, 1.0, 2.0]); dirs.append([0.0, 0.0, -1.0])
    return np.array(tris).astype(F), np.array(org).astype(F), np.array(dirs).astype(F)


def offset_scene(F, offset, seed=3, n=300, m=600):
    """Random triangles of size ~1 .. 20 in a cube of side 200 moved to `offset` (1e4 .. 1e7 in f32, 1e12 and beyond in f64),
    with rays from inside the cube aimed at triangle centroids."""
    rng = np.random.default_rng(seed)
    ctr = rng.uniform(-100, 100, (n, 3))
    tris = (ctr[:, None, :] + rng.normal(size=(n, 3, 3)) * rng.uniform(1, 20, (n, 1, 1))).reshape(n, 9) + offset
    tris = tris.astype(F)
    tgt = tris.astype(np.float64).reshape(n, 3, 3).mean(axis=1)[rng.integers(0, n, m)]
    org = offset + rng.uniform(-150, 150, (m, 3))
    return tris, org.astype(F), _unit(tgt - org).astype(F)


# ---- boxes and points ------------------------------------------------------------------------------------------------------------
# The reference's Aabb::min_distance_squared at ~1e7 in f32: box X is at reference distance^2 0.25 from p, exact distance^2 1; the
# point box Y is at distance^2 0.5.  Under the reference distance X is the nearest shape.
ISSUE_X = ([-5985717.0, -121811.69, -7219457.0], [-3879675.5, 14336917.0, 3772881.0])
ISSUE_P = [-4558777.5, 14336918.0, -5193557.0]


def large_coordinates(F, D, seed=4, n=200, m=96):
    """Boxes of extent up to 1e7 at coordinates up to 1e7 (1e15 in f64), points a few ulps to 1e-3 (relative) outside a face, and
    point boxes next to some of them; in 3-D f32 the first shapes and point are the concrete X, Y, p above."""
    rng = np.random.default_rng(seed + D)
    big = 1e7 if F == np.float32 else 1e15
    lo = rng.uniform(-big, big, (n, D))
    mn, mx = lo.astype(F), (lo + rng.uniform(0, big, (n, D))).astype(F)
    pick = rng.integers(0, n, m)
    axis = rng.integers(0, D, m)
    p = (mn[pick].astype(np.float64) + mx[pick]) / 2
    face = np.where(rng.uniform(size=m) < 0.5, mn[pick, axis], mx[pick, axis]).astype(F)
    sign = np.where(face == mx[pick, axis], 1, -1)
    ulps = rng.integers(0, 5, m)
    p = p.astype(F)
    for j in range(m):
        x = face[j]
        if j % 2 == 0:
            for _ in range(ulps[j]):
                x = np.nextafter(x, F(np.inf) * sign[j])
        else:
            x = F(float(x) + sign[j] * abs(float(x)) * 10.0 ** rng.uniform(-7, -3))
        p[j, axis[j]] = x
    # point boxes half a unit (f32) away from some points: the distance the reference's cancellation gets wrong
    k = n // 4
    mn[:k] = mx[:k] = (p[:k].astype(np.float64) + rng.choice([-0.5, 0.5, 1.0], (k, D))).astype(F)
    if D == 3 and F == np.float32:
        mn[k], mx[k] = np.array(ISSUE_X[0], F), np.array(ISSUE_X[1], F)
        p[0] = np.array(ISSUE_P, F)
        mn[k + 1] = mx[k + 1] = p[0] + np.array([0.5, 0, 0.5], F)
    return mn, mx, p


def ties(F, D, seed=5, n=160, m=64):
    """Point boxes, coincident boxes and exact ties: unit boxes on an integer lattice (some repeated), points on the lattice's
    half-integers, where several boxes are at the same exact distance."""
    rng = np.random.default_rng(seed + D)
    c = rng.integers(-6, 6, (n, D)).astype(np.float64)
    c[n // 2: n // 2 + 20] = c[:20]                                  # coincident boxes
    mn, mx = (c - 0.5).astype(F), (c + 0.5).astype(F)
    mn[-30:] = mx[-30:] = c[-30:].astype(F)                          # point boxes
    p = (rng.integers(-12, 12, (m, D)) / 2.0).astype(F)
    return mn, mx, p


def mixed_scales(F, D, seed=6, n=200, m=64):
    """Extents from 1e-3 to 1e6 side by side, and subnormal extents at subnormal-to-tiny coordinates."""
    rng = np.random.default_rng(seed + D)
    lo = rng.uniform(-1e6, 1e6, (n, D))
    ext = 10.0 ** rng.uniform(-3, 6, (n, D))
    mn, mx = lo.astype(F), (lo + ext).astype(F)
    tiny = float(np.finfo(F).tiny)
    k = n // 4
    sub = rng.uniform(-64, 64, (k, D)) * tiny
    mn[:k], mx[:k] = sub.astype(F), (sub + rng.uniform(0, 8, (k, D)) * tiny * 2.0 ** -20).astype(F)
    p = np.concatenate([rng.uniform(-1e6, 1e6, (m // 2, D)), rng.uniform(-80, 80, (m - m // 2, D)) * tiny]).astype(F)
    return mn, mx, p


def overflow(F, D, seed=7, n=120, m=48):
    """Coordinates where every squared farthest-corner distance overflows (1e30 in f32, 1e160 in f64; surface areas overflow too,
    so the builder falls back to "no split wins" nodes): U = inf and every shape must be listed."""
    rng = np.random.default_rng(seed + D)
    big = 1e30 if F == np.float32 else 1e160
    lo = rng.uniform(-big, big, (n, D))
    mn, mx = lo.astype(F), (lo + rng.uniform(0, 0.1, (n, D)) * big).astype(F)
    p = rng.uniform(-big, big, (m, D)).astype(F)
    return mn, mx, p


BOX_FAMILIES = {"large": large_coordinates, "ties": ties, "mixed": mixed_scales, "overflow": overflow}
