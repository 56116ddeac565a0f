"""tests/edge_dims.py -- the edge-case inputs of tests/edge_inputs.py in any dimension D in {2, 3, 4}, f32 and f64, and the points,
radii, limits and triangles of the queries added after it (test infrastructure).

edge_inputs.edge_scene / edge_rays and dimref.scene / dimorder.rays are left as they are (other tests depend on their exact outputs);
everything here draws from its own seeds.

    scene       "huge" (HUGE[prec]: surface areas overflow in f32 and f64, "no split wins", empty child boxes), "mixed" (half such boxes,
                half unit-scale clusters) and "subnormal" (every coordinate below the smallest normal number), as edge_scene builds them
    rays        the six FAMILIES with D components through Ray::new (normalise in T, inv = 1 / d in T); axis, face, tiny and subdir pick
                their axis among all D
    points      random, on box faces and corners, +-0 components, just off a face by ~sqrt(smallest subnormal) (keys of a few subnormal
                steps), and far outside (keys that overflow to +inf at huge scale)
    radii       0, -0, +inf, r * r overflowing, r * r underflowing to 0, fl(r * r) rounded up onto a key, r * r a key exactly, random
    queries     Aabb / Point / Ball records of dimref's query kinds on those points, the balls with those radii
    limits      anyhit.tmax_families plus the smallest subnormal and each ray's exit distance of its closest shape
    triangles   one triangle inside every box of a 3-D edge scene (vertices at points of the box)

Scale limit: every centroid extent stays finite; beyond that the reference panics on a NaN bucket index."""
import numpy as np

from tests import anyhit, dimorder, dimref
from tests.edge_inputs import FAMILIES, HUGE, SUB_DIR, SUBNORMAL, TINY_DIR, _rng

SCENE_KINDS = ("huge", "mixed", "subnormal")
DIMS = (2, 3, 4)
PRECS = ("f32", "f64")
FT = {"f32": np.float32, "f64": np.float64}


def scene(kind, n, D, prec):
    """(mn, mx), (n, D) arrays of T."""
    rng = _rng("edge_dims_scene", kind, n, D, prec)
    if kind == "huge":
        s = HUGE[prec]
        mn = rng.uniform(-s, s, (n, D))
        mx = mn + rng.uniform(0, s / 10, (n, D))
    elif kind == "mixed":
        s, h = HUGE[prec], n // 2
        big = rng.uniform(-s, s, (h, D))
        centres = rng.uniform(-50, 50, (4, D))
        small = centres[rng.integers(0, 4, n - h)] + rng.normal(0, 3, (n - h, D))
        mn = np.concatenate([big, small])
        mx = mn + np.concatenate([rng.uniform(0, s / 10, (h, D)), rng.uniform(0.05, 2.0, (n - h, D))])
        perm = rng.permutation(n)
        mn, mx = mn[perm], mx[perm]
    elif kind == "subnormal":
        t = SUBNORMAL[prec]
        mn = rng.uniform(-t, t, (n, D))
        mx = mn + rng.uniform(0, t / 2, (n, D))
    else:
        raise KeyError(kind)
    F = FT[prec]
    return mn.astype(F), mx.astype(F)


def unit_directions(d):
    """Unit vectors in f64 without overflow (largest |component| first, then the norm); signs of zero components are kept."""
    d = np.asarray(d, dtype=np.float64)
    m = np.abs(d).max(axis=1, keepdims=True)
    assert np.all(m > 0), "zero direction"
    d = d / m
    return d / np.sqrt((d * d).sum(axis=1, keepdims=True))


def ray_new(o, d, F):
    """Ray::new in any D, elementwise in T: d / sqrt(dot(d, d)) with the dot summed left to right, inv = 1 / d.  (o, d, inv)."""
    o, d = np.asarray(o, dtype=F), np.asarray(d, dtype=F)
    with np.errstate(all="ignore"):
        acc = d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]
        for k in range(2, d.shape[1]):
            acc = acc + d[:, k] * d[:, k]
        d = (d / np.sqrt(acc)[:, None]).astype(F)
        inv = (F(1) / d).astype(F)
    return np.ascontiguousarray(o), np.ascontiguousarray(d), np.ascontiguousarray(inv)


def rays(mn, mx, family, m, prec, seed=0):
    """(o, d, inv), (m, D) each, of one family through the boxes (mn, mx); see edge_inputs.edge_rays for the families."""
    n, D = mn.shape
    rng = _rng("edge_dims_rays", family, m, D, prec, seed, n)
    mn, mx = mn.astype(np.float64), mx.astype(np.float64)
    lo, hi = mn.min(axis=0), mx.max(axis=0)
    pad = (hi - lo) * 0.1
    pick = rng.integers(0, n, m)
    centre = mn[pick] * 0.5 + mx[pick] * 0.5
    rows = np.arange(m)
    if family == "random":
        org = rng.uniform(lo - pad, hi + pad, (m, D))
        tgt = np.where(rng.random((m, 1)) < 0.5, rng.uniform(lo, hi, (m, D)), centre)
        dirs = unit_directions(tgt - org)
    elif family in ("axis", "face"):
        axis = rows % D                                      # every axis, the 4th included
        sign = rng.choice([-1.0, 1.0], m)
        dirs = np.zeros((m, D))
        dirs[1::2] = -0.0
        dirs[rows, axis] = sign
        org = centre.copy()
        org[rows, axis] = np.where(sign > 0, lo[axis] - pad[axis], hi[axis] + pad[axis])
        if family == "face":
            corner = np.where(rng.random((m, D)) < 0.5, mn[pick], mx[pick])
            off = np.arange(D)[None, :] != axis[:, None]
            org[off] = corner[off]
    elif family == "inside":
        org = mn[pick] + rng.random((m, D)) * (mx[pick] - mn[pick])
        dirs = unit_directions(rng.normal(size=(m, D)))
        on = rows[1::2]                                      # every other origin on a face of its box, moving inwards: o = max
        ax = on // 2 % D                                     # with d < 0 folds the entry to -0 before the clamp, o = min with d > 0 to +0
        up = rng.random(len(on)) < 0.5
        org[on, ax] = np.where(up, mx[pick[on], ax], mn[pick[on], ax])
        out = on % 4 == 3                                    # and every fourth one moving outwards: the box is met at t = 0 only
        dirs[on, ax] = np.where(up != out, -1.0, 1.0) * np.maximum(np.abs(dirs[on, ax]), 0.25)
        dirs = unit_directions(dirs)
    elif family in ("tiny", "subdir"):
        org = rng.uniform(lo - pad, hi + pad, (m, D))
        dirs = unit_directions(np.where(rng.random((m, 1)) < 0.5, centre - org, rng.normal(size=(m, D))))
        k = rows % D
        if family == "tiny":
            v = TINY_DIR[prec]
        else:
            v = np.where(rows // D % 2 == 0, SUB_DIR[prec][0], SUB_DIR[prec][1])
        sign = rng.choice([-1.0, 1.0], m)
        if family == "subdir":                               # every other finite-inverse ray starts on a face plane of its box along
            face = (rows // D % 2 == 0) & (rows // (2 * D) % 2 == 0)   # k, moving inwards: (b - o) * inv = 0 * inv is 0, not NaN
            org[face, k[face]] = np.where(sign[face] > 0, mn[pick[face], k[face]], mx[pick[face], k[face]])
            dirs[face] = unit_directions(centre[face] - org[face] + (org[face] == centre[face]))
        dirs[rows, k] = sign * v
    else:
        raise KeyError(family)
    return ray_new(org, dirs, FT[prec])


def ray_batch(mn, mx, per_family, prec, seed=0):
    """All families concatenated: (o, d, inv, family name of every ray)."""
    parts = [rays(mn, mx, f, per_family, prec, seed) for f in FAMILIES]
    o, d, inv = (np.concatenate([p[i] for p in parts]) for i in range(3))
    return o, d, inv, np.repeat(np.array(FAMILIES), per_family)


POINT_KINDS = ("random", "face", "zero", "near", "far")


def points(mn, mx, m, prec, seed=0):
    """(points (m, D) of T, kind of every point), the POINT_KINDS in turn: random around the scene; on faces and corners of a box;
    +-0 components on random ones; off a face of a box by a few sqrt(smallest subnormal) along one axis (keys of a few subnormal
    steps where the coordinates are small enough to keep the offset); far outside the scene (keys that overflow at huge scale)."""
    n, D = mn.shape
    F = FT[prec]
    rng = _rng("edge_dims_points", m, D, prec, seed, n)
    a, b = mn.astype(np.float64), mx.astype(np.float64)
    lo, hi = a.min(axis=0), b.max(axis=0)
    span = hi - lo
    pick = rng.integers(0, n, m)
    kind = np.array(POINT_KINDS)[np.arange(m) % len(POINT_KINDS)]
    p = rng.uniform(lo - 0.1 * span, hi + 0.1 * span, (m, D))
    f = kind == "face"
    p[f] = np.where(rng.random((int(f.sum()), D)) < 0.5, a[pick[f]], b[pick[f]])
    z = kind == "zero"
    p[z] = np.where(rng.random((int(z.sum()), D)) < 0.5, p[z], np.where(rng.random((int(z.sum()), D)) < 0.5, 0.0, -0.0))
    nr = np.flatnonzero(kind == "near")
    step = np.sqrt(float(np.finfo(F).smallest_subnormal))
    p[nr] = a[pick[nr]] * 0.5 + b[pick[nr]] * 0.5
    ax = nr % D
    out = rng.random(len(nr)) < 0.5
    p[nr, ax] = np.where(out, b[pick[nr], ax] + step * rng.uniform(0.5, 4, len(nr)), a[pick[nr], ax] - step * rng.uniform(0.5, 4, len(nr)))
    fr = kind == "far"
    p[fr] = hi + span * rng.uniform(1, 3, (int(fr.sum()), D)) * rng.choice([-1.0, 1.0], (int(fr.sum()), D))
    return np.ascontiguousarray(p.astype(F)), kind


def keys(mn, mx, p):
    """Aabb::min_distance_squared of every box for one point (knnref.keys)."""
    from tests import knnref

    return knnref.keys(mn, mx, p)


RADIUS_KINDS = ("zero", "negzero", "inf", "overflow", "underflow", "roundup", "exact", "random")


def _roundup_radius(key, F):
    """The smallest r >= 0 with fl(r * r) == key, found by bisection over the bit patterns of T (fl(r * r) is monotone in r), or None
    when no r rounds onto key.  Where key is not a square, r * r is below key in exact arithmetic."""
    U = np.uint32 if F == np.float32 else np.uint64
    lo, hi = 0, int(np.array([np.inf], dtype=F).view(U)[0])
    with np.errstate(all="ignore"):
        while lo < hi:                                       # smallest bit pattern with fl(r * r) >= key
            mid = (lo + hi) // 2
            r = np.array([mid], dtype=U).view(F)[0]
            if r * r >= key:
                hi = mid
            else:
                lo = mid + 1
        r = np.array([lo], dtype=U).view(F)[0]
        return r if r * r == key else None


def ball_keys(mn, mx, p):
    """Ball::intersects_aabb's squared distance of every box for one point: clamp p into the box, then the squares of (x - p) summed
    left to right, in T."""
    F = mn.dtype.type
    p = np.asarray(p, dtype=F)
    with np.errstate(all="ignore"):
        x = np.where(p < mn, mn, p)
        x = np.where(x > mx, mx, x)
        d = (x - p).astype(F)
        acc = d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]
        for k in range(2, mn.shape[1]):
            acc = acc + d[:, k] * d[:, k]
    return acc


def radii(mn, mx, pts, prec, seed=0, key_fn=None):
    """(one limit per point, kind of every limit), the RADIUS_KINDS in turn.  overflow: fl(r * r) = +inf, so every key qualifies, +inf
    ones included; underflow: r > 0 with fl(r * r) = 0; roundup: the smallest r whose fl(r * r) is the point's least non-zero finite key
    (r * r is below it in exact arithmetic wherever that key is not a square); exact: r * r equal to a key.  The keys are
    key_fn(p) (default: the boxes' Aabb::min_distance_squared; pass the triangle or the ball keys to reach their edges)."""
    F = FT[prec]
    rng = _rng("edge_dims_radii", len(pts), prec, seed, len(mn))
    fi = np.finfo(F)
    big = F(np.sqrt(float(fi.max)) * 4)
    small = F(np.sqrt(float(fi.smallest_subnormal)) / 4)
    out = np.zeros(len(pts), dtype=F)
    kind = np.array(RADIUS_KINDS)[np.arange(len(pts)) % len(RADIUS_KINDS)]
    for i, p in enumerate(pts):
        k = kind[i]
        d2 = key_fn(p) if key_fn is not None else keys(mn, mx, p)
        pos = d2[(d2 > 0) & np.isfinite(d2)]
        if k == "zero":
            out[i] = 0.0
        elif k == "negzero":
            out[i] = -0.0
        elif k == "inf":
            out[i] = np.inf
        elif k == "overflow":
            out[i] = big
        elif k == "underflow":
            out[i] = small
        elif k == "roundup" and len(pos):
            r = _roundup_radius(pos.min(), F)
            out[i] = r if r is not None else F(np.sqrt(np.float64(pos.min())))
        elif k == "exact" and len(pos):
            key = pos[rng.integers(0, len(pos))]
            r = F(np.sqrt(np.float64(key)))
            for c in (r, np.nextafter(r, F(np.inf)), np.nextafter(r, F(0))):
                with np.errstate(all="ignore"):
                    if c * c == key:
                        r = c
                        break
            out[i] = r
        else:
            span = float(np.max(mx.astype(np.float64) - mn.astype(np.float64)))
            out[i] = F(rng.uniform(0, 1) * span)
    return out, kind


def queries(kind, mn, mx, m, prec, seed=0):
    """(m, stride) records of dimref's query kinds on the points of `points`: POINT the points; AABB boxes [p, p + e] with e a random
    fraction of a shape's own extent (a quarter of them degenerate, e = 0); BALL centres p with the radii of `radii` keyed by
    ball_keys, so r * r overflows, underflows and rounds up onto a ball distance."""
    F = FT[prec]
    p, _ = points(mn, mx, m, prec, seed)
    if kind == dimref.POINT:
        return p
    rng = _rng("edge_dims_queries", kind, m, mn.shape[1], prec, seed, len(mn))
    if kind == dimref.AABB:
        ext = (mx.astype(np.float64) - mn.astype(np.float64))[rng.integers(0, len(mn), m)] * rng.uniform(0, 1.5, (m, mn.shape[1]))
        ext[np.arange(m) % 4 == 1] = 0
        with np.errstate(all="ignore"):
            hi = (p.astype(np.float64) + ext).astype(F)
        return np.ascontiguousarray(np.concatenate([p, hi], axis=1), dtype=F)
    r, _ = radii(mn, mx, p, prec, seed, key_fn=lambda q: ball_keys(mn, mx, q))
    return np.ascontiguousarray(np.concatenate([p, r[:, None]], axis=1), dtype=F)


def limits(tree, o, inv, prec, seed=0):
    """{name: per-ray limits or None}: anyhit.tmax_families of each ray's closest entry d* (dimorder.Tree.closest), plus "subnormal"
    (the smallest subnormal for every ray) and "exit" (the exit distance of the ray's closest shape; +inf without one)."""
    F = FT[prec]
    m = len(o)
    dstar = np.full(m, np.inf, dtype=F)
    exit_ = np.full(m, np.inf, dtype=F)
    for i in range(m):
        ray = (list(o[i]), list(inv[i]))
        s, e = tree.closest(ray)
        if e is not None:
            dstar[i] = e
            exit_[i] = dimorder.slice(ray, *tree.shapes[s])[1]
    fam = anyhit.tmax_families(dstar, F, _rng("edge_dims_limits", m, prec, seed))
    fam["subnormal"] = np.full(m, np.finfo(F).smallest_subnormal, dtype=F)
    fam["exit"] = exit_
    return fam, dstar


def triangles(mn, mx, prec, seed=0):
    """One triangle per box of a 3-D scene, its vertices at random points of the box (computed in f64, rounded to T, clamped into the
    box): (n, 9) of T.  The shapes for the tree are the triangles' own boxes (O.tri_aabbs), which lie inside the scene's boxes."""
    F = FT[prec]
    rng = _rng("edge_dims_triangles", len(mn), prec, seed)
    a, b = mn.astype(np.float64), mx.astype(np.float64)
    v = a[:, None, :] + rng.random((len(mn), 3, 3)) * (b - a)[:, None, :]
    v = np.clip(v.astype(F), mn[:, None, :], mx[:, None, :])
    return np.ascontiguousarray(v.reshape(-1, 9), dtype=F)


# ---- precondition counters ---------------------------------------------------------------------------------------------------------
def empty_child_boxes(nodes) -> int:
    """Inner nodes with an Aabb::empty() child box (what "no split wins" stores), any D."""
    inner = nodes["child_l"] != 0xFFFFFFFF
    e = (nodes["l_aabb"]["min"][:, 0] > nodes["l_aabb"]["max"][:, 0]) | (nodes["r_aabb"]["min"][:, 0] > nodes["r_aabb"]["max"][:, 0])
    return int(np.sum(inner & e))


def ray_facts(o, d, inv, mn, mx) -> dict:
    """Counts of the arithmetic a batch of rays exercises against the boxes, in the rays' own precision (edge_inputs.ray_facts in D)."""
    F = o.dtype.type
    tiny = np.finfo(F).tiny
    zero = d == 0
    sub = (d != 0) & (np.abs(d) < tiny)
    facts = {
        "nonzero_direction": int(np.sum(np.any(d != 0, axis=1))),
        "neg_zero": int(np.sum(zero & np.signbit(d))),
        "pos_zero": int(np.sum(zero & ~np.signbit(d))),
        "inv_neg_inf": int(np.sum(inv == -np.inf)),
        "inv_pos_inf": int(np.sum(inv == np.inf)),
        "subnormal_dir_finite_inv": int(np.sum(sub & np.isfinite(inv))),
        "subnormal_dir_inf_inv": int(np.sum(sub & np.isinf(inv))),
        "axes_special": sorted(set(np.nonzero(sub | zero)[1].tolist())),
    }
    ovf = nan = subn = 0
    with np.errstate(all="ignore"):
        for b in (mn, mx):
            for k in range(o.shape[1]):
                diff = (b[None, :, k] - o[:, k, None]).astype(F)
                prod = (diff * inv[:, k, None]).astype(F)
                ovf += int(np.sum(np.isinf(prod) & np.isfinite(diff) & np.isfinite(inv[:, k, None])))
                nan += int(np.sum(np.isnan(prod) & zero[:, k, None]))
                subn += int(np.sum((diff != 0) & (np.abs(diff) < tiny)))
    facts["overflowing_products"] = ovf
    facts["face_plane_nan"] = nan
    facts["subnormal_differences"] = subn
    return facts
