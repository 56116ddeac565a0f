"""tests/crosswalk.py -- restatement of crossings_walk (closest.cu) over any node array, with and without a per-ray limit, vectorised
over rays with numpy.float32 / numpy.float64 (one rounding per operation, no FMA).  TEST INFRASTRUCTURE: pinned by
tests/test_crosswalk_cpu.py and compared with the device on every row by tests/test_gpu_crossings_edges.py.

The walk, as the kernel does it:
- a root leaf (n = 1) tests the shape's own box (the slab test only, no limit), then counts the triangle;
- otherwise a child is entered when crossings.slab hits the box its parent stores for it and the entry is <= fl(tmax * fl(1 + 2^-16))
  (+inf without a limit: every child whose slab test passes, Bvh::traverse's set; NaN: nothing is entered);
- at every reached leaf both windings are counted with d < tmax (crossings.mt).

    model           (front, back) u32 per ray.  The candidates are the oracle's Bvh::traverse set over the same node array (every stored
                    box on the path passes the slab test); each (ray, shape) pair then climbs the parent links and keeps the pair only if
                    every stored box on the path is entered at <= the bound.  Scales to 10^5 shapes and 10^4 rays.
    model_preorder  the same walk as a per-node loop over the tree from the root, for small scenes (an independent restatement)
    contains_model  the vote (crossings.vote) over the counts of crossings.point_rays
    crossing_distances / kth_limits  each ray's crossing distances (both windings) from a candidate CSR, and limits built around a
                    per-ray k-th one

Scenes (deterministic; their closed-form answers are checked by tests/test_crosswalk_cpu.py):
    layer_stack     4096 two-triangle quads at z = 0 .. 4095, odd layers flipped, rays nearly along +z away from every edge
    stale           triangles whose boxes are moved by twice their extent along +x, rays mostly along +x: every hit triangle lies in
                    front of the box the walk enters for it
    ball_pairs      two overlapping icospheres, nested ones with the same orientation and with the inner one flipped, with points at
                    least a margin away from every surface and their EVEN_ODD / NONZERO truths"""
import numpy as np

from oracle import oracle as O
from tests import crossings as X

U32_MAX = 0xFFFFFFFF


def _prec(F):
    return "f32" if F == np.float32 else "f64"


def bound(tmax, F, m):
    """fl(tmax * fl(1 + 2^-16)) per ray (+inf without a limit)."""
    lim = X._limit(tmax, F, m)
    with np.errstate(all="ignore"):
        return (lim * (F(1) + F(1.0 / 65536.0))).astype(F)


def candidates(nodes, shapes, rays):
    """(rows, shapes) int64 of the oracle's Bvh::traverse (MODE_RECURSIVE) over the node array: the pairs an unlimited walk counts."""
    if len(shapes) == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    F = rays["origin"].dtype.type
    tr = O.traverse(nodes, shapes, rays, O.MODE_RECURSIVE, _prec(F), count_stats=False)
    return X._rows(tr.offsets), tr.hits.astype(np.int64)


def _count(rays, tris, r, s, tmax):
    F = rays["origin"].dtype.type
    m = len(rays)
    lim = X._limit(tmax, F, m)
    tr = np.ascontiguousarray(tris, dtype=F).reshape(-1, 3, 3)
    df, db = X._windings(rays, tr, r, s)
    return (np.bincount(r[df < lim[r]], minlength=m).astype(np.uint32), np.bincount(r[db < lim[r]], minlength=m).astype(np.uint32))


def entered(nodes, rays, r, s, tmax, skip_empty=False):
    """bool per (ray, shape) pair of the Bvh::traverse set: every stored box on the path from the root to the shape's leaf is entered at
    <= the bound (always true at a root leaf and without a limit).  skip_empty: also refuse stored boxes with min > max, the mutant that
    treats the Aabb::empty() child boxes of "no split wins" nodes as empty (their slab test passes)."""
    F = rays["origin"].dtype.type
    keep = np.ones(len(r), dtype=bool)
    if len(nodes) <= 1 or len(r) == 0:
        return keep
    bd = bound(tmax, F, len(rays))
    # an Aabb::empty() stored box (min +inf, max -inf) passes crossings.slab at entry 0, as it passes slab_slice
    leafs = np.flatnonzero(nodes["child_l"] == U32_MAX)
    leaf_of = np.full(int(nodes["shape"][leafs].max()) + 1, -1, dtype=np.int64)
    leaf_of[nodes["shape"][leafs]] = leafs
    cur = leaf_of[s]
    assert np.all(cur >= 0)
    parent, cl = nodes["parent"].astype(np.int64), nodes["child_l"].astype(np.int64)
    o, inv = rays["origin"], rays["inv_direction"]
    act = np.flatnonzero(cur != 0)
    while len(act):
        c = cur[act]
        p = parent[c]
        left = (cl[p] == c)[:, None]
        mn = np.where(left, nodes["l_aabb"]["min"][p], nodes["r_aabb"]["min"][p])
        mx = np.where(left, nodes["l_aabb"]["max"][p], nodes["r_aabb"]["max"][p])
        rr = r[act]
        hit, e = X.slab(o[rr], inv[rr], mn, mx)
        keep[act] &= hit & (e <= bd[rr])
        if skip_empty:
            keep[act] &= ~(mn > mx).any(axis=1)
        cur[act] = p
        act = act[keep[act] & (p != 0)]
    return keep


def model(nodes, shapes, tris, rays, tmax=None, cand=None, skip_empty=False):
    """(front, back) u32 per ray of crossings_walk over the node array; tmax None, per ray or a scalar.  cand: the (rows, shapes) of
    candidates() if already computed."""
    r, s = candidates(nodes, shapes, rays) if cand is None else cand
    k = entered(nodes, rays, r, s, tmax, skip_empty)
    return _count(rays, tris, r[k], s[k], tmax)


def unlimited_walk(nodes, shapes, tris, rays, tmax=None, cand=None):
    """The mutant that ignores the bound when entering children: the loop over Bvh::traverse's set with d < tmax."""
    r, s = candidates(nodes, shapes, rays) if cand is None else cand
    return _count(rays, tris, r, s, tmax)


def model_preorder(nodes, shapes, tris, rays, tmax=None):
    """model as a loop over the nodes from the root (children after their parent), every ray at once: (n_nodes, m) reach flags."""
    F = rays["origin"].dtype.type
    m, n = len(rays), len(shapes)
    if n == 0:
        return np.zeros(m, np.uint32), np.zeros(m, np.uint32)
    o, inv = rays["origin"], rays["inv_direction"]
    if n == 1:
        s0 = int(nodes["shape"][0])
        hit, _ = X.slab(o, inv, np.broadcast_to(shapes["min"][s0], (m, 3)), np.broadcast_to(shapes["max"][s0], (m, 3)))
        r = np.flatnonzero(hit)
        return _count(rays, tris, r, np.full(len(r), s0, np.int64), tmax)
    bd = bound(tmax, F, m)
    reach = np.zeros((len(nodes), m), dtype=bool)
    reach[0] = True
    rr, ss = [], []
    stack = [0]
    while stack:
        i = stack.pop()
        if nodes["child_l"][i] == U32_MAX:
            r = np.flatnonzero(reach[i])
            rr.append(r)
            ss.append(np.full(len(r), nodes["shape"][i], np.int64))
            continue
        for side, key in (("child_l", "l_aabb"), ("child_r", "r_aabb")):
            c = int(nodes[side][i])
            hit, e = X.slab(o, inv, np.broadcast_to(nodes[key]["min"][i], (m, 3)), np.broadcast_to(nodes[key]["max"][i], (m, 3)))
            reach[c] = reach[i] & hit & (e <= bd)
            stack.append(c)
    return _count(rays, tris, np.concatenate(rr), np.concatenate(ss), tmax)


def contains_model(nodes, shapes, tris, points, rule, cand=None):
    """bool per point: the vote of its three rays (crossings.point_rays) counted by the model without a limit."""
    F = shapes["min"].dtype.type
    rays = X.point_rays(points, F)
    return X.vote(*model(nodes, shapes, tris, rays, None, cand), rule)


# ---- limits ---------------------------------------------------------------------------------------------------------------------------
def crossing_distances(rays, tris, r, s):
    """(rows, distances) of every finite crossing distance of the pairs (r, s), both windings, sorted by row then distance."""
    F = rays["origin"].dtype.type
    df, db = X._windings(rays, np.ascontiguousarray(tris, dtype=F).reshape(-1, 3, 3), r, s)
    rows, d = np.concatenate([r, r]), np.concatenate([df, db])
    fin = np.isfinite(d)
    rows, d = rows[fin], d[fin]
    order = np.lexsort((d, rows))
    return rows[order], d[order]


def kth_limits(rays, tris, cand, rng):
    """{name: limits} around each ray's k-th crossing distance d_k of the loop (k uniform per ray; +inf without a crossing): the
    families of anyhit.tmax_families on d_k, the last crossing's nextafter above, the smallest subnormal, the largest finite value
    (its bound overflows to +inf) and a scalar."""
    from tests import anyhit

    F = rays["origin"].dtype.type
    m = len(rays)
    rows, d = crossing_distances(rays, tris, *cand)
    cnt = np.bincount(rows, minlength=m)
    start = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    k = np.floor(rng.uniform(0, 1, m) * cnt).astype(np.int64)
    dk = np.full(m, np.inf, dtype=F)
    has = cnt > 0
    dk[has] = d[start[has] + k[has]]
    last = np.full(m, np.inf, dtype=F)
    last[has] = d[start[has] + cnt[has] - 1]
    fam = anyhit.tmax_families(dk, F, rng)
    fam["above_last"] = np.nextafter(last, F(np.inf)).astype(F)
    fam["subnormal"] = np.full(m, np.finfo(F).smallest_subnormal, dtype=F)
    fam["max_finite"] = np.full(m, np.finfo(F).max, dtype=F)
    fin = np.isfinite(dk)
    fam["scalar"] = F(np.median(dk[fin])) if fin.any() else F(1)
    return fam


# ---- scenes ---------------------------------------------------------------------------------------------------------------------------
EDGE_SHAPES, EDGE_PER_FAMILY = 160, 8


def ray_records(o, d, inv, prec):
    """Ray records of the C ABI from (o, d, inv) computed elsewhere (tests/edge_dims.ray_new keeps -0 and subnormal directions)."""
    from bvh_b200.dtypes import BY_PREC

    rays = np.zeros(len(o), dtype=BY_PREC[prec]["ray"])
    rays["origin"], rays["direction"], rays["inv_direction"] = o, d, inv
    return rays


def triangle_scenes(prec):
    """{name: (tris (n, 9), rays)}: the triangle families of tests/adversarial.py (grazing, shared edges, degenerate, the offset scene at
    two offsets) and the huge / mixed / subnormal edge scenes of tests/edge_dims.py with one triangle per box and the six ray families
    through the triangles' boxes."""
    from tests import adversarial as A
    from tests import edge_dims as ED

    F = np.float32 if prec == "f32" else np.float64
    out = {}
    for name, fn in (("grazing", A.grazing), ("shared_edges", A.shared_edges), ("degenerate", A.degenerate)):
        t, o, d = fn(F)[:3]
        out[name] = (np.ascontiguousarray(t, dtype=F).reshape(-1, 9), O.ray_new(o, d, prec))
    for off in ((1e4, 1e7) if prec == "f32" else (1e12, 1e15)):
        t, o, d = A.offset_scene(F, off)
        out[f"offset_{off:g}"] = (t, O.ray_new(o, d, prec))
    for kind in ED.SCENE_KINDS:
        mn, mx = ED.scene(kind, EDGE_SHAPES, 3, prec)
        t = ED.triangles(mn, mx, prec)
        s = O.tri_aabbs(t, prec)
        o, d, inv, _ = ED.ray_batch(s["min"], s["max"], EDGE_PER_FAMILY, prec)
        out[f"edge_{kind}"] = (t, ray_records(o, d, inv, prec))
    return out


LAYERS = 4096


def layer_stack(F, m=128, seed=0):
    """(tris (2 * LAYERS, 9), rays, z0): quads [-10, 10]^2 at z = 0 .. LAYERS - 1 split along y = x, odd layers with both triangles
    flipped; rays from z = z0 = -0.5 along (a, a, 1), |a| <= 1e-4, so x - y stays put and the drift stays below 0.5: every origin is at
    least 0.6 from the diagonal and 9.4 from the quads' edges.  A ray crosses every layer once, even layers through the back face."""
    rng = np.random.default_rng(seed)
    z = np.arange(LAYERS, dtype=np.float64)
    q = np.array([[-10, -10, 0], [10, -10, 0], [10, 10, 0], [-10, -10, 0], [10, 10, 0], [-10, 10, 0]], dtype=np.float64)
    t = np.repeat(q[None], LAYERS, axis=0)
    t[:, :, 2] = z[:, None]
    t = t.reshape(LAYERS, 2, 3, 3)
    odd = (np.arange(LAYERS) % 2 == 1)
    t[odd] = t[odd][:, :, [0, 2, 1]]
    tris = t.reshape(-1, 9).astype(F)
    x = rng.uniform(-9, 9, m)
    y = rng.uniform(-9, 9, m)
    bad = np.abs(x - y) < 0.6
    y[bad] = np.clip(x[bad] + np.where(x[bad] > 0, -1.0, 1.0) * rng.uniform(0.6, 2, int(bad.sum())), -9, 9)
    a = rng.uniform(-1e-4, 1e-4, m)
    a[: m // 8] = 0.0
    org = np.stack([x, y, np.full(m, -0.5)], axis=1)
    dirs = np.stack([a, a, np.ones(m)], axis=1)
    return tris, O.ray_new(org.astype(F), dirs.astype(F), _prec(F)), -0.5


def layer_limits(rays, j):
    """Per ray, the limit half a layer past layer j[r] (the origin is half a layer below layer 0): front + back == j + 1 below it."""
    F = rays["origin"].dtype.type
    dz = rays["direction"][:, 2].astype(np.float64)
    return ((np.asarray(j, dtype=np.float64) + 1.0) / dz).astype(F)


def stale(F, n=400, m=3000, seed=0):
    """(tris (n, 9), own boxes, moved boxes, rays): random triangles in a 200-unit cube, their boxes moved along +x by twice their x
    extent, rays mostly along +x aimed at triangle centroids from 5 .. 60 units before them.  A ray enters the moved box only after it
    has crossed the triangle."""
    rng = np.random.default_rng(seed)
    c = rng.uniform(-100, 100, (n, 1, 3))
    tris = (c + rng.normal(size=(n, 3, 3)) * rng.uniform(0.5, 4, (n, 1, 1))).astype(F)
    own = O.tri_aabbs(tris, _prec(F))
    moved = own.copy()
    ext = (own["max"][:, 0].astype(np.float64) - own["min"][:, 0])
    moved["min"][:, 0] = (own["min"][:, 0] + 2 * ext).astype(F)
    moved["max"][:, 0] = (own["max"][:, 0] + 2 * ext).astype(F)
    pick = rng.integers(0, n, m)
    w = rng.dirichlet([1, 1, 1], m)
    tgt = np.einsum("ij,ijk->ik", w, tris[pick].astype(np.float64))
    dirs = np.concatenate([np.ones((m, 1)), rng.normal(0, 0.02, (m, 2))], axis=1)
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    org = tgt - rng.uniform(5, 60, (m, 1)) * dirs
    return tris.reshape(n, 9), own, moved, O.ray_new(org.astype(F), dirs.astype(F), _prec(F))


def _ball_points(centres, radii, rng, m, margin):
    """Points in the box around the balls, at least `margin` from every sphere, and per ball the inside flag (m, k)."""
    lo = (np.asarray(centres) - np.asarray(radii)[:, None]).min(axis=0) - 0.3
    hi = (np.asarray(centres) + np.asarray(radii)[:, None]).max(axis=0) + 0.3
    p = rng.uniform(lo, hi, (6 * m, 3))
    r = np.stack([np.linalg.norm(p - c, axis=1) for c in centres], axis=1)
    ok = np.all(np.abs(r - np.asarray(radii)) > margin, axis=1)
    p, r = p[ok][:m], r[ok][:m]
    return p, r < np.asarray(radii)


def ball_pairs(F, level=3, m=6000, seed=0, margin=0.03):
    """{name: (tris (k, 3, 3), points (m, 3), truth EVEN_ODD, truth NONZERO)} for two unit icospheres overlapping at centre distance 0.8
    (EVEN_ODD: XOR, NONZERO: union), an icosphere of radius 0.5 inside one of radius 1 with the same outward orientation (EVEN_ODD: the
    shell, NONZERO: the whole ball) and the same with the inner one flipped (both: the shell).  The level-3 icosphere lies within 0.003
    of its sphere."""
    rng = np.random.default_rng(seed)
    ico = X.icosphere(level, np.float64)
    out = {}
    c2 = np.array([0.8, 0.0, 0.0])
    p, ins = _ball_points([np.zeros(3), c2], np.array([1.0, 1.0]), rng, m, margin)
    out["overlapping"] = (np.concatenate([ico, ico + c2]).astype(F), p.astype(F), ins[:, 0] ^ ins[:, 1], ins[:, 0] | ins[:, 1])
    p, ins = _ball_points([np.zeros(3), np.zeros(3)], np.array([1.0, 0.5]), rng, m, margin)
    shell = ins[:, 0] & ~ins[:, 1]
    out["nested"] = (np.concatenate([ico, 0.5 * ico]).astype(F), p.astype(F), shell, ins[:, 0])
    out["nested_flipped"] = (np.concatenate([ico, (0.5 * ico)[:, [0, 2, 1]]]).astype(F), p.astype(F), shell, shell)
    return out
