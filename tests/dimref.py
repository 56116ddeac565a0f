"""tests/dimref.py -- restatement of the reference's non-ray IntersectsAabb queries and nearest_to, generic in the dimension D, with
numpy.float32 / numpy.float64 scalars (every operation rounds in T, in the reference's order, no FMA possible).  TEST INFRASTRUCTURE:
checked against the C++ oracle at D = 3 (tests/test_dim_queries_cpu.py) and then used as the oracle for D = 2 and D = 4.

    predicates       Aabb::intersects_aabb (src/aabb/aabb_impl.rs:240-248), Aabb::contains (:175-177), Ball::intersects_aabb
                     (src/ball.rs:85-99): clamp, then a left-to-right sum of squares <= r * r
    min_distance_sq  Aabb::min_distance_squared (aabb_impl.rs:618-629)
    query_bvh        Bvh::traverse with a query (src/bvh/bvh_node.rs:288-319): a root leaf tests the shape's own AABB
    query_flat       FlatBvh::traverse (src/flat_bvh.rs:396-431): every leaf tests the shape's own AABB
    nearest_bvh      Bvh::nearest_to (src/bvh/bvh_impl.rs:221-238) / nearest_to_recursive (src/bvh/bvh_node.rs:327-372)
    nearest_flat     FlatBvh::nearest_to (src/flat_bvh.rs:513-562)

Trees are the C ABI's node and flat arrays (numpy structured arrays of any D); shapes are AABB arrays with "min" / "max" fields.
Shapes are unit boxes in the reference's sense: their distance is their AABB's min_distance_squared.
Query records: kind 1 Aabb {min, max} (2D), kind 2 Point (D), kind 3 Ball {center, radius} (D + 1)."""
import numpy as np

U32_MAX = 0xFFFFFFFF
AABB, POINT, BALL = 1, 2, 3


def stride(kind, D):
    return {AABB: 2 * D, POINT: D, BALL: D + 1}[kind]


def predicate(kind, rec):
    """The query's intersects_aabb(mn, mx) for one record (a sequence of T scalars)."""
    rec = list(rec)
    if kind == AABB:
        D = len(rec) // 2
        qmn, qmx = rec[:D], rec[D:]

        def hit(mn, mx):
            for i in range(D):
                if qmx[i] < mn[i] or mx[i] < qmn[i]:
                    return False
            return True
    elif kind == POINT:
        p = rec

        def hit(mn, mx):
            return all(p[i] >= mn[i] for i in range(len(p))) and all(p[i] <= mx[i] for i in range(len(p)))
    else:
        c, r = rec[:-1], rec[-1]

        def hit(mn, mx):
            with np.errstate(all="ignore"):
                d2 = type(r)(0)
                for i in range(len(c)):
                    x = c[i]
                    if x < mn[i]:
                        x = mn[i]
                    if x > mx[i]:
                        x = mx[i]
                    d = x - c[i]
                    d2 = d2 + d * d
                return bool(d2 <= r * r)
    return hit


def min_distance_sq(p, mn, mx):
    F = type(mn[0])
    with np.errstate(all="ignore"):
        o = []
        for k in range(len(p)):
            hs = (mx[k] - mn[k]) * F(0.5)
            c = mn[k] + hs
            q = abs(p[k] - c) - hs
            o.append(q if q > F(0) else F(0))              # T::max(q, 0): NaN gives 0
        acc = o[0] * o[0] + o[1] * o[1]
        for k in range(2, len(o)):
            acc = acc + o[k] * o[k]
    return acc


def _nodes(nodes):
    return [(int(nd["child_l"]), int(nd["child_r"]), int(nd["shape"]), list(nd["l_aabb"]["min"]), list(nd["l_aabb"]["max"]),
             list(nd["r_aabb"]["min"]), list(nd["r_aabb"]["max"])) for nd in nodes]


def _flat(flat):
    return [(list(f["aabb"]["min"]), list(f["aabb"]["max"]), int(f["entry_index"]), int(f["exit_index"]), int(f["shape_index"])) for f in flat]


def _shapes(shapes):
    return [(list(s["min"]), list(s["max"])) for s in shapes]


class Tree:
    """A node array (and optionally its flat array) with the shapes, unpacked once into Python lists of T scalars."""

    def __init__(self, nodes, shapes, flat=None):
        self.nodes, self.shapes = _nodes(nodes), _shapes(shapes)
        self.flat = _flat(flat) if flat is not None else None

    def query_bvh(self, kind, rec):
        hit, out, N = predicate(kind, rec), [], self.nodes
        if not N:
            return out
        if N[0][0] == U32_MAX:
            return [N[0][2]] if hit(*self.shapes[N[0][2]]) else []

        def rec_(i):
            cl, cr, shape, lmn, lmx, rmn, rmx = N[i]
            if cl == U32_MAX:
                out.append(shape)
                return
            if hit(lmn, lmx):
                rec_(cl)
            if hit(rmn, rmx):
                rec_(cr)

        rec_(0)
        return out

    def query_flat(self, kind, rec):
        hit, out, i = predicate(kind, rec), [], 0
        while i < len(self.flat):
            mn, mx, entry, exit_, shape = self.flat[i]
            if entry == U32_MAX:
                if hit(*self.shapes[shape]):
                    out.append(shape)
                i = exit_
            else:
                i = entry if hit(mn, mx) else exit_
        return out

    def nearest_bvh(self, p):
        """(shape, sqrt(distance squared)) or (U32_MAX, None) for an empty tree."""
        N, best = self.nodes, [None, None]
        if not N:
            return U32_MAX, None

        def rec_(i):
            cl, cr, shape, lmn, lmx, rmn, rmx = N[i]
            if cl == U32_MAX:
                d = min_distance_sq(p, *self.shapes[shape])
                if best[0] is None or d < best[1]:
                    best[:] = [shape, d]
                return
            ch = [(cl, min_distance_sq(p, lmn, lmx)), (cr, min_distance_sq(p, rmn, rmx))]
            if ch[0][1] > ch[1][1]:
                ch.reverse()
            for idx, cd in ch:
                if best[0] is None or cd < best[1]:
                    rec_(idx)

        rec_(0)
        return best[0], np.sqrt(best[1])

    def nearest_flat(self, p):
        if not self.flat:
            return U32_MAX, None
        best, i = [None, None], 0
        while i < len(self.flat):
            mn, mx, entry, exit_, shape = self.flat[i]
            if entry == U32_MAX:
                d = min_distance_sq(p, *self.shapes[shape])
                if best[0] is None or d < best[1]:
                    best = [shape, d]
                i = exit_
            else:
                md = min_distance_sq(p, mn, mx)
                i = entry if (best[0] is None or md < best[1]) else exit_
        return best[0], np.sqrt(best[1])


# ---- inputs -------------------------------------------------------------------------------------------------------------------
SCENES = ("random", "coincident", "axis", "peel", "overflow")


def scene(kind, n, D, F, rng, axis=0):
    """(n, D) min / max arrays in T.  overflow: f32 surface areas overflow, so the builder stores empty child boxes."""
    if kind == "random":
        mn = rng.uniform(-100, 100, (n, D))
        mx = mn + rng.uniform(0, 8, (n, D)) ** 2 / 8
    elif kind == "coincident":                                # zero centroid extent: halving all the way down
        mn = mx = np.tile(np.arange(1, D + 1, dtype=np.float64), (n, 1))
    elif kind == "axis":                                      # all centres on one axis
        c = np.zeros((n, D)); c[:, axis] = rng.uniform(-50, 50, n)
        mn, mx = c - 0.5, c + 0.5
    elif kind == "peel":                                      # geometric centroids: a few shapes split off per level
        c = np.zeros((n, D)); c[:, 0] = 1.12 ** np.arange(n); c[:, 1:] = rng.uniform(-1, 1, (n, D - 1))
        mn = mx = c
    elif kind == "overflow":
        c = rng.uniform(-3e19, 3e19, (n, D))
        mn, mx = c - 1e18, c + 1e18
    else:
        raise ValueError(kind)
    return np.asarray(mn, dtype=F), np.asarray(mx, dtype=F)


def queries(kind, mn, mx, m, F, rng, nan=True):
    """(m, stride) records: random ones, points on box faces and corners, +0 / -0 components, degenerate boxes, zero-radius balls,
    and (nan=True) a few NaN components."""
    n, D = mn.shape
    lo, hi = (mn.min(axis=0).astype(np.float64), mx.max(axis=0).astype(np.float64)) if n else (np.full(D, -1.0), np.full(D, 1.0))
    span = np.maximum(hi - lo, 1.0)
    p = lo - 0.1 * span + rng.uniform(0, 1.2, (m, D)) * span
    if n:
        pick = rng.integers(0, n, m)
        face = rng.random((m, D)) < 0.5
        on = rng.random(m) < 0.4                              # on a face / corner of a shape's box
        p[on] = np.where(face[on], mn[pick[on]], mx[pick[on]])
    z = rng.random(m) < 0.08                                  # signed zeros
    p[z] = np.where(rng.random((int(z.sum()), D)) < 0.5, 0.0, -0.0)
    p = p.astype(F)
    if kind == POINT:
        rec = p
    elif kind == AABB:
        ext = (rng.uniform(0, 0.3, (m, D)) * span).astype(F)
        ext[rng.random(m) < 0.25] = 0                         # degenerate boxes: min == max
        rec = np.concatenate([p, (p + ext).astype(F)], axis=1)
    else:
        r = (rng.uniform(0, 0.2, m) * float(np.max(span))).astype(F)
        r[rng.random(m) < 0.25] = 0                           # zero radius
        rec = np.concatenate([p, r[:, None]], axis=1)
    rec = np.ascontiguousarray(rec, dtype=F)
    if nan and m >= 8:
        rows = rng.choice(m, max(1, m // 32), replace=False)
        rec[rows, rng.integers(0, rec.shape[1], len(rows))] = np.nan
    return rec


def points(mn, mx, m, F, rng):
    """Nearest_to query points: no NaN (the reference's nearest_to has no rule for it)."""
    return queries(POINT, mn, mx, m, F, rng, nan=False)
