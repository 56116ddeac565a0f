"""tests/knnref.py -- two models of the k-nearest-shapes query (bvhgpu_knn_*), any dimension D, numpy.float32 / numpy.float64 scalars.

    brute   the contract itself: key d2_s = dimref.min_distance_sq of shape s's own box; s qualifies with no limit, or with a limit r
            when r >= 0 (-0 included) and d2_s <= fl(r * r); row = the first k qualifying shapes of a stable sort by (d2_s, s), their
            distances fl(sqrt(d2_s)), then (U32_MAX, +inf) padding.  Vectorised over the shapes (elementwise numpy ops round in T, one
            rounding per operation, in the reference's order).
    walk    a restatement of knn_walk<D, T, K> (queries.cuh) with numpy scalars: children ordered by the slacked lower bound
            box_lower_d2 (nearer first, left on ties), a child entered when its box is empty or its bound is <= min(k-th key, r * r),
            the far child decided after the near subtree is done.  Returns the row and the number of nodes visited.

D = 2 runs on the device through the z = 0 lift, whose z terms are exactly +0, so the 2-D restatement is this one with D = 2."""
import numpy as np

from tests import dimref
from tests.prunedmodel import box_lower_d2

U32_MAX = 0xFFFFFFFF


def keys(mn, mx, p):
    """d2 of every shape for one point p (D,): Aabb::min_distance_squared, vectorised over the (n, D) boxes."""
    F = mn.dtype.type
    with np.errstate(all="ignore"):
        hs = (mx - mn) * F(0.5)
        c = mn + hs
        q = np.abs(np.asarray(p, dtype=F) - c) - hs
        o = np.where(q > F(0), q, F(0)).astype(F)
        acc = o[:, 0] * o[:, 0] + o[:, 1] * o[:, 1]
        for a in range(2, mn.shape[1]):
            acc = acc + o[:, a] * o[:, a]
    return acc


def brute(mn, mx, pts, k, max_dist=None):
    """(shape (m, k) u32, dist (m, k) T) by the contract."""
    F = mn.dtype.type
    m = len(pts)
    out_s = np.full((m, k), U32_MAX, dtype=np.uint32)
    out_d = np.full((m, k), np.inf, dtype=F)
    for i in range(m):
        if len(mn) == 0:
            continue
        d2 = keys(mn, mx, pts[i])
        if max_dist is not None:
            r = F(max_dist[i])
            if not r >= F(0):
                continue
            with np.errstate(all="ignore"):
                ok = d2 <= r * r
        else:
            ok = np.ones(len(d2), dtype=bool)
        idx = np.flatnonzero(ok)
        order = idx[np.argsort(d2[idx], kind="stable")][:k]
        out_s[i, : len(order)] = order
        with np.errstate(all="ignore"):
            out_d[i, : len(order)] = np.sqrt(d2[order])
    return out_s, out_d


class Walk:
    """knn_walk over a node array in any dimension (C-ABI field names) and the shapes' current boxes ((n, D) min / max arrays)."""

    def __init__(self, nodes, mn, mx):
        self.par = [int(x) for x in nodes["parent"]]
        self.cl = [int(x) for x in nodes["child_l"]]
        self.cr = [int(x) for x in nodes["child_r"]]
        self.sh = [int(x) for x in nodes["shape"]]
        self.box = [(list(nodes["l_aabb"]["min"][i]), list(nodes["l_aabb"]["max"][i]), list(nodes["r_aabb"]["min"][i]),
                     list(nodes["r_aabb"]["max"][i])) for i in range(len(nodes))]
        self.shapes = [(list(a), list(b)) for a, b in zip(mn, mx)]
        self.F = mn.dtype.type

    def row(self, p, k, r=None):
        """(shapes, dists, visits) of one point p (sequence of T), k slots, limit r (None: none)."""
        F = self.F
        p = [F(x) for x in p]
        inf = F(np.inf)
        lst = []                                               # ascending (d2, s), at most k entries
        visits = 0
        with np.errstate(all="ignore"):
            r2 = inf if r is None else F(r) * F(r)
        if self.cl and (r is None or F(r) >= F(0)):
            def thr():
                return lst[-1][0] if len(lst) == k else inf

            def enter(b, e):
                t = thr()
                return e or (b <= t and b <= r2)

            def leaf(s):
                key = dimref.min_distance_sq(p, *self.shapes[s])
                if key <= r2 and (len(lst) < k or (key, s) < lst[-1]):
                    lst.append((key, s))
                    lst.sort()
                    del lst[k:]

            # the parent-link walk as a stack of pending decisions: ("node", i) expands node i; ("try", i, bound, empty) decides a
            # child when it is popped, i.e. after the subtree pushed above it has been walked
            stack = [("node", 0)]
            while stack:
                item = stack.pop()
                if item[0] == "try":
                    if enter(item[2], item[3]):
                        stack.append(("node", item[1]))
                    continue
                i = item[1]
                visits += 1
                if self.cl[i] == U32_MAX:
                    leaf(self.sh[i])
                    continue
                lmn, lmx, rmn, rmx = self.box[i]
                dl, dr = box_lower_d2(p, lmn, lmx), box_lower_d2(p, rmn, rmx)
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

    def rows(self, pts, k, max_dist=None):
        out = [self.row(p, k, None if max_dist is None else max_dist[i]) for i, p in enumerate(pts)]
        return np.array([o[0] for o in out]).reshape(len(pts), k), np.array([o[1] for o in out], dtype=self.F).reshape(len(pts), k), [o[2] for o in out]
