"""tests/multihit.py -- restatement of the device's multi-hit walk (multi_hit_kernel<D, T, TRI, K>, closest.cu), with numpy.float32 /
numpy.float64 scalars (one rounding per operation, no FMA), and the brute force it is held to.  TEST INFRASTRUCTURE: pinned to the C++
oracle at D = 3 by tests/test_multi_hit_cpu.py and compared with the device bit for bit by tests/test_gpu_multi_hit.py.

The walk is closest_kernel's (near child first by slab entry, left on ties, a missed box counts as entry +inf; the far child is judged
when the walk comes back to it, against the list as it is then) keeping the k smallest keys in key_less order:
    AABB mode       key (entry of the shape's own box, the leaf's node index); a leaf qualifies when its own box passes the slab test
                    and, with a limit, entry < tmax.  A child is entered when its slab test passes, entry <= kth and, with a limit,
                    entry < tmax.
    triangle mode   key (Moeller-Trumbore distance d, shape); a leaf qualifies when d < tmax (+inf without a limit).  A child is entered
                    when its slab test passes, entry <= fl(kth * (1 + 2^-16)) and entry <= fl(tmax * (1 + 2^-16)).
kth is the k-th key's distance once the list holds k entries, +inf before.  A root leaf (n = 1) first tests the shape's own box.

    aabb / aabb_batch          AABB mode in any D on a dimref.Tree (the slice of tests/dimorder.py)
    triangles                  triangle mode in D = 3 on a C-ABI node array (moeller_trumbore / slice_entry of tests/prunedmodel.py)
    brute_aabb / brute_aabb_batch, brute_triangles
                               the loop over Bvh::traverse's set (BVH semantics), stably sorted by key; brute_triangles also returns
                               per ray whether every triangle of its row is bounded: the box its parent stores for it (the own box at a
                               root leaf) passes the slab test with entry <= fl(d * (1 + 2^-16)).
Rows are (shape (m, k) u32, dist (m, k), uv (m, k, 2) or None), padded with (U32_MAX, +inf, 0, 0)."""
import numpy as np

from tests import dimorder
from tests import prunedmodel as M

U32_MAX = 0xFFFFFFFF


def _less(a, ia, b, ib):
    return a < b or (a == b and ia < ib)


def _offer(lst, k, key, i):
    """knn_insert on an ascending list of at most k (key, id) pairs."""
    if len(lst) == k and not _less(key, i, *lst[-1]):
        return
    pos = len(lst)
    while pos > 0 and _less(key, i, *lst[pos - 1]):
        pos -= 1
    lst.insert(pos, (key, i))
    del lst[k:]


def _kth(lst, k, F):
    return lst[-1][0] if len(lst) == k else F(np.inf)


def _walk(n_nodes, root_leaf, children, leaf, enter):
    """The stackless walk with an explicit stack.  children(i) -> [(child, slab hit, entry)] near first, or None at a leaf; a child is
    judged by enter(hit, entry) when it is popped, i.e. when the device's walk reaches it."""
    if n_nodes == 0:
        return
    if root_leaf is not None:
        root_leaf()
        return
    stack = [(0, True, None)]
    while stack:
        i, ok, e = stack.pop()
        if e is not None and not enter(ok, e):
            continue
        cs = children(i)
        if cs is None:
            leaf(i)
            continue
        stack.append(cs[1])
        stack.append(cs[0])


def _order(cl, cr, hl, el, hr, er, F):
    el, er = (el if hl else F(np.inf)), (er if hr else F(np.inf))
    left, right = (cl, hl, el), (cr, hr, er)
    return [left, right] if el <= er else [right, left]


def _pad(rows, k, F, uv):
    m = len(rows)
    sh = np.full((m, k), U32_MAX, dtype=np.uint32)
    di = np.full((m, k), np.inf, dtype=F)
    u = np.zeros((m, k, 2), dtype=F) if uv else None
    for r, row in enumerate(rows):
        for j, e in enumerate(row):
            sh[r, j], di[r, j] = e[0], e[1]
            if uv:
                u[r, j] = e[2], e[3]
    return sh, di, u


# ---- AABB mode, any D ---------------------------------------------------------------------------------------------------------------
def aabb(tree, ray, k, tmax):
    """One ray: ray = (origin, inv_direction) as T sequences, tmax a T scalar or None.  [(shape, entry)] ascending, at most k."""
    N = tree.nodes
    F = type(ray[1][0])
    lst = []

    def leaf(i):
        s = N[i][2]
        sl = dimorder.slice(ray, *tree.shapes[s])
        if sl is not None and (tmax is None or sl[0] < tmax):
            _offer(lst, k, sl[0], i)

    def children(i):
        cl, cr, _, lmn, lmx, rmn, rmx = N[i]
        if cl == U32_MAX:
            return None
        sl, sr = dimorder.slice(ray, lmn, lmx), dimorder.slice(ray, rmn, rmx)
        return _order(cl, cr, sl is not None, sl[0] if sl else F(0), sr is not None, sr[0] if sr else F(0), F)

    def enter(ok, e):
        return ok and e <= _kth(lst, k, F) and (tmax is None or e < tmax)

    def root_leaf():
        if dimorder.slice(ray, *tree.shapes[N[0][2]]) is not None:
            leaf(0)

    _walk(len(N), root_leaf if N and N[0][0] == U32_MAX else None, children, leaf, enter)
    return [(N[i][2], e) for e, i in lst]


def _limits(m, tmax):
    return [None] * m if tmax is None else list(tmax)


def aabb_batch(nodes, shapes, o, inv, k, tmax):
    """aabb over a batch: o, inv (m, D) arrays of T; tmax (m,) of T or None.  (shape (m, k), dist (m, k), None)."""
    tree = dimorder.Tree(nodes, shapes)
    F = o.dtype.type
    tm = _limits(len(o), tmax)
    rows = [aabb(tree, (list(o[r]), list(inv[r])), k, tm[r]) for r in range(len(o))]
    return _pad(rows, k, F, False)


def _leaves(N, ray):
    """Bvh::traverse with a ray, DFS order: [node index of each candidate leaf].  A root leaf tests the shape's own box; every other leaf
    is reached through the child boxes its ancestors store."""
    if not N:
        return []
    if N[0][0] == U32_MAX:
        return [0]
    out, stack = [], [0]
    while stack:
        i = stack.pop()
        cl, cr, _, lmn, lmx, rmn, rmx = N[i]
        if cl == U32_MAX:
            out.append(i)
            continue
        if dimorder.slice(ray, rmn, rmx) is not None:
            stack.append(cr)
        if dimorder.slice(ray, lmn, lmx) is not None:
            stack.append(cl)
    return out


def brute_aabb(tree, ray, k, tmax):
    """[(shape, entry)]: the candidates whose own box the ray enters (before tmax), stably sorted by (entry, node index), first k."""
    q = []
    for i in _leaves(tree.nodes, ray):
        s = tree.nodes[i][2]
        sl = dimorder.slice(ray, *tree.shapes[s])
        if sl is not None and (tmax is None or sl[0] < tmax):
            q.append((sl[0], i, s))
    q.sort(key=lambda t: (t[0], t[1]))
    return [(s, e) for e, _, s in q[:k]]


def brute_aabb_batch(nodes, shapes, o, inv, k, tmax):
    tree = dimorder.Tree(nodes, shapes)
    F = o.dtype.type
    tm = _limits(len(o), tmax)
    rows = [brute_aabb(tree, (list(o[r]), list(inv[r])), k, tm[r]) for r in range(len(o))]
    return _pad(rows, k, F, False)


# ---- triangle mode, D = 3 -----------------------------------------------------------------------------------------------------------
class _Tris:
    """A C-ABI node array, its shapes and triangles unpacked once."""

    def __init__(self, nodes, shapes, tris):
        self.F = shapes["min"].dtype.type
        self.tr = np.ascontiguousarray(tris, dtype=self.F).reshape(-1, 3, 3)
        self.cl, self.cr, self.sh = (nodes[a].astype(np.int64).tolist() for a in ("child_l", "child_r", "shape"))
        self.box = [[nodes[a][b][i] for a in ("l_aabb", "r_aabb") for b in ("min", "max")] for i in range(len(nodes))]
        self.own_mn, self.own_mx = shapes["min"], shapes["max"]
        self.n = len(nodes)

    def ray(self, rays, r):
        return list(rays["origin"][r]), list(rays["direction"][r]), list(rays["inv_direction"][r])

    def stored(self):
        """shape -> (min, max) of the box the walk tests last before its leaf."""
        if self.n == 1:
            s = self.sh[0]
            return {s: (self.own_mn[s], self.own_mx[s])}
        out = {}
        for i in range(self.n):
            if self.cl[i] != U32_MAX:
                lmn, lmx, rmn, rmx = self.box[i]
                for c, mn, mx in ((self.cl[i], lmn, lmx), (self.cr[i], rmn, rmx)):
                    if self.cl[c] == U32_MAX:
                        out[self.sh[c]] = (mn, mx)
        return out


def triangles(nodes, shapes, tris, rays, k, tmax):
    """Triangle mode over a batch of 3-D C-ABI rays: (shape (m, k), dist (m, k), uv (m, k, 2))."""
    t = _Tris(nodes, shapes, tris)
    F = t.F
    margin = F(1) + F(1.0 / 65536.0)
    tm = _limits(len(rays), tmax)
    rows = []
    for r in range(len(rays)):
        o, d, inv = t.ray(rays, r)
        lim = F(np.inf) if tm[r] is None else tm[r]
        with np.errstate(all="ignore"):
            tbound = lim * margin
        lst = []

        def leaf(i):
            s = t.sh[i]
            dist = M.moeller_trumbore(o, d, *t.tr[s])[0]
            if dist < lim:
                _offer(lst, k, dist, s)

        def children(i):
            if t.cl[i] == U32_MAX:
                return None
            lmn, lmx, rmn, rmx = t.box[i]
            hl, el = M.slice_entry(o, inv, lmn, lmx)
            hr, er = M.slice_entry(o, inv, rmn, rmx)
            return _order(t.cl[i], t.cr[i], hl, el, hr, er, F)

        def enter(ok, e):
            with np.errstate(all="ignore"):
                return ok and e <= _kth(lst, k, F) * margin and e <= tbound

        def root_leaf():
            s = t.sh[0]
            if M.slice_entry(o, inv, t.own_mn[s], t.own_mx[s])[0]:
                leaf(0)

        _walk(t.n, root_leaf if t.n == 1 else None, children, leaf, enter)
        rows.append([(s, dist) + tuple(M.moeller_trumbore(o, d, *t.tr[s])[1:]) for dist, s in lst])
    return _pad(rows, k, F, True)


def brute_triangles(nodes, shapes, tris, rays, k, tmax):
    """The unpruned row: the loop over Bvh::traverse's set with intersects_triangle, qualifying d < tmax (+inf without a limit), stably
    sorted by (d, s), first k.  (shape, dist, uv, bounded (m,) bool: every triangle of the row is bounded)."""
    t = _Tris(nodes, shapes, tris)
    F = t.F
    margin = F(1) + F(1.0 / 65536.0)
    stored = t.stored()
    tm = _limits(len(rays), tmax)
    rows, bounded = [], np.ones(len(rays), dtype=bool)
    for r in range(len(rays)):
        o, d, inv = t.ray(rays, r)
        lim = F(np.inf) if tm[r] is None else tm[r]
        q = []
        for i in _tri_leaves(t, o, inv):
            s = t.sh[i]
            dist, u, v = M.moeller_trumbore(o, d, *t.tr[s])
            if dist < lim:
                q.append((dist, s, u, v))
        q.sort(key=lambda e: (e[0], e[1]))
        row = [(s, dist, u, v) for dist, s, u, v in q[:k]]
        for s, dist, _, _ in row:
            hit, e = M.slice_entry(o, inv, *stored[s])
            with np.errstate(all="ignore"):
                if not (hit and e <= dist * margin):
                    bounded[r] = False
        rows.append(row)
    return _pad(rows, k, F, True) + (bounded,)


def _tri_leaves(t, o, inv):
    if t.n == 0:
        return []
    if t.n == 1:
        s = t.sh[0]
        return [0] if M.slice_entry(o, inv, t.own_mn[s], t.own_mx[s])[0] else []
    out, stack = [], [0]
    while stack:
        i = stack.pop()
        if t.cl[i] == U32_MAX:
            out.append(i)
            continue
        lmn, lmx, rmn, rmx = t.box[i]
        if M.slice_entry(o, inv, rmn, rmx)[0]:
            stack.append(t.cr[i])
        if M.slice_entry(o, inv, lmn, lmx)[0]:
            stack.append(t.cl[i])
    return out


def weak_ok(shape, dist, tris, rays, tmax, cand):
    """The guarantee off the bounded rows, per ray: the filled slots come first, each is a distinct candidate s with
    dist == intersects_triangle(s) < tmax, in ascending (dist, s) order.  Returns the rays that break it."""
    F = dist.dtype.type
    tr = np.ascontiguousarray(tris, dtype=F).reshape(-1, 3, 3)
    bad = []
    for r in range(len(shape)):
        o, d = list(rays["origin"][r]), list(rays["direction"][r])
        lim = F(np.inf) if tmax is None else tmax[r]
        n = int(np.sum(shape[r] != U32_MAX))
        ok = np.all(shape[r, n:] == U32_MAX) and np.all(np.isposinf(dist[r, n:])) and len(set(shape[r, :n].tolist())) == n
        for j in range(n):
            s = int(shape[r, j])
            ok = ok and s in cand[r] and M.moeller_trumbore(o, d, *tr[s])[0] == dist[r, j] and dist[r, j] < lim
            if j:
                ok = ok and _less(dist[r, j - 1], int(shape[r, j - 1]), dist[r, j], s)
        if not ok:
            bad.append(r)
    return bad
