"""tests/pyref.py -- second, independent restatement of the reference build/flatten/traverse
in pure Python with numpy.float32 / numpy.float64 scalars (every operation rounds in T, no
FMA possible).  TEST INFRASTRUCTURE: used to cross-check the C++ oracle on small scenes, so
that an oracle bug cannot hide behind "GPU == oracle".  Follows SURVEY.md Appendix A and the
reference lines cited there (src/bvh/bvh_node.rs:81-279, src/flat_bvh.rs:60-143,
src/ray/intersect_default.rs:16-37)."""
import numpy as np

U32_MAX = 0xFFFFFFFF


def _dot(v):
    """nalgebra small-vector dot, left to right: (x*x + y*y) [+ z*z]."""
    acc = v[0] * v[0] + v[1] * v[1]
    for k in range(2, len(v)):
        acc = acc + v[k] * v[k]
    return acc


def _sa(F, mn, mx):
    s = [F(mx[k]) - F(mn[k]) for k in range(len(mn))]
    return F(2) * _dot(s)


def _center(F, mn, mx):
    return [F(mn[k]) * F(0.5) + F(mx[k]) * F(0.5) for k in range(len(mn))]


def _join(a, b):
    return ([x if x <= y else y for x, y in zip(a[0], b[0])], [x if x >= y else y for x, y in zip(a[1], b[1])])


def _grow(a, p):
    return ([x if x <= y else y for x, y in zip(a[0], p)], [x if x >= y else y for x, y in zip(a[1], p)])


def build(aabbs, F=np.float32, root_aabb=None):
    """Returns (nodes, node_index): nodes[i] = ('leaf', parent, shape) | ('node', parent, cl, cr, laabb, raabb).
    root_aabb = (min, max): the box the root's split costs are divided by, instead of the joint box of the shapes (Bvh::build's).
    The device's in-place rebuild of a subtree takes the join of the root's two stored child boxes there (tests/rebuildref.py)."""
    n = len(aabbs)
    if n == 0:
        return [], []
    inf = F(np.inf)
    D = len(aabbs[0]["min"])
    EMPTY = ([inf] * D, [-inf] * D)
    boxes = [([F(v) for v in a["min"]], [F(v) for v in a["max"]]) for a in aabbs]
    ctrs = [_center(F, *b) for b in boxes]
    nodes = [None] * (2 * n - 1)
    node_index = [0] * n
    eps = np.finfo(F).eps
    K = F(6) - F(0.01)

    def joint(ids):
        ab, cb = EMPTY, EMPTY
        for i in ids:
            ab = _join(ab, boxes[i])
            cb = _grow(cb, ctrs[i])
        return ab, cb

    ab, cb = joint(range(n))
    if root_aabb is not None:
        ab = ([F(v) for v in root_aabb[0]], [F(v) for v in root_aabb[1]])
    stack = [(list(range(n)), 0, 0, ab, cb)]
    with np.errstate(all="ignore"):
        while stack:
            I, parent, me, AB, CB = stack.pop()
            if len(I) == 1:
                nodes[me] = ("leaf", parent, I[0])
                node_index[I[0]] = me
                continue
            size = [CB[1][k] - CB[0][k] for k in range(D)]
            axis = 0
            for k in range(1, D):
                if size[k] > size[axis]:
                    axis = k
            ext = size[axis]
            if ext < eps:
                h = len(I) // 2
                L, R = I[:h], I[h:]
                (LAB, LCB), (RAB, RCB) = joint(L), joint(R)
            else:
                bk = [[0, EMPTY, EMPTY, []] for _ in range(6)]
                for i in I:
                    rel = (ctrs[i][axis] - CB[0][axis]) / ext
                    b = int(rel * K)
                    bk[b][0] += 1
                    bk[b][1] = _join(bk[b][1], boxes[i])
                    bk[b][2] = _grow(bk[b][2], ctrs[i])
                    bk[b][3].append(i)
                best, min_cost = 0, inf
                LAB = LCB = RAB = RCB = EMPTY
                for s in range(5):
                    Ln, La, Lc = 0, EMPTY, EMPTY
                    for b in range(s + 1):
                        Ln += bk[b][0]; La = _join(La, bk[b][1]); Lc = _join(Lc, bk[b][2])
                    Rn, Ra, Rc = 0, EMPTY, EMPTY
                    for b in range(s + 1, 6):
                        Rn += bk[b][0]; Ra = _join(Ra, bk[b][1]); Rc = _join(Rc, bk[b][2])
                    cost = (F(Ln) * _sa(F, *La) + F(Rn) * _sa(F, *Ra)) / _sa(F, *AB)
                    if cost < min_cost:
                        best, min_cost = s, cost
                        LAB, LCB, RAB, RCB = La, Lc, Ra, Rc
                order = [i for b in range(6) for i in bk[b][3]]
                nl = sum(bk[b][0] for b in range(best + 1))
                L, R = order[:nl], order[nl:]
            cl = me + 1
            cr = cl + 2 * len(L) - 1
            nodes[me] = ("node", parent, cl, cr, LAB, RAB)
            stack.append((R, me, cr, RAB, RCB))
            stack.append((L, me, cl, LAB, LCB))
    return nodes, node_index


def flatten(nodes):
    """Literal recursion of src/flat_bvh.rs:60-143 (python recursion; small trees only)."""
    out = []
    if not nodes:
        return out

    def flat(i):
        nd = nodes[i]
        if nd[0] == "leaf":
            out.append((None, U32_MAX, len(out) + 1, nd[2]))
            return
        for child, aabb in ((nd[2], nd[4]), (nd[3], nd[5])):
            me = len(out)
            out.append(None)
            flat(child)
            out[me] = (aabb, me + 1, len(out), U32_MAX)

    flat(0)
    return out


def hit(F, ray, mn, mx):
    o, inv = ray
    with np.errstate(all="ignore"):
        l = [(F(mn[k]) - o[k]) * inv[k] for k in range(len(o))]
        r = [(F(mx[k]) - o[k]) * inv[k] for k in range(len(o))]
    if any(np.isnan(v) for v in l + r):
        return False
    lo = [min(a, b) for a, b in zip(l, r)]
    hi = [max(a, b) for a, b in zip(l, r)]
    tmin, tmax = max(lo), min(hi)
    z = F(0)
    return bool(tmax >= (tmin if tmin > z else z))


def ray_new(F, o, d):
    o = [F(v) for v in o]
    d = [F(v) for v in d]
    with np.errstate(all="ignore"):
        n = np.sqrt(_dot(d))
        d = [v / n for v in d]
        inv = [F(1) / v for v in d]
    return o, d, inv


def traverse_recursive(nodes, aabbs, ray, F=np.float32):
    out = []
    if not nodes:
        return out

    def rec(i):
        nd = nodes[i]
        if nd[0] == "node":
            if hit(F, ray, *nd[4]):
                rec(nd[2])
            if hit(F, ray, *nd[5]):
                rec(nd[3])
        else:
            if i != 0 or hit(F, ray, aabbs[nd[2]]["min"], aabbs[nd[2]]["max"]):
                out.append(nd[2])

    rec(0)
    return out


def traverse_flat(flat, aabbs, ray, F=np.float32):
    """FlatBvh::traverse (src/flat_bvh.rs:396-431) over flatten()'s output: a leaf re-tests its shape's own AABB."""
    out = []
    i = 0
    while i < len(flat):
        box, entry, exit_, shape = flat[i]
        if entry == U32_MAX:
            if hit(F, ray, aabbs[shape]["min"], aabbs[shape]["max"]):
                out.append(shape)
            i = exit_
        elif hit(F, ray, *box):
            i = entry
        else:
            i = exit_
    return out
