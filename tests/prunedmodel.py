"""A deterministic restatement of the device's two distance-pruned walks, in T with one rounding per operation (numpy scalars,
no FMA), in the operation order of the CUDA sources.  The GPU tests compare the device with it bit for bit; the CPU tests use it
to show that each adversarial family really reaches the case it is meant to reach.

- closest_triangles: closest_kernel<T, true> (closest.cu): the front-to-back walk over a node array with the pruning bound
  best * (1 + 2^-16), ties to the lower shape index, and the n = 1 root leaf;
- nearest_candidates: nearest_bound_kernel / nearest_bound4_kernel (U from the farthest corners) and the QUERY_WITHIN pass over the
  traversal records in FLAT semantics (queries.cuh), any dimension.  D = 2 runs through the z = 0 lift on the device, whose z terms
  are exactly +0, so the 2-D restatement is this one with D = 2.  slack=False restates the bound before the per-axis rounding
  slack existed (lower bound max(min - p, p - max, 0), U from the plain farthest corner)."""
import numpy as np

U32_MAX = 0xFFFFFFFF


def _eps(F):
    return F(np.finfo(F).eps)


# ---- closest hit, triangle mode ---------------------------------------------------------------------------------------------------
def slice_entry(o, inv, mn, mx):
    """Ray::intersection_slice_for_aabb as the device evaluates it: (hit, entry clamped at 0)."""
    F = type(o[0])
    with np.errstate(all="ignore"):
        ls = [(mn[k] - o[k]) * inv[k] for k in range(3)]
        rs = [(mx[k] - o[k]) * inv[k] for k in range(3)]
    if any(x != x for x in ls + rs):
        return False, F(0)
    tmin = max(max(min(ls[0], rs[0]), min(ls[1], rs[1])), min(ls[2], rs[2]))
    tmax = min(min(max(ls[0], rs[0]), max(ls[1], rs[1])), max(ls[2], rs[2]))
    entry = tmin if tmin > F(0) else F(0)
    return not (entry > tmax), entry


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def moeller_trumbore(o, d, a, b, c):
    """Ray::intersects_triangle: (distance or +inf, u, v)."""
    F = type(o[0])
    inf, eps = F(np.inf), _eps(F)
    with np.errstate(all="ignore"):
        ab = [b[k] - a[k] for k in range(3)]
        ac = [c[k] - a[k] for k in range(3)]
        uvec = _cross(d, ac)
        det = _dot(ab, uvec)
        if det < eps:
            return inf, F(0), F(0)
        inv_det = F(1) / det
        ao = [o[k] - a[k] for k in range(3)]
        u = _dot(ao, uvec) * inv_det
        if not (u >= F(0) and u <= F(1)):
            return inf, u, F(0)
        vvec = _cross(ao, ab)
        v = _dot(d, vvec) * inv_det
        if v < F(0) or u + v > F(1):
            return inf, u, v
        dist = _dot(ac, vvec) * inv_det
    return (dist if dist > eps else inf), u, v


def closest_triangles(nodes, shapes, tris, rays):
    """closest_kernel<T, true> per ray: (shape u32, distance, uv (n, 2))."""
    F = shapes["min"].dtype.type
    tr = np.ascontiguousarray(tris, dtype=F).reshape(-1, 3, 3)
    n = len(shapes)
    out_s = np.full(len(rays), U32_MAX, dtype=np.uint32)
    out_d = np.full(len(rays), np.inf, dtype=F)
    out_uv = np.zeros((len(rays), 2), dtype=F)
    if n == 0:
        return out_s, out_d, out_uv
    margin = F(1) + F(1.0 / 65536.0)
    lmn, lmx, rmn, rmx = (nodes[a][b] for a in ("l_aabb", "r_aabb") for b in ("min", "max"))
    cl, cr, sh = nodes["child_l"], nodes["child_r"], nodes["shape"]
    for r in range(len(rays)):
        o, d, inv = list(rays["origin"][r]), list(rays["direction"][r]), list(rays["inv_direction"][r])
        best = [U32_MAX, F(np.inf), F(0), F(0)]

        def leaf(s):
            t, u, v = moeller_trumbore(o, d, *tr[s])
            if t < best[1] or (t == best[1] and t < np.inf and s < best[0]):
                best[:] = [s, t, u, v]

        if n == 1:
            s = int(sh[0])
            if slice_entry(o, inv, shapes["min"][s], shapes["max"][s])[0]:
                leaf(s)
        else:
            stack = [(0, None)]                      # (node, entry to re-check against the bound when popped, None: go)
            while stack:
                i, e = stack.pop()
                if e is not None and not (e <= best[1] * margin):
                    continue
                if cl[i] == U32_MAX:
                    leaf(int(sh[i]))
                    continue
                hl, el = slice_entry(o, inv, lmn[i], lmx[i])
                hr, er = slice_entry(o, inv, rmn[i], rmx[i])
                el, er = (el if hl else F(np.inf)), (er if hr else F(np.inf))
                left_first = el <= er
                near, far = (int(cl[i]), int(cr[i])) if left_first else (int(cr[i]), int(cl[i]))
                ne, fe = (el, er) if left_first else (er, el)
                nok, fok = (hl, hr) if left_first else (hr, hl)
                if fok:
                    stack.append((far, fe))
                if nok:
                    stack.append((near, ne))
        out_s[r], out_d[r], out_uv[r] = best[0], best[1], (best[2], best[3])
    return out_s, out_d, out_uv


# ---- nearest_candidates ------------------------------------------------------------------------------------------------------------
def _floor(F):
    return F(2.0 ** -145) if F == np.float32 else F(2.0 ** -1070)


def axis_magnitude(p, mn, mx):
    with np.errstate(all="ignore"):
        m, nmn, ext = abs(p), -mn, mx - mn
    m = nmn if nmn > m else m
    m = mx if mx > m else m
    return ext if ext > m else m


def axis_slack(m):
    F = type(m)
    with np.errstate(all="ignore"):
        return m * (F(16) * _eps(F)) + _floor(F)


def box_lower_d2(p, mn, mx, slack=True):
    F = type(p[0])
    d2 = F(0)
    with np.errstate(all="ignore"):
        for k in range(len(p)):
            a, b = mn[k] - p[k], p[k] - mx[k]
            d = a if a > b else b
            if slack:
                d = d - axis_slack(axis_magnitude(p[k], mn[k], mx[k]))
            d = d if d > F(0) else F(0)
            d2 = d2 + d * d
    return d2


def box_upper_d2(p, mn, mx, g, slack=True):
    F = type(p[0])
    d2 = F(0)
    with np.errstate(all="ignore"):
        for k in range(len(p)):
            a, b = abs(p[k] - mn[k]), abs(p[k] - mx[k])
            d = a if a > b else b
            if slack and d > F(0):
                m = axis_magnitude(p[k], mn[k], mx[k])
                d = d + axis_slack(g[k] if g[k] > m else m)
            d2 = d2 + d * d
    return d2


class Tree:
    """A node array in any dimension (the device's own) with its shapes' AABBs, as lists of T scalars."""

    def __init__(self, nodes, shapes):
        self.cl = [int(x) for x in nodes["child_l"]]
        self.cr = [int(x) for x in nodes["child_r"]]
        self.sh = [int(x) for x in nodes["shape"]]
        self.box = [(list(nodes["l_aabb"]["min"][i]), list(nodes["l_aabb"]["max"][i]), list(nodes["r_aabb"]["min"][i]),
                     list(nodes["r_aabb"]["max"][i])) for i in range(len(nodes))]
        self.shapes = [(list(s["min"]), list(s["max"])) for s in shapes]

    def bound(self, p, slack=True):
        """nearest_bound_kernel: U for point p (T scalars), before nothing is listed for an empty tree."""
        F = type(p[0])
        if slack:
            lmn, lmx, rmn, rmx = self.box[0]
            g = []
            for k in range(len(p)):
                lm, rm = axis_magnitude(p[k], lmn[k], lmx[k]), axis_magnitude(p[k], rmn[k], rmx[k])
                g.append(lm if lm > rm else rm)
        else:
            g = None
        best = [None, None]

        def leaf(s):
            d = box_upper_d2(p, *self.shapes[s], g, slack)
            if best[0] is None or d < best[1]:
                best[:] = [s, d]

        stack = [(0, None)]
        while stack:
            i, dd = stack.pop()
            if dd is not None and not (best[0] is None or dd <= best[1]):
                continue
            if self.cl[i] == U32_MAX:
                leaf(self.sh[i])
                continue
            lmn, lmx, rmn, rmx = self.box[i]
            dl, dr = box_lower_d2(p, lmn, lmx, slack), box_lower_d2(p, rmn, rmx, slack)
            if dl > dr:
                stack += [(self.cl[i], dl), (self.cr[i], dr)]
            else:
                stack += [(self.cr[i], dr), (self.cl[i], dl)]
        with np.errstate(all="ignore"):
            return best[1] * (F(1) + F(16) * _eps(F))

    def candidates(self, p, slack=True):
        """The CSR list of point p in the device's order (preorder of the traversal records)."""
        if not self.cl:
            return []
        u = self.bound(p, slack)

        def hit(mn, mx):                                  # Query<T, QUERY_WITHIN, D>::hit: empty boxes are always entered
            return any(a > b for a, b in zip(mn, mx)) or box_lower_d2(p, mn, mx, slack) <= u

        if self.cl[0] == U32_MAX:                         # root leaf: its record is the shape's own AABB
            s = self.sh[0]
            return [s] if hit(*self.shapes[s]) else []
        out, stack = [], [0]
        while stack:
            i = stack.pop()
            if self.cl[i] == U32_MAX:
                if hit(*self.shapes[self.sh[i]]):         # FLAT semantics: a reached leaf re-tests the shape's own AABB
                    out.append(self.sh[i])
                continue
            lmn, lmx, rmn, rmx = self.box[i]
            if hit(rmn, rmx):
                stack.append(self.cr[i])
            if hit(lmn, lmx):
                stack.append(self.cl[i])
        return out
