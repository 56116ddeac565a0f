"""tests/anyhit.py -- restatement of the device's any-hit walk (closest_kernel<D, T, TRI, true>, closest.cu), with numpy.float32 /
numpy.float64 scalars (one rounding per operation, no FMA).  TEST INFRASTRUCTURE: pinned to the C++ oracle at D = 3 by
tests/test_any_hit_cpu.py and compared with the device bit for bit by tests/test_gpu_any_hit.py.

The walk is the closest-hit walk with a per-ray constant bound: at an inner node both stored child boxes are sliced, the near one
(smaller entry, left on ties; a missed box counts as entry +inf) is opened first, then the far one, each only if the slab test
passes and
    AABB mode       entry < tmax                         (exact: no box entered at or beyond tmax holds a qualifying shape)
    triangle mode   entry <= fl(tmax * (1 + 2^-16))
A leaf is accepted when the shape's own AABB is entered at e < tmax (AABB mode) or its Moeller-Trumbore distance is < tmax
(triangle mode, the leaf is reached through its stored box only), and the first accepted leaf is the result.  A root leaf (n = 1)
first tests the shape's own box, as Bvh::traverse does (bvh_node.rs:314).

    aabb        AABB mode in any D, on a dimref.Tree (the slice of tests/dimorder.py)
    triangles   triangle mode in D = 3 on a C-ABI node array (moeller_trumbore / slice_entry of tests/prunedmodel.py)
    tmax_families  the per-ray limits the tests sweep, from each ray's own closest distance"""
import numpy as np

from tests import dimorder
from tests import prunedmodel as M

U32_MAX = 0xFFFFFFFF


def _walk(n_nodes, root_leaf, children, leaf):
    """The stackless walk's visiting order with an explicit stack: children(i) -> [(child, entered?)] near first, None
    at a leaf; leaf(i) -> the shape if it is accepted, else None."""
    if n_nodes == 0:
        return U32_MAX
    if root_leaf is not None:
        return root_leaf()
    stack = [0]
    while stack:
        i = stack.pop()
        cs = children(i)
        if cs is None:
            s = leaf(i)
            if s is not None:
                return s
            continue
        for c, ok in reversed(cs):                   # far pushed first: the near subtree is finished before the far one is opened
            if ok:
                stack.append(c)
    return U32_MAX


def aabb(tree, ray, tmax):
    """AABB mode, one ray: ray = (origin, inv_direction) as T sequences, tmax a T scalar.  Returns the witness shape or U32_MAX."""
    N = tree.nodes
    F = type(tmax)
    inf = F(np.inf)

    def own(s):
        sl = dimorder.slice(ray, *tree.shapes[s])
        return s if sl is not None and sl[0] < tmax else None

    def children(i):
        cl, cr, _, lmn, lmx, rmn, rmx = N[i]
        if cl == U32_MAX:
            return None
        sl, sr = dimorder.slice(ray, lmn, lmx), dimorder.slice(ray, rmn, rmx)
        el, er = (sl[0] if sl is not None else inf), (sr[0] if sr is not None else inf)
        left = (cl, sl is not None and el < tmax)
        right = (cr, sr is not None and er < tmax)
        return [left, right] if el <= er else [right, left]

    def root_leaf():
        s = N[0][2]
        r = own(s)
        return U32_MAX if r is None else r

    return _walk(len(N), root_leaf if N and N[0][0] == U32_MAX else None, children, lambda i: own(N[i][2]))


def aabb_batch(nodes, shapes, o, inv, tmax):
    """aabb over a batch: o, inv (m, D) arrays of T; tmax (m,) of T or None (+inf).  u32 array."""
    tree = dimorder.Tree(nodes, shapes)
    F = o.dtype.type
    tm = np.full(len(o), np.inf, dtype=F) if tmax is None else tmax
    return np.array([aabb(tree, (list(o[i]), list(inv[i])), tm[i]) for i in range(len(o))], dtype=np.uint32)


def triangles(nodes, shapes, tris, rays, tmax):
    """Triangle mode over a batch of 3-D C-ABI rays: nodes / shapes C-ABI arrays, tris (n, 9), tmax (m,) of T or None.  u32 array."""
    F = shapes["min"].dtype.type
    tr = np.ascontiguousarray(tris, dtype=F).reshape(-1, 3, 3)
    tm = np.full(len(rays), np.inf, dtype=F) if tmax is None else tmax
    margin = F(1) + F(1.0 / 65536.0)
    cl, cr, sh = nodes["child_l"], nodes["child_r"], nodes["shape"]
    lmn, lmx, rmn, rmx = (nodes[a][b] for a in ("l_aabb", "r_aabb") for b in ("min", "max"))
    out = np.full(len(rays), U32_MAX, dtype=np.uint32)
    for r in range(len(rays)):
        o, d, inv = list(rays["origin"][r]), list(rays["direction"][r]), list(rays["inv_direction"][r])
        t = tm[r]
        with np.errstate(all="ignore"):
            bound = t * margin

        def hit(s):
            return s if M.moeller_trumbore(o, d, *tr[s])[0] < t else None

        def children(i):
            if cl[i] == U32_MAX:
                return None
            hl, el = M.slice_entry(o, inv, lmn[i], lmx[i])
            hr, er = M.slice_entry(o, inv, rmn[i], rmx[i])
            el, er = (el if hl else F(np.inf)), (er if hr else F(np.inf))
            left, right = (int(cl[i]), hl and el <= bound), (int(cr[i]), hr and er <= bound)
            return [left, right] if el <= er else [right, left]

        def root_leaf():
            s = int(sh[0])
            w = hit(s) if M.slice_entry(o, inv, shapes["min"][s], shapes["max"][s])[0] else None
            return U32_MAX if w is None else w

        out[r] = _walk(len(nodes), root_leaf if len(nodes) == 1 else None, children, lambda i: hit(int(sh[i])))
    return out


def tmax_families(dstar, F, rng):
    """{name: per-ray limits (m,) of T, or None} from each ray's own closest distance d* (+inf without a hit): NULL and +inf; d*
    exactly (AABB mode: no hit); nextafter(d*, +inf) (a hit where d* is finite) and nextafter(d*, 0); 0, -0, negative and NaN (no hit);
    uniform in (0, 2 d*) (rays without a hit: (0, 2 * the largest finite d*))."""
    dstar = np.asarray(dstar, dtype=F)
    m = len(dstar)
    fin = np.isfinite(dstar)
    top = F(2) * (dstar[fin].max() if fin.any() else F(1))
    span = np.where(fin, F(2) * dstar, top).astype(F)
    rnd = (rng.uniform(0, 1, m) * span.astype(np.float64)).astype(F)
    rnd = np.where(rnd > 0, rnd, np.nextafter(F(0), F(1))).astype(F)
    return {
        "null": None,
        "inf": np.full(m, np.inf, dtype=F),
        "exact": dstar.copy(),
        "above": np.nextafter(dstar, F(np.inf)).astype(F),
        "below": np.nextafter(dstar, F(0)).astype(F),
        "zero": np.zeros(m, dtype=F),
        "negzero": np.full(m, -0.0, dtype=F),
        "negative": -(rng.uniform(0.5, 10, m)).astype(F),
        "nan": np.full(m, np.nan, dtype=F),
        "random": rnd,
    }
