"""tests/dimcheck.py -- the reference's tree invariants, generic in the dimension D and vectorised with numpy, for node arrays of the
C ABI (any D) and shape AABB arrays with "min" / "max" fields.  TEST INFRASTRUCTURE: checked against the C++ oracle at D = 3
(tests/test_dim_update_cpu.py) and then used for D = 2 and D = 4 (tests/test_gpu_dim_update.py).

    is_consistent   Bvh::is_consistent (src/bvh/bvh_impl.rs:280-485): every node is reached once from the root, every parent field
                    names the node it was reached from, and every child box (a leaf: its shape's box) lies in the box its parent stores
                    for it, up to T::EPSILON (Aabb::approx_contains_aabb_eps, src/aabb/aabb_impl.rs:198-224), arithmetic in T
    is_tight        Bvh::assert_tight: the join of every inner node's two child boxes equals the box its parent stores for it
    layout_ok       Bvh::build's preorder layout: child_l = i + 1, child_r = i + 2 n_l, `shape` of an inner node = shapes below it,
                    and node_index names leaves that hold their own shape
    sah_cost        the whole-tree SAH cost (DESIGN.md): sum over non-root nodes of SA(box in the parent) / SA(root box), in double,
                    with the reference's surface area 2 * |size|^2
"""
import numpy as np

U32_MAX = 0xFFFFFFFF


def _reach(nodes):
    """Nodes reached from the root breadth first, with the node each was reached from; None when a node is reached twice or a link
    leaves the array."""
    nn = len(nodes)
    cl, cr = nodes["child_l"].astype(np.int64), nodes["child_r"].astype(np.int64)
    seen = np.zeros(nn, dtype=np.int64)
    frm = np.zeros(nn, dtype=np.int64)
    front = np.array([0], dtype=np.int64)
    seen[0] = 1
    while len(front):
        inner = front[cl[front] != U32_MAX]
        kids = np.concatenate([cl[inner], cr[inner]])
        par = np.concatenate([inner, inner])
        if len(kids) and (kids.max() >= nn or kids.min() < 0):
            return None
        np.add.at(seen, kids, 1)
        if len(kids) and seen[kids].max() > 1:
            return None
        frm[kids] = par
        front = kids
    return seen.astype(bool), frm


def _slot(nodes, i, frm):
    """The box node i's parent stores for it: (min, max) arrays of shape (len(i), D)."""
    p = frm[i]
    left = nodes["child_l"][p] == i
    mn = np.where(left[:, None], nodes["l_aabb"]["min"][p], nodes["r_aabb"]["min"][p])
    mx = np.where(left[:, None], nodes["l_aabb"]["max"][p], nodes["r_aabb"]["max"][p])
    return mn, mx


def _contains(omn, omx, mn, mx, eps):
    with np.errstate(all="ignore"):
        ok = ((mn - omn) > -eps) & ((mn - omx) < eps) & ((mx - omn) > -eps) & ((mx - omx) < eps)
    return ok.all(axis=1)


def is_consistent(nodes, shapes) -> bool:
    nn = len(nodes)
    if nn == 0:
        return True
    F = nodes["l_aabb"]["min"].dtype.type
    eps = F(np.finfo(F).eps)
    r = _reach(nodes)
    if r is None:
        return False
    seen, frm = r
    if not seen.all() or nodes["parent"][0] != 0:
        return False
    i = np.arange(1, nn)
    if not np.array_equal(nodes["parent"][i].astype(np.int64), frm[i]):
        return False
    omn, omx = _slot(nodes, i, frm)
    leaf = nodes["child_l"][i] == U32_MAX
    ok = np.ones(len(i), dtype=bool)
    s = nodes["shape"][i[leaf]]
    ok[leaf] = _contains(omn[leaf], omx[leaf], shapes["min"][s], shapes["max"][s], eps)
    inn = ~leaf
    for side in ("l_aabb", "r_aabb"):
        ok[inn] &= _contains(omn[inn], omx[inn], nodes[side]["min"][i[inn]], nodes[side]["max"][i[inn]], eps)
    if nodes["child_l"][0] != U32_MAX:                     # the root's outer box is [-inf, inf]: only NaN can fail it
        inf = np.full((1, nodes["l_aabb"]["min"].shape[1]), np.inf, dtype=F)
        for side in ("l_aabb", "r_aabb"):
            ok = ok.all() & _contains(-inf, inf, nodes[side]["min"][:1], nodes[side]["max"][:1], eps).all()
    else:
        s0 = nodes["shape"][0]
        inf = np.full((1, shapes["min"].shape[1]), np.inf, dtype=F)
        ok = ok.all() & _contains(-inf, inf, shapes["min"][s0:s0 + 1], shapes["max"][s0:s0 + 1], eps).all()
    return bool(np.all(ok))


def is_tight(nodes) -> bool:
    nn = len(nodes)
    if nn == 0 or nodes["child_l"][0] == U32_MAX:
        return True
    r = _reach(nodes)
    if r is None:
        return False
    seen, frm = r
    i = np.flatnonzero(seen)
    i = i[(i != 0) & (nodes["child_l"][i] != U32_MAX)]
    jmn = np.minimum(nodes["l_aabb"]["min"][i], nodes["r_aabb"]["min"][i])
    jmx = np.maximum(nodes["l_aabb"]["max"][i], nodes["r_aabb"]["max"][i])
    omn, omx = _slot(nodes, i, frm)
    return bool(np.array_equal(jmn, omn) and np.array_equal(jmx, omx))


def counts(nodes):
    leaf = nodes["child_l"] == U32_MAX
    return np.where(leaf, 1, nodes["shape"]).astype(np.int64)


def layout_ok(nodes, node_index) -> bool:
    """Bvh::build's preorder layout, and node_index[s] is a leaf holding shape s."""
    nn = len(nodes)
    n = len(node_index)
    if nn != max(2 * n - 1, 0):
        return False
    if n == 0:
        return True
    ni = node_index.astype(np.int64)
    if ni.max() >= nn or not np.all(nodes["child_l"][ni] == U32_MAX) or not np.array_equal(nodes["shape"][ni], np.arange(n)):
        return False
    c = counts(nodes)
    i = np.flatnonzero(nodes["child_l"] != U32_MAX)
    if c[0] != n or not np.all(nodes["child_l"][i] == i + 1):
        return False
    nl = c[i + 1]
    return bool(np.all(nodes["child_r"][i] == i + 2 * nl) and np.all(c[i] == nl + c[nodes["child_r"][i].astype(np.int64)]))


def sah_cost(nodes) -> float:
    nn = len(nodes)
    if nn < 3:
        return 0.0
    i = np.flatnonzero(nodes["child_l"] != U32_MAX)
    with np.errstate(all="ignore"):
        tot = 0.0
        for side in ("l_aabb", "r_aabb"):
            s = nodes[side]["max"][i].astype(np.float64) - nodes[side]["min"][i].astype(np.float64)
            tot += float((2.0 * (s * s).sum(axis=1)).sum())
        rs = np.maximum(nodes["l_aabb"]["max"][0], nodes["r_aabb"]["max"][0]).astype(np.float64) - \
            np.minimum(nodes["l_aabb"]["min"][0], nodes["r_aabb"]["min"][0]).astype(np.float64)
        return float(np.float64(tot) / (2.0 * (rs * rs).sum()))      # a zero-size root: nan or inf, as in the oracle
