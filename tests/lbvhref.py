"""tests/lbvhref.py -- restatement of the LBVH builders (BVHGPU_BUILD_LBVH, BVHGPU_BUILD_LBVH_TREELET; lbvh.cu, DESIGN §4.3b) in numpy,
on the C ABI's node arrays, for D = 3 and the D = 2 lift (z = [0, 0]).  TEST INFRASTRUCTURE: the device's LBVH trees must equal these
node arrays and node_index exactly (tests/test_gpu_lbvh_exact.py); tests/test_lbvh_cpu.py pins the restatement itself.

    centroids     center1 in T: min*0.5 + max*0.5, no FMA; their bounds in the order-preserving key order (-0 < +0), as prep_only
    Morton code   per axis in float64: u = (c - lo) / (hi - lo) if hi > lo else 0; where hi - lo overflows to +inf, both operands are
                  halved first: (c*0.5 - lo*0.5) / (hi*0.5 - lo*0.5); a NaN u becomes 0, then u is clamped to [0, 1];
                  q = min(trunc(u * 2097151), 2097151); code |= expand21(q) << (2 - k): x on bit 2, y on bit 1, z on bit 0 of a triple
    sort          stable by code (cub radix sort over bits [0, 63) with values 0..n-1): ties keep the lower shape index first
    Karras tree   the binary radix tree over the augmented key (code, sorted position): delta = clz64(a ^ b), or 64 + clz32(i ^ j) when
                  a == b.  Internal vertex 0 is the root; the children of the vertex with range [f, l] split after gamma are gamma
                  (leaf f + ... if f == gamma) and gamma + 1.  Restated twice: karras() follows karras_kernel, karras_recursive() splits
                  at the highest differing bit of the augmented keys
    emit          vertex v lands at index(v) = 2*first(v) + L(v) (L = left edges on its root path); child boxes are joins in the
                  min_t / max_t order (-0 below +0)
    treelets      (mode 2) every inner vertex with <= TILE shapes whose parent has > TILE shapes, or that is the root, is replaced by
                  Bvh::build of its shapes taken in Morton order (the oracle for D = 3, tests/pyref.py for D = 2), relocated: links +
                  the vertex's index, the local root's parent = the LBVH parent, shapes through the Morton order; leaves directly
                  below a vertex with > TILE shapes stay LBVH leaves
"""
import numpy as np

from tests import rebuildref as RR

U32_MAX = 0xFFFFFFFF
TILE = 512
QMAX = 2097151


# ---- bit helpers -----------------------------------------------------------------------------------------------------------------
def expand21(q):
    v = np.asarray(q, dtype=np.uint64) & np.uint64(0x1FFFFF)
    for s, m in ((32, 0x1F00000000FFFF), (16, 0x1F0000FF0000FF), (8, 0x100F00F00F00F00F), (4, 0x10C30C30C30C30C3), (2, 0x1249249249249249)):
        v = (v | (v << np.uint64(s))) & np.uint64(m)
    return v


def clz64(x):
    """__clzll of the unsigned 64-bit integers x (64 for x == 0)."""
    x = np.array(x, dtype=np.uint64)
    n = np.zeros(x.shape, dtype=np.int64)
    zero = x == 0
    for s in (32, 16, 8, 4, 2, 1):
        top = (x >> np.uint64(64 - s)) == 0
        n[top] += s
        x[top] <<= np.uint64(s)
    n[zero] = 64
    return n


def clz32(x):
    """__clz of unsigned 32-bit integers."""
    return clz64(np.asarray(x, dtype=np.uint64) & np.uint64(0xFFFFFFFF)) - 32


def _keys(x):
    """Order-preserving unsigned keys of floats (min / max of keys == min / max of the floats with -0 < +0)."""
    x = np.ascontiguousarray(x)
    U, top = (np.uint32, np.uint32(0x80000000)) if x.dtype == np.float32 else (np.uint64, np.uint64(0x8000000000000000))
    u = x.view(U)
    return np.where(u & top, ~u, u | top)


def min_t(a, b):
    """min with -0 below +0 (fminf / fmin on the device, min_t)."""
    return np.where(_keys(a) <= _keys(b), a, b)


def max_t(a, b):
    return np.where(_keys(a) >= _keys(b), a, b)


def key_bounds(c):
    """(lo, hi) per column of c in the key order: -0 < +0."""
    k = _keys(c)
    lo = c[np.argmin(k, axis=0), np.arange(c.shape[1])]
    hi = c[np.argmax(k, axis=0), np.arange(c.shape[1])]
    return lo, hi


# ---- stages ------------------------------------------------------------------------------------------------------------------------
def lift(mn, mx):
    """(n, D) boxes of D = 2 or 3 as 3-D boxes (z = [0, 0] for D = 2)."""
    if mn.shape[1] == 3:
        return mn, mx
    z = np.zeros((len(mn), 1), dtype=mn.dtype)
    return np.concatenate([mn, z], axis=1), np.concatenate([mx, z], axis=1)


def centroids(mn, mx):
    F = mn.dtype.type
    return mn * F(0.5) + mx * F(0.5)


def quantise(c, lo, hi):
    """q in [0, 2097151] of one axis: c float64 array, lo / hi float64 scalars.  Returns (q, facts)."""
    c, lo, hi = np.asarray(c, dtype=np.float64), np.float64(lo), np.float64(hi)
    facts = {"overflow": False, "nan_u_unhalved": 0}
    if not hi > lo:
        return np.zeros(len(c), dtype=np.uint64), facts
    with np.errstate(all="ignore"):
        num, den = c - lo, hi - lo
        if np.isinf(den):
            facts["overflow"] = True
            facts["nan_u_unhalved"] = int(np.sum(np.isnan(num / den)))
            num, den = c * 0.5 - lo * 0.5, hi * 0.5 - lo * 0.5
        u = num / den
        u = np.where(u >= 0.0, np.minimum(u, 1.0), 0.0)         # NaN -> 0
        q = np.trunc(u * float(QMAX)).astype(np.uint64)
    return np.minimum(q, np.uint64(QMAX)), facts


def morton(mn, mx):
    """63-bit codes of the (n, 3) boxes in T, and per-axis facts."""
    c = centroids(mn, mx)
    lo, hi = key_bounds(c)
    code = np.zeros(len(c), dtype=np.uint64)
    facts = []
    for k in range(3):
        q, f = quantise(c[:, k], lo[k], hi[k])
        code |= expand21(q) << np.uint64(2 - k)
        facts.append(f)
    return code, facts


def _delta(code, i, j):
    """Common prefix length of sorted positions i and j (arrays), -1 where j is out of range."""
    n = len(code)
    ok = (j >= 0) & (j < n)
    jj = np.where(ok, j, 0)
    a, b = code[i], code[jj]
    same = a == b
    d = np.where(same, 64 + clz32(i ^ jj), clz64(a ^ b))
    return np.where(ok, d, -1)


def karras(code):
    """karras_kernel over sorted codes, vectorised: (left, right, first, count) of the internal vertices 0..n-2; children >= n-1 are
    leaves (leaf n-1+p holds sorted position p)."""
    n = len(code)
    i = np.arange(n - 1, dtype=np.int64)
    d = np.where(_delta(code, i, i + 1) - _delta(code, i, i - 1) >= 0, 1, -1)
    dmin = _delta(code, i, i - d)
    lmax = np.full(n - 1, 2, dtype=np.int64)
    grow = _delta(code, i, i + lmax * d) > dmin
    while grow.any():
        lmax[grow] <<= 1
        grow = grow & (_delta(code, i, i + lmax * d) > dmin)
    l = np.zeros(n - 1, dtype=np.int64)
    t = int(lmax.max()) >> 1
    while t >= 1:
        act = t <= (lmax >> 1)
        hit = act & (_delta(code, i, i + (l + t) * d) > dmin)
        l[hit] += t
        t >>= 1
    j = i + l * d
    dnode = _delta(code, i, j)
    s = np.zeros(n - 1, dtype=np.int64)
    t = (l + 1) >> 1
    act = np.ones(n - 1, dtype=bool)
    while act.any():
        hit = act & (_delta(code, i, i + (s + t) * d) > dnode)
        s[hit] += t[hit]
        act = act & (t != 1)
        t = np.where(act, (t + 1) >> 1, t)
    gamma = i + s * d + np.where(d < 0, -1, 0)
    lo, hi = np.minimum(i, j), np.maximum(i, j)
    left = np.where(lo == gamma, n - 1 + gamma, gamma)
    right = np.where(hi == gamma + 1, n - 1 + gamma + 1, gamma + 1)
    return left, right, lo, hi - lo + 1


def karras_recursive(code):
    """The same tree from its definition: a vertex over sorted positions [f, l] splits at the highest bit in which the augmented keys
    (code, position) of f and l differ; its left child is vertex gamma (a leaf if f == gamma), its right child gamma + 1."""
    n = len(code)
    code = np.asarray(code, dtype=np.uint64)
    left = np.zeros(n - 1, dtype=np.int64)
    right = np.zeros(n - 1, dtype=np.int64)
    first = np.zeros(n - 1, dtype=np.int64)
    count = np.zeros(n - 1, dtype=np.int64)
    stack = [(0, 0, n - 1)]
    while stack:
        v, f, l = stack.pop()
        a, b = int(code[f]), int(code[l])
        if a != b:
            bit = (a ^ b).bit_length() - 1
            hi_half = np.searchsorted(code[f:l + 1] >> np.uint64(bit), np.uint64(b >> bit))   # first position with the bit set
            gamma = f + int(hi_half) - 1
        else:
            bit = (f ^ l).bit_length() - 1
            gamma = ((l >> bit) << bit) - 1
        first[v], count[v] = f, l - f + 1
        for side, (cf, cl, cv) in ((left, (f, gamma, gamma)), (right, (gamma + 1, l, gamma + 1))):
            if cf == cl:
                side[v] = n - 1 + cf
            else:
                side[v] = cv
                stack.append((cv, cf, cl))
    return left, right, first, count


class Karras:
    """The radix tree of sorted codes as vertex arrays: vertices 0..n-2 internal, n-1+p the leaf of sorted position p."""

    def __init__(self, left, right, first, count, n):
        self.n = n
        tot = 2 * n - 1
        self.left, self.right = left, right
        self.first = np.concatenate([first, np.arange(n)])
        self.count = np.concatenate([count, np.ones(n, dtype=np.int64)])
        self.parent = np.zeros(tot, dtype=np.int64)
        self.isleft = np.zeros(tot, dtype=bool)
        self.parent[left] = np.arange(n - 1)
        self.parent[right] = np.arange(n - 1)
        self.isleft[left] = True
        self.levels = []                                          # vertices by depth
        self.L = np.zeros(tot, dtype=np.int64)                    # left edges on the root path
        self.depth = np.zeros(tot, dtype=np.int64)
        front = np.zeros(1, dtype=np.int64)
        while len(front):
            self.levels.append(front)
            inner = front[front < n - 1]
            cl, cr = left[inner], right[inner]
            self.L[cl], self.L[cr] = self.L[inner] + 1, self.L[inner]
            self.depth[cl] = self.depth[cr] = self.depth[inner] + 1
            front = np.concatenate([cl, cr])
        self.index = 2 * self.first + self.L


def restate(a, prec, mode):
    """(nodes, node_index, info) of bvhgpu_build_* with BVHGPU_BUILD_LBVH (mode 1) or BVHGPU_BUILD_LBVH_TREELET (mode 2) on the AABB
    array `a` of dimension D = 2 or 3.  info: codes, sorted order, the Karras vertices, treelet roots (node indices) and Morton facts."""
    F = RR._F(prec)
    D = a["min"].shape[1]
    n = len(a)
    nodes = np.zeros(max(2 * n - 1, 0), dtype=RR.node_dtype(D, prec))
    node_index = np.zeros(n, dtype=np.uint32)
    info = {"treelets": [], "order": np.arange(n), "code": np.zeros(n, dtype=np.uint64), "morton": None, "tree": None}
    if n == 0:
        return nodes, node_index, info
    mn, mx = lift(np.asarray(a["min"], dtype=F), np.asarray(a["max"], dtype=F))
    for side in ("l_aabb", "r_aabb"):
        nodes[side]["min"], nodes[side]["max"] = F(np.inf), F(-np.inf)
    if n == 1:
        nodes["child_l"] = nodes["child_r"] = U32_MAX
        return nodes, node_index, info
    code, mf = morton(mn, mx)
    order = np.argsort(code, kind="stable")
    sc = code[order]
    info.update(code=code, order=order, morton=mf)
    K = Karras(*karras(sc), n)
    info["tree"] = K
    # bottom-up boxes of every vertex, joined with min_t / max_t
    tot = 2 * n - 1
    bmn = np.empty((tot, 3), dtype=F)
    bmx = np.empty((tot, 3), dtype=F)
    bmn[n - 1:], bmx[n - 1:] = mn[order], mx[order]
    for lvl in reversed(K.levels):
        v = lvl[lvl < n - 1]
        bmn[v] = min_t(bmn[K.left[v]], bmn[K.right[v]])
        bmx[v] = max_t(bmx[K.left[v]], bmx[K.right[v]])
    # emit every vertex at its preorder index
    v = np.arange(tot)
    idx = K.index
    inner = v < n - 1
    nodes["parent"][idx] = np.where(v == 0, 0, idx[K.parent])
    iv, ii = v[inner], idx[inner]
    nodes["child_l"][ii] = ii + 1
    nodes["child_r"][ii] = ii + 2 * K.count[K.left[iv]]
    nodes["shape"][ii] = K.count[iv]
    for side, ch in (("l_aabb", K.left), ("r_aabb", K.right)):
        nodes[side]["min"][ii] = bmn[ch[iv]][:, :D]
        nodes[side]["max"][ii] = bmx[ch[iv]][:, :D]
    lv, li = v[~inner], idx[~inner]
    nodes["child_l"][li] = nodes["child_r"][li] = U32_MAX
    nodes["shape"][li] = order[lv - (n - 1)]
    node_index[order[lv - (n - 1)]] = li
    if mode == 2:
        roots = treelet_roots(K)
        info["treelets"] = [int(idx[r]) for r in roots]
        for r in roots:
            _treelet(nodes, node_index, a, prec, order[K.first[r]:K.first[r] + K.count[r]], int(idx[r]),
                     0 if r == 0 else int(idx[K.parent[r]]))
    return nodes, node_index, info


def treelet_roots(K):
    """Inner vertices with <= TILE shapes whose parent has > TILE shapes, or that are the root."""
    v = np.arange(K.n - 1)
    small = K.count[v] <= TILE
    return v[small & ((v == 0) | (K.count[K.parent[v]] > TILE))]


def _treelet(nodes, node_index, a, prec, shapes, at, parent):
    loc, lidx = RR.build(np.ascontiguousarray(a[shapes]), prec)
    k = len(shapes)
    out = np.array(loc, dtype=nodes.dtype)
    leaf = out["child_l"] == U32_MAX
    out["child_l"][~leaf] += at
    out["child_r"][~leaf] += at
    out["parent"] += at
    out["parent"][0] = parent
    out["shape"][leaf] = shapes[out["shape"][leaf]]
    nodes[at:at + 2 * k - 1] = out
    node_index[shapes] = np.asarray(lidx, dtype=np.int64) + at


# ---- facts about restated trees ---------------------------------------------------------------------------------------------------
def depth(nodes):
    """The longest root path in edges."""
    return len(RR.levels(nodes)) - 1


def preorder_ok(nodes):
    """child_l = i + 1, child_r = i + 2 * n_l, parents point back, inner `shape` = number of shapes below."""
    n = (len(nodes) + 1) // 2
    if len(nodes) == 1:
        return nodes["child_l"][0] == U32_MAX
    cl, cr = nodes["child_l"].astype(np.int64), nodes["child_r"].astype(np.int64)
    inner = np.flatnonzero(cl != U32_MAX)
    cnt = np.where(cl == U32_MAX, 1, nodes["shape"].astype(np.int64))
    ok = np.array_equal(cl[inner], inner + 1) and np.array_equal(cr[inner], inner + 2 * cnt[inner + 1])
    ok = ok and np.array_equal(cnt[inner], cnt[cl[inner]] + cnt[cr[inner]]) and cnt[0] == n
    par = nodes["parent"].astype(np.int64)
    return bool(ok and np.all(par[cl[inner]] == inner) and np.all(par[cr[inner]] == inner) and par[0] == 0)


def subtree_shapes(nodes, i):
    """Shapes of the leaves in the node range of node i."""
    k = 1 if nodes["child_l"][i] == U32_MAX else int(nodes["shape"][i])
    rng = np.arange(i, i + 2 * k - 1)
    return nodes["shape"][rng[nodes["child_l"][rng] == U32_MAX]].astype(np.int64)


def mixed_zero_signs(nodes):
    """Inner nodes whose two child boxes hold -0.0 and +0.0 in the same coordinate."""
    inner = nodes["child_l"] != U32_MAX
    hits = 0
    for mm in ("min", "max"):
        a, b = nodes["l_aabb"][mm][inner], nodes["r_aabb"][mm][inner]
        hits += int(np.sum(np.any((a == 0) & (b == 0) & (np.signbit(a) != np.signbit(b)), axis=1)))
    return hits


# ---- scenes shared by tests/test_lbvh_cpu.py and tests/test_gpu_lbvh_exact.py ----------------------------------------------------
def identical_scene(n, D, prec, rng):
    """Boxes of different sizes around one common centre: every code is 0 and only the position orders the shapes."""
    h = rng.choice([0.5, 1.0, 2.0, 4.0], (n, 1)) * np.ones((1, D))
    return RR.make_boxes(3.0 - h, 3.0 + h, D, prec)


def comb_scene(D, prec, low_bits=17):
    """Centroids whose codes are 0, every single-bit code and 2^63 - 1, with 2^low_bits shapes on code 0 and 8 on a few single-bit
    codes: a chain of single-bit splits above a balanced position subtree, root paths of at least 63 + low_bits edges.  Centroids sit
    at q + 0.5 in bounds [0, 2097151] per axis (so trunc(u * 2097151) is q for certain); boxes are q + 0.5 -+ 0.5."""
    bits = range(63) if D == 3 else [b for b in range(63) if b % 3 != 0]      # D = 2: z (bit 0 of each triple) is always 0
    q = [np.zeros(3)]
    for b in bits:
        v = np.zeros(3)
        v[2 - b % 3] = 1 << (b // 3)
        q += [v] * (8 if b % 7 == 3 else 1)
    q += [np.zeros(3)] * ((1 << low_bits) - 1)
    q = np.array(q)
    c = q + 0.5
    c = np.concatenate([c, np.zeros((1, 3)), np.full((1, 3), float(QMAX))])   # the bounds: one centroid at 0, one at 2097151
    if D == 2:
        c = c[:, :2]
    return RR.make_boxes(c - 0.5, c + 0.5, D, prec)


def signed_zero_scene(n, D, prec, rng):
    """Every box's min.x is -0.0 or +0.0 and half of the boxes are flat at y = -0.0 or +0.0: both signs of zero meet in one
    coordinate at almost every join."""
    mn = rng.uniform(-100, 100, (n, D))
    mx = mn + rng.uniform(0.5, 8, (n, D))
    mn[:, 0] = np.where(rng.random(n) < 0.5, -0.0, 0.0)
    mx[:, 0] = rng.uniform(0.5, 8, n)
    flat = rng.random(n) < 0.5
    z = np.where(rng.random(n) < 0.5, -0.0, 0.0)
    mn[flat, 1] = z[flat]
    mx[flat, 1] = z[flat]
    return RR.make_boxes(mn, mx, D, prec)


def overflow_centroid_scene(n, D, rng):
    """f64 boxes whose x centroids span (-1.5e308, 1.5e308): hi - lo overflows, and (c - lo) / (hi - lo) is inf / inf = NaN for
    centroids near hi.  Both ends are present."""
    mn = rng.uniform(-100, 100, (n, D))
    mn[:, 0] = rng.uniform(-1.5, 1.5, n) * 1e308
    mn[:2, 0] = (-1.5e308, 1.5e308)
    return RR.make_boxes(mn, mn + rng.uniform(0.5, 8, (n, D)), D, "f64")
