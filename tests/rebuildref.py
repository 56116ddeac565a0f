"""tests/rebuildref.py -- restatement of the update step every dynamic entry point rests on (DESIGN §4.5 / §4.12; flatten.cu: optimize,
update_incremental, rebuild_degraded; update.cuh; dim4.cu: rebuild_degraded4), generic in the dimension D, on the C ABI's node arrays
with numpy scalars of type T.  TEST INFRASTRUCTURE: the device's optimize / update_shapes must produce these node arrays, node_index
and `rebuilt` counts exactly (tests/test_gpu_rebuild_exact.py); tests/test_rebuild_cpu.py pins the restatement itself.

    refit and climb   every parent slot becomes the join of its child's two stored slots (a leaf: its shape's box).  The full form
                      (optimize) refits every node; the incremental form (update_shapes) only the root paths of the changed leaves,
                      and the off-path slots keep what they stored
    surface area      2 * (sum of the squared extents, left to right) in T, no FMA (surface_area / surface_area4)
    baseline          taken at the first rebuilding call from the tree as it stands then (ensure_sa_base, node_sa_kernel), refreshed
                      only over the node ranges of rebuilt subtrees (rebase_kernel / rebase4_kernel)
    growth test       SA(new join) > fl_T(max_growth * base), on the refitted nodes; max_growth <= 0: boxes only
    roots             rebuild_candidate (not degraded but a child is, or the degraded tree root), outermost candidates only
    rebuild           the node range [r, r + 2k - 1) of a root with k shapes becomes Bvh::build of its shapes in leaf order, seeded
                      with the join of the root's two stored child slots after the refit (tests/pyref.py build(root_aabb=...); for D = 3
                      the oracle's build wherever that seed is the joint box of the shapes), relocated: links + r, the local root's
                      parent = r's old parent, leaves through the leaf-order list; node_index follows
"""
import numpy as np

from tests import pyref

U32_MAX = 0xFFFFFFFF


def surface_area(mn, mx):
    """Aabb::surface_area of the rows of (m, D) arrays in their own type: 2 * (((sx*sx + sy*sy) + sz*sz) + ...), no FMA."""
    F = mn.dtype.type
    with np.errstate(all="ignore"):
        s = mx - mn
        acc = s[:, 0] * s[:, 0] + s[:, 1] * s[:, 1]
        for k in range(2, s.shape[1]):
            acc = acc + s[:, k] * s[:, k]
        return F(2) * acc


def levels(nodes):
    """Node indices by depth, root first."""
    cl, cr = nodes["child_l"].astype(np.int64), nodes["child_r"].astype(np.int64)
    out, front = [], np.zeros(1, dtype=np.int64)
    while len(front):
        out.append(front)
        inner = front[cl[front] != U32_MAX]
        front = np.concatenate([cl[inner], cr[inner]])
    return out


class Tree:
    """A tree as the device holds it (nodes, node_index, the growth baseline), stepped by optimize() / update()."""

    def __init__(self, nodes, node_index):
        self.nodes = np.array(nodes, copy=True)
        self.node_index = np.array(node_index, dtype=np.uint32, copy=True)
        self.base = None
        self.D = self.nodes["l_aabb"]["min"].shape[1]
        self.F = self.nodes["l_aabb"]["min"].dtype.type
        self.facts = {}

    # ---- helpers over the node array ----
    def _join(self, i):
        nd = self.nodes
        return (np.minimum(nd["l_aabb"]["min"][i], nd["r_aabb"]["min"][i]), np.maximum(nd["l_aabb"]["max"][i], nd["r_aabb"]["max"][i]))

    def _node_sa(self, i):
        """SA of the join of an inner node's two slots, 0 for leaves (node_sa_kernel / rebase_kernel)."""
        out = np.zeros(len(i), dtype=self.F)
        inner = self.nodes["child_l"][i] != U32_MAX
        out[inner] = surface_area(*self._join(i[inner]))
        return out

    def _child_box(self, c, bmn, bmx):
        """The box a child's slot gets in the climb: its shape's box for a leaf, the join of its two slots otherwise."""
        leaf = self.nodes["child_l"][c] == U32_MAX
        mn = np.empty((len(c), self.D), dtype=self.F)
        mx = np.empty_like(mn)
        s = self.nodes["shape"][c[leaf]].astype(np.int64)
        mn[leaf], mx[leaf] = bmn[s], bmx[s]
        mn[~leaf], mx[~leaf] = self._join(c[~leaf])
        return mn, mx

    # ---- the step ----
    def optimize(self, boxes, max_growth):
        """bvhgpu_optimize (3-D only): full refit, growth test on every inner node.  Returns `rebuilt`."""
        assert max_growth >= 1.0
        return self._step(boxes, None, max_growth)

    def update(self, changed, boxes, max_growth):
        """bvhgpu_update (any D): `boxes` are all shapes' boxes after the motion, `changed` the indices sent.  Returns `rebuilt`."""
        return self._step(boxes, np.asarray(changed, dtype=np.int64).reshape(-1), max_growth)

    def _step(self, boxes, changed, max_growth):
        nd, F = self.nodes, self.F
        n, nn = len(self.node_index), len(nd)
        bmn, bmx = np.asarray(boxes["min"], dtype=F), np.asarray(boxes["max"], dtype=F)
        self.facts = {"roots": [], "seed_differs": 0}
        if n == 0 or (changed is not None and len(changed) == 0):
            return 0
        if n < 3:                                                      # one or two shapes: a full refit, nothing a rebuild could change
            changed, max_growth = None, 0.0
        rebuild = max_growth > 0
        if rebuild and self.base is None:                              # the baseline is the tree before this call's motion
            self.base = self._node_sa(np.arange(nn))
        cl, cr, par = (nd[f].astype(np.int64) for f in ("child_l", "child_r", "parent"))
        inner_all = cl != U32_MAX
        if changed is None:
            touched = inner_all.copy()                                 # every inner node is refit
            onpath = np.ones(nn, dtype=bool)
        else:
            touched = np.zeros(nn, dtype=bool)
            leaves = self.node_index[changed].astype(np.int64)
            onpath = np.zeros(nn, dtype=bool)
            onpath[leaves] = True
            cur = np.unique(par[leaves[leaves != 0]])
            while len(cur):
                cur = cur[~touched[cur]]
                touched[cur] = True
                cur = np.unique(par[cur[cur != 0]])
            onpath |= touched
        for lvl in reversed(levels(nd)):                               # bottom up: a child's slots are final before its parent's
            i = lvl[touched[lvl]]
            for side, ch in (("l_aabb", cl), ("r_aabb", cr)):
                c = ch[i]
                sel = onpath[c]
                mn, mx = self._child_box(c[sel], bmn, bmx)
                nd[side]["min"][i[sel]] = mn
                nd[side]["max"][i[sel]] = mx
        if not rebuild:
            return 0
        bad = np.zeros(nn, dtype=bool)
        t = np.flatnonzero(touched)
        with np.errstate(all="ignore"):
            bad[t] = surface_area(*self._join(t)) > F(max_growth) * self.base[t]
        cand = np.zeros(nn, dtype=bool)
        ii = np.flatnonzero(inner_all)
        cand[ii] = np.where(bad[ii], ii == 0, bad[cl[ii]] | bad[cr[ii]])
        outer = np.zeros(nn, dtype=bool)                               # some proper ancestor is a candidate
        for lvl in levels(nd):
            i = lvl[inner_all[lvl]]
            flag = outer[i] | cand[i]
            outer[cl[i]] = flag
            outer[cr[i]] = flag
        roots = np.flatnonzero(cand & ~outer)
        rebuilt = 0
        for r in roots:
            k = int(nd["shape"][r])
            self._rebuild(int(r), k, bmn, bmx, boxes)
            rng = np.arange(r, r + 2 * k - 1)
            self.base[rng] = self._node_sa(rng)
            rebuilt += k
        return rebuilt

    def _rebuild(self, r, k, bmn, bmx, boxes):
        from oracle import oracle as O

        nd, F, D = self.nodes, self.F, self.D
        rng = np.arange(r, r + 2 * k - 1)
        order = nd["shape"][rng[nd["child_l"][rng] == U32_MAX]].astype(np.int64)     # preorder = leaf order
        seed = self._join(np.array([r]))
        seed = (seed[0][0], seed[1][0])
        jmn, jmx = bmn[order].min(axis=0), bmx[order].max(axis=0)
        same = bool(np.array_equal(seed[0], jmn) and np.array_equal(seed[1], jmx))
        ctr = bmn[order] * F(0.5) + bmx[order] * F(0.5)
        ext = ctr.max(axis=0) - ctr.min(axis=0)                        # largest_axis of the root's centre bounds: the first maximum
        self.facts["roots"].append({"root": r, "count": k, "axis": int(np.argmax(ext)) if np.all(np.isfinite(ext)) else -1})
        self.facts["seed_differs"] += 0 if same else 1
        parent = int(nd["parent"][r])
        if D == 3 and same:
            prec = "f32" if F is np.float32 else "f64"
            sub = np.ascontiguousarray(boxes[order], dtype=O._DT[prec]["aabb"])
            b = O.build(sub, prec)
            loc, lidx = b.nodes, b.node_index.astype(np.int64)
            leaf = loc["child_l"] == U32_MAX
            out = np.array(loc, dtype=nd.dtype)
            out["child_l"][~leaf] += r
            out["child_r"][~leaf] += r
            out["parent"] += r
            out["parent"][0] = parent
            out["shape"][leaf] = order[loc["shape"][leaf]]
            nd[r:r + 2 * k - 1] = out
            self.node_index[order] = lidx + r
            return
        pa = [{"min": bmn[s], "max": bmx[s]} for s in order]
        pn, pidx = pyref.build(pa, F, root_aabb=seed)
        self._place(r, pn, pidx, order, parent)

    def _place(self, r, pn, pidx, order, parent):
        """Writes tests/pyref.py's tree over local shapes 0..k-1 into the node range from r: links + r, the local root's parent =
        `parent`, shapes through `order`; leaves store Aabb::empty() child boxes, inner nodes the number of shapes below them."""
        nd, F, D = self.nodes, self.F, self.D
        empty_mn, empty_mx = np.full(D, np.inf, dtype=F), np.full(D, -np.inf, dtype=F)
        cnt = np.zeros(len(pn), dtype=np.int64)
        for j in range(len(pn) - 1, -1, -1):                             # children follow their parent in preorder
            w, g = pn[j], r + j
            nd["parent"][g] = parent if j == 0 else r + w[1]
            if w[0] == "leaf":
                cnt[j] = 1
                nd["child_l"][g] = nd["child_r"][g] = U32_MAX
                nd["shape"][g] = order[w[2]]
                for side in ("l_aabb", "r_aabb"):
                    nd[side]["min"][g], nd[side]["max"][g] = empty_mn, empty_mx
            else:
                cnt[j] = cnt[w[2]] + cnt[w[3]]
                nd["child_l"][g], nd["child_r"][g], nd["shape"][g] = r + w[2], r + w[3], cnt[j]
                for side, box in (("l_aabb", w[4]), ("r_aabb", w[5])):
                    nd[side]["min"][g] = np.array(box[0], dtype=F)
                    nd[side]["max"][g] = np.array(box[1], dtype=F)
        self.node_index[order] = np.asarray(pidx, dtype=np.int64) + r


def halving_pairs(nodes, boxes, roots):
    """Inner nodes with two leaf children of identical centres inside the given rebuilt subtrees: each was split by the halving branch,
    and which leaf holds which shape follows the order the builder was given."""
    F = nodes["l_aabb"]["min"].dtype.type
    bmn, bmx = np.asarray(boxes["min"], dtype=F), np.asarray(boxes["max"], dtype=F)
    c = bmn * F(0.5) + bmx * F(0.5)
    total = 0
    for ro in roots:
        r, k = ro["root"], ro["count"]
        i = np.arange(r, r + 2 * k - 1)
        i = i[(nodes["child_l"][i] != U32_MAX) & (nodes["shape"][i] == 2)]
        a, b = nodes["shape"][i + 1].astype(np.int64), nodes["shape"][i + 2].astype(np.int64)
        total += int(np.sum(np.all(c[a] == c[b], axis=1)))
    return total


# ---- scenes and motions shared by tests/test_rebuild_cpu.py and tests/test_gpu_rebuild_exact.py ----------------------------------
def aabb_dtype(D, prec):
    from bvh_b200.dtypes import BY_PREC, BY_PREC_2D, BY_PREC_4D

    return {2: BY_PREC_2D, 3: BY_PREC, 4: BY_PREC_4D}[D][prec]["aabb"]


def _F(prec):
    return np.float32 if prec == "f32" else np.float64


def make_boxes(mn, mx, D, prec):
    a = np.zeros(len(mn), dtype=aabb_dtype(D, prec))
    a["min"], a["max"] = mn, mx
    return a


def random_scene(n, D, prec, rng, w_scale=1.0):
    """Boxes in [-100, 100]^D with sizes up to 8; w_scale > 1 stretches the fourth axis so that it wins largest_axis."""
    mn = rng.uniform(-100, 100, (n, D))
    if D == 4:
        mn[:, 3] *= w_scale
    return make_boxes(mn, mn + rng.uniform(0, 8, (n, D)) ** 2 / 8, D, prec)


def clustered_scene(n, D, prec, rng, per=6):
    """Clusters of `per` boxes with one shared centre (boxes of different sizes around it): subtrees over a cluster halve."""
    c = rng.uniform(-100, 100, (n // per + 1, D))[np.arange(n) // per]
    h = rng.choice([0.25, 0.5, 1.0, 2.0], (n, 1)) * np.ones((1, D))
    return make_boxes(c - h, c + h, D, prec)


def jitter(a, idx, scale, rng):
    """Move the boxes idx by uniform offsets in [-scale, scale] (computed in f64, rounded to T)."""
    b = a.copy()
    F = a["min"].dtype.type
    D = a["min"].shape[1]
    off = rng.uniform(-scale, scale, (len(idx), D))
    b["min"][idx] = (a["min"][idx].astype(np.float64) + off).astype(F)
    b["max"][idx] = (a["max"][idx].astype(np.float64) + off).astype(F)
    return b


def scramble_region(a, centre_of, k, rng):
    """The k shapes nearest to shape `centre_of` get new random places inside their joint box: every subtree inside the region is
    degraded, the node above the region is not."""
    c = (a["min"].astype(np.float64) + a["max"].astype(np.float64)) / 2
    idx = np.argsort(((c - c[centre_of]) ** 2).sum(axis=1), kind="stable")[:k]
    lo, hi = c[idx].min(axis=0), c[idx].max(axis=0)
    b = a.copy()
    F = a["min"].dtype.type
    new = rng.uniform(lo, hi, (k, len(lo)))
    half = (a["max"][idx].astype(np.float64) - a["min"][idx].astype(np.float64)) / 2
    b["min"][idx], b["max"][idx] = (new - half).astype(F), (new + half).astype(F)
    return np.sort(idx), b


def mixed_motion(a, rng, regions=(1500, 300, 200, 120, 80, 40), singles=80, single_scale=4.0):
    """One call's motion with rebuild roots of every size: scrambled regions of the given sizes, plus single shapes jittered a little."""
    b, moved = a, []
    n = len(a)
    for k in regions:
        idx, b = scramble_region(b, int(rng.integers(0, n)), k, rng)
        moved.append(idx)
    s = rng.choice(n, singles, replace=False)
    b = jitter(b, s, single_scale, rng)
    moved.append(s)
    return np.unique(np.concatenate(moved)).astype(np.uint32), b


def node_dtype(D, prec):
    from bvh_b200.dtypes import BY_PREC, BY_PREC_2D, BY_PREC_4D

    return {2: BY_PREC_2D, 3: BY_PREC, 4: BY_PREC_4D}[D][prec]["node"]


def build(a, prec):
    """Bvh::build of an AABB array as (nodes, node_index) in the C ABI layout: the oracle for D = 3, tests/pyref.py otherwise."""
    from oracle import oracle as O

    D = a["min"].shape[1]
    if D == 3:
        b = O.build(np.ascontiguousarray(a, dtype=O._DT[prec]["aabb"]), prec)
        return np.array(b.nodes, dtype=node_dtype(3, prec)), b.node_index
    F = _F(prec)
    pn, pidx = pyref.build([{"min": r["min"], "max": r["max"]} for r in a], F)
    nodes = np.zeros(len(pn), dtype=node_dtype(D, prec))
    t = Tree(nodes, np.zeros(len(pidx), dtype=np.uint32))
    t._place(0, pn, pidx, np.arange(len(pidx)), 0)
    return t.nodes, t.node_index
