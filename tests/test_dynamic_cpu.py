"""Batched add / remove without a GPU: the renumbering rule, and the oracle's sequential add_shape / remove_shape (the
device's reference) on built trees, re-emitted in preorder."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import dynoracle as D
from tests.scenes import scene


def _sequential_swap_remove(n, i):
    """shapes.swap_remove(i) as Bvh::remove_shape(i, true) + pop() leaves the ids: the last one takes slot i."""
    ids = list(range(n))
    ids[i] = ids[-1]
    ids.pop()
    return ids


@pytest.mark.parametrize("seed", range(20))
def test_swap_rule_is_remove_shape_swap_then_pop_for_one_index(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 200))
    i = int(rng.integers(0, n))
    assert D.apply_moves(np.arange(n), [i]).tolist() == _sequential_swap_remove(n, i)


def test_swap_rule_for_several_indices_fills_holes_in_ascending_order():
    assert D.apply_moves(np.arange(5), [0, 1, 2]).tolist() == [3, 4]
    assert D.apply_moves(np.arange(6), [4, 1]).tolist() == [0, 5, 2, 3]
    from bvh_b200.api import swap_moves                 # the product's copy of the rule
    for seed in range(10):
        rng = np.random.default_rng(seed)
        n = int(rng.integers(1, 300))
        idx = rng.choice(n, int(rng.integers(1, n + 1)), replace=False)
        assert np.array_equal(swap_moves(n, idx), D.swap_moves(n, idx))


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("name", ["random500", "points300", "cubes20"])
def test_oracle_remove_in_any_order_gives_one_tree(name, prec):
    """The contraction does not depend on removal order -- what lets the device remove all k at once."""
    shapes = scene(name, prec)
    b = O.build(shapes, prec)
    rng = np.random.default_rng(3)
    for k in (1, 2, len(shapes) // 3, len(shapes) - 1, len(shapes)):
        idx = rng.choice(len(shapes), k, replace=False)
        n1, i1, s1 = D.remove_shapes(b.nodes, b.node_index, shapes, idx, prec)
        n2, i2, s2 = D.remove_shapes(b.nodes, b.node_index, shapes, idx[::-1], prec)
        assert D.same_tree(n1, n2) and np.array_equal(i1, i2)
        if len(s1) > 1:
            assert O.is_consistent(n1, s1, prec) and O.is_tight(n1, prec)
            f = n1[n1["child_l"] != O.U32_MAX]                   # preorder layout
            assert np.array_equal(f["child_l"], np.flatnonzero(n1["child_l"] != O.U32_MAX) + 1)


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_oracle_mixed_add_remove_stays_consistent(prec):
    """The fuzz target's Add / Remove mutations (push + add_shape(len-1); remove_shape(i, true) + pop) through the oracle."""
    rng = np.random.default_rng(7)
    shapes = scene("random300", prec)
    b = O.build(shapes, prec)
    nodes, ni = b.nodes, b.node_index
    for step in range(150):
        if len(shapes) > 1 and rng.random() < 0.45:
            i = int(rng.integers(0, len(shapes)))
            nodes, ni, shapes = D.remove_shapes(nodes, ni, shapes, [i], prec)
        else:
            mn = rng.uniform(-1000, 1000, (1, 3)) * (1000 if rng.random() < 0.1 else 1)
            new = O.make_aabbs(mn, mn + rng.uniform(0, 20, (1, 3)), prec)
            shapes = np.concatenate([shapes, new])
            nodes, ni = D.add_shapes(nodes, ni, shapes, 1, prec)
        assert O.is_consistent(nodes, shapes, prec) and O.is_tight(nodes, prec), step
        assert np.array_equal(nodes["shape"][ni], np.arange(len(shapes)))


# ---- numpy restatement of the device's index arithmetic (dynamic.cu), checked against the oracle before any GPU time ----------
def _counts_starts(nodes):
    nn = len(nodes)
    leaf = nodes["child_l"] == O.U32_MAX
    c = np.where(leaf, 1, nodes["shape"]).astype(np.int64)
    start = np.zeros(nn, dtype=np.int64)
    for i in range(nn):
        if not leaf[i]:
            start[i + 1] = start[i]
            start[nodes["child_r"][i]] = start[i] + c[i + 1]
    return leaf, c, start


def _box(nodes, shapes, j):
    nd = nodes[j]
    if nd["child_l"] == O.U32_MAX:
        return shapes["min"][nd["shape"]].copy(), shapes["max"][nd["shape"]].copy()
    return np.minimum(nd["l_aabb"]["min"], nd["r_aabb"]["min"]), np.maximum(nd["l_aabb"]["max"], nd["r_aabb"]["max"])


def _refit_affected(nw, aff, shapes):
    """climb_affected_kernel: both slots of every affected node from its children's boxes, children first (higher index first)."""
    for j in np.flatnonzero(aff)[::-1]:
        l, r = nw["child_l"][j], nw["child_r"][j]
        nw["l_aabb"]["min"][j], nw["l_aabb"]["max"][j] = _box(nw, shapes, l)
        nw["r_aabb"]["min"][j], nw["r_aabb"]["max"][j] = _box(nw, shapes, r)


def contract(nodes, shapes, idx):
    """remove_shapes: survive flags over R (removed leaves by position), exclusive scan = new index, swap-rule relabel."""
    n, k = len(shapes), len(idx)
    leaf, c, start = _counts_starts(nodes)
    rm = np.zeros(n + 1, dtype=np.int64); rm[idx] = 1
    ni = np.zeros(n, dtype=np.int64); ni[nodes["shape"][leaf]] = np.flatnonzero(leaf)
    kpos = np.zeros(n + 1, dtype=np.int64); kpos[start[ni[idx]]] = 1
    R = np.concatenate([[0], np.cumsum(kpos)[:-1]])
    Rm = np.concatenate([[0], np.cumsum(rm)[:-1]])
    m = n - k
    holes = np.flatnonzero(rm[:m])
    relabel = lambda s: s if s < m else holes[(s - m) - (Rm[s] - Rm[m])]
    nc = c - (R[start + c] - R[start])
    cl = np.where(leaf, 0, c[np.minimum(np.arange(len(nodes)) + 1, len(nodes) - 1)])
    ncl = cl - (R[start + cl] - R[start])
    survive = np.where(leaf, nc == 1, (ncl > 0) & (nc > ncl))
    newidx = np.concatenate([[0], np.cumsum(survive)])
    nw = np.zeros(max(2 * m - 1, 0), dtype=nodes.dtype)
    aff = np.zeros(len(nw), dtype=bool)
    node_index = np.zeros(m, dtype=np.uint32)
    for i in np.flatnonzero(survive):
        j = newidx[i]
        par = nw["parent"][j]                                 # written by the surviving parent, as on the device
        nw[j] = nodes[i]
        nw["parent"][j] = par
        if leaf[i]:
            s = relabel(int(nodes["shape"][i])); nw["shape"][j] = s; node_index[s] = j
        else:
            nw["child_l"][j] = j + 1; nw["child_r"][j] = j + 2 * ncl[i]; nw["shape"][j] = nc[i]
            nw["parent"][j + 1] = j; nw["parent"][j + 2 * ncl[i]] = j
            aff[j] = nc[i] != c[i]
        if j == 0:
            nw["parent"][0] = 0
    rest = D.apply_moves(shapes, idx)
    _refit_affected(nw, aff, rest)
    return nw, node_index, rest


def _descend(nodes, box, prec):
    F = O._DT[prec]["f"]
    sa = lambda mn, mx: F(2) * ((F(mx[0] - mn[0]) * F(mx[0] - mn[0]) + F(mx[1] - mn[1]) * F(mx[1] - mn[1])) + F(mx[2] - mn[2]) * F(mx[2] - mn[2]))
    smn, smx = box["min"], box["max"]
    i = 0
    with np.errstate(over="ignore", invalid="ignore"):
        while nodes["child_l"][i] != O.U32_MAX:
            l, r = nodes["l_aabb"][i], nodes["r_aabb"][i]
            send_left = F(sa(r["min"], r["max"]) + sa(np.minimum(l["min"], smn), np.maximum(l["max"], smx)))
            send_right = F(sa(l["min"], l["max"]) + sa(np.minimum(r["min"], smn), np.maximum(r["max"], smx)))
            merged = F(sa(np.minimum(r["min"], l["min"]), np.maximum(r["max"], l["max"])) + sa(smn, smx))
            min_send = send_left if send_left < send_right else send_right
            if merged < F(F(min_send * F(3)) / F(10)):
                break
            i = int(nodes["child_l"][i] if send_left < send_right else nodes["child_r"][i])
    return i


def graft(nodes, shapes, prec):
    """add_shapes with k = 1 and max_growth 0: base(i) = i + 2 (S(i) - a_i), content -> i + 2 S(i), start += S(i), then the climb."""
    n = len(shapes) - 1
    p = _descend(nodes, shapes[n], prec)
    leaf, c, start = _counts_starts(nodes)
    nn = len(nodes)
    a = np.zeros(nn, dtype=np.int64); a[p] = 1
    S = np.cumsum(a)
    nw = np.zeros(nn + 2, dtype=nodes.dtype)
    aff = np.zeros(nn + 2, dtype=bool)
    node_index = np.zeros(n + 1, dtype=np.uint32)
    for i in range(nn):
        base = i + 2 * (S[i] - a[i]); pos = base + 2 * a[i]
        par = nodes["parent"][i] + 2 * S[nodes["parent"][i]] if i else 0
        o = nodes[i].copy()
        o["parent"] = base if a[i] else par
        if not leaf[i]:
            below = S[i + 2 * c[i] - 2] - S[i]
            o["child_l"] = pos + 1; cr = nodes["child_r"][i]; o["child_r"] = cr + 2 * (S[cr] - a[cr]); o["shape"] = c[i] + below
            aff[pos] = below > 0
        else:
            node_index[o["shape"]] = pos
        nw[pos] = o
        if a[i]:
            g = nw[base]
            g["parent"] = par; g["child_l"] = base + 1; g["child_r"] = pos; g["shape"] = 1 + (1 if leaf[i] else o["shape"])
            nw[base] = g
            lf = nodes[0].copy()
            lf["parent"] = base; lf["child_l"] = lf["child_r"] = O.U32_MAX; lf["shape"] = n
            for s_ in ("l_aabb", "r_aabb"):
                lf[s_]["min"] = np.inf; lf[s_]["max"] = -np.inf
            nw[base + 1] = lf
            node_index[n] = base + 1
            aff[base] = True
    _refit_affected(nw, aff, shapes)
    return nw, node_index


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("name", ["random300", "points200", "cubes10"])
def test_numpy_contraction_equals_oracle_remove(name, prec):
    shapes = scene(name, prec)
    b = O.build(shapes, prec)
    rng = np.random.default_rng(8)
    for k in (1, 2, len(shapes) // 10, len(shapes) // 2, len(shapes) - 1):
        idx = rng.choice(len(shapes), k, replace=False)
        wn, wi, ws = D.remove_shapes(b.nodes, b.node_index, shapes, idx, prec)
        gn, gi, gs = contract(b.nodes, shapes, idx)
        assert D.same_tree(gn, wn) and np.array_equal(gi, wi) and np.array_equal(gs, ws), k


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_numpy_graft_equals_oracle_add_shape(prec):
    rng = np.random.default_rng(10)
    shapes = scene("random300", prec)
    b = O.build(shapes, prec)
    nodes, ni = b.nodes, b.node_index
    for step in range(60):
        mn = rng.uniform(-1000, 1000, (1, 3)) * (1e4 if step % 3 == 1 else 1.0)
        shapes = np.concatenate([shapes, O.make_aabbs(mn, mn + rng.uniform(0, 30, (1, 3)), prec)])
        gn, gi = graft(nodes, shapes, prec)
        nodes, ni = D.add_shapes(nodes, ni, shapes, 1, prec)
        assert D.same_tree(gn, nodes) and np.array_equal(gi, ni), step
