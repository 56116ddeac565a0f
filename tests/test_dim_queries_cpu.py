"""CPU checks behind the 2-D and 4-D queries and nearest_to:
- the header declares the 14 entry points and the binding sees them;
- the dimension-generic restatement (tests/dimref.py) equals the C++ oracle at D = 3 on random, coincident and f32 overflow scenes,
  in BVH and FLAT mode, f32 and f64: the same hit lists in the same order, the same nearest shape and the same distance bits.  That
  makes it an oracle for D = 2 and D = 4 (tests/test_gpu_dim_queries.py);
- the lift identities the 2-D embedding and the 4-D tests rely on hold in the restatement: a 3-D scene with a constant fourth axis
  gives the 3-D results, a 2-D scene with z = [0, 0] gives the 2-D results."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import dimref, pyref

PRECS = ("f32", "f64")
FT = {"f32": np.float32, "f64": np.float64}
KINDS = (dimref.AABB, dimref.POINT, dimref.BALL)
NEW = [f"bvhgpu_{f}_{p}x{d}" for d in (2, 4) for p in ("f32", "f64") for f in ("query", "nearest", "nearest_candidates")]
NEW += [f"bvhgpu_query_dev_{p}x4" for p in ("f32", "f64")]


def test_header_declares_the_new_entry_points():
    from bvh_b200 import capi

    assert len(NEW) == 14
    assert set(NEW) <= set(capi.declared_symbols())


def _oracle_tree(mn, mx, prec):
    shapes = np.zeros(len(mn), dtype=O.AABB3F if prec == "f32" else O.AABB3D)
    shapes["min"], shapes["max"] = mn, mx
    nodes = O.build(shapes, prec).nodes
    return shapes, nodes, O.flatten(nodes, prec)


def _same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.tobytes() == b.tobytes()


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("scene", ["random", "coincident", "overflow"])
def test_restatement_equals_the_oracle_in_3d(scene, prec):
    F = FT[prec]
    rng = np.random.default_rng(5)
    mn, mx = dimref.scene(scene, 300, 3, F, rng)
    shapes, nodes, flat = _oracle_tree(mn, mx, prec)
    if scene == "overflow" and prec == "f32":
        assert np.any(nodes["l_aabb"]["min"][:, 0] == np.inf)       # the builder stored empty child boxes
    tree = dimref.Tree(nodes, shapes, flat)
    for kind in KINDS:
        q = dimref.queries(kind, mn, mx, 120, F, rng)
        for use_flat in (False, True):
            off, hits = O.query(kind, q, nodes, shapes, flat=flat if use_flat else None, prec=prec)
            for i in range(len(q)):
                want = hits[off[i]:off[i + 1]].tolist()
                got = tree.query_flat(kind, q[i]) if use_flat else tree.query_bvh(kind, q[i])
                assert got == want, (kind, use_flat, i)
    p = dimref.points(mn, mx, 120, F, rng)
    for use_flat in (False, True):
        s, d = O.nearest_to(flat if use_flat else nodes, shapes, p, prec=prec, flat=use_flat)
        for i in range(len(p)):
            gs, gd = tree.nearest_flat(p[i]) if use_flat else tree.nearest_bvh(p[i])
            assert gs == s[i] and _same_bits(gd, d[i]), (use_flat, i)


def _lift(mn, mx, c, F):
    col = np.full((len(mn), 1), c, dtype=F)
    return np.concatenate([mn, col], axis=1), np.concatenate([mx, col], axis=1)


def _lift_rec(kind, q, c, F):
    D = q.shape[1] - (1 if kind == dimref.BALL else 0)
    D = D // 2 if kind == dimref.AABB else D
    col = np.full((len(q), 1), c, dtype=F)
    if kind == dimref.AABB:
        return np.concatenate([q[:, :D], col, q[:, D:], col], axis=1)
    if kind == dimref.POINT:
        return np.concatenate([q, col], axis=1)
    return np.concatenate([q[:, :D], col, q[:, D:]], axis=1)


def _pyref_tree(mn, mx, F, dtype_table):
    """Nodes / flat arrays of the reference's build (tests/pyref.py) in the C ABI layout of the dimension of mn."""
    n, D = mn.shape
    d = dtype_table
    nodes_l, index = pyref.build([{"min": list(mn[i]), "max": list(mx[i])} for i in range(n)], F)
    nodes = np.zeros(len(nodes_l), dtype=d["node"])
    for i, w in enumerate(nodes_l):
        nodes["parent"][i] = w[1]
        if w[0] == "leaf":
            nodes["child_l"][i] = nodes["child_r"][i] = dimref.U32_MAX
            nodes["shape"][i] = w[2]
            nodes["l_aabb"]["min"][i] = nodes["r_aabb"]["min"][i] = np.inf
            nodes["l_aabb"]["max"][i] = nodes["r_aabb"]["max"][i] = -np.inf
        else:
            nodes["child_l"][i], nodes["child_r"][i] = w[2], w[3]
            nodes["l_aabb"]["min"][i], nodes["l_aabb"]["max"][i] = w[4]
            nodes["r_aabb"]["min"][i], nodes["r_aabb"]["max"][i] = w[5]
    flat_l = pyref.flatten(nodes_l)
    flat = np.zeros(len(flat_l), dtype=d["flat"])
    for i, (box, entry, exit_, shape) in enumerate(flat_l):
        flat["aabb"]["min"][i], flat["aabb"]["max"][i] = box if box is not None else ([np.inf] * D, [-np.inf] * D)
        flat["entry_index"][i], flat["exit_index"][i], flat["shape_index"][i] = entry, exit_, shape
    shapes = np.zeros(n, dtype=d["aabb"])
    shapes["min"], shapes["max"] = mn, mx
    return dimref.Tree(nodes, shapes, flat), nodes_l


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("low", [2, 3])
def test_lift_identities_in_the_restatement(low, prec):
    """D -> D + 1 with a constant last axis (w = [1.5, 1.5] for 3 -> 4, z = [0, 0] for 2 -> 3): same tree, same hits, same nearest
    shape and distance bits."""
    from bvh_b200.dtypes import BY_PREC, BY_PREC_2D, BY_PREC_4D

    F = FT[prec]
    c = F(1.5) if low == 3 else F(0)
    table = {2: BY_PREC_2D, 3: BY_PREC, 4: BY_PREC_4D}
    rng = np.random.default_rng(11 + low)
    for scene in ("random", "coincident"):
        mn, mx = dimref.scene(scene, 120, low, F, rng)
        lo, nodes_lo = _pyref_tree(mn, mx, F, table[low][prec])
        hi, nodes_hi = _pyref_tree(*_lift(mn, mx, c, F), F, table[low + 1][prec])
        assert [(w[0],) + tuple(w[1:4]) for w in nodes_lo] == [(w[0],) + tuple(w[1:4]) for w in nodes_hi]   # same topology
        for kind in KINDS:
            q = dimref.queries(kind, mn, mx, 60, F, rng)
            ql = _lift_rec(kind, q, c, F)
            for i in range(len(q)):
                assert lo.query_bvh(kind, q[i]) == hi.query_bvh(kind, ql[i])
                assert lo.query_flat(kind, q[i]) == hi.query_flat(kind, ql[i])
        p = dimref.points(mn, mx, 60, F, rng)
        pl = _lift_rec(dimref.POINT, p, c, F)
        for i in range(len(p)):
            for f in ("nearest_bvh", "nearest_flat"):
                a, b = getattr(lo, f)(p[i]), getattr(hi, f)(pl[i])
                assert a[0] == b[0] and _same_bits(a[1], b[1]), (scene, f, i)
