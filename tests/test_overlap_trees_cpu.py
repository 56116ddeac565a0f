"""CPU checks behind the overlap pairs between two trees (bvhgpu_overlap_trees_*):
- the header declares the 10 entry points and the binding sees them;
- the brute-force model of tests/crossref.py equals the C++ oracle's Aabb query of A's boxes on an oracle-built B, offsets and hits,
  on trees without empty child boxes (dimref scenes and the adversarial box families), f32 and f64;
- hand-made cases: touching faces and corners, empty and inverted boxes, infinite coordinates, identical boxes;
- the transpose identity: pairs(A, B) are the pairs of (B, A) reversed;
- the a == b identity: row s is s's self-overlap row, the earlier leaves whose rows list s, and s itself when its box meets itself,
  in leaf order."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import adversarial as A, dimref, edge_dims, overlapref as R
from tests.crossref import cross_rows

FT = {"f32": np.float32, "f64": np.float64}
NEW = [f"bvhgpu_overlap_trees_{p}x{d}" for d in (2, 3, 4) for p in ("f32", "f64")]
NEW += [f"bvhgpu_overlap_trees_dev_{p}x{d}" for d in (3, 4) for p in ("f32", "f64")]


def test_header_declares_the_new_entry_points():
    from bvh_b200 import capi

    assert len(NEW) == 10
    assert set(NEW) <= set(capi.declared_symbols())


def _check_against_oracle(amn, amx, bmn, bmx, prec):
    shapes = np.zeros(len(bmn), dtype=O.AABB3F if prec == "f32" else O.AABB3D)
    shapes["min"], shapes["max"] = bmn, bmx
    b = O.build(shapes, prec)
    assert edge_dims.empty_child_boxes(b.nodes) == 0
    off, hits = cross_rows(amn, amx, bmn, bmx, b.node_index)
    qoff, qhits = O.query(O.QUERY_AABB, np.concatenate([amn, amx], axis=1), b.nodes, shapes, prec=prec)
    assert np.array_equal(np.asarray(qoff, dtype=np.uint64), off.astype(np.uint64))
    assert np.array_equal(np.asarray(qhits, dtype=np.uint32), hits)
    return len(hits)


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("scene_b", ["random", "coincident", "axis", "peel"])
@pytest.mark.parametrize("scene_a", ["random", "axis"])
def test_model_equals_the_oracle_query(scene_a, scene_b, prec):
    F = FT[prec]
    amn, amx = dimref.scene(scene_a, 230, 3, F, np.random.default_rng(12))
    bmn, bmx = dimref.scene(scene_b, 300, 3, F, np.random.default_rng(13))
    _check_against_oracle(amn, amx, bmn, bmx, prec)


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("family", ["large", "ties", "mixed"])
def test_model_equals_the_oracle_query_on_adversarial_boxes(family, prec):
    F = FT[prec]
    bmn, bmx, _ = A.BOX_FAMILIES[family](F, 3)
    rng = np.random.default_rng(8)
    ext = bmx.astype(np.float64) - bmn
    d = rng.uniform(-0.5, 0.5, bmn.shape) * ext
    amn, amx = (bmn + d).astype(F), (bmx + d).astype(F)
    assert _check_against_oracle(amn, amx, bmn, bmx, prec) > 0


def _boxes(F, rows_):
    a = np.array(rows_, dtype=np.float64)
    return a[:, 0].astype(F), a[:, 1].astype(F)


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_hand_made_cases(prec):
    F = FT[prec]
    inf = np.inf
    amn, amx = _boxes(F, [
        ([0, 0, 0], [1, 1, 1]),                  # a0
        ([inf, inf, inf], [-inf, -inf, -inf]),   # a1 Aabb::empty(): overlaps nothing finite
        ([0.5, 0.5, 0.5], [0.25, 0.75, 0.75]),   # a2 inverted in x
        ([-inf, 5, 5], [inf, 6, 6]),             # a3 infinite in x
        ([7, 7, 7], [8, 8, 8]),                  # a4 alone
    ])
    bmn, bmx = _boxes(F, [
        ([1, 0, 0], [2, 1, 1]),                  # b0 touches a0 on a face
        ([1, 1, 1], [3, 2, 2]),                  # b1 touches a0 on a corner
        ([10, 5, 5], [10, 5, 5]),                # b2 point on a3's face
        ([0, 0, 0], [1, 1, 1]),                  # b3 identical to a0
        ([0.2, 0.6, 0.6], [0.6, 0.7, 0.7]),      # b4 inside a0, spans inverted a2's x range [0.25, 0.5]: the formula holds
        ([inf, inf, inf], [-inf, -inf, -inf]),   # b5 empty
    ])
    leaf = np.array([9, 3, 5, 1, 7, 11], dtype=np.uint32)    # B's DFS order: b3, b1, b2, b4, b0, b5
    off, hits = cross_rows(amn, amx, bmn, bmx, leaf)
    assert off.tolist() == [0, 4, 4, 6, 7, 7]
    assert hits.tolist() == [3, 1, 4, 0, 3, 4, 2]
    # n_a = 0, n_b = 0, n_b = 1
    o, h = cross_rows(amn[:0], amx[:0], bmn, bmx, leaf)
    assert o.tolist() == [0] and len(h) == 0
    o, h = cross_rows(amn, amx, bmn[:0], bmx[:0], leaf[:0])
    assert o.tolist() == [0] * 6 and len(h) == 0
    o, h = cross_rows(amn, amx, bmn[3:4], bmx[3:4], leaf[3:4])
    assert o.tolist() == [0, 1, 1, 2, 2, 2] and h.tolist() == [0, 0]


@pytest.mark.parametrize("D", [2, 3, 4])
@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_transpose_identity(prec, D):
    F = FT[prec]
    rng = np.random.default_rng(30 + D)
    amn, amx = dimref.scene("random", 300, D, F, rng)
    bmn, bmx = dimref.scene("random", 200, D, F, rng)
    amx, bmx = (amn + (amx - amn) * 5).astype(F), (bmn + (bmx - bmn) * 5).astype(F)
    leaf_a, leaf_b = rng.permutation(600)[:300], rng.permutation(400)[:200]
    ab = cross_rows(amn, amx, bmn, bmx, leaf_b)
    ba = cross_rows(bmn, bmx, amn, amx, leaf_a)
    p_ab = set(map(tuple, R.pairs(*ab).tolist()))
    p_ba = {(a, b) for b, a in R.pairs(*ba).tolist()}
    assert p_ab == p_ba and len(p_ab) == len(ab[1]) > 0


@pytest.mark.parametrize("scene", ["random", "coincident", "peel"])
@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_self_identity(prec, scene):
    F = FT[prec]
    rng = np.random.default_rng(50)
    mn, mx = dimref.scene(scene, 250, 3, F, rng)
    mn[:5], mx[:5] = mx[:5], mn[:5]                            # inverted boxes do not meet themselves (unless flat)
    leaf = rng.permutation(500)[:250].astype(np.uint32)
    off, hits = cross_rows(mn, mx, mn, mx, leaf)
    so, sh = R.rows(mn, mx, leaf)
    earlier = [[] for _ in range(len(mn))]
    for s, t in R.pairs(so, sh).tolist():
        earlier[t].append(s)
    for s in range(len(mn)):
        want = list(sh[so[s]:so[s + 1]]) + earlier[s]
        if R.intersects(mn[s], mx[s], mn[s:s + 1], mx[s:s + 1])[0]:
            want.append(s)
        want = sorted(want, key=lambda t: leaf[t])
        assert hits[off[s]:off[s + 1]].tolist() == want, s
