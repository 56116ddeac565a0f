"""CPU checks behind the self-overlap pairs (bvhgpu_overlap_pairs_*):
- the header declares the 10 entry points and the binding sees them;
- the brute-force model of tests/overlapref.py, closed symmetrically, equals the C++ oracle's Aabb query with every shape's own box
  minus the shape itself, on oracle-built 3-D trees without empty child boxes (dimref scenes and the adversarial box families),
  f32 and f64;
- every pair appears once, in the row of the earlier leaf, with ascending leaves in each row;
- hand-made cases: touching faces and corners, empty and inverted boxes, infinite coordinates, identical boxes."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import adversarial as A, dimref, edge_dims, overlapref as R

FT = {"f32": np.float32, "f64": np.float64}
NEW = [f"bvhgpu_overlap_pairs_{p}x{d}" for d in (2, 3, 4) for p in ("f32", "f64")]
NEW += [f"bvhgpu_overlap_pairs_dev_{p}x{d}" for d in (3, 4) for p in ("f32", "f64")]


def test_header_declares_the_new_entry_points():
    from bvh_b200 import capi

    assert len(NEW) == 10
    assert set(NEW) <= set(capi.declared_symbols())


def _oracle_tree(mn, mx, prec):
    shapes = np.zeros(len(mn), dtype=O.AABB3F if prec == "f32" else O.AABB3D)
    shapes["min"], shapes["max"] = mn, mx
    b = O.build(shapes, prec)
    return shapes, b.nodes, b.node_index


def _check_against_oracle(mn, mx, prec):
    shapes, nodes, leaf = _oracle_tree(mn, mx, prec)
    assert edge_dims.empty_child_boxes(nodes) == 0
    off, hits = R.rows(mn, mx, leaf)
    p = R.pairs(off, hits)
    assert (leaf[p[:, 1]] > leaf[p[:, 0]]).all()                       # the row of the earlier leaf
    for s in range(len(mn)):                                            # DFS order inside a row
        assert (np.diff(leaf[hits[off[s]:off[s + 1]]].astype(np.int64)) > 0).all()
    q = np.concatenate([mn, mx], axis=1)
    qoff, qhits = O.query(O.QUERY_AABB, q, nodes, shapes, prec=prec)
    got = R.closure(off, hits, len(mn))
    for s in range(len(mn)):
        want = sorted(int(t) for t in qhits[qoff[s]:qoff[s + 1]] if t != s)
        assert got[s] == want, s
    return len(p)


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("scene", ["random", "coincident", "axis", "peel"])
def test_model_equals_the_oracle_query(scene, prec):
    F = FT[prec]
    mn, mx = dimref.scene(scene, 300, 3, F, np.random.default_rng(11))
    npairs = _check_against_oracle(mn, mx, prec)
    if scene == "coincident":
        assert npairs == 300 * 299 // 2


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("family", ["large", "ties", "mixed"])
def test_model_equals_the_oracle_query_on_adversarial_boxes(family, prec):
    mn, mx, _ = A.BOX_FAMILIES[family](FT[prec], 3)
    assert _check_against_oracle(mn, mx, prec) > 0


def _boxes(F, rows_):
    a = np.array(rows_, dtype=np.float64)
    return a[:, 0].astype(F), a[:, 1].astype(F)


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_hand_made_cases(prec):
    F = FT[prec]
    inf = np.inf
    mn, mx = _boxes(F, [
        ([0, 0, 0], [1, 1, 1]),          # 0
        ([1, 0, 0], [2, 1, 1]),          # 1 touches 0 on a face
        ([2, 1, 1], [3, 2, 2]),          # 2 touches 1 on an edge / corner
        ([inf, inf, inf], [-inf, -inf, -inf]),   # 3 Aabb::empty(): overlaps nothing finite
        ([0.5, 0.5, 0.5], [0.25, 0.75, 0.75]),   # 4 inverted in x: [0.25, 0.5] of 0 spans it, the formula holds
        ([-inf, 5, 5], [inf, 6, 6]),     # 5 infinite in x
        ([10, 5, 5], [10, 5, 5]),        # 6 point on 5's face
        ([0, 0, 0], [1, 1, 1]),          # 7 identical to 0
        ([7, 7, 7], [8, 8, 8]),          # 8 alone
    ])
    leaf = np.arange(len(mn), dtype=np.uint32) * 2 + 1                  # leaves in index order
    off, hits = R.rows(mn, mx, leaf)
    got = {(int(s), int(t)) for s, t in R.pairs(off, hits)}
    assert got == {(0, 1), (0, 4), (0, 7), (1, 2), (1, 7), (4, 7), (5, 6)}
    assert len(R.pairs(off, hits)) == len(got)
    # the same scene in reverse leaf order: the same pairs, each in the other row
    off2, hits2 = R.rows(mn, mx, leaf[::-1].copy())
    assert {(int(t), int(s)) for s, t in R.pairs(off2, hits2)} == got
    # n = 0 and n = 1
    off0, hits0 = R.rows(mn[:0], mx[:0], leaf[:0])
    assert off0.tolist() == [0] and len(hits0) == 0
    off1, hits1 = R.rows(mn[:1], mx[:1], leaf[:1])
    assert off1.tolist() == [0, 0] and len(hits1) == 0


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_lifts_in_the_model(prec):
    """2-D rows equal the 3-D rows of the scene lifted to z = [0, 0]; a constant fourth axis leaves the 3-D rows unchanged."""
    F = FT[prec]
    mn, mx = dimref.scene("random", 200, 2, F, np.random.default_rng(3))
    leaf = np.random.default_rng(4).permutation(400)[:200].astype(np.uint32)
    z = lambda a, v: np.concatenate([a, np.full((len(a), 1), v, dtype=F)], axis=1)   # noqa: E731
    o2, h2 = R.rows(mn, mx, leaf)
    o3, h3 = R.rows(z(mn, 0), z(mx, 0), leaf)
    o4, h4 = R.rows(z(z(mn, 0), 3.5), z(z(mx, 0), 3.5), leaf)
    assert np.array_equal(o2, o3) and np.array_equal(h2, h3) and np.array_equal(o3, o4) and np.array_equal(h3, h4)
    assert len(h2) > 0
