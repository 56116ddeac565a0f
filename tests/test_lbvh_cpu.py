"""Pins tests/lbvhref.py, the restatement of the LBVH builders: the two Karras forms agree, restated trees are valid preorder trees
that pass the reference's consistency and tightness checks, treelet mode on one treelet is Bvh::build, and the special scenes of
tests/test_gpu_lbvh_exact.py have what they claim.  CPU only."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import lbvhref as LR
from tests import rebuildref as RR
from tests.scenes import scene


def _sorted_codes(codes):
    return np.sort(np.asarray(codes, dtype=np.uint64), kind="stable")


def _same_karras(codes):
    a, b = LR.karras(codes), LR.karras_recursive(codes)
    for x, y, what in zip(a, b, ("left", "right", "first", "count")):
        assert np.array_equal(x, y), (what, len(codes))


@pytest.mark.parametrize("n", [2, 3, 4, 5, 17, 1000, 4097])
def test_karras_forms_agree_on_random_codes(n):
    rng = np.random.default_rng(n)
    _same_karras(_sorted_codes(rng.integers(0, 1 << 63, n, dtype=np.uint64)))


@pytest.mark.parametrize("n", [2, 3, 7, 64, 1000, 3001])
def test_karras_forms_agree_with_many_duplicates(n):
    rng = np.random.default_rng(100 + n)
    base = rng.integers(0, 1 << 63, max(n // 20, 1), dtype=np.uint64)
    _same_karras(_sorted_codes(base[rng.integers(0, len(base), n)]))
    small = rng.integers(0, 4, n).astype(np.uint64)                # codes differing in the lowest bits only
    _same_karras(_sorted_codes(small))


@pytest.mark.parametrize("n", [2, 3, 512, 513, 1025])
def test_karras_forms_agree_on_equal_codes(n):
    _same_karras(np.zeros(n, dtype=np.uint64))
    _same_karras(np.full(n, (1 << 63) - 1, dtype=np.uint64))


def test_karras_forms_agree_on_single_bit_codes():
    codes = np.array([0] + [1 << b for b in range(63)] + [(1 << 63) - 1], dtype=np.uint64)
    _same_karras(np.repeat(codes, 3))
    _same_karras(codes)


def test_clz_and_expand21():
    x = np.array([0, 1, 2, 3, 1 << 31, 1 << 32, (1 << 63) | 5, (1 << 64) - 1], dtype=np.uint64)
    want = [64 - int(v).bit_length() for v in x.tolist()]
    assert LR.clz64(x).tolist() == want
    assert LR.clz32(np.array([0, 1, 1 << 31])).tolist() == [32, 31, 0]
    for q in (1, 2, 0x1FFFFF, 0x155555, 12345):
        want = sum(((q >> b) & 1) << (3 * b) for b in range(21))
        assert int(LR.expand21(q)) == want


def test_quantisation_rule():
    q, f = LR.quantise([0.5, 1.5, 2097151.5], 0.0, 2097151.0)
    assert q.tolist() == [0, 1, 2097151] and not f["overflow"]
    q, _ = LR.quantise([3.0, 3.0], 3.0, 3.0)                       # no extent: code 0
    assert q.tolist() == [0, 0]
    q, f = LR.quantise([-1.5e308, 0.0, 1.5e308], -1.5e308, 1.5e308)
    assert f["overflow"] and f["nan_u_unhalved"] == 1               # c - lo overflows too at the top: inf / inf
    assert q.tolist() == [0, 1048575, 2097151]
    q, _ = LR.quantise([np.inf, 1.0], 0.0, np.inf)                 # an infinite centroid: NaN u -> 0, finite / inf -> 0
    assert q.tolist() == [0, 0]


def _check_tree(nodes, idx, a, prec, D):
    n = len(a)
    assert len(nodes) == 2 * n - 1 and LR.preorder_ok(nodes)
    leaves = nodes["child_l"] == LR.U32_MAX
    assert np.array_equal(np.sort(nodes["shape"][leaves]), np.arange(n))
    assert np.array_equal(nodes["shape"][idx], np.arange(n))
    if D == 3:
        assert O.is_consistent(nodes, a, prec) and O.is_tight(nodes, prec)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("D,prec", [(3, "f32"), (3, "f64"), (2, "f32"), (2, "f64")])
@pytest.mark.parametrize("n", [2, 3, 511, 513, 3000])
def test_restated_trees_are_valid(n, D, prec, mode):
    a = RR.random_scene(n, D, prec, np.random.default_rng(n + D))
    nodes, idx, info = LR.restate(a, prec, mode)
    _check_tree(nodes, idx, a, prec, D)
    if mode == 1:                                                   # without treelets: the Morton order is the leaf order
        assert np.array_equal(nodes["shape"][nodes["child_l"] == LR.U32_MAX], info["order"])


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("name", ["random2", "random3", "random33", "random257", "random513"])
def test_one_treelet_is_build(name, prec):
    a = scene(name, prec)
    if len(a) > LR.TILE:
        a = a[:LR.TILE]
    nodes, idx, info = LR.restate(a, prec, 2)
    want = O.build(a, prec)
    assert info["treelets"] == [0]
    for f in ("parent", "child_l", "child_r", "shape"):
        assert np.array_equal(nodes[f], want.nodes[f])
    for s in ("l_aabb", "r_aabb"):
        for m in ("min", "max"):
            assert np.array_equal(nodes[s][m], want.nodes[s][m])
    assert np.array_equal(idx, want.node_index)


def test_treelet_roots_follow_the_tile_rule():
    a = RR.random_scene(20000, 3, "f32", np.random.default_rng(3))
    nodes, idx, info = LR.restate(a, "f32", 2)
    _check_tree(nodes, idx, a, "f32", 3)
    K = info["tree"]
    roots = LR.treelet_roots(K)
    assert len(roots) > 20
    assert np.all(K.count[roots] <= LR.TILE) and np.all(K.count[K.parent[roots]] > LR.TILE)
    covered = np.zeros(len(a), dtype=int)                           # every shape lies in at most one treelet
    for r in info["treelets"]:
        covered[LR.subtree_shapes(nodes, r)] += 1
    assert covered.max() == 1
    comb = LR.comb_scene(3, "f32", low_bits=12)                     # the chain's single-bit leaves hang below vertices of > TILE shapes
    nodes, idx, info = LR.restate(comb, "f32", 2)
    _check_tree(nodes, idx, comb, "f32", 3)
    inside = np.concatenate([LR.subtree_shapes(nodes, r) for r in info["treelets"]])
    assert len(np.unique(inside)) == len(inside) and 40 < len(comb) - len(inside) < 100


@pytest.mark.parametrize("D", [2, 3])
def test_comb_scene_is_deep(D):
    a = LR.comb_scene(D, "f32")
    nodes, idx, info = LR.restate(a, "f32", 1)
    _check_tree(nodes, idx, a, "f32", D)
    d = LR.depth(nodes)
    assert d <= 128                                                  # path_kernel's 7 rounds of pointer jumping
    assert d >= (80 if D == 3 else 55), d
    distinct = np.unique(info["code"])
    want = {0, (1 << 63) - 1 if D == 3 else sum(1 << b for b in range(63) if b % 3)}
    want |= {1 << b for b in range(63) if D == 3 or b % 3}
    assert set(distinct.tolist()) == want
    f64 = LR.comb_scene(D, "f64")
    assert np.array_equal(LR.restate(f64, "f64", 1)[2]["code"], info["code"])


def test_identical_centroids_give_one_code():
    a = LR.identical_scene(1025, 3, "f32", np.random.default_rng(1))
    nodes, idx, info = LR.restate(a, "f32", 1)
    assert np.all(info["code"] == 0) and np.array_equal(info["order"], np.arange(len(a)))
    assert LR.depth(nodes) == 11                                    # a balanced tree over positions 0..1024


@pytest.mark.parametrize("D", [2, 3])
def test_signed_zero_scene_mixes_signs(D):
    a = LR.signed_zero_scene(3000, D, "f32", np.random.default_rng(4))
    for mode in (1, 2):
        nodes, idx, info = LR.restate(a, "f32", mode)
        _check_tree(nodes, idx, a, "f32", D)
        assert LR.mixed_zero_signs(nodes) > 100
        if mode == 1:                                               # -0 wins every min join: a child box's min.x is -0 iff a shape below has it
            neg = np.signbit(a["min"][:, 0])
            for i in np.flatnonzero(nodes["child_l"] != LR.U32_MAX)[:400]:
                for side, c in (("l_aabb", nodes["child_l"][i]), ("r_aabb", nodes["child_r"][i])):
                    assert np.signbit(nodes[side]["min"][i][0]) == neg[LR.subtree_shapes(nodes, c)].any()


@pytest.mark.parametrize("D", [2, 3])
def test_overflow_scene_quantises_with_halved_operands(D):
    a = LR.overflow_centroid_scene(3000, D, np.random.default_rng(5))
    nodes, idx, info = LR.restate(a, "f64", 1)
    f = info["morton"][0]
    assert f["overflow"] and f["nan_u_unhalved"] > 0
    assert len(np.unique(info["code"] >> np.uint64(62))) == 2       # the top x bit still splits the shapes (all 0 without the halving)
    _check_tree(nodes, idx, a, "f64", D)
