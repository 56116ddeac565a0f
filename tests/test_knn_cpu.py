"""CPU side of the k-nearest-shapes query: the restatement of knn_walk (tests/knnref.py) returns the brute-force rows bit for bit on
the oracle's trees (D = 3) and the reference build restated in any dimension (tests/pyref.py, D = 2 and 4), on every dimref scene
and every adversarial box family, with and without per-point limits.  This is the pruning argument of DESIGN.md section 4.16 checked
before any GPU run: the slacked lower bound, ties entered and empty boxes always entered lose nothing."""
import numpy as np
import pytest

from tests import adversarial as A, dimref, knnref as K
from tests.test_pruned_walks_cpu import tree_for

FT = {"f32": np.float32, "f64": np.float64}
KS = (1, 3, 16, 64)


def limits(mn, mx, pts, rng):
    """One limit per point: 0, -1, -0, NaN, +inf, a random radius, and radii whose square is some shape's key exactly (the
    boundary is included), in turn."""
    F = mn.dtype.type
    out = np.zeros(len(pts), dtype=F)
    for i, p in enumerate(pts):
        kind = i % 7
        if kind < 5:
            out[i] = [0.0, -1.0, -0.0, np.nan, np.inf][kind]
        elif kind == 5 or len(mn) == 0:
            out[i] = F(rng.uniform(0, 1) * float(np.max(np.abs(mx - mn))) if len(mn) else 1.0)
        else:
            d2 = K.keys(mn, mx, p)
            key = d2[rng.integers(0, len(d2))]
            r = F(np.sqrt(key))
            for c in (r, np.nextafter(r, F(np.inf)), np.nextafter(r, F(0))):
                with np.errstate(all="ignore"):
                    if c * c == key:
                        r = c
                        break
            out[i] = r
    return out


def odd_points(D, F):
    """Points with NaN and infinite coordinates: every key is then 0 or +inf on that axis, and the row is still the brute force."""
    p = np.zeros((4, D), dtype=F)
    p[0, 0] = np.nan
    p[1, -1] = np.inf
    p[2, 0] = -np.inf
    p[3, :] = np.nan
    return p


def check(nodes, mn, mx, pts, rng, ks=KS):
    walk = K.Walk(nodes, mn, mx)
    lim = limits(mn, mx, pts, rng)
    for k in ks:
        for md in (None, lim):
            ws, wd, _ = walk.rows(pts, k, md)
            bs, bd = K.brute(mn, mx, pts, k, md)
            assert np.array_equal(ws, bs), (k, md is None)
            assert wd.tobytes() == bd.tobytes(), (k, md is None)


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("D", [2, 3, 4])
@pytest.mark.parametrize("scene", dimref.SCENES)
def test_walk_equals_brute_force_on_every_scene(scene, D, prec):
    F = FT[prec]
    rng = np.random.default_rng(100 * dimref.SCENES.index(scene) + 10 * D + (prec == "f64"))
    mn, mx = dimref.scene(scene, 90, D, F, rng)
    nodes, _ = tree_for(mn, mx, prec)
    pts = np.concatenate([dimref.points(mn, mx, 10, F, rng), odd_points(D, F)])
    check(nodes, mn, mx, pts, rng)


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("D", [2, 3, 4])
@pytest.mark.parametrize("family", sorted(A.BOX_FAMILIES))
def test_walk_equals_brute_force_on_adversarial_boxes(family, D, prec):
    """large: the reference's rounded distance cancels (the concrete X / Y / p case in 3-D f32); ties: equal keys broken by index;
    mixed: subnormal extents; overflow: "no split wins" empty child boxes."""
    F = FT[prec]
    mn, mx, pts = A.BOX_FAMILIES[family](F, D)
    nodes, _ = tree_for(mn, mx, prec)
    check(nodes, mn, mx, pts[:24], np.random.default_rng(3))


def test_issue_case_k1_is_the_brute_force_minimum():
    """3-D f32: X is at rounded key 0.25 (exact distance^2 1) and the point box Y at 0.5; k = 1 returns X, the brute-force minimum
    of min_distance_squared, and the walk keeps it although its exact distance is the larger one."""
    mn = np.array([A.ISSUE_X[0], np.array(A.ISSUE_P) + [0.5, 0, 0.5]], dtype=np.float32)
    mx = np.array([A.ISSUE_X[1], np.array(A.ISSUE_P) + [0.5, 0, 0.5]], dtype=np.float32)
    p = np.array([A.ISSUE_P], dtype=np.float32)
    assert list(K.keys(mn, mx, p[0])) == [0.25, 0.5]
    nodes, _ = tree_for(mn, mx, "f32")
    s, d, _ = K.Walk(nodes, mn, mx).rows(p, 2)
    assert s.tolist() == [[0, 1]] and d.tolist() == [[0.5, np.float32(np.sqrt(np.float32(0.5)))]]


def test_pruning_skips_most_of_the_tree():
    """On a random 3-D scene the walk visits a small part of the tree for k = 8, and all of it with a NaN-free +inf limit only
    when k reaches n: pruning is real, not a full scan."""
    rng = np.random.default_rng(11)
    mn, mx = dimref.scene("random", 400, 3, np.float32, rng)
    nodes, _ = tree_for(mn, mx, "f32")
    pts = dimref.points(mn, mx, 16, np.float32, rng)
    _, _, visits = K.Walk(nodes, mn, mx).rows(pts, 8)
    assert np.mean(visits) < len(nodes) / 4, np.mean(visits)


def test_empty_and_single_shape_trees():
    F = np.float32
    mn = np.array([[0.0, 0, 0]], dtype=F)
    mx = np.array([[1.0, 1, 1]], dtype=F)
    nodes, _ = tree_for(mn, mx, "f32")
    pts = np.array([[2.0, 0.5, 0.5], [0.5, 0.5, 0.5]], dtype=F)
    s, d, _ = K.Walk(nodes, mn, mx).rows(pts, 3)
    assert s.tolist() == [[0, K.U32_MAX, K.U32_MAX]] * 2
    assert d.tolist() == [[1.0, np.inf, np.inf], [0.0, np.inf, np.inf]]
    bs, bd = K.brute(mn[:0], mx[:0], pts, 2)
    assert (bs == K.U32_MAX).all() and np.isinf(bd).all()
