"""The exact restatement of the triangle-pair predicate (tests/tritri.py) on cases with known answers, against a second formulation
(separating axes in fractions.Fraction) on random small-grid triangles, and its vectorised filter against the integer path.  No GPU."""
import itertools
from fractions import Fraction

import numpy as np
import pytest

from tests import tritri as T

FT = {"f32": np.float32, "f64": np.float64}
P0 = [(0, 0, 0), (2, 0, 0), (0, 2, 0)]             # the reference triangle in z = 0, legs along x and y, hypotenuse x + y = 2


def _moved(q, v, k, F, up):
    """q with coordinate k of vertex v moved one ulp of F up or down."""
    q = np.array(q, dtype=F)
    q[v, k] = np.nextafter(q[v, k], F(np.inf) if up else F(-np.inf))
    return q


# (P, Q, meets, (vertex, axis) to move, meets after moving it up, meets after moving it down); None: nothing to move
HAND = {
    "separated": (P0, [(0, 0, 1), (2, 0, 1), (0, 2, 1)], False, None, None, None),
    "crossing": (P0, [(0.25, 0.25, -1), (0.25, 0.25, 1), (1, 0.25, 0)], True, None, None, None),
    "vertex_on_face": (P0, [(0.5, 0.5, 0), (1, 0.5, 1), (0.5, 1, 1)], True, (0, 2), False, True),
    "edge_on_edge": (P0, [(1, 0, 1), (1, 0, -1), (1, -1, 0)], True, (0, 1), True, False),
    "edge_through_vertex": (P0, [(2, 0, 1), (2, 0, -1), (3, 0.5, 0)], True, (0, 0), False, True),
    "parallel_planes": ([(0, 0, 1), (2, 0, 1), (0, 2, 1)], [(0.5, 0.5, 1), (1.5, 0.5, 1), (0.5, 1.5, 1)], True, None, None, None),
    "coplanar_overlap": (P0, [(0.5, 0.5, 0), (3, 0.5, 0), (0.5, 3, 0)], True, None, None, None),
    "coplanar_vertex_touch": (P0, [(1, 1, 0), (2, 2, 0), (1, 3, 0)], True, (0, 0), False, True),
    "coplanar_shared_edge_part": (P0, [(0.5, 1.5, 0), (1.5, 0.5, 0), (2, 2, 0)], True, (0, 0), True, True),
    "coplanar_inside": (P0, [(0.25, 0.25, 0), (0.5, 0.25, 0), (0.25, 0.5, 0)], True, None, None, None),
    "coplanar_disjoint": (P0, [(3, 3, 0), (4, 3, 0), (3, 4, 0)], False, None, None, None),
    "coplanar_star": ([(0, 0, 0), (4, 0, 0), (2, 3, 0)], [(0, 2, 0), (4, 2, 0), (2, -1, 0)], True, None, None, None),
}


@pytest.mark.parametrize("prec", FT)
@pytest.mark.parametrize("case", HAND)
def test_hand_cases(case, prec):
    F = FT[prec]
    p, q, want, move, up, down = HAND[case]
    p, q = np.array(p, dtype=F) + 1, np.array(q, dtype=F) + 1              # off zero, whose f64 neighbours are out of range
    for a, b in ((p, q), (q, p), (p[[1, 2, 0]], q[[2, 1, 0]])):         # symmetric, and independent of the vertex order
        assert T.meets(a, b, F) == want
    if case == "parallel_planes":                                         # the planes z = 1 and z = 1 + ulp: apart
        assert not T.meets(p, _lift(q, F), F) and not T.meets(_lift(q, F), p, F)
    elif move:
        assert T.meets(p, _moved(q, *move, F, True), F) == up
        assert T.meets(p, _moved(q, *move, F, False), F) == down


def _lift(q, F):
    """q with every z moved one ulp up."""
    q = np.array(q, dtype=F)
    q[:, 2] = np.nextafter(q[:, 2], F(np.inf))
    return q


@pytest.mark.parametrize("prec", FT)
def test_excluded_triangles_meet_nothing(prec):
    F = FT[prec]
    crossing = np.array([(0.25, 0.25, -1), (0.25, 0.25, 1), (1, 0.25, 0)], dtype=F)
    bad = {
        "collinear": [(0, 0, 0), (1, 1, 1), (2, 2, 2)],
        "repeated": [(0, 0, 0), (1, 0, 0), (1, 0, 0)],
        "point": [(0.5, 0.25, 0)] * 3,
        "nan": [(0, 0, 0), (2, 0, 0), (0, np.nan, 0)],
        "inf": [(0, 0, 0), (np.inf, 0, 0), (0, 2, 0)],
        "collinear_ulp": [(0, 0, 0), (1, 1, 0), (3, 3, 0)],
    }
    for name, t in bad.items():
        t = np.array(t, dtype=F)
        assert T.classify(t, F)[0] == T.EXCLUDED, name
        for other in (np.array(P0, dtype=F), crossing, t):
            assert not T.meets(t, other, F) and not T.meets(other, t, F), name
            assert not T.meets(t, other, F, skip_shared=False)
    # one ulp off the line is a triangle again
    t = np.array([(0, 0, 0), (1, 1, 0), (3, 3, 0)], dtype=F)
    t[2, 1] = np.nextafter(t[2, 1], F(4))
    assert T.classify(t, F)[0] == T.OK


@pytest.mark.parametrize("prec", FT)
def test_shared_vertex_rule_with_signed_zero(prec):
    F = FT[prec]
    p = np.array([(0, 0, 0), (1, 0, 0), (0, 1, 0)], dtype=F)
    q = np.array([(-0.0, -0.0, 0), (-1, 0, 1), (0, -1, 1)], dtype=F)     # -0 == +0: the vertex at the origin is shared
    assert T.shares_vertex(p, q)
    assert T.meets(p, q, F, skip_shared=False) and not T.meets(p, q, F, skip_shared=True)
    r = q.copy()
    r[0, 0] = -np.finfo(F).smallest_subnormal if F == np.float32 else -2.0 ** -300   # not shared, and then apart
    assert not T.shares_vertex(p, r)
    assert not T.meets(p, r, F, skip_shared=False) and not T.meets(p, r, F, skip_shared=True)
    # a fold-over through a shared vertex is a contact without skip_shared and is dropped with it
    fold = np.array([(0, 0, 0), (1, 0.5, 0.25), (1, 0.5, -0.25)], dtype=F)
    assert T.meets(p, fold, F) is True and T.meets(p, fold, F, skip_shared=True) is False


def test_f64_range_rule():
    F = np.float64
    far = np.array([(10, 10, 10), (11, 10, 10), (10, 11, 10)], dtype=F)
    for x in (2.0 ** -301, 2.0 ** 301, -(2.0 ** 400), 5e-324):
        t = far.copy()
        t[1, 2] = x
        assert T.classify(t, F)[0] == T.UNCHECKED
        assert T.meets(np.array(P0, dtype=F), t, F) and T.meets(t, np.array(P0, dtype=F), F, skip_shared=True)
        deg = np.array([(x, 0, 0), (x, 0, 0), (x, 0, 0)], dtype=F)      # a point, but unchecked: never excluded as degenerate
        assert T.meets(deg, np.array(P0, dtype=F), F)
        nan = deg.copy()
        nan[0, 1] = np.nan                                                # non-finite stays excluded
        assert not T.meets(nan, t, F)
    for x in (2.0 ** -300, 2.0 ** 300, 0.0, -0.0):                        # the range's ends and zero are decided exactly
        t = far.copy()
        t[1, 2] = x
        assert T.classify(t, F)[0] == T.OK
    # f32 has no range rule: its smallest subnormal and largest value are decided
    t = np.array([(np.finfo(np.float32).smallest_subnormal, 0, 0), (np.finfo(np.float32).max, 0, 0), (0, 1, 0)], dtype=np.float32)
    assert T.classify(t, np.float32)[0] == T.OK


# ---- the second formulation: separating axes in fractions.Fraction ----
def _sub(a, b):
    return tuple(x - y for x, y in zip(a, b))


def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def _dot(a, b):
    return sum(x * y for x, y in zip(a, b))


def sat_meets(p, q):
    """Closed non-degenerate triangles meet unless an axis separates their projections strictly: the two normals, the nine edge
    crosses and, when the triangles are coplanar, the in-plane normals of the six edges."""
    p = [tuple(Fraction(x) for x in v) for v in p]
    q = [tuple(Fraction(x) for x in v) for v in q]
    ep = [_sub(p[(k + 1) % 3], p[k]) for k in range(3)]
    eq = [_sub(q[(k + 1) % 3], q[k]) for k in range(3)]
    n_p, n_q = _cross(ep[0], ep[1]), _cross(eq[0], eq[1])
    axes = [n_p, n_q] + [_cross(a, b) for a in ep for b in eq]
    coplanar = _cross(n_p, n_q) == (0, 0, 0) and _dot(n_p, _sub(q[0], p[0])) == 0
    if coplanar:
        axes += [_cross(n_p, e) for e in ep] + [_cross(n_q, e) for e in eq]
    for ax in axes:
        if ax == (0, 0, 0):
            continue
        a = [_dot(ax, v) for v in p]
        b = [_dot(ax, v) for v in q]
        if max(a) < min(b) or max(b) < min(a):
            return False
    return True


def _grid_pairs(rng, m, grid):
    """m pairs on a grid of half-integers; every fourth pair flattened into one plane z = x + 1, where pairs are coplanar."""
    pts = rng.integers(0, grid, size=(m, 2, 3, 3)).astype(np.float64) / 2
    pts[::4, :, :, 2] = pts[::4, :, :, 0] + 1
    return pts


def test_agrees_with_separating_axes_on_small_grids():
    rng = np.random.default_rng(11)
    n = checked = touching = coplanar = 0
    for grid in (3, 4, 5):
        for p, q in _grid_pairs(rng, 5000, grid):
            ip = [tuple(T.to_int(x, np.float64) for x in v) for v in p]
            iq = [tuple(T.to_int(x, np.float64) for x in v) for v in q]
            if not T.projection(ip)[2] or not T.projection(iq)[2]:
                continue
            n += 1
            want = sat_meets(p, q)
            assert T.tri_tri(ip, iq) == want, (p.tolist(), q.tolist())
            checked += 1
            if want and (all(T.orient3(*ip, v) >= 0 for v in iq) or all(T.orient3(*ip, v) <= 0 for v in iq)):
                touching += 1
            coplanar += all(T.orient3(*ip, v) == 0 for v in iq)
    assert checked >= 10_000 and coplanar >= 200 and touching >= 1000


@pytest.mark.parametrize("prec", FT)
def test_filter_and_model_agree_with_the_integer_path(prec):
    F = FT[prec]
    rng = np.random.default_rng(5)
    # near-coplanar and near-touching pairs: a grid plus a few ulps of noise, and some exact grid pairs
    base = rng.integers(0, 4, size=(3000, 2, 3, 3)).astype(F)
    noise = rng.integers(-2, 3, size=base.shape)
    tri = base.copy()
    for s in (1, -1):
        sel = noise * s > 0
        tri[sel] = np.nextafter(tri[sel], F(s * np.inf))
    tri[:1000] = base[:1000]
    a, b = tri[:, 0], tri[:, 1]
    model = T.Model(a, F, b)
    idx = np.arange(len(a))
    for skip in (False, True):
        got = model.keep(idx, idx, skip)
        want = np.array([T.meets(a[k], b[k], F, skip) for k in idx])
        assert np.array_equal(got, want)
    # the filter's decided signs are the exact ones
    P, Q = a.astype(np.float64), b.astype(np.float64)
    s = T.orient3_filter(P[:, 0], P[:, 1], P[:, 2], Q[:, 0])
    for k in np.nonzero(s)[0][:2000]:
        ip = [tuple(T.to_int(x, F) for x in v) for v in a[k]]
        assert s[k] == T.orient3(*ip, tuple(T.to_int(x, F) for x in b[k][0]))


def test_csr_model_is_the_filtered_overlap_rows():
    F = np.float64
    rng = np.random.default_rng(3)
    tris = rng.integers(0, 6, size=(300, 3, 3)).astype(F) / 2
    mn, mx = T.tri_boxes(tris, F)
    leaf = rng.permutation(len(tris)) + 10
    for skip in (False, True):
        off, hits = T.self_rows(tris, mn, mx, leaf, F, skip)
        from tests import overlapref
        o0, h0 = overlapref.rows(mn, mx, leaf)
        got = {(int(s), int(t)) for s, t in overlapref.pairs(off, hits)}
        want = {(int(s), int(t)) for s, t in overlapref.pairs(o0, h0) if T.meets(tris[s], tris[t], F, skip)}
        assert got == want and len(hits) == len(got)
        assert np.all(np.diff(off.astype(np.int64)) >= 0)
    # between trees: the same filter of the cross rows
    other = tris[::-1] + 0.5
    bmn, bmx = T.tri_boxes(other, F)
    off, hits = T.cross_tri_rows(tris, mn, mx, other, bmn, bmx, leaf, F)
    got = {(int(s), int(t)) for s, t in overlapref.pairs(off, hits)}
    want = {(s, t) for s, t in itertools.product(range(len(tris)), range(len(other)))
            if np.all(~((mx[s] < bmn[t]) | (bmx[t] < mn[s]))) and T.meets(tris[s], other[t], F)}
    assert got == want
