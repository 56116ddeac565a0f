"""Pins the polygon model of tests/polygons.py on its own (no GPU): hand cases with known answers and one-ulp moves, the vectorised
filter against the exact integer restatement, an independent cell count on integer grids, the f64 range, the segment key, and the
boundedness of the key against the walk's slacked box bound on adversarial segments."""
import numpy as np
import pytest

from tests import polygons as P

PRECS = [np.float32, np.float64]


def _cls(segs, pts, F, rule=P.EVEN_ODD):
    segs = np.asarray(segs, dtype=F).reshape(-1, 4)
    pts = np.asarray(pts, dtype=F).reshape(-1, 2)
    fast = P.classes(segs, pts, F, rule)
    exact = P.contains_exact(segs, pts, F, rule)
    assert np.array_equal(fast[0], exact[0]) and np.array_equal(fast[1], exact[1])
    return fast


def _square(x0, y0, x1, y1, ccw=True):
    v = np.array([[x0, y0], [x1, y0], [x1, y1], [x0, y1]], dtype=np.float64)
    return P.loop(v if ccw else v[::-1])


def _ulps(x, F):
    x = F(x)
    return [np.nextafter(x, F(-np.inf)), x, np.nextafter(x, F(np.inf))]


@pytest.mark.parametrize("F", PRECS)
def test_unit_squares_ccw_and_cw(F):
    pts = [[0.5, 0.5], [1.5, 0.5], [-0.5, 0.5], [0.5, 1.5]]
    cls, w = _cls(_square(0, 0, 1, 1), pts, F)
    assert list(w) == [1, 0, 0, 0] and list(cls) == [1, 0, 0, 0]
    cls, w = _cls(_square(0, 0, 1, 1, ccw=False), pts, F, P.NONZERO)
    assert list(w) == [-1, 0, 0, 0] and list(cls) == [1, 0, 0, 0]


@pytest.mark.parametrize("F", PRECS)
def test_square_with_hole(F):
    segs = np.vstack([_square(0, 0, 4, 4), _square(1, 1, 3, 3, ccw=False)])
    cls, w = _cls(segs, [[0.5, 0.5], [2, 2], [3.5, 2], [5, 2]], F, P.NONZERO)
    assert list(w) == [1, 0, 1, 0] and list(cls) == [1, 0, 1, 0]


@pytest.mark.parametrize("F", PRECS)
def test_pentagram_centre_winds_twice(F):
    t = np.pi / 2 + np.arange(5) * 4 * np.pi / 5
    segs = P.loop(np.stack([np.cos(t), np.sin(t)], axis=1))
    cls_eo, w = _cls(segs, [[0.0, 0.0]], F, P.EVEN_ODD)
    cls_nz, _ = _cls(segs, [[0.0, 0.0]], F, P.NONZERO)
    assert w[0] == 2 and cls_eo[0] == P.OUTSIDE and cls_nz[0] == P.INSIDE


@pytest.mark.parametrize("F", PRECS)
def test_vertices_edges_and_horizontal_rows(F):
    sq = _square(0, 0, 1, 1)
    for p in ([0, 0], [1, 1], [0, 1], [0.5, 0], [0.5, 1], [1, 0.25], [0, 0.75]):
        cls, _ = _cls(sq, [p], F)
        assert cls[0] == P.BOUNDARY, p
        # one ulp each way on each coordinate: never a wrong inside / outside, boundary only where still on the edge
        for ax in (0, 1):
            for v in _ulps(p[ax], F):
                q = list(map(F, p)); q[ax] = v
                c, _ = _cls(sq, [q], F)
                inside = 0 < q[0] < 1 and 0 < q[1] < 1
                on = (0 <= q[0] <= 1 and 0 <= q[1] <= 1) and not inside
                want = P.BOUNDARY if on else P.INSIDE if inside else P.OUTSIDE
                if not (P.in_range(q[0], F) and P.in_range(q[1], F)):
                    want = P.UNDECIDED                                   # f64: one ulp off zero is subnormal
                assert c[0] == want, q
    # a point on the row of a horizontal edge, outside it
    cls, w = _cls(sq, [[-1, 0], [-1, 1], [2, 0]], F)
    assert list(cls) == [0, 0, 0] and list(w) == [0, 0, 0]


@pytest.mark.parametrize("F", PRECS)
def test_collinear_vertices_and_cancelling_edges(F):
    # collinear consecutive vertices along the bottom edge
    v = np.array([[0, 0], [0.25, 0], [0.5, 0], [1, 0], [1, 1], [0, 1]], dtype=np.float64)
    cls, w = _cls(P.loop(v), [[0.5, 0.5], [0.25, 0], [0.5, -0.1]], F)
    assert list(cls) == [1, 2, 0]
    # two unit squares sharing an edge, traversed both ways: the shared edges cancel inside, remain boundary on them
    segs = np.vstack([_square(0, 0, 1, 1), _square(1, 0, 2, 1)])
    cls, w = _cls(segs, [[0.5, 0.5], [1.5, 0.5], [1, 0.5]], F, P.NONZERO)
    assert list(w[:2]) == [1, 1] and cls[2] == P.BOUNDARY


@pytest.mark.parametrize("F", PRECS)
def test_excluded_segments(F):
    sq = _square(0, 0, 1, 1)
    extra = np.array([[0.5, 0.5, 0.5, 0.5], [np.nan, 0, 1, 1], [0, 0.5, np.inf, 0.5]])
    cls, w = _cls(np.vstack([sq, extra]), [[0.5, 0.5], [0.25, 0.5]], F)
    assert list(cls) == [1, 1] and list(w) == [1, 1]
    cls, w = _cls(sq, [[np.nan, 0.5], [0.5, np.inf]], F)
    assert list(cls) == [0, 0] and list(w) == [0, 0]


def test_f64_range():
    F = np.float64
    lo, hi = 2.0 ** -300, 2.0 ** 300
    s = hi / 2
    sq = _square(-s, -s, s, s)
    for x, want in ((np.nextafter(lo, 0), P.UNDECIDED), (lo, P.INSIDE), (hi * 0.75, P.OUTSIDE), (np.nextafter(hi, np.inf), P.UNDECIDED)):
        cls, w = _cls(sq, [[x, 0.0]], F)
        assert cls[0] == want, x
        if want == P.UNDECIDED:
            assert w[0] == 0
    # a relevant segment with an out-of-range coordinate makes the point undecided unless it is boundary
    big = np.array([[1.0, -1.0, 2.0 ** 301, 1.0]])
    cls, _ = _cls(np.vstack([_square(0, 0, 1, 1), big]), [[0.5, 0.5], [1.0, 0.5], [0.5, 5.0]], F)
    assert list(cls) == [P.UNDECIDED, P.BOUNDARY, P.OUTSIDE]
    tiny = np.array([[2.0 ** -301, -1.0, 0.5, 1.0]])
    cls, _ = _cls(np.vstack([_square(0, 0, 1, 1), tiny]), [[0.25, 0.0]], F)
    assert cls[0] == P.BOUNDARY


@pytest.mark.parametrize("F", PRECS)
def test_rectilinear_grid_polygons_against_cell_count(F):
    """Random unions of unit cells traced as loops of cell edges (each cell a CCW square, shared edges cancel): the winding at every
    cell centre is the number of covering cells; points on grid lines are boundary when a covering cell touches them."""
    rng = np.random.default_rng(1)
    cover = rng.integers(0, 3, size=(7, 6))
    segs = [_square(x, y, x + 1, y + 1) for x in range(7) for y in range(6) for _ in range(cover[x, y])]
    segs = np.vstack(segs)
    cx, cy = np.meshgrid(np.arange(7) + 0.5, np.arange(6) + 0.5, indexing="ij")
    pts = np.stack([cx.ravel(), cy.ravel()], axis=1)
    cls, w = _cls(segs, pts, F, P.NONZERO)
    assert np.array_equal(w, cover.ravel())
    assert np.array_equal(cls, (cover.ravel() > 0).astype(np.uint8))


@pytest.mark.parametrize("F", PRECS)
def test_vectorised_filter_agrees_with_the_integer_rule_on_snapped_scenes(F):
    rng = np.random.default_rng(7)
    v = rng.integers(-4, 5, size=(60, 2)).astype(np.float64) / 4
    segs = P.loop(v)
    pts = rng.integers(-5, 6, size=(300, 2)).astype(np.float64) / 4
    pts[::7] += rng.uniform(-1e-7, 1e-7, size=pts[::7].shape)
    for rule in (P.EVEN_ODD, P.NONZERO):
        _cls(segs, pts, F, rule)


def test_koch_and_map_scenes():
    k = P.koch(3)
    assert len(k) == 3 * 4 ** 3
    cls, w = P.classes(k, np.array([[0.5, 0.3], [0.5, -0.5], [5, 5]]), np.float64, P.EVEN_ODD)
    assert list(w) == [1, 0, 0]
    m = P.star_map(4, 5)
    assert len(m) == 4 * 20
    cls, w = P.classes(m, np.array([[0.0, 0.0], [1.0, 0.0], [10.0, 10.0]]), np.float64, P.NONZERO)
    assert list(w) == [0, 1, 0]


@pytest.mark.parametrize("F", PRECS)
def test_segment_key(F):
    segs = np.array([[0, 0, 2, 0], [0, 0, 0, 0], [1, 1, 1, 1], [0, 0, np.nan, 1]], dtype=F)
    key, q = P.keys_and_closest(np.array([1, 1], dtype=F), segs)
    assert key[0] == 1 and list(q[0]) == [1, 0]
    assert key[1] == 2 and list(q[1]) == [0, 0]
    assert key[2] == 0
    assert np.isnan(key[3])
    # the endpoint branches return the end points themselves
    key, q = P.keys_and_closest(np.array([5, 3], dtype=F), segs[:1])
    assert list(q[0]) == [2, 0] and key[0] == F(9) + F(9)


def _adversarial_segments(F, rng):
    m = 400
    fam = []
    a = rng.uniform(-1, 1, (m, 2))
    fam.append(np.hstack([a, a + rng.uniform(-1, 1, (m, 2)) * 1e-6]))                  # near-degenerate
    fam.append(np.hstack([a * 1e3, a * 1e3 + rng.uniform(-1e-3, 1e-3, (m, 2))]))      # long and thin (far from the origin)
    b = rng.uniform(-1, 1, (m, 2)) * 10.0 ** rng.integers(-6, 7, (m, 1))
    fam.append(np.hstack([b, b * rng.uniform(-3, 3, (m, 1))]))                        # mixed scale
    big = float(np.finfo(F).max) / 4
    fam.append(np.hstack([a * big, -a * big]))                                        # overflow scale (ex may overflow)
    tiny = float(np.finfo(F).smallest_subnormal) * 64
    fam.append(np.hstack([a * tiny, rng.uniform(-1, 1, (m, 2)) * tiny]))             # subnormal
    return [f.astype(F) for f in fam]


@pytest.mark.parametrize("F", PRECS)
def test_finite_segments_inside_their_box_are_bounded(F):
    rng = np.random.default_rng(3)
    for segs in _adversarial_segments(F, rng):
        mn, mx = P.seg_boxes(segs)
        scale = float(np.nanmax(np.abs(segs)))
        for p in rng.uniform(-1.5, 1.5, (24, 2)) * scale:
            p = p.astype(F)
            assert P.bounded(p, segs, mn, mx).all()
            key, q = P.keys_and_closest(p, segs)
            fin = np.isfinite(q).all(1)
            # the closest point lies in the box, up to a few ulps (inside the bound's 16-eps slack)
            eps = float(np.finfo(F).eps)
            m = np.maximum(np.abs(mn), np.abs(mx)).astype(np.float64)
            slack = 4 * eps * m + 4 * float(np.finfo(F).smallest_subnormal)
            assert ((q[fin] >= mn[fin] - slack[fin]) & (q[fin] <= mx[fin] + slack[fin])).all()
