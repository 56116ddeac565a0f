"""Exact-arithmetic restatements of the distances the pruned walks compare (fractions.Fraction on the T-valued inputs).

The device's distance-pruned walks (triangle-mode closest_hit, nearest_candidates) compare two differently rounded computations of
one quantity.  What they guarantee is stated against the exact quantity, so the tests need it exactly:
- ray_triangle: the ray parameter of the exact ray-plane intersection, with exact barycentric inside / outside and the back-face
  rule (det > 0 is a front face);
- slab_entry: the exact entry distance of a ray into a box, from `direction` (not the rounded inv_direction);
- box_lower_d2 / box_far_d2 / point_triangle_d2: exact squared distances from a point to a box, to its farthest corner and to a
  triangle, in any dimension.
Fractions are slow: use them on the rays and points a test singles out, not on whole batches.  Non-finite inputs are the caller's
business (these functions raise on them)."""
from fractions import Fraction


def fr(x):
    """The exact value of a finite T scalar."""
    return Fraction(float(x))


def _v(a):
    return [fr(x) for x in a]


def _sub(a, b):
    return [x - y for x, y in zip(a, b)]


def _dot(a, b):
    return sum((x * y for x, y in zip(a, b)), Fraction(0))


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def ray_triangle(o, d, a, b, c):
    """(t, u, v) of the exact intersection of the line o + t d with the triangle's plane, or None where the exact Moeller-Trumbore
    test rejects it: det <= 0 (back face or ray parallel to the plane), or the point outside the closed triangle.  t may be <= 0
    (the plane lies behind the origin); the caller decides what a hit behind the origin means."""
    o, d, a, b, c = _v(o), _v(d), _v(a), _v(b), _v(c)
    ab, ac, ao = _sub(b, a), _sub(c, a), _sub(o, a)
    uvec = _cross(d, ac)
    det = _dot(ab, uvec)
    if det <= 0:
        return None
    u = _dot(ao, uvec) / det
    vvec = _cross(ao, ab)
    v = _dot(d, vvec) / det
    if u < 0 or v < 0 or u + v > 1:
        return None
    return _dot(ac, vvec) / det, u, v


def slab_entry(o, d, mn, mx):
    """(entry, exit) of the ray o + t d (t >= 0) through the closed box, entry clamped at 0; None if it misses.  A zero direction
    component passes its slab when the origin lies inside it."""
    lo, hi = Fraction(0), None
    for ok, dk, a, b in zip(_v(o), _v(d), _v(mn), _v(mx)):
        if dk == 0:
            if ok < a or ok > b:
                return None
            continue
        t1, t2 = (a - ok) / dk, (b - ok) / dk
        if t1 > t2:
            t1, t2 = t2, t1
        lo = max(lo, t1)
        hi = t2 if hi is None else min(hi, t2)
    if hi is not None and lo > hi:
        return None
    return lo, hi


def box_lower_d2(p, mn, mx):
    """Exact squared distance from p to the closed box (0 inside)."""
    s = Fraction(0)
    for x, a, b in zip(_v(p), _v(mn), _v(mx)):
        g = max(a - x, x - b, Fraction(0))
        s += g * g
    return s


def box_far_d2(p, mn, mx):
    """Exact squared distance from p to the box's farthest corner."""
    s = Fraction(0)
    for x, a, b in zip(_v(p), _v(mn), _v(mx)):
        g = max(abs(x - a), abs(x - b))
        s += g * g
    return s


def _seg_d2(p, a, b):
    ab, ap = _sub(b, a), _sub(p, a)
    den = _dot(ab, ab)
    s = Fraction(0) if den == 0 else min(max(_dot(ab, ap) / den, Fraction(0)), Fraction(1))
    q = [x + s * y for x, y in zip(a, ab)]
    dd = _sub(p, q)
    return _dot(dd, dd)


def point_triangle_d2(p, a, b, c):
    """Exact squared distance from p to the closed triangle abc in any dimension (Voronoi regions of Ericson's
    closest_point_triangle, evaluated exactly).  A zero-area triangle is the union of its edges."""
    p, a, b, c = _v(p), _v(a), _v(b), _v(c)
    ab, ac = _sub(b, a), _sub(c, a)
    g11, g12, g22 = _dot(ab, ab), _dot(ab, ac), _dot(ac, ac)
    if g11 * g22 - g12 * g12 == 0:
        return min(_seg_d2(p, a, b), _seg_d2(p, b, c), _seg_d2(p, a, c))
    ap, bp, cp = _sub(p, a), _sub(p, b), _sub(p, c)
    d1, d2 = _dot(ab, ap), _dot(ac, ap)
    d3, d4 = _dot(ab, bp), _dot(ac, bp)
    d5, d6 = _dot(ab, cp), _dot(ac, cp)
    vc, vb, va = d1 * d4 - d3 * d2, d5 * d2 - d1 * d6, d3 * d6 - d5 * d4
    if d1 <= 0 and d2 <= 0:
        q = a
    elif d3 >= 0 and d4 <= d3:
        q = b
    elif d6 >= 0 and d5 <= d6:
        q = c
    elif vc <= 0 and d1 >= 0 and d3 <= 0:
        w = d1 / (d1 - d3)
        q = [x + w * y for x, y in zip(a, ab)]
    elif vb <= 0 and d2 >= 0 and d6 <= 0:
        w = d2 / (d2 - d6)
        q = [x + w * y for x, y in zip(a, ac)]
    elif va <= 0 and d4 - d3 >= 0 and d5 - d6 >= 0:
        w = (d4 - d3) / ((d4 - d3) + (d5 - d6))
        q = [x + w * (z - x) for x, z in zip(b, c)]
    else:
        den = va + vb + vc
        v, w = vb / den, vc / den
        q = [x + v * y + w * z for x, y, z in zip(a, ab, ac)]
    dd = _sub(p, q)
    return _dot(dd, dd)
