"""The guarantees of the two distance-pruned walks, as checks shared by the CPU and GPU tests.

closest_hit, triangle mode (include/bvh_b200.h, DESIGN.md 4.7): the result G differs from the reference's loop over Bvh::traverse
(W = oracle.closest_hit) only where W's Moeller-Trumbore distance lies more than 2^-16 in front of W's own box entry.  On every ray
with G != W:
  - G's distance, u and v are the reference's Moeller-Trumbore result for G, bit for bit;
  - d_W <= d_G;
  - the slab entry of W's own AABB is greater than fl(d_G * (1 + 2^-16));
  - in exact arithmetic W's intersection (if it has one) lies farther than d_G.

nearest_candidates (include/bvh_b200.h, DESIGN.md 4.6): every list contains every shape at the minimal exact distance, the shape
Bvh::nearest_to returns, and the shape a brute force over Aabb::min_distance_squared picks."""
import numpy as np

from oracle import oracle as O
from tests import dimref, exactref as E

MARGIN = {"f32": np.float32(1) + np.float32(2.0 ** -16), "f64": np.float64(1) + np.float64(2.0 ** -16)}


def check_closest(gs, gd, guv, ws, wd, tris, shapes, rays, prec):
    """Assert the triangle-mode contract; returns the number of rays where G != W."""
    tris = np.ascontiguousarray(tris).reshape(-1, 9)
    diff = np.flatnonzero(gs != ws)
    for r in diff:
        g, w = int(gs[r]), int(ws[r])
        ctx = (int(r), g, w, gd[r], wd[r])
        assert g != O.U32_MAX, ctx                              # a hit the reference finds is never lost outright
        t, u, v = O.ray_triangle(rays[r], tris[g], prec)
        assert (np.array([t, u, v]).tobytes() == np.array([gd[r], guv[r, 0], guv[r, 1]]).tobytes()), ctx
        assert wd[r] <= gd[r], ctx
        sl = O.ray_slice(rays[r], shapes[w], prec)
        entry = max(sl[0], type(gd[r])(0))
        assert entry > gd[r] * MARGIN[prec], ctx
        ex = E.ray_triangle(rays["origin"][r], rays["direction"][r], *tris[w].reshape(3, 3))
        assert ex is None or ex[0] > E.fr(gd[r]), ctx
    return len(diff)


def _ref_nearest(nodes, shapes, p, D, prec):
    """(the shape Bvh::nearest_to returns, the first shape of minimal Aabb::min_distance_squared) for point p."""
    if D == 3:
        s, _ = O.nearest_to(nodes, shapes, p[None], prec)
        d2 = O.shape_distances_squared(shapes, p, prec)
        return int(s[0]), int(np.argmin(d2))
    s, _ = dimref.Tree(nodes, shapes).nearest_bvh(list(p))
    d2 = [dimref.min_distance_sq(list(p), list(a), list(b)) for a, b in zip(shapes["min"], shapes["max"])]
    return int(s), int(np.argmin(d2))


def check_candidates(lists, nodes, shapes, pts, prec):
    """Assert the nearest_candidates contract for every point; lists[i] is point i's list.  Returns how many points had more
    than one shape at the minimal exact distance and how many had a reference nearest shape that is not an exact nearest."""
    D = pts.shape[1]
    ties = rounded = 0
    for i, p in enumerate(pts):
        lst = set(int(x) for x in lists[i])
        ex = [E.box_lower_d2(p, a, b) for a, b in zip(shapes["min"], shapes["max"])]
        m = min(ex)
        exact_min = {j for j, x in enumerate(ex) if x == m}
        walk, brute = _ref_nearest(nodes, shapes, p, D, prec)
        assert exact_min <= lst, (i, sorted(exact_min - lst))
        assert walk in lst and brute in lst, (i, walk, brute)
        ties += len(exact_min) > 1
        rounded += brute not in exact_min or walk not in exact_min
    return ties, rounded

