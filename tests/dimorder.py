"""tests/dimorder.py -- restatement of the reference's distance-ordered walks over rays, generic in the dimension D, with
numpy.float32 / numpy.float64 scalars (every operation rounds in T, in the reference's order, no FMA possible).  TEST INFRASTRUCTURE:
checked against the C++ oracle at D = 3 (tests/test_dim_ordered_cpu.py) and then used as the oracle for D = 2 and D = 4
(tests/test_gpu_dim_ordered.py).  Builds on the node / shape unpacking of tests/dimref.py.

    slice            Ray::intersection_slice_for_aabb (src/ray/ray_impl.rs:118-145), axes folded left to right with nalgebra's
                     inf / sup (`if a <= b {a} else {b}` / `a >= b`), as the oracle's ray_slice_for_aabb
    Tree.ordered     Bvh::nearest_traverse_iterator / farthest_traverse_iterator made perfectly sorted: the Bvh::traverse set, stably
                     sorted by the slice of the child box the tree stores for each leaf (entry ascending / exit descending)
    Tree.closest     the shape whose own AABB the ray enters first among Bvh::traverse's candidates, key (entry, DFS order)
    rays             ray batches for a scene of dimref.scene

Rays: (origin, inv_direction) pairs of T sequences."""
import numpy as np

from tests import dimref
from tests.dimref import U32_MAX


def slice(ray, mn, mx):
    """(entry, exit) or None.  Any NaN in (b - o) * inv rejects; entry = max(tmin, 0)."""
    o, inv = ray
    F = type(mn[0])
    with np.errstate(all="ignore"):
        lr = [((mn[k] - o[k]) * inv[k], (mx[k] - o[k]) * inv[k]) for k in range(len(o))]
    if any(np.isnan(l) or np.isnan(r) for l, r in lr):
        return None
    inf_ = lambda a, b: a if a <= b else b                    # nalgebra inf / sup
    sup_ = lambda a, b: a if a >= b else b
    tmin, tmax = inf_(*lr[0]), sup_(*lr[0])
    for l, r in lr[1:]:
        tmin, tmax = sup_(tmin, inf_(l, r)), inf_(tmax, sup_(l, r))
    lo = tmin if tmin > F(0) else F(0)                        # fast_max(tmin, 0)
    return None if lo > tmax else (lo, tmax)


class Tree(dimref.Tree):
    """dimref.Tree (nodes and shapes of any D) with the ray walks."""

    def _candidates(self, ray):
        """Bvh::traverse with a ray, DFS order: [(shape, slice of the box the walk tested last)].  A root leaf tests the shape's own
        box (bvh_node.rs:314); every other leaf is reported with the child box its parent stores."""
        N, out = self.nodes, []
        if not N:
            return out
        if N[0][0] == U32_MAX:
            s = slice(ray, *self.shapes[N[0][2]])
            return [(N[0][2], s)] if s is not None else []

        def rec_(i, box_slice):
            cl, cr, shape, lmn, lmx, rmn, rmx = N[i]
            if cl == U32_MAX:
                out.append((shape, box_slice))
                return
            for child, mn, mx in ((cl, lmn, lmx), (cr, rmn, rmx)):
                s = slice(ray, mn, mx)
                if s is not None:
                    rec_(child, s)

        rec_(0, None)
        return out

    def ordered(self, ray, ascending=True):
        """[(shape, distance)]: entry distance ascending or exit distance descending, stable (ties in DFS order)."""
        c = self._candidates(ray)
        key = (lambda e: e[1][0]) if ascending else (lambda e: -e[1][1])
        return [(s, sl[0] if ascending else sl[1]) for s, sl in sorted(c, key=key)]

    def closest(self, ray):
        """(shape, entry distance) of the first strict minimum over the candidates whose own box the ray enters, (U32_MAX, None)."""
        best = (U32_MAX, None)
        for s, _ in self._candidates(ray):
            sl = slice(ray, *self.shapes[s])
            if sl is not None and (best[1] is None or sl[0] < best[1]):
                best = (s, sl[0])
        return best


def rays(mn, mx, m, F, rng):
    """(origins, inv_directions), (m, D) each, with Ray::new's reciprocal of a normalised direction: random rays through the scene,
    axis-aligned rays that start on box faces and corners (the z / w planes of the other axes give 0 * inf = NaN: the NaN rule; the
    moving axis can exit at +0 or -0), and rays with -0.0 direction or origin components (inv = -inf)."""
    n, D = mn.shape
    lo, hi = (mn.min(axis=0).astype(np.float64), mx.max(axis=0).astype(np.float64)) if n else (np.full(D, -1.0), np.full(D, 1.0))
    span = np.maximum(hi - lo, 1.0)
    o = lo - 0.2 * span + rng.uniform(0, 1.4, (m, D)) * span
    d = rng.normal(size=(m, D))
    if n:
        aim = rng.random(m) < 0.7                             # most random rays are aimed at a shape's centre
        tgt = rng.integers(0, n, m)
        c = 0.5 * mn[tgt].astype(np.float64) + 0.5 * mx[tgt].astype(np.float64)
        d[aim] = c[aim] - o[aim] + (rng.random((int(aim.sum()), 1)) < 0.5) * 1e-3 * span * d[aim]   # half of them exactly
        aligned = rng.random(m) < 0.35
        pick = rng.integers(0, n, m)
        face = rng.random((m, D)) < 0.5
        o[aligned] = np.where(face[aligned], mn[pick[aligned]], mx[pick[aligned]])
        axis = rng.integers(0, D, m)
        d[aligned] = 0.0
        d[aligned, axis[aligned]] = np.where(rng.random(int(aligned.sum())) < 0.5, 1.0, -1.0)
    z = rng.random(m) < 0.1                                   # -0.0 components: direction (inv = -inf) and origin
    d[z, 0] = -0.0
    o[z, -1] = -0.0
    o, d = o.astype(F), d.astype(F)
    with np.errstate(all="ignore"):
        nrm = np.sqrt(np.sum(d.astype(F) * d.astype(F), axis=1, dtype=F)).astype(F)
        d = (d / nrm[:, None]).astype(F)
        inv = (F(1) / d).astype(F)
    return o, d, inv
