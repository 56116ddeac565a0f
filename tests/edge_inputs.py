"""Seeded edge-case inputs for the parity tests (test infrastructure): overflow-scale, mixed-scale and subnormal scenes, and
finite unit rays whose slab arithmetic reaches those scales.

scenes.py's scene() / rays_for() are left as they are (existing tests depend on their exact outputs).  Those rays are built from
`targets - origins`; on an f32 scene at 1e30 the square of that difference overflows in Ray::new, so the direction becomes 0 and
every such ray is a point-in-box test.  The rays here are normalised in f64 without overflow before Ray::new sees them, so they
keep a finite unit direction at every scale.

Scale limits: every centroid extent stays finite (|coords| far below FLT_MAX / 2 resp. DBL_MAX / 2).  Where it overflows the
reference panics on a NaN bucket index, so such inputs are outside the contract."""
import zlib

import numpy as np

from oracle import oracle as O

SCENE_KINDS = ("huge", "mixed", "subnormal")
FAMILIES = ("random", "axis", "face", "inside", "tiny", "subdir")

HUGE = {"f32": 1e30, "f64": 1e160}            # squared extents overflow T (surface area = inf): "no split wins" nodes
SUBNORMAL = {"f32": 1e-39, "f64": 1e-309}     # coordinate scale below the smallest normal number of T
TINY_DIR = {"f32": 1e-30, "f64": 1e-160}      # a direction component whose inverse times an overflow-scale extent overflows T
SUB_DIR = {"f32": (3e-39, 1e-45), "f64": (1e-308, 5e-324)}   # subnormal direction components: finite inverse, infinite inverse


def _rng(*key) -> np.random.Generator:
    return np.random.default_rng(zlib.crc32("/".join(map(str, key)).encode()))


def edge_scene(kind: str, n: int, prec: str = "f32") -> np.ndarray:
    """huge: boxes at HUGE[prec] (every surface area overflows); mixed: half such boxes, half unit-scale clusters (no-split nodes at
    the top, ordinary subtrees below them); subnormal: every coordinate within +-SUBNORMAL[prec] (every node halves)."""
    rng = _rng("edge_scene", kind, n, prec)
    if kind == "huge":
        s = HUGE[prec]
        mn = rng.uniform(-s, s, (n, 3))
        mx = mn + rng.uniform(0, s / 10, (n, 3))
    elif kind == "mixed":
        s, h = HUGE[prec], n // 2
        big = rng.uniform(-s, s, (h, 3))
        centres = rng.uniform(-50, 50, (4, 3))
        small = centres[rng.integers(0, 4, n - h)] + rng.normal(0, 3, (n - h, 3))
        mn = np.concatenate([big, small])
        mx = mn + np.concatenate([rng.uniform(0, s / 10, (h, 3)), rng.uniform(0.05, 2.0, (n - h, 3))])
        perm = rng.permutation(n)
        mn, mx = mn[perm], mx[perm]
    elif kind == "subnormal":
        t = SUBNORMAL[prec]
        mn = rng.uniform(-t, t, (n, 3))
        mx = mn + rng.uniform(0, t / 2, (n, 3))
    else:
        raise KeyError(kind)
    return O.make_aabbs(mn, mx, prec)


def unit_directions(d) -> np.ndarray:
    """Unit vectors in f64 without overflow: divide by the largest |component| first, then by the norm (a plain norm of a 1e160
    vector overflows and gives zero directions).  Signs of zero components are kept."""
    d = np.asarray(d, dtype=np.float64).reshape(-1, 3)
    m = np.abs(d).max(axis=1, keepdims=True)
    assert np.all(m > 0), "zero direction"
    d = d / m
    return d / np.sqrt((d * d).sum(axis=1, keepdims=True))


def edge_rays(shapes: np.ndarray, family: str, n: int, prec: str = "f32", seed: int = 0) -> np.ndarray:
    """`n` rays of one family through `shapes`, built by Ray::new (O.ray_new) from a unit direction:
    random  - random origins around the scene, aimed at random points of the bounds or at box centres;
    axis    - axis-parallel from outside the scene towards a box centre; zero components are +0.0 for even rays, -0.0 for odd ones;
    face    - the rays of `axis` with the origin moved onto face planes (min or max) of a random box: 0 * +-inf = NaN (miss);
    inside  - origins inside boxes, random directions;
    tiny    - random directions with one component TINY_DIR[prec]: (b - o) * inv overflows to +-inf on overflow-scale scenes;
    subdir  - random directions with one subnormal component, alternately with a finite and an infinite inverse."""
    rng = _rng("edge_rays", family, n, prec, seed, len(shapes))
    mn, mx = shapes["min"].astype(np.float64), shapes["max"].astype(np.float64)
    lo, hi = mn.min(axis=0), mx.max(axis=0)
    pad = (hi - lo) * 0.1
    pick = rng.integers(0, len(shapes), n)
    centre = mn[pick] * 0.5 + mx[pick] * 0.5
    if family == "random":
        org = rng.uniform(lo - pad, hi + pad, (n, 3))
        tgt = np.where(rng.random((n, 1)) < 0.5, rng.uniform(lo, hi, (n, 3)), centre)
        dirs = unit_directions(tgt - org)
    elif family in ("axis", "face"):
        axis = rng.integers(0, 3, n)
        sign = rng.choice([-1.0, 1.0], n)
        dirs = np.zeros((n, 3))
        dirs[1::2] = -0.0
        dirs[np.arange(n), axis] = sign
        org = centre.copy()
        org[np.arange(n), axis] = np.where(sign > 0, lo[axis] - pad[axis], hi[axis] + pad[axis])
        if family == "face":
            corner = np.where(rng.random((n, 1)) < 0.5, mn[pick], mx[pick])
            off = np.arange(3)[None, :] != axis[:, None]
            org[off] = corner[off]
        dirs = unit_directions(dirs)
    elif family == "inside":
        org = mn[pick] + rng.random((n, 3)) * (mx[pick] - mn[pick])
        dirs = unit_directions(rng.normal(size=(n, 3)))
    elif family in ("tiny", "subdir"):
        org = rng.uniform(lo - pad, hi + pad, (n, 3))
        dirs = unit_directions(np.where(rng.random((n, 1)) < 0.5, centre - org, rng.normal(size=(n, 3))))
        k = rng.integers(0, 3, n)
        if family == "tiny":
            v = TINY_DIR[prec]
        else:
            v = np.where(np.arange(n) % 2 == 0, SUB_DIR[prec][0], SUB_DIR[prec][1])
        dirs[np.arange(n), k] = rng.choice([-1.0, 1.0], n) * v
    else:
        raise KeyError(family)
    return O.ray_new(org, dirs, prec)


def edge_ray_batch(shapes: np.ndarray, per_family: int, prec: str = "f32", seed: int = 0):
    """All families concatenated: (rays, family name of every ray)."""
    rays = np.concatenate([edge_rays(shapes, f, per_family, prec, seed) for f in FAMILIES])
    return rays, np.repeat(np.array(FAMILIES), per_family)


# ---- precondition counters: what a scene / a family actually contains ---------------------------------------------------------
def empty_child_boxes(nodes) -> int:
    """Inner nodes with an Aabb::empty() child box (what "no split wins" stores)."""
    inner = nodes["child_l"] != O.U32_MAX
    e = (nodes["l_aabb"]["min"][:, 0] > nodes["l_aabb"]["max"][:, 0]) | (nodes["r_aabb"]["min"][:, 0] > nodes["r_aabb"]["max"][:, 0])
    return int(np.sum(inner & e))


def ray_facts(rays: np.ndarray, shapes: np.ndarray) -> dict:
    """Counts of the arithmetic a batch of rays exercises against `shapes`, evaluated in the rays' own precision."""
    F = rays["origin"].dtype.type
    d, inv, o = rays["direction"], rays["inv_direction"], rays["origin"]
    tiny = np.finfo(F).tiny
    zero = d == 0
    sub = (d != 0) & (np.abs(d) < tiny)
    facts = {
        "nonzero_direction": int(np.sum(np.any(d != 0, axis=1))),
        "neg_zero": int(np.sum(zero & np.signbit(d))),
        "pos_zero": int(np.sum(zero & ~np.signbit(d))),
        "inv_neg_inf": int(np.sum(inv == -np.inf)),
        "inv_pos_inf": int(np.sum(inv == np.inf)),
        "subnormal_dir": int(np.sum(sub)),
        "subnormal_dir_finite_inv": int(np.sum(sub & np.isfinite(inv))),
        "subnormal_dir_inf_inv": int(np.sum(sub & np.isinf(inv))),
    }
    # slab products (b - o) * inv over every ray x box x axis, in F
    ovf = nan = subn = 0
    with np.errstate(all="ignore"):
        for b in (shapes["min"], shapes["max"]):
            for k in range(3):
                diff = (b[None, :, k] - o[:, k, None]).astype(F)
                prod = (diff * inv[:, k, None]).astype(F)
                ovf += int(np.sum(np.isinf(prod) & np.isfinite(diff) & np.isfinite(inv[:, k, None])))
                nan += int(np.sum(np.isnan(prod) & zero[:, k, None]))
                subn += int(np.sum((diff != 0) & (np.abs(diff) < tiny)))
    facts["overflowing_products"] = ovf
    facts["face_plane_nan"] = nan
    facts["subnormal_differences"] = subn
    return facts
