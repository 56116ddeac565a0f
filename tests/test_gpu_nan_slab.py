"""GPU test of the f32 slab test's NaN rule (a NaN product means a miss) where exactly one of the six products is NaN: a ray whose
origin lies on a box plane and whose direction has a zero of either sign on that axis computes (b - o) * inv = 0 * ±inf.  The f32
slab test folds with NaN-propagating min / max instead of testing the products for NaN (DESIGN §2), so the hit sets and the visit
counter are checked against the oracle, the original formulation, not against another device kernel: walk_count_kernel,
walk_persistent_kernel and walk_top_kernel (the whole top in shared memory, and a 64-entry top whose fringe subtrees are walked
in the global records), BVH and FLAT semantics, full and origin + direction ray layouts.
Run on an H100:  python -m pytest tests -m gpu"""
import numpy as np
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu
F = np.float32
SUB = F(1e-40)                                                       # subnormal in f32
BIG = F(3e38)                                                        # BIG + BIG overflows to inf in f32


def nan_scene(seed=0):
    """Boxes on an integer lattice (some shrunk to a half-integer max plane), subnormal boxes around the origin and boxes with
    one overflow-scale coordinate.  (Infinite coordinates themselves are not buildable: the reference's bucket index of an
    infinite centroid is NaN.)"""
    rng = np.random.default_rng(seed)
    g = np.stack(np.meshgrid(np.arange(14), np.arange(14), np.arange(14), indexing="ij"), -1).reshape(-1, 3).astype(F)
    mn, mx = g.copy(), g + F(1)
    half = rng.random(g.shape) < 0.3
    mx[half] = g[half] + F(0.5)
    sub_mn = rng.choice(np.array([-SUB, -SUB / 4, F(0), SUB / 8], dtype=F), size=(48, 3))
    sub_mx = sub_mn + rng.choice(np.array([SUB / 8, SUB / 2, SUB], dtype=F), size=(48, 3))
    inf_mn = rng.uniform(0, 14, size=(12, 3)).astype(F).round()
    inf_mx = inf_mn + F(1)
    for k in range(12):                                              # b - o overflows to ±inf for the far origins of nan_rays
        if k % 2:
            inf_mx[k, k % 3] = BIG
        else:
            inf_mn[k, k % 3] = -BIG
    shapes = np.zeros(len(g) + 48 + 12, dtype=O.AABB3F)
    shapes["min"] = np.concatenate([mn, sub_mn, inf_mn])
    shapes["max"] = np.concatenate([mx, sub_mx, inf_mx])
    return shapes


def nan_rays(seed=0, per=120):
    """Families: origin on an integer (min and max) or half-integer (max) plane of axis a with direction component ±0 on a, for
    every axis and sign; origin on a lattice corner with ±0 and outward components (boxes met only at t = 0); subnormal origins
    and direction components at the subnormal boxes; rays that cross the infinite boxes."""
    rng = np.random.default_rng(seed)
    oo, dd, fam = [], [], []
    for a in range(3):
        for s in (F(0.0), F(-0.0)):
            for plane in ("int", "half"):
                o = rng.uniform(-1, 15, size=(per, 3)).astype(F)
                o[:, a] = rng.integers(0, 14, per).astype(F) + (F(0.5) if plane == "half" else F(0))
                d = rng.normal(size=(per, 3)).astype(F)
                d[:, a] = s
                oo.append(o); dd.append(d); fam += [f"plane{a}{'-' if np.signbit(s) else '+'}{plane}"] * per
    o = rng.integers(0, 15, size=(per, 3)).astype(F)
    d = rng.choice(np.array([0.0, -0.0, 1.0, -1.0, 0.25, -3.0], dtype=F), size=(per, 3))
    d[np.all(d == 0, axis=1), 0] = F(1)
    oo.append(o); dd.append(d); fam += ["touch_t0"] * per
    o = rng.choice(np.array([0.0, -0.0, SUB, -SUB, SUB / 4], dtype=F), size=(per, 3))
    d = rng.choice(np.array([0.0, -0.0, SUB, -SUB, 1.0, -1.0], dtype=F), size=(per, 3))
    d[np.all(d == 0, axis=1), 1] = F(-1)
    oo.append(o); dd.append(d); fam += ["subnormal"] * per
    o = rng.uniform(-3, 17, size=(per, 3)).astype(F)
    axis = np.arange(per) % 3
    o[np.arange(per), axis] = np.where(np.arange(per) % 2, -BIG, BIG)  # far origins: b - o = ±inf at the overflow-scale boxes
    d = rng.normal(size=(per, 3)).astype(F)
    d[::4, 0] = F(-0.0)
    d[1::4, 1] = F(0.0)
    oo.append(o); dd.append(d); fam += ["infinite_products"] * per
    rays = O.ray_new(np.concatenate(oo), np.concatenate(dd))
    return rays, np.array(fam)


def single_nan_products(rays, shapes):
    """Per ray: the number of (shape, axis) pairs where exactly one of the axis's two products is 0 * ±inf."""
    o, inv = rays["origin"][:, None, :], rays["inv_direction"][:, None, :]
    with np.errstate(all="ignore"):
        nl = np.isnan((shapes["min"][None] - o) * inv)
        nr = np.isnan((shapes["max"][None] - o) * inv)
    return (nl ^ nr).sum(axis=(1, 2))


def _assert_preconditions(rays, shapes, fam):
    single = single_nan_products(rays, shapes)
    for f in set(fam.tolist()):
        if f.startswith("plane"):
            assert (single[fam == f] > 0).all(), f                   # every plane ray meets the 0 * inf product
    assert (single[fam == "touch_t0"] > 0).sum() > 0 and (single[fam == "subnormal"] > 0).sum() > 0
    d = rays["direction"]
    assert (np.signbit(d) & (d == 0)).any() and (~np.signbit(d) & (d == 0)).any()
    with np.errstate(all="ignore"):
        far = rays["origin"][fam == "infinite_products"][:, None, :]
        assert np.isinf(shapes["max"][None] - far).any() and np.isinf(shapes["min"][None] - far).any()
    sub = np.abs(shapes["min"])
    assert ((sub > 0) & (sub < np.finfo(F).tiny)).any()


def test_single_nan_products_match_the_oracle():
    from bvh_b200 import api, capi

    shapes = nan_scene()
    rays, fam = nan_rays()
    _assert_preconditions(rays, shapes, fam)
    built = O.build(shapes)
    want = {capi.TRAVERSE_BVH: O.traverse(built.nodes, shapes, rays, O.MODE_RECURSIVE),
            capi.TRAVERSE_FLAT: O.traverse(O.flatten(built.nodes), shapes, rays, O.MODE_FLAT)}
    # the device walk visits one record per child box the recursive walk tests
    visits = want[capi.TRAVERSE_BVH].slab_tests
    assert len(want[capi.TRAVERSE_BVH].hits) > 0
    bvh = api.Bvh.build(shapes)
    ctx = bvh.ctx
    try:
        ctx.set_option("traverse_stream", 0)
        for mode, r in want.items():
            # walk_count_kernel, walk_persistent_kernel, walk_top_kernel with the whole top and with a 64-entry top
            for pers, top in ((0, 0), (1, 0), (1, 1), (1, 64)):
                ctx.set_option("traverse_persistent", pers); ctx.set_option("traverse_top", top)
                for compact in (False, True):
                    off, hits = bvh.traverse_batch(rays, mode=mode, compact=compact)
                    what = f"mode {mode} persistent {pers} top {top} compact {compact}"
                    if not (np.array_equal(off.astype(np.uint64), r.offsets) and np.array_equal(hits, r.hits)):
                        got, exp = O.per_ray_lists(off, hits), O.per_ray_lists(r.offsets, r.hits)
                        bad = [i for i in range(len(fam)) if not np.array_equal(got[i], exp[i])]
                        pytest.fail(f"{what}: {len(bad)} rays differ, families {sorted(set(fam[bad].tolist()))}")
                    assert bvh.traverse_stats()[0] == visits, what
    finally:
        ctx.set_option("traverse_top", -1); ctx.set_option("traverse_persistent", 2); ctx.set_option("traverse_stream", -1)
        bvh.free()
