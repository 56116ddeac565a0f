"""GPU test of the shared-memory top-of-tree walk's form for trees beyond L2: walk_top_kernel votes on idle lanes after every
visit there (after every 4 visits on L2-resident trees, which the other top-walk tests cover).  Same CSR and visit counter as the
plain persistent walk (traverse_top = 0), BVH and FLAT semantics.
Run on an H100:  python -m pytest tests -m gpu"""
import numpy as np
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu


def test_top_walk_on_a_tree_beyond_l2_is_bit_identical():
    from bvh_b200 import api, capi, scenes

    shapes = scenes.create_n_cubes_aabbs(50_000)                   # 600 000 triangles: 1.2 M records, 38 MB (> 32 MB)
    oo, dd = scenes.ray_endpoints(100_000, 3)
    rays = O.ray_new(oo, dd)
    bvh = api.Bvh.build(shapes)
    ctx = bvh.ctx
    try:
        ctx.set_option("traverse_persistent", 1); ctx.set_option("traverse_stream", 0)
        for mode in (capi.TRAVERSE_BVH, capi.TRAVERSE_FLAT):
            got = []
            for top in (0, 1):
                ctx.set_option("traverse_top", top)
                off, hits = bvh.traverse_batch(rays, mode=mode)
                got.append((off, hits, bvh.traverse_stats()[0]))
            assert np.array_equal(got[0][0], got[1][0]) and np.array_equal(got[0][1], got[1][1]), mode
            assert got[0][2] == got[1][2], mode
    finally:
        ctx.set_option("traverse_top", -1); ctx.set_option("traverse_persistent", 2); ctx.set_option("traverse_stream", -1)
        bvh.free()
