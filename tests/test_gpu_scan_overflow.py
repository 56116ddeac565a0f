"""A tile of 2048 counts whose sum passes 2^32: 2^21 + 1 boxes that all contain the origin and 2048 rays (or Point queries) through
it, 2^32 + 2048 hits in one tile.  The scans add tile sums in 64 bits, so every entry point reports the exact total 2048 n, leaves
every offset below 2^32 exact and the closing one at 0xFFFFFFFF, and returns BVHGPU_ERR_CAPACITY ("hits overflow the u32 CSR
offsets"); the sharded step's fetch raises.  Control: 2047 rays give the exact total 2047 n and offsets[i] == i n.  The truth is
analytic.  Each call walks every leaf for every ray (2^32 leaf visits and more), so the calls are few.
Run on an H100:  python -m pytest tests/test_gpu_scan_overflow.py -m gpu"""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O
from tests import shardref as S

pytestmark = pytest.mark.gpu
N_BOXES = (1 << 21) + 1
CAP = 1 << 16                     # far below the total: the hit lists are cut at cap, the offsets stay exact


@pytest.fixture(scope="module")
def pile():
    """(api, capi, bvh, shapes): the f32 tree of N_BOXES boxes around the origin."""
    from bvh_b200 import api, capi

    rng = np.random.default_rng(21)
    half = rng.uniform(1.0, 2.0, (N_BOXES, 3))
    shapes = O.make_aabbs(-half * rng.uniform(0.25, 1.0, (N_BOXES, 3)), half)
    bvh = api.Bvh.build(shapes)
    yield api, capi, bvh, shapes
    bvh.free()


def _rays(n):
    """n rays from a sphere of radius 10 through the origin."""
    rng = np.random.default_rng(n)
    org = rng.normal(size=(n, 3))
    org *= 10.0 / np.linalg.norm(org, axis=1, keepdims=True)
    return O.ray_new(org, -org)


def _assert_offsets(off, nrays, total):
    want = np.arange(nrays + 1, dtype=np.uint64) * np.uint64(N_BOXES)
    want[want > 0xFFFFFFFF] = 0xFFFFFFFF
    assert int(total) == nrays * N_BOXES
    assert np.array_equal(np.asarray(off, dtype=np.uint64), want)


def _device_call(pile, nrays, fn_name, payload):
    import torch

    api, capi, bvh, _shapes = pile
    dev = torch.device("cuda", 0)
    bvh.ctx.set_stream(torch.cuda.current_stream().cuda_stream)
    d_in = torch.from_numpy(payload.view(np.uint8).reshape(-1)).to(dev)
    d_off = torch.zeros(nrays + 1, dtype=torch.int32, device=dev)
    d_hits = torch.zeros(CAP, dtype=torch.int32, device=dev)
    total = C.c_size_t(0)
    return d_in, d_off, d_hits, total


@pytest.mark.parametrize("nrays", [2048, 2047])
def test_traverse_dev_total_does_not_wrap(pile, nrays):
    import torch

    api, capi, bvh, _ = pile
    rays = _rays(nrays)
    d_in, d_off, d_hits, total = _device_call(pile, nrays, None, rays)
    st = capi.lib().bvhgpu_traverse_dev_f32x3(bvh._h, capi.TRAVERSE_BVH, C.c_void_p(d_in.data_ptr()), nrays, C.c_void_p(d_off.data_ptr()),
                                              C.c_void_p(d_hits.data_ptr()), CAP, C.byref(total))
    torch.cuda.synchronize()
    assert st == capi.ERR_CAPACITY                  # 2048: the u32 offsets overflow; 2047: the hits do not fit CAP
    _assert_offsets(d_off.cpu().numpy().view(np.uint32), nrays, total.value)
    assert np.all(d_hits.cpu().numpy().view(np.uint32) < N_BOXES)


def test_host_traverse_total_does_not_wrap(pile):
    api, capi, bvh, _ = pile
    rays = _rays(2048)
    off = np.zeros(2049, dtype=np.uint32)
    hits = np.zeros(CAP, dtype=np.uint32)
    total = C.c_size_t(0)
    st = capi.lib().bvhgpu_traverse_f32x3(bvh._h, capi.TRAVERSE_BVH, rays.ctypes.data_as(C.c_void_p), 2048, off.ctypes.data_as(C.c_void_p),
                                          hits.ctypes.data_as(C.c_void_p), CAP, C.byref(total))
    assert st == capi.ERR_CAPACITY
    _assert_offsets(off, 2048, total.value)


def test_point_query_total_does_not_wrap(pile):
    import torch

    api, capi, bvh, _ = pile
    pts = np.zeros((2048, 3), dtype=np.float32)
    d_in, d_off, d_hits, total = _device_call(pile, 2048, None, pts)
    st = capi.lib().bvhgpu_query_dev_f32x3(bvh._h, capi.TRAVERSE_BVH, capi.QUERY_POINT, C.c_void_p(d_in.data_ptr()), 2048,
                                           C.c_void_p(d_off.data_ptr()), C.c_void_p(d_hits.data_ptr()), CAP, C.byref(total))
    torch.cuda.synchronize()
    assert st == capi.ERR_CAPACITY
    _assert_offsets(d_off.cpu().numpy().view(np.uint32), 2048, total.value)


def test_sharded_step_total_does_not_wrap(pile):
    """A world-1 step of the fused exchange: offsets saturate past 2^32, the mailbox carries the exact 64-bit total, the fetch
    raises ERR_CAPACITY, and nothing lands past cap."""
    _api, capi, _bvh, shapes = pile
    vs = S.VirtualShards(shapes, [2048], CAP)
    try:
        d_rays = vs.upload(_rays(2048))
        vs.step(d_rays)
        vs.synchronize()
        _assert_offsets(vs.offsets(0), 2048, 2048 * N_BOXES)
        assert int(vs.mailbox(0)[S.MB_TOT + (S.MAX_PEERS * 1 + 0) * 4 + 1]) == 2048 * N_BOXES
        with pytest.raises(capi.BvhGpuError) as e:
            vs.fetch(0)
        assert e.value.status == capi.ERR_CAPACITY
        assert vs.guards_intact()
    finally:
        vs.close()
