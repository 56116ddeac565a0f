"""tests/launch_edges.py reads the launch constants from the CUDA sources: every one is found (a renamed constant fails here instead of
silently shrinking the GPU sweep of tests/test_gpu_launch_edges.py), and the restated chunk bounds of the streamed host path cover
every batch it streams without an empty chunk."""
import pytest

from tests import launch_edges as LE


def test_every_constant_is_found():
    want = ("BVH_MAX_CHUNKS", "CSR_SCAN_TILE", "CSR_SCAN_THREADS", "SCAN_ITEMS", "SCAN_THREADS", "SCAN_TILE", "TOP_BUDGET", "SCAN_BLOCKS_STEP",
            "SCAN_BLOCKS_THREADS", "SCAN_POST_STEP", "STREAM_MIN", "CHUNK_RAYS", "SLICE_MIN", "TOP_RAYS_PER_CTA", "PERSISTENT_THREADS",
            "TOP_UNROLL_MAX_BYTES", "TNODE_F32_BYTES")
    for k in want:
        assert isinstance(LE.CONST.get(k), int) and LE.CONST[k] > 0, k
    assert LE.CONST["SCAN_TILE"] == LE.CONST["CSR_SCAN_TILE"] and LE.CONST["SCAN_THREADS"] == LE.CONST["CSR_SCAN_THREADS"]
    assert LE.CONST["SCAN_BLOCKS_STEP"] == LE.CONST["SCAN_BLOCKS_THREADS"]          # the loop step is the block the carry assumes
    for k in LE.PER_ITEM_128 + LE.PER_ITEM_256:                                    # every per-item kernel's launch is found
        assert LE.BLOCK.get(k), k
    assert all(LE.BLOCK[k] == {128} for k in LE.PER_ITEM_128) and all(LE.BLOCK[k] == {256} for k in LE.PER_ITEM_256)


def test_edges():
    small = LE.edges("small")
    assert small == sorted(set(small)) and small[0] == 1 and small[-1] == 2 * LE.CONST["SCAN_TILE"] + 1
    for b in (32, 128, 256, LE.CONST["TOP_RAYS_PER_CTA"], LE.CONST["SCAN_TILE"]):
        assert {b - 1, b, b + 1} <= set(small), b
    assert LE.edges("scan_post")[1] == LE.CONST["SCAN_TILE"] * LE.CONST["SCAN_THREADS"]
    assert LE.edges("scan_blocks")[1] == LE.CONST["CSR_SCAN_TILE"] * LE.CONST["SCAN_BLOCKS_THREADS"]
    host = LE.edges("host")
    assert [LE.chunks_for(R) for R in host[:2]] == [1, 2]
    big = host[-1]
    assert LE.chunks_for(big) == LE.CONST["BVH_MAX_CHUNKS"] and big % LE.CONST["BVH_MAX_CHUNKS"] and big % 24
    assert LE.edges("top", 132) == [135167, 135168, 135169]
    with pytest.raises(ValueError):
        LE.edges("top")


def test_chunk_bounds_restate_the_source():
    """chunk_bounds is a restatement of the lambda in traverse.cu: a change there must be made here too."""
    units, body = LE.bound_source()
    assert units == "sched == 1 ? nchunks + nhalf : nchunks"
    assert body == "const uint32_t u = sched == 1 ? (c <= nhalf ? 2 * c : nhalf + c) : c; return (uint32_t)((uint64_t)R * u / units);"


@pytest.mark.parametrize("sched", [0, 1])
def test_chunk_bounds_cover_every_streamed_batch(sched):
    sizes = sorted(set(LE.edges("host") + [LE.CONST["STREAM_MIN"], 250_001, 1_000_000, 2**31 - 1]))
    for R in sizes:
        if R < LE.CONST["STREAM_MIN"]:
            continue
        for n in range(2, LE.CONST["BVH_MAX_CHUNKS"] + 1):
            b = LE.chunk_bounds(R, n, sched)
            assert len(b) == n + 1 and b[0] == 0 and b[-1] == R, (R, n)
            assert all(lo < hi for lo, hi in zip(b, b[1:])), (R, n)          # monotone, no empty chunk
    assert LE.chunks_for(10**9, 17) == LE.CONST["BVH_MAX_CHUNKS"] and LE.chunks_for(10, 3) == 3
