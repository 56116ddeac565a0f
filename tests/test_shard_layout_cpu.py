"""The staging layout of the fused multi-GPU step (tests/shardref.py) against the size the header reserves for it, the shard split of
dist.shard_range, and the count-width rule at its thresholds.  No GPU."""
import os
import re

import numpy as np
import pytest

from bvh_b200 import capi
from bvh_b200.dist import shard_range
from tests import shardref as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_stage_bytes():
    """BVHGPU_SHARD_STAGE_BYTES as the header defines it, evaluated by Python."""
    text = open(os.path.join(ROOT, "include", "bvh_b200.h")).read()
    body = re.search(r"#define BVHGPU_SHARD_STAGE_BYTES\(nrays_global\)\s*(.+)", text)[1]
    expr = body.replace("(size_t)", "").replace("BVHGPU_MAX_PEERS", str(S.MAX_PEERS)).replace("/", "//")
    return lambda n: eval(expr, {"nrays_global": n})


def _splits():
    """Shard sizes for every W <= 8: even and uneven splits, and the adversarial ones (every shard 1 ray, every shard 2049 rays,
    one large shard with seven 1-ray shards, shards just past a tile)."""
    out = []
    for w in range(1, S.MAX_PEERS + 1):
        out += [[1] * w, [2049] * w, [2048] * w, [2047] * w, [4097] * w, [1] * (w - 1) + [10 ** 6], [10 ** 6 + 1] + [1] * (w - 1)]
        for n in (1, 7, 2047, 2048, 2049, 4099, 3 * 2048 + 5, 1_000_003):
            if n >= w:
                out.append([b - a for a, b in (shard_range(n, r, w) for r in range(w))])
    out.append([10 ** 6] + [1] * 7)
    return out


@pytest.mark.parametrize("sizes", _splits(), ids=lambda s: f"W{len(s)}-{sum(s)}")
def test_stage_bytes_cover_the_layout(sizes):
    ng = sum(sizes)
    need = S.layout_bytes(sizes)
    assert S.stage_bytes(ng) == capi.shard_stage_bytes(ng) == _header_stage_bytes()(ng)
    assert capi.shard_stage_bytes(ng) >= need, (sizes, need)
    assert capi.shard_stage_bytes(ng) % 256 == 0


def test_stage_bytes_at_every_tile_boundary():
    """The tightest case of the rule: each shard adds at most one partial tile, so 8 shards past a tile boundary need the most."""
    for ng in range(8, 64 * 2048, 509):
        for w in range(1, S.MAX_PEERS + 1):
            sizes = [b - a for a, b in (shard_range(ng, r, w) for r in range(w))]
            assert capi.shard_stage_bytes(ng) >= S.layout_bytes(sizes)
            worst = [1] * (w - 1) + [ng - (w - 1)]
            assert capi.shard_stage_bytes(ng) >= S.layout_bytes(worst)


@pytest.mark.parametrize("n", [1, 2, 7, 8, 9, 2047, 2048, 2049, 4099, 1_000_003])
def test_shard_range_covers_every_ray_once(n):
    for w in range(1, S.MAX_PEERS + 1):
        if n < w:
            continue
        seen = np.zeros(n, dtype=np.int64)
        prev = 0
        for r in range(w):
            lo, hi = shard_range(n, r, w)
            assert lo == prev and hi >= lo
            seen[lo:hi] += 1
            prev = hi
        assert prev == n and np.all(seen == 1)
        sizes = [shard_range(n, r, w)[1] - shard_range(n, r, w)[0] for r in range(w)]
        assert max(sizes) - min(sizes) <= 1


def test_width_thresholds():
    assert [S.width(c) for c in (0, 1, 255, 256, 65535, 65536, 2 ** 32 - 1)] == [1, 1, 1, 2, 2, 4, 4]


def test_staging_image_encodes_each_width():
    """A 3-rank batch whose tiles peak at 255, 256, 65535 and 65536: the image holds the counts little-endian in the tile's width
    and the table holds each tile's offset inside its source's list with the width in the top byte."""
    sizes = [4099, 2049, 1]
    counts = np.zeros(sum(sizes), dtype=np.int64)
    counts[[0, 5]] = [255, 3]              # rank 0, tile 0: width 1
    counts[2048 + 7] = 256                 # rank 0, tile 1: width 2
    counts[4096 + 2] = 65536               # rank 0, tile 2: width 4
    counts[4099 + 2048] = 65535            # rank 1, tile 1: width 2
    img, written = S.staging_image(sizes, counts)
    got = S.tiles(sizes, counts)
    assert [(g, s, w) for g, s, _lo, _n, _m, w, _o in got] == [(0, 0, 1), (1, 0, 2), (2, 0, 4), (3, 1, 1), (4, 1, 2), (5, 2, 1)]
    nt = 6
    table = img[S.TILE_BYTES * nt:].view("<u8")
    assert [int(e) & ((1 << 56) - 1) for e in table] == [0, 258, 514, 0, 0, 0]
    assert [int(e) >> 56 for e in table] == [1, 2, 4, 1, 2, 1]
    assert img[0] == 255 and img[5] == 3
    assert img[S.TILE_BYTES + 14: S.TILE_BYTES + 16].view("<u2")[0] == 256
    assert img[2 * S.TILE_BYTES + 8: 2 * S.TILE_BYTES + 12].view("<u4")[0] == 65536
    assert img[4 * S.TILE_BYTES: 4 * S.TILE_BYTES + 2].view("<u2")[0] == 65535
    assert written.sum() == S.TILE * (1 + 2 + 4 + 1 + 2 + 1) + 8 * nt


def test_mailbox_words():
    w = S.mailbox_words(3, [10, 0, 7])
    assert w[(8 + 0) * 4] == 3 and w[(8 + 0) * 4 + 1] == 10 and w[(8 + 2) * 4 + 1] == 7
    assert w[64 + 8 + 1] == 3 and w[128 + 3 * 4] == 3
    w = S.mailbox_words(1024, [1])
    assert w[0] == 1024 and w[1] == 1 and w[64] == 1024 and w[128] == 1024
