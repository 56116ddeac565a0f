"""tests/overlapref.py -- the brute-force model of the self-overlap pairs (bvhgpu_overlap_pairs_*), generic in D, f32 / f64 (test
infrastructure).

leaf[s] is the preorder node index of shape s's leaf.  Row s lists every shape t with leaf[t] > leaf[s] whose box intersects s's box,
in ascending leaf[t] order; `intersects` is Aabb::intersects_aabb taken literally: for every axis !(a.max < b.min || b.max < a.min),
compared in the boxes' own precision.  Rows are computed in leaf order (argsort of leaf) and vectorised over the partners."""
import numpy as np

U32_MAX = 0xFFFFFFFF


def intersects(amn, amx, bmn, bmx):
    """Aabb::intersects_aabb of box a against every box of b (broadcast over the leading axes of b)."""
    return np.all(~((amx < bmn) | (bmx < amn)), axis=-1)


def rows(mn, mx, leaf):
    """CSR (offsets u32[n + 1], hits u32) of the contract.  The offsets saturate at 0xFFFFFFFF as the device's do."""
    mn, mx, leaf = np.asarray(mn), np.asarray(mx), np.asarray(leaf)
    n = len(mn)
    order = np.argsort(leaf, kind="stable")
    lists = [None] * n
    for r, s in enumerate(order):
        cand = order[r + 1:]
        lists[s] = cand[intersects(mn[s], mx[s], mn[cand], mx[cand])]
    counts = np.array([len(x) for x in lists], dtype=np.uint64)
    offsets = np.zeros(n + 1, dtype=np.uint64)
    np.cumsum(counts, out=offsets[1:])
    hits = np.concatenate(lists).astype(np.uint32) if n else np.zeros(0, dtype=np.uint32)
    return np.minimum(offsets, U32_MAX).astype(np.uint32), hits


def pairs(offsets, hits):
    """The rows as an (m, 2) array of (s, t), in row order."""
    offsets = np.asarray(offsets, dtype=np.int64)
    s = np.repeat(np.arange(len(offsets) - 1), np.diff(offsets))
    return np.stack([s, np.asarray(hits, dtype=np.int64)], axis=1)


def closure(offsets, hits, n):
    """The symmetric closure: for every shape, the sorted list of all shapes it overlaps (itself excluded)."""
    p = pairs(offsets, hits)
    out = [[] for _ in range(n)]
    for s, t in p:
        out[s].append(int(t))
        out[t].append(int(s))
    return [sorted(x) for x in out]
