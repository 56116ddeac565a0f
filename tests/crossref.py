"""tests/crossref.py -- the brute-force model of the overlap pairs between two trees (bvhgpu_overlap_trees_*), generic in D, f32 / f64
(test infrastructure).

leaf_b[b] is the preorder node index of shape b's leaf in tree B.  Row a (a shape of tree A) lists every shape b of B whose box
intersects a's box, in ascending leaf_b[b] order; `intersects` is Aabb::intersects_aabb taken literally (tests/overlapref.py), compared
in the boxes' own precision.  Rows are computed a chunk of A at a time against all of B in leaf order."""
import numpy as np

from tests.overlapref import U32_MAX, intersects


def cross_rows(amn, amx, bmn, bmx, leaf_b, chunk=256):
    """CSR (offsets u32[n_a + 1], hits u32) of the contract.  The offsets saturate at 0xFFFFFFFF as the device's do."""
    amn, amx, bmn, bmx = (np.asarray(x) for x in (amn, amx, bmn, bmx))
    order = np.argsort(np.asarray(leaf_b), kind="stable")
    omn, omx = bmn[order], bmx[order]
    n = len(amn)
    counts = np.zeros(n, dtype=np.uint64)
    lists = []
    for s in range(0, n, chunk):
        m = intersects(amn[s:s + chunk, None, :], amx[s:s + chunk, None, :], omn[None], omx[None])
        r, c = np.nonzero(m)                                   # row-major: rows in order, partners in B's leaf order
        counts[s:s + len(m)] = np.bincount(r, minlength=len(m))
        lists.append(order[c])
    offsets = np.zeros(n + 1, dtype=np.uint64)
    np.cumsum(counts, out=offsets[1:])
    hits = np.concatenate(lists).astype(np.uint32) if lists else np.zeros(0, dtype=np.uint32)
    return np.minimum(offsets, U32_MAX).astype(np.uint32), hits
