"""Test infrastructure: the oracle's sequential Bvh::add_shape / Bvh::remove_shape (oracle/bvh_oracle.hpp), re-emitted in Bvh::build's
preorder layout (tests/cpp/dyn_oracle.cpp), plus the renumbering rule of a batched removal."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

from oracle import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def lib():
    global _lib
    if _lib is None:
        tmp = tempfile.mkdtemp(prefix="bvh_dyn_oracle_")
        atexit.register(shutil.rmtree, tmp, True)              # the loaded library stays mapped until the process ends
        out = os.path.join(tmp, "libdynoracle.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
                        os.path.join(HERE, "cpp", "dyn_oracle.cpp"), "-o", out], check=True)
        _lib = C.CDLL(out)
        for p in ("f32", "f64"):
            getattr(_lib, f"dyn_add_{p}").restype = C.c_uint32
            getattr(_lib, f"dyn_remove_{p}").restype = C.c_uint32
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def add_shapes(nodes, node_index, shapes, k, prec="f32"):
    """shapes = all n + k AABBs; the tree over the first n gets shapes n .. n+k-1 by sequential add_shape.  Returns (nodes, node_index)."""
    d = O._DT[prec]
    n = len(shapes) - k
    out = np.zeros(2 * len(shapes) - 1, dtype=d["node"])
    out[: len(nodes)] = nodes
    ni = np.zeros(len(shapes), dtype=np.uint32)
    ni[:n] = node_index
    shapes = np.ascontiguousarray(shapes, dtype=d["aabb"])
    m = getattr(lib(), f"dyn_add_{prec}")(_p(out), C.c_uint32(len(nodes)), _p(ni), C.c_uint32(n), _p(shapes), C.c_uint32(k))
    assert m == len(out)
    return out, ni


def remove_shapes(nodes, node_index, shapes, indices, prec="f32"):
    """remove_shape(i, swap=false) for every index of the tree over `shapes`, then the swap rule's renumbering.  Returns
    (nodes, node_index, new shapes)."""
    d = O._DT[prec]
    n = len(shapes)
    idx = np.ascontiguousarray(indices, dtype=np.uint32)
    out = np.array(nodes, dtype=d["node"], copy=True)
    ni = np.array(node_index, dtype=np.uint32, copy=True)
    shapes = np.ascontiguousarray(shapes, dtype=d["aabb"])
    m = getattr(lib(), f"dyn_remove_{prec}")(_p(out), C.c_uint32(len(nodes)), _p(ni), C.c_uint32(n), _p(shapes), _p(idx), C.c_uint32(len(idx)))
    assert m == max(2 * (n - len(idx)) - 1, 0)
    return out[:m], ni[: n - len(idx)], apply_moves(shapes, idx)


def swap_moves(n, indices):
    """(new, old) pairs: survivors >= n-k fill the vacated indices < n-k, both in ascending order."""
    rm = np.zeros(n, dtype=bool)
    rm[np.asarray(indices, dtype=np.int64)] = True
    m = n - int(rm.sum())
    return np.stack([np.flatnonzero(rm[:m]), m + np.flatnonzero(~rm[m:])], axis=1).reshape(-1, 2)


def apply_moves(items, indices):
    items = np.array(items, copy=True)
    mv = swap_moves(len(items), indices)
    items[mv[:, 0]] = items[mv[:, 1]]
    return items[: len(items) - len(indices)]


def same_tree(a, b):
    """Node arrays equal field for field (AABB coordinates with ==)."""
    if len(a) != len(b):
        return False
    for f in ("parent", "child_l", "child_r", "shape"):
        if not np.array_equal(a[f], b[f]):
            return False
    for s in ("l_aabb", "r_aabb"):
        for e in ("min", "max"):
            if not np.array_equal(a[s][e], b[s][e]):
                return False
    return True
