"""The Python layer without a GPU: the ctypes signatures capi.py reads from include/bvh_b200.h, and the C calls the CSR methods of
Bvh, Bvh2 and Bvh4 make, recorded by a fake library that reports scripted statuses and totals."""
import ctypes as C

import numpy as np
import pytest

from bvh_b200 import api, capi
from bvh_b200.dtypes import U32_MAX

CLASSES = {3: api.Bvh, 2: api.Bvh2, 4: api.Bvh4}
N_SHAPES = 700                     # what tree_num_shapes reports; Bvh2 / Bvh4 are built knowing it


# ---- signatures ------------------------------------------------------------------------------------------------------------------

def test_every_declared_symbol_is_typed_from_the_header():
    sigs = capi.signatures()
    assert sorted(sigs) == capi.declared_symbols() and len(sigs) >= 232
    L = capi.lib()
    for name, (restype, argtypes) in sigs.items():
        fn = getattr(L, name)
        assert fn.argtypes is not None and list(fn.argtypes) == argtypes, name
        assert fn.restype is restype, name


@pytest.mark.parametrize("fn, index, want", [
    ("bvhgpu_create", 0, C.c_int),                                       # int
    ("bvhgpu_memcpy_d2h", 3, C.c_size_t),                                # size_t
    ("bvhgpu_knn_f32x3", 3, C.c_uint32),                                 # uint32_t
    ("bvhgpu_set_option", 2, C.c_int64),                                 # int64_t
    ("bvhgpu_update_f64x3", 4, C.c_double),                              # double
    ("bvhgpu_update_f64x3", 5, C.POINTER(C.c_size_t)),                   # size_t*
    ("bvhgpu_traverse_stats_f32x3", 1, C.POINTER(C.c_uint64)),           # uint64_t*
    ("bvhgpu_traverse_sharded_dev_f32x3", 4, C.POINTER(capi.Shard)),     # const bvhgpu_shard*
    ("bvhgpu_traverse_sharded_dev_f64x3", 4, C.POINTER(capi.Shard)),
    ("bvhgpu_set_option", 1, C.c_char_p),                                # const char*
    ("bvhgpu_create", 1, C.POINTER(C.c_void_p)),                         # bvhgpu_ctx**
    ("bvhgpu_build_f32x2", 4, C.POINTER(C.c_void_p)),                    # bvhgpu_tree2f**
    ("bvhgpu_peer_alloc", 2, C.POINTER(C.c_void_p)),                     # void**
    ("bvhgpu_get_metric", 2, C.c_void_p),                                # double*: every other pointer
    ("bvhgpu_traverse_f32x4", 0, C.c_void_p),                            # bvhgpu_tree4f*
    ("bvhgpu_traverse_f32x4", 2, C.c_void_p),                            # const bvh_ray4f*
])
def test_parameter_types(fn, index, want):
    assert capi.signatures()[fn][1][index] is want


@pytest.mark.parametrize("fn, want", [
    ("bvhgpu_last_error", C.c_char_p), ("bvhgpu_version", C.c_char_p), ("bvhgpu_destroy", None), ("bvhgpu_tree_free_f64x4", None),
    ("bvhgpu_tree_num_shapes_f32x2", C.c_size_t), ("bvhgpu_tree_num_nodes_f64x3", C.c_size_t), ("bvhgpu_launch_count", C.c_uint64),
    ("bvhgpu_traverse_f32x3", C.c_int),
])
def test_return_types(fn, want):
    assert capi.signatures()[fn][0] is want


def test_void_parameter_lists_and_multi_line_prototypes(tmp_path):
    h = tmp_path / "h.h"
    h.write_text("/* bvhgpu_commented(int x); */\nconst char* bvhgpu_a(void);\nvoid bvhgpu_b();\nsize_t\n  bvhgpu_c(const bvhgpu_ctx *ctx,\n"
                 "           uint32_t k,   /* a comment */\n           bvhgpu_tree3f **out);\nint bvhgpu_d(size_t, int*);\n")
    assert capi.signatures(str(h)) == {"bvhgpu_a": (C.c_char_p, []), "bvhgpu_b": (None, []),
                                       "bvhgpu_c": (C.c_size_t, [C.c_void_p, C.c_uint32, C.POINTER(C.c_void_p)]),
                                       "bvhgpu_d": (C.c_int, [C.c_size_t, C.c_void_p])}
    assert capi.signatures()["bvhgpu_last_error"] == (C.c_char_p, [])


@pytest.mark.parametrize("proto, ctype", [("int bvhgpu_f(float x);", "float"), ("long bvhgpu_f(int x);", "long"),
                                          ("int bvhgpu_f(int x, unsigned y);", "unsigned"), ("uint32_t bvhgpu_f(void);", "uint32_t")])
def test_unknown_type_raises(tmp_path, proto, ctype):
    h = tmp_path / "h.h"
    h.write_text("int bvhgpu_ok(int x);\n" + proto + "\n")
    with pytest.raises(ImportError, match=rf"bvhgpu_f uses the C type '{ctype}'"):
        capi.signatures(str(h))


def test_unreadable_prototype_raises(tmp_path):
    h = tmp_path / "h.h"
    h.write_text("int bvhgpu_ok(int x);\nint bvhgpu_g(void (*callback)(int));\n")
    with pytest.raises(ImportError, match=r"cannot read the prototypes of \['bvhgpu_g'\]"):
        capi.signatures(str(h))


# ---- the CSR methods through a recording library ------------------------------------------------------------------------------------

class _Handle:
    """A tree handle only the fake library sees.  It is false, so a tree's __del__ never hands it to the real library."""

    def __init__(self, name):
        self.name = name

    def __bool__(self):
        return False


class FakeLib:
    """Records every C call.  A CSR call reports `total` hits, with ERR_CAPACITY when they exceed the capacity it was given."""

    def __init__(self, total):
        self.total, self.calls = total, []

    def __getattr__(self, name):
        if not name.startswith("bvhgpu_"):
            raise AttributeError(name)

        def call(*args):
            self.calls.append((name, args))
            if name == "bvhgpu_last_error":
                return b"scripted failure"
            if name.startswith("bvhgpu_tree_num_shapes_"):
                return N_SHAPES
            if name.startswith("bvhgpu_traverse_fetch_") or not hasattr(args[-1], "_obj"):
                return capi.OK
            args[-1]._obj.value = self.total
            return capi.ERR_CAPACITY if self.total > args[-2] else capi.OK
        return call

    def csr_calls(self):
        """(entry point without its suffix, capacity) of every call but the shape count and the error message."""
        return [(n.rsplit("_", 1)[0], a[-1] if "fetch" in n else a[-2]) for n, a in self.calls
                if "num_shapes" not in n and n != "bvhgpu_last_error"]


def _tree(D, prec="f32", name="a"):
    cls = CLASSES[D]
    return cls(_Handle(name), prec, None) if D == 3 else cls(_Handle(name), prec, None, N_SHAPES)


def _rays(D, n, prec="f32"):
    return np.zeros(n, dtype=_tree(D, prec)._d["ray"])


def _points(D, n):
    return np.zeros((n, D))


# (method, stem of its entry point, items, arguments, starting capacity of each dimension)
CSR = [
    ("traverse_batch", "traverse", 300, lambda D: (_rays(D, 300),), {3: 1200, 2: 4800, 4: 4800}),
    ("traverse_batch", "traverse", 2, lambda D: (_rays(D, 2),), {3: 1024, 2: 1024, 4: 1024}),
    ("query_batch", "query", 100, lambda D: (capi.QUERY_POINT, _points(D, 100)), {D: 1600 for D in (2, 3, 4)}),
    ("query_batch", "query", 50, lambda D: (capi.QUERY_AABB, np.zeros((50, 2 * D))), {D: 1024 for D in (2, 3, 4)}),
    ("query_batch", "query", 70, lambda D: (capi.QUERY_BALL, np.zeros((70, D + 1))), {D: 1120 for D in (2, 3, 4)}),
    ("overlap_pairs", "overlap_pairs", N_SHAPES, lambda D: (), {D: 4 * N_SHAPES for D in (2, 3, 4)}),
    ("overlap_pairs", "overlap_pairs", N_SHAPES, lambda D: (33,), {D: 33 for D in (2, 3, 4)}),
    ("overlap_pairs_with", "overlap_trees", N_SHAPES, lambda D: (_tree(D, name="b"),), {D: 4 * N_SHAPES for D in (2, 3, 4)}),
    ("overlap_pairs_with", "overlap_trees", N_SHAPES, lambda D: (_tree(D, name="b"), 40), {D: 40 for D in (2, 3, 4)}),
    ("nearest_candidates", "nearest_candidates", 20, lambda D: (_points(D, 20),), {D: 1280 for D in (2, 3, 4)}),
    ("nearest_candidates", "nearest_candidates", 3, lambda D: (_points(D, 3),), {D: 1024 for D in (2, 3, 4)}),
    ("traverse_ordered", "traverse_ordered", 200, lambda D: (_rays(D, 200),), {D: 1600 for D in (2, 3, 4)}),
]


def _call(monkeypatch, D, method, args, total):
    lib = FakeLib(total)
    monkeypatch.setattr(capi, "lib", lambda: lib)
    return lib, getattr(_tree(D), method)(*args)


@pytest.mark.parametrize("D", [2, 3, 4])
@pytest.mark.parametrize("method, stem, n, args, cap0", CSR)
def test_csr_call_that_fits(monkeypatch, D, method, stem, n, args, cap0):
    lib, out = _call(monkeypatch, D, method, args(D), 17)
    assert lib.csr_calls() == [(f"bvhgpu_{stem}", cap0[D])]
    assert len(out) == (3 if method == "traverse_ordered" else 2)
    assert len(out[0]) == n + 1 and all(len(a) == 17 for a in out[1:])


@pytest.mark.parametrize("D", [2, 3, 4])
@pytest.mark.parametrize("method, stem, n, args, cap0", CSR)
def test_csr_call_with_a_short_capacity(monkeypatch, D, method, stem, n, args, cap0):
    """3-D: one walk, then the retained list is copied with bvhgpu_traverse_fetch_*(total).  2-D and 4-D, and the distance-ordered
    lists of every dimension: one more call with cap = total."""
    total = 10 * cap0[D] + 3
    lib, out = _call(monkeypatch, D, method, args(D), total)
    fetch = D == 3 and method != "traverse_ordered"
    again = ("bvhgpu_traverse_fetch", total) if fetch else (f"bvhgpu_{stem}", total)
    assert lib.csr_calls() == [(f"bvhgpu_{stem}", cap0[D]), again]
    assert len(out[0]) == n + 1 and all(len(a) == total for a in out[1:])


@pytest.mark.parametrize("D", [2, 3, 4])
@pytest.mark.parametrize("method, stem, n, args, cap0", CSR)
def test_csr_total_beyond_u32_raises_without_a_retry(monkeypatch, D, method, stem, n, args, cap0):
    with pytest.raises(capi.BvhGpuError) as e:
        _call(monkeypatch, D, method, args(D), U32_MAX + 1)
    assert e.value.status == capi.ERR_CAPACITY and "scripted failure" in str(e.value)
    lib = capi.lib()
    assert lib.csr_calls() == [(f"bvhgpu_{stem}", cap0[D])]


def test_the_cap_argument_of_the_3d_traversal(monkeypatch):
    lib, _ = _call(monkeypatch, 3, "traverse_batch", (_rays(3, 300), capi.TRAVERSE_BVH, 40), 17)
    assert lib.csr_calls() == [("bvhgpu_traverse", 40)]
    lib, _ = _call(monkeypatch, 3, "traverse_batch", (_rays(3, 300), capi.TRAVERSE_BVH, 40, True), 41)
    assert lib.csr_calls() == [("bvhgpu_traverse_od", 40), ("bvhgpu_traverse_fetch", 41)]


def test_overlap_pairs_with_passes_both_trees(monkeypatch):
    for D in (2, 3, 4):
        other = _tree(D, name="b")
        lib, _ = _call(monkeypatch, D, "overlap_pairs_with", (other,), 1)
        name, args = lib.calls[-1]
        assert args[0].name == "a" and args[1] is other._h


# ---- the limits helper -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("D", [2, 3, 4])
def test_limits(D, prec):
    t = _tree(D, prec)
    F = np.float32 if prec == "f32" else np.float64
    assert t._limits(None, 5) is None
    for x, want in ((2.5, [2.5] * 5), (np.arange(5.0)[::-1], [4, 3, 2, 1, 0]), ([1, 2, 3, 4, 5], [1, 2, 3, 4, 5])):
        got = t._limits(x, 5)
        assert got.dtype == F and got.shape == (5,) and got.flags.c_contiguous and got.tolist() == want
    with pytest.raises(ValueError):
        t._limits(np.arange(4.0), 5)


@pytest.mark.parametrize("D", [2, 3, 4])
def test_no_limit_is_a_null_pointer(monkeypatch, D):
    lib = FakeLib(0)
    monkeypatch.setattr(capi, "lib", lambda: lib)
    t = _tree(D)
    t.any_hit(_rays(D, 4))
    t.knn(_points(D, 4), 2)
    t.any_hit(_rays(D, 4), 7.0)
    (_, a0), (_, a1), (_, a2) = lib.calls
    assert a0[3] is None and a1[4] is None and a2[3].value
