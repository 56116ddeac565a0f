"""ctypes binding of libbvh_b200.so (include/bvh_b200.h).  There is no fallback: if the shared
library is missing or a symbol cannot be resolved, importing the product API raises."""
from __future__ import annotations

import ctypes as C
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(_HERE, "libbvh_b200.so")
HEADER = os.path.join(os.path.dirname(_HERE), "include", "bvh_b200.h")

OK, ERR_INVALID, ERR_CUDA, ERR_NAN, ERR_CAPACITY, ERR_TIMEOUT, ERR_UNSUPPORTED, ERR_INTERNAL = range(8)
BUILD_EXACT_SAH, BUILD_LBVH, BUILD_LBVH_TREELET = 0, 1, 2
TRAVERSE_BVH, TRAVERSE_FLAT = 0, 1
QUERY_AABB, QUERY_POINT, QUERY_BALL = 1, 2, 3


RAYS_FULL, RAYS_OD = 0, 1
FILL_EVEN_ODD, FILL_NONZERO = 0, 1
MAX_PEERS, MAILBOX_BYTES, IPC_HANDLE_BYTES = 8, 65536, 64
MB_TRACE_WORD, MB_TRACE_LEN = 128, 1024          # mailbox trace ring (u64 words), see traverse.cu


def shard_stage_bytes(nrays_global: int) -> int:
    """BVHGPU_SHARD_STAGE_BYTES"""
    return (8200 * (nrays_global // 2048 + 2 * MAX_PEERS) + 255) & ~255


class Shard(C.Structure):
    """bvhgpu_shard (include/bvh_b200.h)."""
    _fields_ = [("rank", C.c_int), ("world", C.c_int),
                ("peer_counts", C.c_void_p * MAX_PEERS), ("peer_hits", C.c_void_p * MAX_PEERS), ("peer_mailbox", C.c_void_p * MAX_PEERS),
                ("offsets", C.c_void_p), ("seq", C.c_uint64), ("shard_rays", C.c_size_t * MAX_PEERS), ("cap", C.c_size_t),
                ("ray_layout", C.c_int)]


class BvhGpuError(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"bvhgpu status {status}: {message}")
        self.status = status


def declared_symbols() -> list[str]:
    """Every function include/bvh_b200.h declares."""
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(bvhgpu_[a-z0-9_]+)\s*\(", text)))


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise ImportError(
            f"{SO_PATH} is missing: build it with `python -m bvh_b200.build` (nvcc, sm_90a). "
            "bvh_b200 has no CPU fallback."
        )
    L = C.CDLL(SO_PATH)
    vp, sz, i32, u64p = C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.c_uint64)
    szp = C.POINTER(C.c_size_t)
    L.bvhgpu_last_error.restype = C.c_char_p
    L.bvhgpu_version.restype = C.c_char_p
    L.bvhgpu_create.argtypes = [i32, C.POINTER(vp)]
    L.bvhgpu_destroy.argtypes = [vp]
    L.bvhgpu_destroy.restype = None
    L.bvhgpu_set_stream.argtypes = [vp, vp]
    L.bvhgpu_reset_stream.argtypes = [vp]
    L.bvhgpu_synchronize.argtypes = [vp]
    L.bvhgpu_launch_count.argtypes = [vp]
    L.bvhgpu_launch_count.restype = C.c_uint64
    L.bvhgpu_set_option.argtypes = [vp, C.c_char_p, C.c_int64]
    L.bvhgpu_get_metric.argtypes = [vp, C.c_char_p, C.POINTER(C.c_double)]
    L.bvhgpu_peer_alloc.argtypes = [vp, sz, C.POINTER(vp), vp]
    L.bvhgpu_peer_open.argtypes = [vp, vp, C.POINTER(vp)]
    L.bvhgpu_peer_close.argtypes = [vp, vp]
    L.bvhgpu_peer_free.argtypes = [vp, vp]
    L.bvhgpu_memcpy_d2h.argtypes = [vp, vp, vp, sz]
    L.bvhgpu_memcpy_h2d_async.argtypes = [vp, vp, vp, sz]
    L.bvhgpu_host_alloc.argtypes = [vp, sz, C.POINTER(vp)]
    L.bvhgpu_host_free.argtypes = [vp, vp]
    for s in ("f32x3", "f64x3"):
        getattr(L, f"bvhgpu_build_{s}").argtypes = [vp, vp, sz, i32, C.POINTER(vp)]
        getattr(L, f"bvhgpu_build_dev_{s}").argtypes = [vp, vp, sz, i32, C.POINTER(vp)]
        getattr(L, f"bvhgpu_tree_from_nodes_{s}").argtypes = [vp, vp, sz, vp, sz, C.POINTER(vp)]
        getattr(L, f"bvhgpu_tree_free_{s}").argtypes = [vp]
        getattr(L, f"bvhgpu_tree_free_{s}").restype = None
        for f in ("num_shapes", "num_nodes"):
            getattr(L, f"bvhgpu_tree_{f}_{s}").argtypes = [vp]
            getattr(L, f"bvhgpu_tree_{f}_{s}").restype = sz
        getattr(L, f"bvhgpu_tree_nodes_{s}").argtypes = [vp, vp, vp]
        getattr(L, f"bvhgpu_flatten_{s}").argtypes = [vp, vp, sz, szp]
        getattr(L, f"bvhgpu_traverse_{s}").argtypes = [vp, i32, vp, sz, vp, vp, sz, szp]
        getattr(L, f"bvhgpu_traverse_fetch_{s}").argtypes = [vp, vp, sz]
        getattr(L, f"bvhgpu_tree_set_triangles_{s}").argtypes = [vp, vp, sz]
        getattr(L, f"bvhgpu_tree_set_triangles_dev_{s}").argtypes = [vp, vp, sz]
        getattr(L, f"bvhgpu_closest_hit_{s}").argtypes = [vp, vp, sz, i32, vp, vp, vp]
        getattr(L, f"bvhgpu_closest_hit_dev_{s}").argtypes = [vp, vp, i32, sz, i32, vp, vp, vp]
        getattr(L, f"bvhgpu_any_hit_{s}").argtypes = [vp, vp, sz, vp, i32, vp]
        getattr(L, f"bvhgpu_any_hit_dev_{s}").argtypes = [vp, vp, i32, sz, vp, i32, vp]
        getattr(L, f"bvhgpu_traverse_od_{s}").argtypes = [vp, i32, vp, sz, vp, vp, sz, szp]
        getattr(L, f"bvhgpu_traverse_od_dev_{s}").argtypes = [vp, i32, vp, sz, vp, vp, sz, szp]
        getattr(L, f"bvhgpu_refit_dev_{s}").argtypes = [vp, vp, sz]
        getattr(L, f"bvhgpu_update_{s}").argtypes = [vp, vp, vp, sz, C.c_double, C.POINTER(C.c_size_t)]
        getattr(L, f"bvhgpu_update_dev_{s}").argtypes = [vp, vp, vp, sz, C.c_double, C.POINTER(C.c_size_t)]
        getattr(L, f"bvhgpu_optimize_dev_{s}").argtypes = [vp, vp, sz, C.c_double, C.POINTER(C.c_size_t)]
        getattr(L, f"bvhgpu_traverse_dev_{s}").argtypes = [vp, i32, vp, sz, vp, vp, sz, szp]
        getattr(L, f"bvhgpu_traverse_stats_{s}").argtypes = [vp, u64p]
        getattr(L, f"bvhgpu_traverse_ordered_{s}").argtypes = [vp, vp, sz, i32, vp, vp, vp, sz, szp]
        getattr(L, f"bvhgpu_query_{s}").argtypes = [vp, i32, i32, vp, sz, vp, vp, sz, szp]
        getattr(L, f"bvhgpu_query_dev_{s}").argtypes = [vp, i32, i32, vp, sz, vp, vp, sz, szp]
        getattr(L, f"bvhgpu_traverse_sharded_dev_{s}").argtypes = [vp, i32, vp, sz, C.POINTER(Shard)]
        getattr(L, f"bvhgpu_rays_new_dev_{s}").argtypes = [vp, vp, vp, sz, vp]
        getattr(L, f"bvhgpu_sah_cost_{s}").argtypes = [vp, C.POINTER(C.c_double)]
        getattr(L, f"bvhgpu_refit_{s}").argtypes = [vp, vp, sz]
        getattr(L, f"bvhgpu_nearest_{s}").argtypes = [vp, C.c_int, vp, sz, vp, vp]
        getattr(L, f"bvhgpu_nearest_triangles_{s}").argtypes = [vp, C.c_int, vp, sz, vp, vp]
        getattr(L, f"bvhgpu_nearest_candidates_{s}").argtypes = [vp, vp, sz, vp, vp, sz, C.POINTER(C.c_size_t)]
        getattr(L, f"bvhgpu_optimize_{s}").argtypes = [vp, vp, sz, C.c_double, C.POINTER(C.c_size_t)]
        for f in ("add_shapes", "add_shapes_dev"):
            getattr(L, f"bvhgpu_{f}_{s}").argtypes = [vp, vp, sz, C.c_double, C.POINTER(C.c_size_t)]
        for f in ("remove_shapes", "remove_shapes_dev"):
            getattr(L, f"bvhgpu_{f}_{s}").argtypes = [vp, vp, sz]
    for s in ("f32x2", "f64x2"):
        getattr(L, f"bvhgpu_build_{s}").argtypes = [vp, vp, sz, i32, C.POINTER(vp)]
        getattr(L, f"bvhgpu_tree_free_{s}").argtypes = [vp]
        getattr(L, f"bvhgpu_tree_free_{s}").restype = None
        getattr(L, f"bvhgpu_tree_num_shapes_{s}").argtypes = [vp]
        getattr(L, f"bvhgpu_tree_num_shapes_{s}").restype = sz
        getattr(L, f"bvhgpu_tree_nodes_{s}").argtypes = [vp, vp, vp]
        getattr(L, f"bvhgpu_flatten_{s}").argtypes = [vp, vp, sz, szp]
        getattr(L, f"bvhgpu_traverse_{s}").argtypes = [vp, i32, vp, sz, vp, vp, sz, szp]
        getattr(L, f"bvhgpu_query_{s}").argtypes = [vp, i32, i32, vp, sz, vp, vp, sz, szp]
        getattr(L, f"bvhgpu_nearest_{s}").argtypes = [vp, i32, vp, sz, vp, vp]
        getattr(L, f"bvhgpu_nearest_candidates_{s}").argtypes = [vp, vp, sz, vp, vp, sz, szp]
        getattr(L, f"bvhgpu_refit_{s}").argtypes = [vp, vp, sz]
        getattr(L, f"bvhgpu_update_{s}").argtypes = [vp, vp, vp, sz, C.c_double, szp]
        getattr(L, f"bvhgpu_add_shapes_{s}").argtypes = [vp, vp, sz, C.c_double, szp]
        getattr(L, f"bvhgpu_remove_shapes_{s}").argtypes = [vp, vp, sz]
    for s in ("f32x2", "f64x2", "f32x4", "f64x4"):
        getattr(L, f"bvhgpu_traverse_ordered_{s}").argtypes = [vp, vp, sz, i32, vp, vp, vp, sz, szp]
        getattr(L, f"bvhgpu_closest_hit_{s}").argtypes = [vp, vp, sz, vp, vp]
        getattr(L, f"bvhgpu_any_hit_{s}").argtypes = [vp, vp, sz, vp, vp]
    for s in ("f32x2", "f64x2", "f32x3", "f64x3", "f32x4", "f64x4"):
        getattr(L, f"bvhgpu_knn_{s}").argtypes = [vp, vp, sz, C.c_uint32, vp, vp, vp]
    for s in ("f32x3", "f64x3", "f32x4", "f64x4"):
        getattr(L, f"bvhgpu_knn_dev_{s}").argtypes = [vp, vp, sz, C.c_uint32, vp, vp, vp]
    for s in ("f32x3", "f64x3"):
        getattr(L, f"bvhgpu_knn_triangles_{s}").argtypes = [vp, vp, sz, C.c_uint32, vp, vp, vp, vp]
        getattr(L, f"bvhgpu_knn_triangles_dev_{s}").argtypes = [vp, vp, sz, C.c_uint32, vp, vp, vp, vp]
        getattr(L, f"bvhgpu_multi_hit_{s}").argtypes = [vp, vp, sz, C.c_uint32, vp, i32, vp, vp, vp]
        getattr(L, f"bvhgpu_multi_hit_dev_{s}").argtypes = [vp, vp, i32, sz, C.c_uint32, vp, i32, vp, vp, vp]
        getattr(L, f"bvhgpu_count_hits_{s}").argtypes = [vp, vp, sz, vp, vp, vp]
        getattr(L, f"bvhgpu_count_hits_dev_{s}").argtypes = [vp, vp, i32, sz, vp, vp, vp]
        getattr(L, f"bvhgpu_contains_points_{s}").argtypes = [vp, vp, sz, i32, vp]
        getattr(L, f"bvhgpu_contains_points_dev_{s}").argtypes = [vp, vp, sz, i32, vp]
        getattr(L, f"bvhgpu_signed_distance_{s}").argtypes = [vp, vp, sz, i32, vp, vp, vp]
        getattr(L, f"bvhgpu_signed_distance_dev_{s}").argtypes = [vp, vp, sz, i32, vp, vp, vp]
    for s in ("f32x2", "f64x2", "f32x4", "f64x4"):
        getattr(L, f"bvhgpu_multi_hit_{s}").argtypes = [vp, vp, sz, C.c_uint32, vp, vp, vp]
    for s in ("f32x4", "f64x4"):
        getattr(L, f"bvhgpu_multi_hit_dev_{s}").argtypes = [vp, vp, sz, C.c_uint32, vp, vp, vp]
        getattr(L, f"bvhgpu_closest_hit_dev_{s}").argtypes = [vp, vp, sz, vp, vp]
        getattr(L, f"bvhgpu_any_hit_dev_{s}").argtypes = [vp, vp, sz, vp, vp]
        for f in ("add_shapes", "add_shapes_dev"):
            getattr(L, f"bvhgpu_{f}_{s}").argtypes = [vp, vp, sz, C.c_double, szp]
        for f in ("remove_shapes", "remove_shapes_dev"):
            getattr(L, f"bvhgpu_{f}_{s}").argtypes = [vp, vp, sz]
        getattr(L, f"bvhgpu_refit_{s}").argtypes = [vp, vp, sz]
        getattr(L, f"bvhgpu_refit_dev_{s}").argtypes = [vp, vp, sz]
        getattr(L, f"bvhgpu_update_{s}").argtypes = [vp, vp, vp, sz, C.c_double, szp]
        getattr(L, f"bvhgpu_update_dev_{s}").argtypes = [vp, vp, vp, sz, C.c_double, szp]
        getattr(L, f"bvhgpu_build_{s}").argtypes = [vp, vp, sz, i32, C.POINTER(vp)]
        getattr(L, f"bvhgpu_tree_free_{s}").argtypes = [vp]
        getattr(L, f"bvhgpu_tree_free_{s}").restype = None
        getattr(L, f"bvhgpu_tree_num_shapes_{s}").argtypes = [vp]
        getattr(L, f"bvhgpu_tree_num_shapes_{s}").restype = sz
        getattr(L, f"bvhgpu_tree_nodes_{s}").argtypes = [vp, vp, vp]
        getattr(L, f"bvhgpu_flatten_{s}").argtypes = [vp, vp, sz, szp]
        getattr(L, f"bvhgpu_traverse_{s}").argtypes = [vp, i32, vp, sz, vp, vp, sz, szp]
        getattr(L, f"bvhgpu_traverse_dev_{s}").argtypes = [vp, i32, vp, sz, vp, vp, sz, szp]
        getattr(L, f"bvhgpu_query_{s}").argtypes = [vp, i32, i32, vp, sz, vp, vp, sz, szp]
        getattr(L, f"bvhgpu_query_dev_{s}").argtypes = [vp, i32, i32, vp, sz, vp, vp, sz, szp]
        getattr(L, f"bvhgpu_nearest_{s}").argtypes = [vp, i32, vp, sz, vp, vp]
        getattr(L, f"bvhgpu_nearest_candidates_{s}").argtypes = [vp, vp, sz, vp, vp, sz, szp]
    for s in ("f32x2", "f64x2", "f32x3", "f64x3", "f32x4", "f64x4"):
        getattr(L, f"bvhgpu_overlap_pairs_{s}").argtypes = [vp, vp, vp, sz, szp]
        getattr(L, f"bvhgpu_overlap_trees_{s}").argtypes = [vp, vp, vp, vp, sz, szp]
    for s in ("f32x3", "f64x3", "f32x4", "f64x4"):
        getattr(L, f"bvhgpu_overlap_pairs_dev_{s}").argtypes = [vp, vp, vp, sz, szp]
        getattr(L, f"bvhgpu_overlap_trees_dev_{s}").argtypes = [vp, vp, vp, vp, sz, szp]
    missing =[n for n in declared_symbols() if not hasattr(L, n)]
    if missing:
        raise ImportError(f"{SO_PATH} does not export {missing}")
    _lib = L
    return L


def check(status: int) -> None:
    if status != OK:
        raise BvhGpuError(status, lib().bvhgpu_last_error().decode("utf-8", "replace"))
