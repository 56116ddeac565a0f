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


# C types of the header's parameters and return values.  Every other pointer parameter is c_void_p, and `T**` (an out-handle) is
# POINTER(c_void_p).  A type outside these tables raises instead of falling back to ctypes' int, which truncates pointers and sizes.
_ARG_TYPES = {"int": C.c_int, "size_t": C.c_size_t, "uint32_t": C.c_uint32, "int64_t": C.c_int64, "double": C.c_double,
              "size_t*": C.POINTER(C.c_size_t), "uint64_t*": C.POINTER(C.c_uint64), "const bvhgpu_shard*": C.POINTER(Shard),
              "const char*": C.c_char_p}
_RET_TYPES = {"int": C.c_int, "size_t": C.c_size_t, "uint64_t": C.c_uint64, "void": None, "const char*": C.c_char_p}


def _ctype(fn: str, ctype: str, table: dict, header: str):
    t = re.sub(r"\s*\*", "*", " ".join(ctype.split()))
    if t in table:
        return table[t]
    if table is _ARG_TYPES and t.endswith("*"):
        return C.POINTER(C.c_void_p) if t.endswith("**") else C.c_void_p
    raise ImportError(f"{header}: {fn} uses the C type {t!r}, which has no ctypes mapping in bvh_b200/capi.py")


def signatures(header: str = HEADER) -> dict:
    """{name: (restype, argtypes)} of every prototype `RET bvhgpu_name(PARAMS);` the header declares."""
    text = re.sub(r"/\*.*?\*/", "", open(header).read(), flags=re.S)
    out = {}
    for ret, name, params in re.findall(r"((?:const\s+)?\w+\s*\**)\s*\b(bvhgpu_[a-z0-9_]+)\s*\(([^()]*)\)\s*;", text):
        args = []
        for p in ([] if params.strip() in ("", "void") else params.split(",")):
            m = re.fullmatch(r"(.+?)\s*\b\w+", p.strip(), flags=re.S)                 # drop the parameter's name
            args.append(_ctype(name, m[1] if m else p, _ARG_TYPES, header))
        out[name] = (_ctype(name, ret, _RET_TYPES, header), args)
    unread = set(re.findall(r"\b(bvhgpu_[a-z0-9_]+)\s*\(", text)) - set(out)
    if unread:
        raise ImportError(f"{header}: cannot read the prototypes of {sorted(unread)}")
    return out


def declared_symbols() -> list[str]:
    """Every function include/bvh_b200.h declares."""
    return sorted(signatures())


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
    sigs = signatures()
    missing = [n for n in sorted(sigs) if not hasattr(L, n)]
    if missing:
        raise ImportError(f"{SO_PATH} does not export {missing}")
    for name, (restype, argtypes) in sigs.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
    _lib = L
    return L


def check(status: int) -> None:
    if status != OK:
        raise BvhGpuError(status, lib().bvhgpu_last_error().decode("utf-8", "replace"))
