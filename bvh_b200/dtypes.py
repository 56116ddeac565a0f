"""numpy views of the C-ABI PODs declared in include/bvh_b200.h."""
import numpy as np

U32_MAX = 0xFFFFFFFF


def _make(f, dims=3):
    aabb = np.dtype([("min", f, (dims,)), ("max", f, (dims,))])
    ray = np.dtype([("origin", f, (dims,)), ("direction", f, (dims,)), ("inv_direction", f, (dims,))])
    node = np.dtype([("parent", "<u4"), ("child_l", "<u4"), ("child_r", "<u4"), ("shape", "<u4"), ("l_aabb", aabb), ("r_aabb", aabb)])
    flat_size = {(3, "<f4"): 36, (3, "<f8"): 64, (2, "<f4"): 28, (2, "<f8"): 48, (4, "<f4"): 44, (4, "<f8"): 80}[(dims, f)]
    flat = np.dtype(
        {
            "names": ["aabb", "entry_index", "exit_index", "shape_index"],
            "formats": [aabb, "<u4", "<u4", "<u4"],
            "offsets": [0, aabb.itemsize, aabb.itemsize + 4, aabb.itemsize + 8],
            "itemsize": flat_size,
        }
    )
    return aabb, ray, node, flat


AABB3F, RAY3F, NODE3F, FLAT3F = _make("<f4")
AABB3D, RAY3D, NODE3D, FLAT3D = _make("<f8")

AABB2F, RAY2F, NODE2F, FLAT2F = _make("<f4", 2)
AABB2D, RAY2D, NODE2D, FLAT2D = _make("<f8", 2)
BY_PREC_2D = {
    "f32": dict(scalar=np.float32, aabb=AABB2F, ray=RAY2F, node=NODE2F, flat=FLAT2F, suffix="f32x2"),
    "f64": dict(scalar=np.float64, aabb=AABB2D, ray=RAY2D, node=NODE2D, flat=FLAT2D, suffix="f64x2"),
}
assert AABB2F.itemsize == 16 and RAY2F.itemsize == 24 and NODE2F.itemsize == 48 and FLAT2F.itemsize == 28
assert AABB2D.itemsize == 32 and RAY2D.itemsize == 48 and NODE2D.itemsize == 80 and FLAT2D.itemsize == 48

AABB4F, RAY4F, NODE4F, FLAT4F = _make("<f4", 4)
AABB4D, RAY4D, NODE4D, FLAT4D = _make("<f8", 4)
BY_PREC_4D = {
    "f32": dict(scalar=np.float32, aabb=AABB4F, ray=RAY4F, node=NODE4F, flat=FLAT4F, suffix="f32x4"),
    "f64": dict(scalar=np.float64, aabb=AABB4D, ray=RAY4D, node=NODE4D, flat=FLAT4D, suffix="f64x4"),
}
assert AABB4F.itemsize == 32 and RAY4F.itemsize == 48 and NODE4F.itemsize == 80 and FLAT4F.itemsize == 44
assert AABB4D.itemsize == 64 and RAY4D.itemsize == 96 and NODE4D.itemsize == 144 and FLAT4D.itemsize == 80

BY_PREC = {
    "f32": dict(scalar=np.float32, aabb=AABB3F, ray=RAY3F, node=NODE3F, flat=FLAT3F, suffix="f32x3"),
    "f64": dict(scalar=np.float64, aabb=AABB3D, ray=RAY3D, node=NODE3D, flat=FLAT3D, suffix="f64x3"),
}
assert AABB3F.itemsize == 24 and RAY3F.itemsize == 36 and NODE3F.itemsize == 64 and FLAT3F.itemsize == 36
assert AABB3D.itemsize == 48 and RAY3D.itemsize == 72 and NODE3D.itemsize == 112 and FLAT3D.itemsize == 64
