"""CPU checks behind the 2-D and 4-D distance-ordered traversal and closest hit:
- the header declares the 10 entry points and the binding sees them;
- the dimension-generic restatement (tests/dimorder.py: slice, Tree.ordered, Tree.closest) equals the C++ oracle at D = 3, bit for bit
  through unsigned views: O.ray_slice, O.traverse (BVH semantics) stably sorted by the oracle's slice of the stored child box, and
  O.closest_hit in AABB mode.  Scenes: random, coincident and f32 overflow-scale (empty child boxes); rays: random, axis-aligned from
  box faces and corners (the NaN rule and +-0 exits), and -0.0 components.  That makes it the oracle of tests/test_gpu_dim_ordered.py
  in D = 2 and D = 4;
- the lift identity the 2-D embedding relies on holds in the restatement: a 2-D scene with z = [-1, +1] records and z = 0 origins with
  inv_direction.z = +inf gives the 2-D distances bit for bit."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import dimorder, dimref

PRECS = ("f32", "f64")
FT = {"f32": np.float32, "f64": np.float64}
UINT = {np.float32: np.uint32, np.float64: np.uint64}
NEW = [f"bvhgpu_{f}_{p}x{d}" for d in (2, 4) for p in ("f32", "f64") for f in ("traverse_ordered", "closest_hit")]
NEW += [f"bvhgpu_closest_hit_dev_{p}x4" for p in ("f32", "f64")]


def test_header_declares_the_new_entry_points():
    from bvh_b200 import capi

    assert len(NEW) == 10
    assert set(NEW) <= set(capi.declared_symbols())


def _bits(x, F):
    return np.asarray([x], dtype=F).view(UINT[F])[0]


def _oracle_scene(scene, n, prec, rng):
    F = FT[prec]
    mn, mx = dimref.scene(scene, n, 3, F, rng)
    shapes = np.zeros(n, dtype=O.AABB3F if prec == "f32" else O.AABB3D)
    shapes["min"], shapes["max"] = mn, mx
    nodes = O.build(shapes, prec).nodes
    o, d, inv = dimorder.rays(mn, mx, 150, F, rng)
    rays = np.zeros(len(o), dtype=O._DT[prec]["ray"])
    rays["origin"], rays["direction"], rays["inv_direction"] = o, d, inv
    return shapes, nodes, rays, o, inv


def _assert_ray_families(o, inv, shapes):
    """The batch holds what the docstring claims: -0 and infinite reciprocals, and origins exactly on a box face."""
    assert np.any(np.isinf(inv)) and np.any(np.signbit(inv) & np.isinf(inv))
    on_face = (o[:, None, :] == shapes["min"][None]) | (o[:, None, :] == shapes["max"][None])
    assert on_face.any()


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("scene", ["random", "coincident", "overflow"])
def test_slice_ordered_and_closest_equal_the_oracle_in_3d(scene, prec):
    F = FT[prec]
    rng = np.random.default_rng(21)
    shapes, nodes, rays, o, inv = _oracle_scene(scene, 300, prec, rng)
    _assert_ray_families(o, inv, shapes)
    if scene == "overflow" and prec == "f32":
        assert np.any(nodes["l_aabb"]["min"][:, 0] == np.inf)       # empty child boxes: entry 0 / exit inf for every ray
    tree = dimorder.Tree(nodes, shapes)
    # slice: every stored child box and every shape box, bit for bit (None = no intersection)
    boxes = [(nd[s]["min"], nd[s]["max"]) for nd in nodes for s in ("l_aabb", "r_aabb")][:200] + [(b["min"], b["max"]) for b in shapes[:100]]
    for i in range(len(rays)):
        ray = (list(o[i]), list(inv[i]))
        for mn, mx in boxes[:: 7]:
            want = O.ray_slice(rays[i], np.array([(mn, mx)], dtype=shapes.dtype), prec)
            got = dimorder.slice(ray, list(mn), list(mx))
            assert (got is None) == (want is None), (i, mn, mx)
            if got is not None:
                assert _bits(got[0], F) == _bits(want[0], F) and _bits(got[1], F) == _bits(want[1], F), (i, got, want)
    # ordered: the oracle's BVH set with its slices, stably sorted
    ref = O.traverse(nodes, shapes, rays, O.MODE_RECURSIVE, prec)
    lists = O.per_ray_lists(ref.offsets, ref.hits)
    leaf_box = {}
    for i, nd in enumerate(nodes):
        if nd["child_l"] != dimref.U32_MAX:
            leaf_box[int(nd["child_l"])] = nd["l_aabb"]; leaf_box[int(nd["child_r"])] = nd["r_aabb"]
    node_of = {int(nd["shape"]): i for i, nd in enumerate(nodes) if nd["child_l"] == dimref.U32_MAX}
    for i, lst in enumerate(lists):
        ray = (list(o[i]), list(inv[i]))
        if len(nodes) == 1:
            sl = [O.ray_slice(rays[i], shapes[int(s)], prec) for s in lst]
        else:
            sl = [O.ray_slice(rays[i], np.array([(leaf_box[node_of[int(s)]]["min"], leaf_box[node_of[int(s)]]["max"])], dtype=shapes.dtype), prec)
                  for s in lst]
        for ascending in (True, False):
            key = [s[0] if ascending else -s[1] for s in sl]
            order = sorted(range(len(lst)), key=lambda j: key[j])
            want = [(int(lst[j]), _bits(sl[j][0] if ascending else sl[j][1], F)) for j in order]
            got = [(int(s), _bits(d, F)) for s, d in tree.ordered(ray, ascending)]
            assert got == want, (i, ascending)
    # closest: O.closest_hit in AABB mode
    ws, wd, _ = O.closest_hit(nodes, shapes, rays, prec=prec)
    assert (ws != O.U32_MAX).sum() > (0 if scene == "coincident" else len(rays) // 10)      # point boxes: only exact aims hit
    for i in range(len(rays)):
        s, d = tree.closest((list(o[i]), list(inv[i])))
        assert s == ws[i], i
        assert _bits(np.inf if d is None else d, F) == _bits(wd[i], F), i


@pytest.mark.parametrize("prec", PRECS)
def test_z_lift_keeps_the_2d_slice(prec):
    """Records with z = [-1, +1] (and empty boxes, z = [+inf, -inf]) sliced by a ray with origin.z = 0, inv_direction.z = +inf give the
    2-D slice bit for bit: the z slab is (-inf, +inf), never NaN, and it is the last axis of the fold."""
    F = FT[prec]
    rng = np.random.default_rng(3)
    mn, mx = dimref.scene("random", 200, 2, F, rng)
    o, _, inv = dimorder.rays(mn, mx, 200, F, rng)
    boxes = [(list(mn[i]), list(mx[i])) for i in range(len(mn))] + [([F(np.inf)] * 2, [F(-np.inf)] * 2)]
    for i in range(len(o)):
        r2 = (list(o[i]), list(inv[i]))
        r3 = (list(o[i]) + [F(0)], list(inv[i]) + [F(np.inf)])
        for bmn, bmx in boxes[::5]:
            z = (F(-1), F(1)) if np.isfinite(bmn[0]) else (F(np.inf), F(-np.inf))
            a, b = dimorder.slice(r2, bmn, bmx), dimorder.slice(r3, bmn + [z[0]], bmx + [z[1]])
            assert (a is None) == (b is None)
            if a is not None:
                assert _bits(a[0], F) == _bits(b[0], F) and _bits(a[1], F) == _bits(b[1], F)
