"""CPU checks of the 2-D and 4-D add_shapes / remove_shapes entry points: the header declares all twelve, the library exports them,
the ctypes table types them, and the Python wrappers reach every one of them."""
import subprocess

SYMBOLS = [f"bvhgpu_{op}_{p}x{d}" for d in (2, 4) for p in ("f32", "f64") for op in ("add_shapes", "remove_shapes")] + \
          [f"bvhgpu_{op}_dev_{p}x4" for p in ("f32", "f64") for op in ("add_shapes", "remove_shapes")]


def test_twelve_entry_points_are_declared_and_exported():
    from bvh_b200 import capi

    assert len(SYMBOLS) == 12
    declared = set(capi.declared_symbols())
    assert set(SYMBOLS) <= declared
    L = capi.lib()
    for s in SYMBOLS:
        assert getattr(L, s).argtypes, s                       # typed in bvh_b200/capi.py
    out = subprocess.run(["nm", "-D", "--defined-only", capi.SO_PATH], capture_output=True, text=True).stdout
    exported = {l.split()[-1] for l in out.splitlines() if " T " in l}
    assert set(SYMBOLS) <= exported
    assert not any(f"bvhgpu_{op}_dev_{p}x2" in declared for p in ("f32", "f64") for op in ("add_shapes", "remove_shapes"))   # host-only


def test_python_wrappers():
    from bvh_b200 import api

    for name in ("add_shapes", "remove_shapes"):
        assert getattr(api.Bvh2, name) is getattr(api.Bvh4, name)
    for name in ("add_shapes_dev", "remove_shapes_dev"):
        assert hasattr(api.Bvh4, name) and not hasattr(api.Bvh2, name)


# ---- tests/dimdyn.py: the dimension-generic restatement of add_shape / remove_shape ----------------------------------------------
import numpy as np  # noqa: E402
import pytest  # noqa: E402

from tests import dimdyn, dynoracle  # noqa: E402

U32_MAX = 0xFFFFFFFF


def _scene3(prec, n, rng):
    from oracle import oracle as O

    mn = rng.uniform(-100, 100, (n, 3))
    return O.make_aabbs(mn, mn + rng.uniform(0, 6, (n, 3)), prec)


def _new3(prec, k, rng):
    """Boxes inside the scene, far away (the merge branch), degenerate points and overflow-scale boxes, in turn."""
    from oracle import oracle as O

    mn = np.zeros((k, 3)); mx = np.zeros((k, 3))
    for j in range(k):
        kind = j % 4
        if kind == 0:
            mn[j] = rng.uniform(-100, 100, 3); mx[j] = mn[j] + rng.uniform(0, 6, 3)
        elif kind == 1:
            mn[j] = rng.uniform(-100, 100, 3) * 1e4; mx[j] = mn[j] + rng.uniform(0, 6, 3)
        elif kind == 2:
            mn[j] = mx[j] = rng.integers(-5, 5, 3)
        else:
            mn[j] = rng.uniform(-1e30, 1e30, 3); mx[j] = mn[j] + 1e29
    return O.make_aabbs(mn, mx, prec)


def _lift_tree(nodes, ni, shapes, D, prec, w=1.5):
    """The 3-D tree and shapes with z = 0 dropped (D = 2) or a constant w = [c, c] appended (D = 4); leaves keep empty slots."""
    from bvh_b200.dtypes import BY_PREC_2D, BY_PREC_4D

    tab = (BY_PREC_2D if D == 2 else BY_PREC_4D)[prec]
    out = np.zeros(len(nodes), dtype=tab["node"])
    for f in ("parent", "child_l", "child_r", "shape"):
        out[f] = nodes[f]
    leaf = nodes["child_l"] == U32_MAX
    for side in ("l_aabb", "r_aabb"):
        for mm, fill in (("min", np.inf), ("max", -np.inf)):
            out[side][mm][:, :min(D, 3)] = nodes[side][mm][:, :min(D, 3)]
            if D == 4:
                out[side][mm][:, 3] = np.where(leaf, fill, w)
    a = np.zeros(len(shapes), dtype=tab["aabb"])
    for mm in ("min", "max"):
        a[mm][:, :min(D, 3)] = shapes[mm][:, :min(D, 3)]
        if D == 4:
            a[mm][:, 3] = w
    return out, np.array(ni, dtype=np.uint32), a


def _same_projected(n3, nd, D):
    assert np.array_equal(n3[["parent", "child_l", "child_r", "shape"]].tolist(), nd[["parent", "child_l", "child_r", "shape"]].tolist())
    for side in ("l_aabb", "r_aabb"):
        for mm in ("min", "max"):
            assert np.array_equal(n3[side][mm][:, :min(D, 3)], nd[side][mm][:, :min(D, 3)])


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_restatement_equals_the_oracle_at_d3(prec):
    from oracle import oracle as O

    rng = np.random.default_rng(3)
    shapes = _scene3(prec, 300, rng)
    want = O.build(shapes, prec)
    new = _new3(prec, 80, rng)
    allshapes = np.concatenate([shapes, new])
    # single adds, one after the other
    dyn = dimdyn.Dyn(want.nodes, want.node_index, shapes)
    dyn.add_many(new)
    got_nodes, got_ni = dyn.canonical()
    ref_nodes, ref_ni = dynoracle.add_shapes(want.nodes, want.node_index, allshapes, len(new), prec)
    assert dynoracle.same_tree(got_nodes, ref_nodes) and np.array_equal(got_ni, ref_ni)
    assert dyn.merges > 0                                        # the far boxes take the merge branch
    # batched removes, in the caller's order, renumbered by the swap rule
    nodes, ni, cur = ref_nodes, ref_ni, allshapes
    for k in (1, 2, 37, 150, None):
        k = len(cur) - 1 if k is None else k
        idx = rng.choice(len(cur), k, replace=False).astype(np.uint32)
        dyn = dimdyn.Dyn(nodes, ni, cur)
        moves = dyn.remove(idx)
        got_nodes, got_ni = dyn.canonical()
        nodes, ni, cur = dynoracle.remove_shapes(nodes, ni, cur, idx, prec)
        assert np.array_equal(moves, dynoracle.swap_moves(len(dyn.shapes) + k, idx))
        assert dynoracle.same_tree(got_nodes, nodes) and np.array_equal(got_ni, ni), k
        assert np.array_equal(dyn.shape_array(cur.dtype).tobytes(), cur.tobytes())
    dyn = dimdyn.Dyn(nodes, ni, cur)                             # the last shape goes: the empty tree, then an add builds a leaf
    dyn.remove([0])
    assert len(dyn.canonical()[0]) == 0
    dyn.add(cur["min"][0], cur["max"][0])
    n1, i1 = dyn.canonical()
    assert len(n1) == 1 and n1["child_l"][0] == U32_MAX and i1.tolist() == [0]


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("D", [2, 4])
def test_restatement_in_d2_and_d4_equals_its_d3_result(D, prec):
    """D = 2 on the z = 0 lift and D = 4 with a constant w: the same topology and the same boxes in the shared axes."""
    from oracle import oracle as O

    rng = np.random.default_rng(D)
    shapes = _scene3(prec, 250, rng)
    shapes["min"][:, 2] = shapes["max"][:, 2] = 0 if D == 2 else shapes["min"][:, 2]
    want = O.build(shapes, prec)
    new = _new3(prec, 60, rng)
    if D == 2:
        new["min"][:, 2] = new["max"][:, 2] = 0
    d3 = dimdyn.Dyn(want.nodes, want.node_index, shapes)
    nd, nid, sd = _lift_tree(want.nodes, want.node_index, shapes, D, prec)
    dd = dimdyn.Dyn(nd, nid, sd)
    _, _, newd = _lift_tree(want.nodes[:0], [], new, D, prec)
    d3.add_many(new)
    dd.add_many(newd)
    n3, i3 = d3.canonical()
    nD, iD = dd.canonical()
    _same_projected(n3, nD, D)
    assert np.array_equal(i3, iD) and d3.merges == dd.merges > 0
    idx = rng.choice(len(d3.shapes), 120, replace=False)
    assert np.array_equal(d3.remove(idx), dd.remove(idx))
    n3, i3 = d3.canonical()
    nD, iD = dd.canonical()
    _same_projected(n3, nD, D)
    assert np.array_equal(i3, iD)
