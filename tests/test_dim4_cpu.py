"""D = 4 checks that need no device: the 4-D PODs of the C ABI against the numpy dtypes, the 14 new entry points, and the
embedding identity the GPU tests rely on -- a 3-D scene lifted to 4-D with a constant w = [c, c] builds the same tree."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from tests import pyref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES4 = [f"bvhgpu_{f}_{s}" for s in ("f32x4", "f64x4")
          for f in ("build", "tree_free", "tree_num_shapes", "tree_nodes", "flatten", "traverse", "traverse_dev")]


def test_4d_pod_sizes_match_the_header_compiled_with_gcc():
    from bvh_b200 import dtypes as D

    names = ["bvh_aabb4f", "bvh_ray4f", "bvh_node4f", "bvh_flat4f", "bvh_aabb4d", "bvh_ray4d", "bvh_node4d", "bvh_flat4d"]
    src = '#include <stdio.h>\n#include "bvh_b200.h"\nint main(void) {\n' + "".join(
        f'    printf("%zu ", sizeof({n}));\n' for n in names) + "    return 0;\n}\n"
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "s.c"), os.path.join(d, "s")
        open(c, "w").write(src)
        subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), c, "-o", exe], check=True)
        sizes = [int(x) for x in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    assert sizes == [32, 48, 80, 44, 64, 96, 144, 80]
    dts = [D.AABB4F, D.RAY4F, D.NODE4F, D.FLAT4F, D.AABB4D, D.RAY4D, D.NODE4D, D.FLAT4D]
    assert [t.itemsize for t in dts] == sizes
    assert D.BY_PREC_4D["f32"]["suffix"] == "f32x4" and D.BY_PREC_4D["f64"]["node"] is D.NODE4D


def test_header_declares_the_14_entry_points_of_d4():
    from bvh_b200 import capi

    assert len(NAMES4) == 14
    assert set(NAMES4) <= set(capi.declared_symbols())


def _scene3(kind, n, F, rng):
    mn = np.zeros((n, 3)); mx = np.zeros((n, 3))
    if kind == "random":
        mn = rng.uniform(-100, 100, (n, 3)); mx = mn + rng.uniform(0, 8, (n, 3)) ** 2 / 8
    elif kind == "coincident":
        mn[:] = [1.0, 2.0, 3.0]; mx[:] = [1.0, 2.0, 3.0]
    elif kind == "overflow":                                 # f32 surface areas overflow: empty child boxes, halving children
        c = rng.uniform(-3e19, 3e19, (n, 3)); mn, mx = c - 1e18, c + 1e18
    return [{"min": [F(v) for v in a], "max": [F(v) for v in b]} for a, b in zip(mn, mx)]


def _lift(aabbs, F, c):
    return [{"min": a["min"] + [F(c)], "max": a["max"] + [F(c)]} for a in aabbs]


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("kind", ["random", "coincident", "overflow"])
def test_a_constant_fourth_axis_does_not_change_the_tree(kind, prec):
    """w = [c, c] for every shape adds an exact +0 to every surface area and never wins largest_axis, so the 4-D restatement builds
    the 3-D tree: same node indices, parents, children, node_index and xyz boxes; children's w is [c, c], or empty where the 3-D box is
    empty.  The 3-D tree is also the C++ oracle's."""
    from oracle import oracle as O

    F = np.float32 if prec == "f32" else np.float64
    rng = np.random.default_rng(600 + len(kind))
    a3 = _scene3(kind, 600, F, rng)
    n3, i3 = pyref.build(a3, F)
    n4, i4 = pyref.build(_lift(a3, F, 1.5), F)
    assert i4 == i3
    for w3, w4 in zip(n3, n4):
        assert w4[:4] == w3[:4]
        if w3[0] == "node":
            for b3, b4 in ((w3[4], w4[4]), (w3[5], w4[5])):
                assert b4[0][:3] == b3[0] and b4[1][:3] == b3[1]
                empty = b3[0][0] == F(np.inf)
                assert (b4[0][3], b4[1][3]) == ((F(np.inf), F(-np.inf)) if empty else (F(1.5), F(1.5)))
    arr = np.zeros(len(a3), dtype=O.AABB3F if prec == "f32" else O.AABB3D)
    arr["min"] = [a["min"] for a in a3]; arr["max"] = [a["max"] for a in a3]
    want = O.build(arr, prec)
    assert list(want.node_index) == i3
    for i, w in enumerate(n3):
        nd = want.nodes[i]
        assert int(nd["parent"]) == w[1]
        if w[0] == "leaf":
            assert int(nd["child_l"]) == pyref.U32_MAX and int(nd["shape"]) == w[2]
        else:
            assert (int(nd["child_l"]), int(nd["child_r"])) == (w[2], w[3])
            assert list(nd["l_aabb"]["min"]) == w[4][0] and list(nd["r_aabb"]["max"]) == w[5][1]
