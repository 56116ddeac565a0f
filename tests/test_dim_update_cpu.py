"""CPU checks behind refit and update_shapes for 2-D and 4-D trees:
- the header declares the 12 entry points and the library exports them;
- the dimension-generic invariant checker (tests/dimcheck.py) agrees with the C++ oracle's is_consistent / is_tight on 3-D node
  arrays: fresh builds, trees after the oracle's update_shapes (not in preorder), and deliberately broken arrays.  That makes it the
  checker of the 2-D and 4-D trees in tests/test_gpu_dim_update.py."""
import subprocess

import numpy as np
import pytest

from oracle import oracle as O
from tests import dimcheck

PRECS = ("f32", "f64")
NEW = [f"bvhgpu_{f}_{p}x{d}" for d in (2, 4) for p in ("f32", "f64") for f in ("refit", "update")]
NEW += [f"bvhgpu_{f}_dev_{p}x4" for p in ("f32", "f64") for f in ("refit", "update")]


def test_header_declares_and_the_library_exports_the_new_entry_points():
    from bvh_b200 import capi

    assert len(NEW) == 12
    assert set(NEW) <= set(capi.declared_symbols())
    L = capi.lib()
    assert all(hasattr(L, n) for n in NEW)
    out = subprocess.run(["nm", "-D", "--defined-only", capi.SO_PATH], capture_output=True, text=True).stdout
    assert set(NEW) <= {l.split()[-1] for l in out.splitlines() if " T " in l}


def _scene(kind, n, prec, rng):
    a = np.zeros(n, dtype=O.AABB3F if prec == "f32" else O.AABB3D)
    if kind == "random":
        mn = rng.uniform(-100, 100, (n, 3))
        a["min"], a["max"] = mn, mn + rng.uniform(0, 5, (n, 3))
    elif kind == "coincident":
        a["min"], a["max"] = [1, 2, 3], [1, 2, 3]
    elif kind == "cubes":
        a = O.create_n_cubes(n // 12 + 1, prec=prec)[:n]
    return a


def _agree(nodes, shapes, prec, want_consistent=None, want_tight=None):
    c, t = O.is_consistent(nodes, shapes, prec), O.is_tight(nodes, prec)
    assert dimcheck.is_consistent(nodes, shapes) == c
    assert dimcheck.is_tight(nodes) == t
    if want_consistent is not None:
        assert c == want_consistent
    if want_tight is not None:
        assert t == want_tight


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("kind,n", [("random", 1), ("random", 2), ("random", 500), ("coincident", 64), ("cubes", 1200)])
def test_checker_agrees_with_the_oracle_on_builds_and_updates(kind, n, prec):
    rng = np.random.default_rng(n + len(kind))
    shapes = _scene(kind, n, prec, rng)
    r = O.build(shapes, prec)
    _agree(r.nodes, shapes, prec, True, True)
    assert dimcheck.layout_ok(r.nodes, r.node_index)
    if n >= 3 and kind != "coincident":
        assert dimcheck.sah_cost(r.nodes) == pytest.approx(O.sah_cost(r.nodes, prec)[0], rel=1e-12)
    # the oracle's update_shapes (remove + re-insert): consistent and tight, but no longer in build's preorder layout
    moved = shapes.copy()
    changed = rng.choice(n, size=max(1, n // 10), replace=False).astype(np.uint32)
    moved["min"][changed] += 7.0
    moved["max"][changed] += 7.0
    nodes, node_index = O.update_shapes(r.nodes, r.node_index, moved, changed, prec)
    _agree(nodes, moved, prec)
    if n >= 2:
        _agree(r.nodes, moved, prec, want_consistent=False)        # the old tree does not hold the moved boxes


@pytest.mark.parametrize("prec", PRECS)
def test_checker_agrees_with_the_oracle_on_broken_arrays(prec):
    rng = np.random.default_rng(7)
    shapes = _scene("random", 300, prec, rng)
    r = O.build(shapes, prec)
    inner = np.flatnonzero(r.nodes["child_l"] != 0xFFFFFFFF)
    cases = []
    a = r.nodes.copy(); a["l_aabb"]["max"][inner[5], 1] -= 1.0; cases.append(a)           # a child box shrunk: not consistent
    a = r.nodes.copy(); a["l_aabb"]["min"][0, 0] -= 1.0; cases.append(a)                 # the root's left box grown: consistent, not tight
    a = r.nodes.copy(); a["parent"][inner[9]] = 0 if r.nodes["parent"][inner[9]] else 1; cases.append(a)   # a wrong parent field
    a = r.nodes.copy(); a["child_r"][inner[3]] = a["child_l"][inner[3]]; cases.append(a)  # a node reached twice
    a = r.nodes.copy(); a["l_aabb"]["min"][0, 2] = np.nan; cases.append(a)                # NaN at the root
    leaf = np.flatnonzero(r.nodes["child_l"] == 0xFFFFFFFF)
    a = r.nodes.copy(); a["shape"][leaf[0]], a["shape"][leaf[1]] = a["shape"][leaf[1]], a["shape"][leaf[0]]; cases.append(a)
    for a in cases:
        try:
            c = O.is_consistent(a, shapes, prec)
        except Exception:                                    # the oracle cannot walk every broken array: the checker must refuse it
            c = False
        assert dimcheck.is_consistent(a, shapes) == c
        if c:
            assert dimcheck.is_tight(a) == O.is_tight(a, prec)
    assert not dimcheck.is_consistent(cases[0], shapes) and dimcheck.is_consistent(cases[1], shapes) and not dimcheck.is_tight(cases[1])
    assert dimcheck.layout_ok(r.nodes, r.node_index) and not dimcheck.layout_ok(cases[5], r.node_index)
