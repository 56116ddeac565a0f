"""The in-place rebuild of optimize / update_shapes is exactly Bvh::build of each rebuilt subtree's shapes (DESIGN §4.5, §4.12): the
device equals tests/rebuildref.py -- integers bit for bit, coordinates with ==, node_index and the `rebuilt` count -- for D = 2, 3 and
4, f32 and f64, in every form that exists for the dimension: Bvh.optimize (3-D), update_shapes with host pointers, and the
device-pointer update (3-D and 4-D).  Every case first asserts, from the restated result, that it reaches what it is about.
Run on an H100:  python -m pytest tests/test_gpu_rebuild_exact.py -m gpu"""
import ctypes as C

import numpy as np
import pytest

from tests import rebuildref as RR

pytestmark = pytest.mark.gpu
PRECS = ("f32", "f64")
FORMS = {2: ("update",), 3: ("optimize", "update", "update_dev"), 4: ("update", "update_dev")}
REGIONS = {2: (1500, 300, 200, 120, 80, 40), 3: (1500, 300, 200, 120, 80, 40), 4: (800, 60)}     # scrambled regions per call


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A

    return A


class _Dev:
    """One device tree of dimension D behind the three forms of the step."""

    def __init__(self, api, D, a, prec):
        self.D, self.prec = D, prec
        self.b = {2: api.Bvh2, 3: api.Bvh, 4: api.Bvh4}[D].build(a, prec=prec)

    def state(self):
        if self.D == 3:
            self.b._nodes = self.b._node_index = None
            return self.b.nodes, self.b.node_index
        return self.b.nodes_and_index()

    def step(self, form, changed, a, mg):
        import torch

        from bvh_b200 import capi

        if form == "optimize":
            return self.b.optimize(a, mg)
        if form == "update":
            return self.b.update_shapes(changed, a, max_growth=mg)
        d_idx = torch.from_numpy(np.ascontiguousarray(changed, dtype=np.uint32).view(np.int32)).to("cuda")
        d_box = torch.from_numpy(np.ascontiguousarray(a[changed]).view(np.uint8)).to("cuda")
        torch.cuda.synchronize()
        if self.D == 4:
            return self.b.update_dev(d_idx.data_ptr(), d_box.data_ptr(), len(changed), max_growth=mg)
        rb = C.c_size_t(0)
        capi.check(getattr(capi.lib(), f"bvhgpu_update_dev_{self.b._d['suffix']}")(self.b._h, C.c_void_p(d_idx.data_ptr()), C.c_void_p(d_box.data_ptr()),
                                                                                  len(changed), C.c_double(mg), C.byref(rb)))
        return int(rb.value)

    def free(self):
        self.b.free()


def _restate(t, form, changed, a, mg):
    return t.optimize(a, mg) if form == "optimize" else t.update(changed, a, mg)


def _assert_same(dev, t, what):
    nodes, idx = dev.state()
    assert np.array_equal(idx, t.node_index), (what, "node_index")
    for f in ("parent", "child_l", "child_r", "shape"):
        bad = np.flatnonzero(nodes[f] != t.nodes[f])
        assert len(bad) == 0, (what, f, bad[:8].tolist())
    for side in ("l_aabb", "r_aabb"):
        for mm in ("min", "max"):                             # == : only the sign of a zero may differ (DESIGN §2)
            bad = np.flatnonzero(np.any(nodes[side][mm] != t.nodes[side][mm], axis=1))
            assert len(bad) == 0, (what, side, mm, bad[:8].tolist())


def _step_both(dev, t, form, changed, a, mg, what):
    want = _restate(t, form, changed, a, mg)
    got = dev.step(form, changed, a, mg)
    assert got == want, (what, got, want)
    _assert_same(dev, t, what)
    return t.facts


def _start(api, D, a, prec):
    dev = _Dev(api, D, a, prec)
    return dev, RR.Tree(*dev.state())


def _sizes(facts):
    return [r["count"] for r in facts["roots"]]


# ---- roots of every size -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("D,form", [(D, f) for D in (2, 3, 4) for f in FORMS[D]])
def test_rebuilt_subtrees_of_every_size_are_build_of_their_shapes(api, D, form, prec):
    """3-D / 2-D: roots of <= 16 shapes (in-register subtrees), 17-512 (SEG) and > 512 (gangs or BIN / SCATTER tiles);
    4-D: roots of <= 256 shapes (small4_kernel) and > 512 (several tiles of the seeded level loop), with w winning largest_axis."""
    rng = np.random.default_rng(100 * D + len(form))
    n = 8000 if D == 4 else 20000
    a = RR.random_scene(n, D, prec, rng, w_scale=3.0)
    dev, t = _start(api, D, a, prec)
    seen = []
    for call in range(2):                                     # the second call runs against the baseline the first one refreshed
        changed, a = RR.mixed_motion(a, rng, regions=REGIONS[D])
        facts = _step_both(dev, t, form, changed, a, 1.5, (D, form, prec, call))
        seen.append(facts)
    _assert_root_sizes(D, seen)
    dev.free()


def _assert_root_sizes(D, seen):
    """Every call rebuilds a root of more than 512 shapes; the small class (and for D < 4 the middle class) appear in some call."""
    for facts in seen:
        assert max(_sizes(facts)) > 512
    assert any(k <= (256 if D == 4 else 16) for f in seen for k in _sizes(f))
    if D == 4:
        assert any(r["axis"] == 3 for f in seen for r in f["roots"])
    else:
        assert any(16 < k <= 512 for f in seen for k in _sizes(f))


@pytest.mark.parametrize("small,subtree,gang", [(0, 0, 0), (0, 1, 0), (0, 0, 1), (0, 1, 1), (1, 1, 1), (1, 0, 1)])
@pytest.mark.parametrize("prec", PRECS)
def test_rebuild_is_exact_under_every_builder_strategy(api, prec, small, subtree, gang):
    """rebuild_subtrees picks its own small / subtree / gang settings; every combination must give the restated subtrees."""
    rng = np.random.default_rng(7)
    a = RR.random_scene(20000, 3, prec, rng)
    ctx = api.Context.default()
    ctx.set_option("build_small", small); ctx.set_option("build_subtree", subtree); ctx.set_option("build_gang", gang)
    try:
        dev, t = _start(api, 3, a, prec)
        seen = []
        for form in ("optimize", "update"):
            changed, a = RR.mixed_motion(a, rng)
            seen.append(_step_both(dev, t, form, changed, a, 1.5, (form, small, subtree, gang)))
        _assert_root_sizes(3, seen)
        dev.free()
    finally:
        ctx.set_option("build_small", -1); ctx.set_option("build_subtree", -1); ctx.set_option("build_gang", -1)


def test_rebuild_of_a_large_scene_without_gangs(api):
    """1.2 M shapes (test_optimize_large_scene_without_gangs' scene and motion): roots above 512 shapes run as queue-mode tile tasks."""
    from bvh_b200 import scenes as S

    a = S.create_n_cubes_aabbs(100000).copy()
    dev, t = _start(api, 3, a, "f32")
    rng = np.random.default_rng(21)
    for form in ("optimize", "update"):
        mv = np.sort(rng.choice(len(a), len(a) // 20, replace=False)).astype(np.uint32)
        dl = rng.uniform(-3000.0, 3000.0, (len(mv), 3)).astype(np.float32)
        a = a.copy()
        a["min"][mv] += dl
        a["max"][mv] += dl
        s = _sizes(_step_both(dev, t, form, mv, a, 1.5, form))
        assert max(s) > 512 and min(s) <= 16, (len(s), max(s))
    dev.free()


def test_4d_update_with_more_than_1024_roots(api):
    """1.2 M random 4-D boxes, 1 % of them jittered by about their own size: thousands of small roots in one call, so root_tiles4's
    tile_scan1024 runs over more than one chunk of 1 024 roots."""
    rng = np.random.default_rng(12)
    a = RR.random_scene(1_200_000, 4, "f32", rng)
    dev, t = _start(api, 4, a, "f32")
    changed = np.sort(rng.choice(len(a), len(a) // 100, replace=False)).astype(np.uint32)
    a = RR.jitter(a, changed, 4.0, rng)
    facts = _step_both(dev, t, "update", changed, a, 1.5, "1.2M")
    assert len(facts["roots"]) > 1024, len(facts["roots"])
    dev.free()


# ---- leaf order ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("D", [2, 3, 4])
def test_leaf_order_decides_the_halving_branch(api, D, prec):
    """Clusters of coincident centres: rebuilt subtrees halve by position, so the shapes must reach the builder in leaf order."""
    rng = np.random.default_rng(D)
    a = RR.clustered_scene(6000, D, prec, rng)
    dev, t = _start(api, D, a, prec)
    for form in FORMS[D]:
        changed, a = RR.mixed_motion(a, rng, regions=(400, 60), singles=30, single_scale=3.0)
        facts = _step_both(dev, t, form, changed, a, 1.5, (D, form))
        assert RR.halving_pairs(t.nodes, a, facts["roots"]) > 0
    dev.free()


# ---- overflow-scale scenes ------------------------------------------------------------------------------------------------------
def _overflow_scene(kind, D, prec):
    from tests import dimref
    from tests.edge_inputs import edge_scene

    if kind == "overflow":
        mn, mx = dimref.scene("overflow", 3000, D, RR._F(prec), np.random.default_rng(9))
        return RR.make_boxes(mn, mx, D, prec)
    return np.ascontiguousarray(edge_scene(kind, 3000, prec), dtype=RR.aabb_dtype(3, prec))


def overflow_motion(a, rng, prec):
    """60 unit-scale boxes jittered inside their clusters and 30 overflow-scale boxes moved at their own scale."""
    sizes = (a["max"].astype(np.float64) - a["min"].astype(np.float64)).max(axis=1)
    small, big = np.flatnonzero(sizes < 10), np.flatnonzero(sizes >= 10)
    s = rng.choice(small, min(len(small), 60), replace=False)
    g = rng.choice(big, 30, replace=False)
    a = RR.jitter(a, s, 20.0, rng)
    a = RR.jitter(a, g, float(np.median(sizes[big])) * 3, rng)
    return np.sort(np.concatenate([s, g])).astype(np.uint32), a


@pytest.mark.parametrize("kind,D,prec", [("huge", 3, "f32"), ("huge", 3, "f64"), ("mixed", 3, "f32"), ("mixed", 3, "f64"), ("overflow", 4, "f32")])
def test_overflow_scale_scenes(api, kind, D, prec):
    """"No split wins" nodes store empty child boxes.  In the incremental form a root's off-path slot may still hold one, and the
    rebuild is seeded with the join of the root's two stored slots, not with the joint box of its shapes (DESIGN §4.5): the mixed
    scenes reach roots where the two differ."""
    differs = overflow_frames(kind, D, prec, lambda form, b: _start(api, D, b, prec), _step_both)
    if kind == "mixed":
        assert differs > 0


def overflow_frames(kind, D, prec, start, step):
    """Six frames of overflow_motion per form, each form on a fresh tree; returns how many incremental-form roots were seeded with a
    box other than the joint box of their shapes."""
    rng = np.random.default_rng(8)
    a = _overflow_scene(kind, D, prec)
    differs = 0
    for form in FORMS[D]:
        b = a
        dev, t = start(form, b)
        before = t.nodes.copy()
        rebuilt = 0
        for frame in range(6):
            changed, b = overflow_motion(b, rng, prec)
            facts = step(dev, t, form, changed, b, 1.5, (kind, form, frame))
            differs += facts["seed_differs"] if form != "optimize" else 0
            assert form != "optimize" or facts["seed_differs"] == 0        # a full refit leaves every seed tight
            rebuilt += len(facts["roots"])
        assert t.nodes.tobytes() != before.tobytes()           # the climb replaced empty boxes, or roots were rebuilt
        assert kind != "mixed" or rebuilt > 0
        if dev is not None:
            dev.free()
    return differs


# ---- drift: the carried baseline and its refresh --------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("D", [2, 3, 4])
def test_drift_over_frames_with_every_max_growth(api, D, prec):
    """16 frames of drift on one tree: 3-D alternates optimize with the two update forms, 2-D and 4-D repeat update_shapes (4-D:
    host and device pointers in turn); max_growth cycles through 1.0, 1.5, 0 (boxes only) and 1e30 (never degraded), and one frame
    sends a repeated index with an identical box."""
    rng = np.random.default_rng(50 + D)
    n = 3000
    a = RR.random_scene(n, D, prec, rng)
    dev, t = _start(api, D, a, prec)
    vel = rng.uniform(-6, 6, (n, D))
    F = RR._F(prec)
    total, with_base = 0, 0
    for frame in range(16):
        changed = np.sort(rng.choice(n, 300, replace=False)).astype(np.uint32)
        a = a.copy()
        a["min"][changed] = (a["min"][changed] + vel[changed]).astype(F)
        a["max"][changed] = (a["max"][changed] + vel[changed]).astype(F)
        if frame == 5:
            changed = np.concatenate([changed, changed[:3], changed[:1]])
        mg = (1.0, 1.5, 0.0, 1e30)[frame % 4]
        forms = FORMS[D]
        form = forms[frame % len(forms)]
        if form == "optimize" and mg <= 0:
            form = "update"
        r = _step_both(dev, t, form, changed, a, mg, (D, prec, frame, form, mg))
        total += sum(_sizes(r))
        with_base += t.base is not None
    assert total > 0 and with_base > 0
    dev.free()
