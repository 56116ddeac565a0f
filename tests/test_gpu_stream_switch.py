"""A context's calls stay in order when its stream changes (bvhgpu_set_stream / bvhgpu_reset_stream).

Every case holds a producer back behind a spin of about 0.1 s on stream P, enqueues it, switches the context to stream Q and runs the
consumers there at once: nothing synchronises P between the producer and the consumers.  Outputs are read back only after the whole
device has been synchronised.  A consumer that did not wait for the producer reads the tree (or the triangles) as they were before.

Switch directions: the context's own stream -> a torch stream, a torch stream -> its own stream (reset_stream), torch stream A ->
torch stream B, and a torch stream -> CUDA's legacy stream 0.  The own stream has no handle outside the library, so the spin reaches
it through a torch feeder stream F: set_stream(F), spin on F, reset_stream(); "still pending" is then asked of F.

Expected values come from a twin tree on a second context that reaches the same state through host calls, each of which returns only
when its work is done.  The other suites hold those host calls to the models (oracle, tests/dimref.py, knnref, knntri, multihit,
anyhit, overlapref, crossref, dynoracle); the 3-D build here is also checked against the oracle directly.  Every case asserts that the
expected result before the producer differs from the one after it, so a consumer that read the old state would fail.

Producers that return before their work has run (build_dev, set_triangles_dev, the _dev walks of the free and synchronize cases) are
witnesses: the case asserts that P was still busy when the producer returned.  Producers that synchronise inside (host forms, and the
_dev refit / update / add / remove, whose box and index checks read a flag back) are ordering checks: they run the same way but
cannot show a pending producer.
Run on an H100:  python -m pytest tests/test_gpu_stream_switch.py -m gpu"""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O
from tests import dimref
from tests.edge_dims import ray_new, unit_directions

pytestmark = pytest.mark.gpu

LONG_SPIN = 200_000_000      # torch.cuda._sleep cycles ahead of the producer (~0.1 s on an H100)
DIRECTIONS = ("own_to_torch", "torch_to_own", "torch_a_to_b", "torch_to_legacy")
PRECS = ("f32", "f64")
N = 2000                     # shapes
NR = 1500                    # rays, points and queries


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A

    return A


@pytest.fixture(scope="module")
def twin_ctx(api):
    ctx = api.Context()
    yield ctx
    ctx.close()


def _F(prec):
    return np.float32 if prec == "f32" else np.float64


def _table(D):
    from bvh_b200.dtypes import BY_PREC, BY_PREC_2D, BY_PREC_4D

    return {2: BY_PREC_2D, 3: BY_PREC, 4: BY_PREC_4D}[D]


def _cls(api, D):
    return {2: api.Bvh2, 3: api.Bvh, 4: api.Bvh4}[D]


def _sfx(D, prec):
    return f"{prec}x{D}"


# ---- streams --------------------------------------------------------------------------------------------------------------------
class Switch:
    """A fresh context on stream P; `spin()` holds back the next call on P, `switch()` moves the context to Q."""

    def __init__(self, api, direction):
        import torch

        self.ctx = api.Context()
        self.direction = direction
        self.a, self.b, self.feeder = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
        self.p_handle = None if direction == "own_to_torch" else self.a.cuda_stream
        self.q_handle = {"own_to_torch": self.b.cuda_stream, "torch_to_own": None, "torch_a_to_b": self.b.cuda_stream,
                         "torch_to_legacy": 0}[direction]
        self.ctx.set_stream(self.p_handle)

    def spin(self):
        """LONG_SPIN ahead of whatever the context enqueues next on P; returns the torch stream that shows whether it is still busy."""
        import torch

        if self.p_handle is None:
            self.ctx.set_stream(self.feeder.cuda_stream)
            with torch.cuda.stream(self.feeder):
                torch.cuda._sleep(LONG_SPIN)
            self.ctx.set_stream(None)
            return self.feeder
        with torch.cuda.stream(self.a):
            torch.cuda._sleep(LONG_SPIN)
        return self.a

    def switch(self):
        self.ctx.set_stream(self.q_handle)

    def close(self):
        import torch

        torch.cuda.synchronize()
        self.ctx.close()


def _drain():
    import torch

    torch.cuda.synchronize()


# ---- scenes and inputs ----------------------------------------------------------------------------------------------------------
def _boxes(D, prec, n, seed, shift=0.0):
    rng = np.random.default_rng(seed)
    mn, mx = dimref.scene("random", n, D, np.float64, rng)
    a = np.zeros(n, dtype=_table(D)[prec]["aabb"])
    a["min"], a["max"] = mn + shift, mx + shift
    return a


def _moved(a, seed):
    """Every box moved by up to a third of the scene: a different tree state for every consumer."""
    rng = np.random.default_rng(seed)
    D = a["min"].shape[1]
    d = rng.uniform(-70, 70, (len(a), D))
    b = a.copy()
    b["min"] = a["min"] + d
    b["max"] = a["max"] + d
    return b


def _rays(D, prec, m, seed):
    rng = np.random.default_rng(seed)
    org = rng.uniform(-130, 130, (m, D))
    tgt = rng.uniform(-90, 90, (m, D))
    o, d, inv = ray_new(org, unit_directions(tgt - org), _F(prec))
    r = np.zeros(m, dtype=_table(D)[prec]["ray"])
    r["origin"], r["direction"], r["inv_direction"] = o, d, inv
    return r


def _inputs(D, prec, seed=7):
    F = _F(prec)
    rng = np.random.default_rng(seed)
    rays = _rays(D, prec, NR, seed)
    pts = rng.uniform(-110, 110, (NR, D)).astype(F)
    amin = rng.uniform(-110, 110, (NR, D))
    aab = np.concatenate([amin, amin + rng.uniform(0, 12, (NR, D))], axis=1).astype(F)
    balls = np.concatenate([rng.uniform(-110, 110, (NR, D)), rng.uniform(5, 25, (NR, 1))], axis=1).astype(F)
    return dict(rays=rays, pts=pts, aab=aab, balls=balls)


def _dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


def _buf(nbytes):
    import torch

    return torch.full((max(int(nbytes), 16),), 0xFF, dtype=torch.uint8, device="cuda")


def _host(t, dtype, count=None):
    a = t.cpu().numpy().view(dtype)
    return a if count is None else a[:count]


def _same(x, y):
    return len(x) == len(y) and all(np.asarray(a).tobytes() == np.asarray(b).tobytes() for a, b in zip(x, y))


# ---- consumers --------------------------------------------------------------------------------------------------------------------
# Host consumers are (name, fn(tree, inputs) -> arrays) and return when their work is done.  _dev consumers enqueue into buffers
# allocated before the spin and are read back after the device synchronised; each one names the host form it must equal: `expect`.
def _nodes(tree):
    if hasattr(tree, "nodes_and_index"):
        return tree.nodes_and_index()
    tree._nodes = None
    return tree.nodes, tree.node_index


def _flat(tree):
    """The flat nodes field by field: the padding bytes of the f64 records are not part of the result."""
    f = tree.flatten()
    f = f if isinstance(f, np.ndarray) else f.nodes
    return (f["aabb"]["min"], f["aabb"]["max"], f["entry_index"], f["exit_index"], f["shape_index"])


def _host_consumers(D, family):
    from bvh_b200 import capi

    rays = [("traverse", lambda t, i: t.traverse_batch(i["rays"])),
            ("traverse_flat", lambda t, i: t.traverse_batch(i["rays"], mode=capi.TRAVERSE_FLAT)),
            ("closest_hit", lambda t, i: t.closest_hit(i["rays"])),
            ("any_hit", lambda t, i: (t.any_hit(i["rays"]),)),
            ("multi_hit", lambda t, i: t.multi_hit(i["rays"], 3)[:2]),
            ("ordered", lambda t, i: t.traverse_ordered(i["rays"]))]
    if D == 3:
        rays.append(("traverse_od", lambda t, i: t.traverse_batch(i["rays"], compact=True)))
    points = [("query_aabb", lambda t, i: t.query_batch(capi.QUERY_AABB, i["aab"])),
              ("query_ball", lambda t, i: t.query_batch(capi.QUERY_BALL, i["balls"])),
              ("nearest_to", lambda t, i: t.nearest_to_batch(i["pts"])),
              ("nearest_candidates", lambda t, i: t.nearest_candidates(i["pts"])),
              ("knn", lambda t, i: t.knn(i["pts"], 4))]
    shape = [("overlap", lambda t, i: t.overlap_pairs()), ("tree_nodes", lambda t, i: _nodes(t)), ("flatten", lambda t, i: _flat(t))]
    if family == "all":
        return rays + points + shape
    if family == "rays_points":
        return rays + points
    return [c for c in rays + points + shape if c[0] in ("traverse", "knn", "overlap", "tree_nodes")]


def _dev_consumers(D, prec, family):
    """(name, prepare(inputs) -> run(tree) -> read(), expect(twin, inputs)) of the _dev forms for D = 3, 4.  prepare uploads the
    inputs and allocates the outputs, then synchronises the device: it runs before the spin."""
    from bvh_b200 import capi

    if D == 2:
        return []
    F = _F(prec)
    lib = capi.lib()

    def traverse_dev(i, od=False):
        n = len(i["rays"])
        src = np.concatenate([i["rays"]["origin"], i["rays"]["direction"]], axis=1) if od else i["rays"]
        d_r, d_off, d_hits = _dev(src), _buf(4 * (n + 1)), _buf(4 * 64 * n)
        _drain()

        def run(t):
            if od:
                capi.check(getattr(lib, f"bvhgpu_traverse_od_dev_{_sfx(D, prec)}")(t._h, capi.TRAVERSE_BVH, C.c_void_p(d_r.data_ptr()), n,
                                                                                   C.c_void_p(d_off.data_ptr()), C.c_void_p(d_hits.data_ptr()),
                                                                                   64 * n, None))
            else:
                t.traverse_dev(d_r.data_ptr(), n, d_off.data_ptr(), d_hits.data_ptr(), 64 * n)

            def read():
                off = _host(d_off, np.uint32, n + 1)
                return off, _host(d_hits, np.uint32, int(off[-1]))
            return read
        return run

    def query_dev(i):
        q = i["aab"]
        n = len(q)
        d_q, d_off, d_hits = _dev(q), _buf(4 * (n + 1)), _buf(4 * 64 * n)
        _drain()

        def run(t):
            capi.check(getattr(lib, f"bvhgpu_query_dev_{_sfx(D, prec)}")(t._h, capi.TRAVERSE_BVH, capi.QUERY_AABB, C.c_void_p(d_q.data_ptr()), n,
                                                                         C.c_void_p(d_off.data_ptr()), C.c_void_p(d_hits.data_ptr()), 64 * n, None))

            def read():
                off = _host(d_off, np.uint32, n + 1)
                return off, _host(d_hits, np.uint32, int(off[-1]))
            return read
        return run

    def knn_dev(i):
        n = len(i["pts"])
        d_p, d_s, d_d = _dev(i["pts"]), _buf(4 * 4 * n), _buf(F().itemsize * 4 * n)
        _drain()

        def run(t):
            t.knn_dev(d_p.data_ptr(), n, 4, 0, d_s.data_ptr(), d_d.data_ptr())
            return lambda: (_host(d_s, np.uint32, 4 * n).reshape(n, 4), _host(d_d, F, 4 * n).reshape(n, 4))
        return run

    out = [("traverse_dev", traverse_dev, lambda w, i: w.traverse_batch(i["rays"])),
           ("knn_dev", knn_dev, lambda w, i: w.knn(i["pts"], 4))]
    if family != "dynamic":
        out.append(("query_dev", query_dev, lambda w, i: w.query_batch(capi.QUERY_AABB, i["aab"])))
        if D == 3:
            out.append(("traverse_od_dev", lambda i: traverse_dev(i, od=True), lambda w, i: w.traverse_batch(i["rays"])))
    return out


def _expect(twin, D, prec, family, inputs):
    hc = {name: fn(twin, inputs) for name, fn in _host_consumers(D, family)}
    dc = {name: expect(twin, inputs) for name, _, expect in _dev_consumers(D, prec, family)}
    return hc, dc


def _run_consumers(tree, D, prec, family, inputs, prepared):
    """Enqueue every consumer on the context's current stream; host forms return at once with their arrays."""
    reads = {}
    for name, fn in _host_consumers(D, family):
        res = fn(tree, inputs)
        reads[name] = (lambda r=res: r)
    for name, _, _ in _dev_consumers(D, prec, family):
        reads[name] = prepared[name](tree)
    return reads


def _prepare_dev(D, prec, family, inputs):
    """Inputs and output buffers of the _dev consumers, allocated and written before the spin."""
    return {name: prep(inputs) for name, prep, _ in _dev_consumers(D, prec, family)}


def _check(reads, before, after):
    """Every consumer: the expected result changed with the producer, and the consumer on Q saw the new one."""
    hb, db = before
    ha, da = after
    want = {**ha, **da}
    old = {**hb, **db}
    for name, read in reads.items():
        got = read()
        if old is not None and name in old:
            assert not _same(old[name], want[name]), f"{name}: the producer does not change the expected result"
        assert _same(got, want[name]), name


def _free(*trees):
    for t in trees:
        if t is not None:
            t.free()


# ---- build, then switch -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("direction", DIRECTIONS)
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("D,form", [(2, "host"), (3, "host"), (3, "dev"), (4, "host")])
def test_build_then_switch(api, twin_ctx, direction, prec, D, form):
    """build (ordering check) / build_dev (witness) on P, every consumer on Q == the twin's; the 3-D twin == the oracle."""
    shapes = _boxes(D, prec, N, seed=11)
    inputs = _inputs(D, prec)
    cls = _cls(api, D)
    twin = cls.build(shapes, prec=prec, ctx=twin_ctx)
    sw, tree = Switch(api, direction), None
    try:
        after = _expect(twin, D, prec, "all", inputs)
        if D == 3:
            want = O.build(shapes, prec)
            r = O.traverse(want.nodes, shapes, inputs["rays"], O.MODE_RECURSIVE, prec)
            off, hits = after[0]["traverse"]
            assert np.array_equal(off.astype(np.uint64), r.offsets) and np.array_equal(hits, r.hits)
        d_shapes = _dev(shapes)
        prepared = _prepare_dev(D, prec, "all", inputs)
        pending = sw.spin()
        if form == "dev":
            tree = cls.build_dev(d_shapes.data_ptr(), N, prec=prec, ctx=sw.ctx)
            assert not pending.query()                            # the build was still waiting when it returned
        else:
            tree = cls.build(shapes, prec=prec, ctx=sw.ctx)
        sw.switch()
        reads = _run_consumers(tree, D, prec, "all", inputs, prepared)
        _drain()
        _check(reads, ({}, {}), after)
    finally:
        _free(tree, twin)
        sw.close()


# ---- refit, then switch -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("direction", DIRECTIONS)
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("D,form", [(2, "host"), (3, "host"), (3, "dev"), (4, "host"), (4, "dev")])
def test_refit_then_switch(api, twin_ctx, direction, prec, D, form):
    """refit / refit_dev of every box on P, the ray and point consumers on Q == the twin's after the same refit."""
    shapes = _boxes(D, prec, N, seed=12)
    new = _moved(shapes, seed=13)
    inputs = _inputs(D, prec)
    cls = _cls(api, D)
    twin = cls.build(shapes, prec=prec, ctx=twin_ctx)
    sw = Switch(api, direction)
    tree = cls.build(shapes, prec=prec, ctx=sw.ctx)
    try:
        before = _expect(twin, D, prec, "rays_points", inputs)
        twin.refit(new)
        after = _expect(twin, D, prec, "rays_points", inputs)
        prepared = _prepare_dev(D, prec, "rays_points", inputs)
        _run_consumers(tree, D, prec, "rays_points", inputs, _prepare_dev(D, prec, "rays_points", inputs))   # build the lazy records
        d_new = _dev(new)
        _drain()
        sw.spin()
        if form == "dev":
            capi_refit_dev(tree, D, prec, d_new, len(new))
        else:
            tree.refit(new)
        sw.switch()
        reads = _run_consumers(tree, D, prec, "rays_points", inputs, prepared)
        _drain()
        _check(reads, before, after)
    finally:
        _free(tree, twin)
        sw.close()


def capi_refit_dev(tree, D, prec, d_new, n):
    from bvh_b200 import capi

    capi.check(getattr(capi.lib(), f"bvhgpu_refit_dev_{_sfx(D, prec)}")(tree._h, C.c_void_p(d_new.data_ptr()), n))
    tree._nodes = None


# ---- update / add / remove, then switch -------------------------------------------------------------------------------------------
def _dynamic(tree, D, prec, op, form, data):
    """One dynamic call on `tree`; `data` holds the host arrays and (form "dev") their device copies."""
    from bvh_b200 import capi

    lib, sfx = capi.lib(), _sfx(D, prec)
    if form == "host":
        if op == "update":
            tree.update_shapes(data["idx"], data["all"], 1.5)
        elif op == "add":
            tree.add_shapes(data["add"], 1.5)
        else:
            tree.remove_shapes(data["rm"])
    else:
        if op == "update":
            capi.check(getattr(lib, f"bvhgpu_update_dev_{sfx}")(tree._h, C.c_void_p(data["d_idx"].data_ptr()), C.c_void_p(data["d_fresh"].data_ptr()),
                                                                len(data["idx"]), C.c_double(1.5), None))
        elif op == "add":
            capi.check(getattr(lib, f"bvhgpu_add_shapes_dev_{sfx}")(tree._h, C.c_void_p(data["d_add"].data_ptr()), len(data["add"]), C.c_double(1.5),
                                                                    None))
        else:
            capi.check(getattr(lib, f"bvhgpu_remove_shapes_dev_{sfx}")(tree._h, C.c_void_p(data["d_rm"].data_ptr()), len(data["rm"])))
        if hasattr(tree, "_sync_n"):
            tree._sync_n()
    if hasattr(tree, "_nodes"):
        tree._nodes = None


@pytest.mark.parametrize("direction", DIRECTIONS)
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("op", ["update", "add", "remove"])
@pytest.mark.parametrize("D,form", [(2, "host"), (3, "host"), (3, "dev"), (4, "host"), (4, "dev")])
def test_dynamic_then_switch(api, twin_ctx, direction, prec, op, D, form):
    """update_shapes / add_shapes / remove_shapes (host or _dev) on P; traverse, knn, overlap and tree_nodes on Q == the twin's."""
    shapes = _boxes(D, prec, N, seed=14)
    rng = np.random.default_rng(15)
    idx = np.sort(rng.choice(N, N // 3, replace=False)).astype(np.uint32)
    moved = _moved(shapes, seed=16)
    allb = shapes.copy()
    allb[idx] = moved[idx]
    data = dict(idx=idx, all=allb, fresh=np.ascontiguousarray(allb[idx]), add=_boxes(D, prec, 400, seed=17, shift=20.0),
                rm=rng.choice(N, 500, replace=False).astype(np.uint32))
    inputs = _inputs(D, prec)
    cls = _cls(api, D)
    twin = cls.build(shapes, prec=prec, ctx=twin_ctx)
    sw = Switch(api, direction)
    tree = cls.build(shapes, prec=prec, ctx=sw.ctx)
    try:
        before = _expect(twin, D, prec, "dynamic", inputs)
        _dynamic(twin, D, prec, op, "host", data)
        after = _expect(twin, D, prec, "dynamic", inputs)
        prepared = _prepare_dev(D, prec, "dynamic", inputs)
        _run_consumers(tree, D, prec, "dynamic", inputs, _prepare_dev(D, prec, "dynamic", inputs))   # build the lazy records
        if form == "dev":
            data.update(d_idx=_dev(idx), d_fresh=_dev(data["fresh"]), d_add=_dev(data["add"]), d_rm=_dev(data["rm"]))
        _drain()
        sw.spin()
        _dynamic(tree, D, prec, op, form, data)
        sw.switch()
        reads = _run_consumers(tree, D, prec, "dynamic", inputs, prepared)
        _drain()
        _check(reads, before, after)
    finally:
        _free(tree, twin)
        sw.close()


# ---- set_triangles_dev over triangles already set, then switch -----------------------------------------------------------------------
def _triangle_scene(prec):
    shapes, tris = O.create_n_cubes(150, prec=prec, want_tris=True)
    tris = np.ascontiguousarray(tris, dtype=_F(prec)).reshape(-1, 9)
    # the same soup point-reflected through each triangle's box centre: every triangle stays in its own box, and on a cube face
    # it becomes the face's other half, so the shape a ray or point finds changes
    v = tris.reshape(-1, 3, 3)
    other = (shapes["min"][:, None, :] + shapes["max"][:, None, :] - v).astype(_F(prec)).reshape(-1, 9)
    rng = np.random.default_rng(5)
    centres = (shapes["min"][::12] + shapes["max"][::12]).astype(np.float64) * 0.5
    tgt = centres[rng.integers(0, len(centres), NR)] + rng.uniform(-0.4, 0.4, (NR, 3))
    org = tgt + rng.normal(0, 1, (NR, 3)) * 3000
    rays = O.ray_new(org, tgt - org, prec)
    pts = (centres[rng.integers(0, len(centres), NR)] + rng.normal(0, 2.0, (NR, 3))).astype(_F(prec))
    return shapes, tris, other, rays, pts


def _triangle_consumers():
    return [("closest_hit", lambda t, r, p: t.closest_hit(r, triangles=True)),
            ("any_hit", lambda t, r, p: (t.any_hit(r, triangles=True),)),
            ("multi_hit", lambda t, r, p: t.multi_hit(r, 3, triangles=True, uv=True)),
            ("knn_triangles", lambda t, r, p: t.knn_triangles(p, 3, closest=True)),
            ("nearest_triangles", lambda t, r, p: t.nearest_triangles_batch(p))]


@pytest.mark.parametrize("direction", DIRECTIONS)
@pytest.mark.parametrize("prec", PRECS)
def test_set_triangles_dev_then_switch(api, twin_ctx, direction, prec):
    """set_triangles_dev (witness) rewrites the triangles in place on P; the triangle-mode consumers on Q == the twin's."""
    from bvh_b200 import capi

    shapes, tris, other, rays, pts = _triangle_scene(prec)
    twin = api.Bvh.build(shapes, prec=prec, ctx=twin_ctx)
    sw = Switch(api, direction)
    tree = api.Bvh.build(shapes, prec=prec, ctx=sw.ctx)
    try:
        twin.set_triangles(tris)
        before = {name: fn(twin, rays, pts) for name, fn in _triangle_consumers()}
        twin.set_triangles(other)
        after = {name: fn(twin, rays, pts) for name, fn in _triangle_consumers()}
        tree.set_triangles(tris)
        for _, fn in _triangle_consumers():                    # every lazily built record exists before the producer runs
            fn(tree, rays, pts)
        d_other = _dev(other)
        _drain()
        pending = sw.spin()
        capi.check(getattr(capi.lib(), f"bvhgpu_tree_set_triangles_dev_{_sfx(3, prec)}")(tree._h, C.c_void_p(d_other.data_ptr()), len(other)))
        assert not pending.query()                              # the rewrite was still waiting when it returned
        sw.switch()
        got = {name: fn(tree, rays, pts) for name, fn in _triangle_consumers()}
        _drain()
        for name in got:
            assert not _same(before[name], after[name]), name
            assert _same(got[name], after[name]), name
    finally:
        _free(tree, twin)
        sw.close()


# ---- overlap_pairs_with after tree B changed on P ----------------------------------------------------------------------------------
@pytest.mark.parametrize("direction", DIRECTIONS)
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("D,form", [(2, "host"), (3, "dev"), (4, "dev")])
def test_overlap_with_after_refit_then_switch(api, twin_ctx, direction, prec, D, form):
    """Tree B refitted on P, overlap_pairs_with (and _dev for D = 3, 4) from tree A on Q == the twins'."""
    a_boxes, b_boxes = _boxes(D, prec, N, seed=18), _boxes(D, prec, N, seed=19)
    b_new = _moved(b_boxes, seed=20)
    cls = _cls(api, D)
    ta, tb = cls.build(a_boxes, prec=prec, ctx=twin_ctx), cls.build(b_boxes, prec=prec, ctx=twin_ctx)
    sw = Switch(api, direction)
    a, b = cls.build(a_boxes, prec=prec, ctx=sw.ctx), cls.build(b_boxes, prec=prec, ctx=sw.ctx)
    try:
        before = ta.overlap_pairs_with(tb)
        tb.refit(b_new)
        after = ta.overlap_pairs_with(tb)
        assert not _same(before, after)
        a.overlap_pairs_with(b)
        cap = 2 * max(len(before[1]), len(after[1])) + 16
        d_off, d_hits, d_new = _buf(4 * (N + 1)), _buf(4 * cap), _dev(b_new)
        _drain()
        sw.spin()
        if form == "dev":
            capi_refit_dev(b, D, prec, d_new, N)
        else:
            b.refit(b_new)
        sw.switch()
        got = a.overlap_pairs_with(b)
        if form == "dev":
            a.overlap_pairs_with_dev(b, d_off.data_ptr(), d_hits.data_ptr(), cap)
        _drain()
        assert _same(got, after)
        if form == "dev":
            off = _host(d_off, np.uint32, N + 1)
            assert _same((off, _host(d_hits, np.uint32, int(off[-1]))), after)
    finally:
        _free(a, b, ta, tb)
        sw.close()


# ---- a tree freed on Q while a walk on P still reads it ------------------------------------------------------------------------------
@pytest.mark.parametrize("direction", DIRECTIONS)
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("D,call", [(3, "traverse_dev"), (3, "knn_dev"), (4, "traverse_dev"), (4, "knn_dev")])
def test_free_across_switch(api, twin_ctx, direction, prec, D, call):
    """A _dev walk (witness) on P behind the spin, then on Q: free its tree and build another one over as many shapes.  The walk's
    output is the first tree's, not the second's: the freed buffers went back to the pool only after the walk."""
    first, second = _boxes(D, prec, N, seed=21), _moved(_boxes(D, prec, N, seed=22), seed=23)
    inputs = _inputs(D, prec)
    cls = _cls(api, D)
    name, prep, expect = next(c for c in _dev_consumers(D, prec, "all") if c[0] == call)
    t1, t2 = cls.build(first, prec=prec, ctx=twin_ctx), cls.build(second, prec=prec, ctx=twin_ctx)
    sw, tree, other = Switch(api, direction), None, None
    try:
        want, old = expect(t1, inputs), expect(t2, inputs)
        assert not _same(want, old)
        tree = cls.build(first, prec=prec, ctx=sw.ctx)
        run = prep(inputs)
        pending = sw.spin()
        read = run(tree)
        assert not pending.query()                              # the walk was still waiting when it returned
        sw.switch()
        tree.free()
        other = cls.build(second, prec=prec, ctx=sw.ctx)
        _drain()
        assert _same(read(), want)
    finally:
        _free(tree, other, t1, t2)
        sw.close()


# ---- synchronize after a switch -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("direction", DIRECTIONS)
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("D", [3, 4])
def test_synchronize_across_switch(api, twin_ctx, direction, prec, D):
    """A _dev walk on P behind the spin, a switch, then Context.synchronize(): P has finished, and so has the walk."""
    shapes = _boxes(D, prec, N, seed=24)
    inputs = _inputs(D, prec)
    cls = _cls(api, D)
    name, prep, expect = _dev_consumers(D, prec, "all")[0]
    twin = cls.build(shapes, prec=prec, ctx=twin_ctx)
    sw = Switch(api, direction)
    tree = cls.build(shapes, prec=prec, ctx=sw.ctx)
    try:
        want = expect(twin, inputs)
        run = prep(inputs)
        pending = sw.spin()
        read = run(tree)
        assert not pending.query()
        sw.switch()
        sw.ctx.synchronize()
        assert pending.query()                                  # synchronize waited for the previous stream too
        assert _same(read(), want)
    finally:
        _free(tree, twin)
        sw.close()
