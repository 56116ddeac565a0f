"""Argument, size, status and empty-tree contract of every tree-taking entry point, for D = 2, 3 and 4, f32 and f64.

One table: for each host-pointer and `_dev` form, the status it returns for a null tree, a null input or output pointer, n = 0,
n = 2^31 against a one-element buffer, a bad mode / kind / k / max_growth / ray layout, an empty tree and a tree whose build failed
on the device (`bvhgpu_build_dev_*` over a NaN box, D = 3), and for the empty tree what it writes (include/bvh_b200.h).
Run on an H100:  python -m pytest tests/test_gpu_entry_points.py -m gpu"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

OK, INVALID, NAN = 0, 1, 3
INV = 0xFFFFFFFF
HUGE = 1 << 31
KNN_MAX_K = 64

SFX = {(2, "f32"): "f32x2", (2, "f64"): "f64x2", (3, "f32"): "f32x3", (3, "f64"): "f64x3", (4, "f32"): "f32x4", (4, "f64"): "f64x4"}
W_RAY = {2: 6, 3: 9, 4: 12}


def _F(prec):
    return np.float32 if prec == "f32" else np.float64


# ---- entry points ------------------------------------------------------------------------------------------------------------
# A row names the operation, host or _dev form, n, the tree and the fault; _invoke lays out the ABI arguments of (D, prec) with
# buffers from Bufs.  Widths are in scalars per item.
class Bufs:
    """Host (numpy) or device (torch) buffers of n_alloc items, outputs prefilled with 0xAB bytes."""

    def __init__(self, dev, D, prec, n_alloc):
        self.dev, self.D, self.F, self.n = dev, D, _F(prec), n_alloc
        self.keep = []

    def arr(self, width, dtype=None, data=None, extra=0):
        """n_alloc * width + extra items of dtype: `data`, or 0xAB bytes."""
        dtype = dtype or self.F
        if data is None:
            a = np.full((self.n * width + extra) * np.dtype(dtype).itemsize, 0xAB, dtype=np.uint8).view(dtype)
        else:
            a = np.ascontiguousarray(data, dtype=dtype).reshape(-1)
        if self.dev:
            import torch

            t = torch.from_numpy(a.view(np.uint8).copy()).to("cuda")
            self.keep.append(t)
            return t
        self.keep.append(a)
        return a

    @staticmethod
    def ptr(b):
        if b is None:
            return None
        return C.c_void_p(b.data_ptr() if hasattr(b, "data_ptr") else b.ctypes.data)

    def host(self, b, dtype):
        if hasattr(b, "data_ptr"):
            import torch

            torch.cuda.synchronize()
            return b.cpu().numpy().view(dtype)
        return b


def _unit_box(D, F):
    return np.concatenate([np.zeros(D), np.ones(D)]).astype(F)


def _ray(D, F):
    """A ray from (-1, 0.5, ..) along +x, in the ABI layout of D (origin, direction[, inv_direction])."""
    o = np.full(D, 0.5); o[0] = -1.0
    d = np.zeros(D); d[0] = 1.0
    if D == 2:                                  # bvh_ray2*: origin, direction, inv_direction
        return np.concatenate([o, d, [1.0, np.inf]]).astype(F)
    inv = np.full(D, np.inf); inv[0] = 1.0
    return np.concatenate([o, d, inv]).astype(F)


def _call(L, name, args):
    return getattr(L, name)(*args)


class Row:
    def __init__(self, op, dev, n=1, tree="ok", nulls=(), mode=0, kind=1, k=1, growth=2.0, layout=0, want=OK, check=None):
        self.op, self.dev, self.n, self.tree, self.nulls = op, dev, n, tree, set(nulls)
        self.mode, self.kind, self.k, self.growth, self.layout = mode, kind, k, growth, layout
        self.want, self.check = want, check


def _invoke(L, D, prec, tree, row):
    """Builds the arguments of row.op for (D, prec) and calls it; returns (status, outputs dict, Bufs)."""
    s = SFX[(D, prec)]
    F = _F(prec)
    dev = row.dev
    n = row.n
    B = Bufs(dev, D, prec, 1 if n == HUGE else max(n, 1))
    ray1 = _ray(D, F)
    box1 = _unit_box(D, F)
    tot = C.c_size_t(12345)
    rebuilt = C.c_size_t(12345)
    outs = {}

    def inp(name, data_one, width, dtype=None):
        if name in row.nulls:
            return None
        return B.arr(width, dtype, data=np.tile(data_one, B.n))

    def out(name, width, dtype=None, extra=0):
        if name in row.nulls:
            return None
        b = B.arr(width, dtype or F, extra=extra)
        outs[name] = (b, dtype or F)
        return b

    P = B.ptr
    op = row.op
    sfx = ("_dev_" if dev else "_") + s
    if op in ("traverse", "traverse_od"):
        w = 6 if op == "traverse_od" else W_RAY[D]
        r = inp("in", ray1[:6] if op == "traverse_od" else ray1, w)
        off = out("out", 1, np.uint32, extra=1)
        hits = B.arr(4, np.uint32)
        name = f"bvhgpu_{op}{sfx}"
        st = _call(L, name, [tree, row.mode, P(r), n, P(off), P(hits), 4 * B.n, C.byref(tot)])
        outs["total"] = tot
    elif op == "query":
        w = {1: 2 * D, 2: D, 3: D + 1}.get(row.kind, 2 * D)
        rec = np.concatenate([box1, [0.5]]).astype(F)[:w] if row.kind != 2 else np.full(D, 0.5, dtype=F)
        q = inp("in", rec, w)
        off = out("out", 1, np.uint32, extra=1)
        hits = B.arr(4, np.uint32)
        st = _call(L, f"bvhgpu_query{sfx}", [tree, row.mode, row.kind, P(q), n, P(off), P(hits), 4 * B.n, C.byref(tot)])
        outs["total"] = tot
    elif op in ("nearest", "nearest_triangles"):
        p = inp("in", np.full(D, 0.5, dtype=F), D)
        sh = out("out", 1, np.uint32)
        di = out("dist", 1)
        st = _call(L, f"bvhgpu_{op}{sfx}", [tree, row.mode, P(p), n, P(sh), P(di)])
    elif op == "nearest_candidates":
        p = inp("in", np.full(D, 0.5, dtype=F), D)
        off = out("out", 1, np.uint32, extra=1)
        cand = B.arr(4, np.uint32)
        st = _call(L, f"bvhgpu_nearest_candidates{sfx}", [tree, P(p), n, P(off), P(cand), 4 * B.n, C.byref(tot)])
        outs["total"] = tot
    elif op == "traverse_ordered":
        r = inp("in", ray1, W_RAY[D])
        off = out("out", 1, np.uint32, extra=1)
        hits = B.arr(4, np.uint32)
        dists = B.arr(4)
        st = _call(L, f"bvhgpu_traverse_ordered{sfx}", [tree, P(r), n, 1, P(off), P(hits), P(dists), 4 * B.n, C.byref(tot)])
        outs["total"] = tot
    elif op == "closest_hit":
        r = inp("in", ray1, W_RAY[D])
        sh = out("out", 1, np.uint32)
        di = out("dist", 1)
        if D == 3 and dev:
            args = [tree, P(r), row.layout, n, 0, P(sh), P(di), None]
        elif D == 3:
            args = [tree, P(r), n, 0, P(sh), P(di), None]
        else:
            args = [tree, P(r), n, P(sh), P(di)]
        st = _call(L, f"bvhgpu_closest_hit{sfx}", args)
    elif op == "any_hit":
        r = inp("in", ray1, W_RAY[D])
        sh = out("out", 1, np.uint32)
        if D == 3 and dev:
            args = [tree, P(r), row.layout, n, None, 0, P(sh)]
        elif D == 3:
            args = [tree, P(r), n, None, 0, P(sh)]
        else:
            args = [tree, P(r), n, None, P(sh)]
        st = _call(L, f"bvhgpu_any_hit{sfx}", args)
    elif op == "knn":
        p = inp("in", np.full(D, 0.5, dtype=F), D)
        kk = row.k
        B2 = Bufs(dev, D, prec, B.n * max(min(kk, KNN_MAX_K), 1))
        sh = None if "out" in row.nulls else B2.arr(1, np.uint32)
        di = B2.arr(1)
        if sh is not None:
            outs["out"] = (sh, np.uint32)
        B.keep.append(B2)
        st = _call(L, f"bvhgpu_knn{sfx}", [tree, P(p), n, kk, None, P(sh), P(di)])
    elif op in ("refit", "optimize"):
        a = inp("in", box1, 2 * D)
        if op == "refit":
            st = _call(L, f"bvhgpu_refit{sfx}", [tree, P(a), n])
        else:
            st = _call(L, f"bvhgpu_optimize{sfx}", [tree, P(a), n, row.growth, C.byref(rebuilt)])
    elif op == "update":
        c = inp("idx", np.zeros(1, np.uint32), 1, np.uint32)
        a = inp("in", box1, 2 * D)
        st = _call(L, f"bvhgpu_update{sfx}", [tree, P(c), P(a), n, row.growth, C.byref(rebuilt)])
    elif op == "add_shapes":
        a = inp("in", box1, 2 * D)
        st = _call(L, f"bvhgpu_add_shapes{sfx}", [tree, P(a), n, row.growth, C.byref(rebuilt)])
    elif op == "remove_shapes":
        c = inp("in", np.zeros(1, np.uint32), 1, np.uint32)
        st = _call(L, f"bvhgpu_remove_shapes{sfx}", [tree, P(c), n])
    elif op == "tree_nodes":
        nodes = B.arr(64, np.uint8)
        idx = B.arr(1, np.uint32)
        st = _call(L, f"bvhgpu_tree_nodes_{s}", [tree, P(nodes), P(idx)])
    elif op == "flatten":
        fl = B.arr(64 * 16, np.uint8)
        ln = C.c_size_t(12345)
        st = _call(L, f"bvhgpu_flatten_{s}", [tree, P(fl), 1024, C.byref(ln)])
        outs["len"] = ln
    elif op == "sah_cost":
        o2 = (C.c_double * 2)()
        st = _call(L, f"bvhgpu_sah_cost_{s}", [tree, o2])
    else:
        raise AssertionError(op)
    return st, outs, B


# ---- the table ---------------------------------------------------------------------------------------------------------------
CSR = ("traverse", "query", "nearest_candidates", "traverse_ordered")
PER_ITEM = ("nearest", "closest_hit", "any_hit", "knn")


def _ops(D, dev):
    """The tree-taking batch / dynamic entry points of D (host or _dev form)."""
    if dev:
        ops = ["traverse", "query", "knn", "closest_hit", "any_hit", "refit", "update", "add_shapes", "remove_shapes"] if D != 2 else []
        if D == 3:
            ops += ["traverse_od", "optimize"]
        return ops
    ops = list(CSR) + list(PER_ITEM) + ["refit", "update", "add_shapes", "remove_shapes", "tree_nodes", "flatten"]
    if D == 3:
        ops += ["traverse_od", "nearest_triangles", "optimize", "sah_cost"]
    return ops


def _empty_check(op):
    def offsets_zero(outs, B):
        o = B.host(outs["out"][0], np.uint32)
        assert (o[: B.n + 1] == 0).all()
        assert outs["total"].value == 0

    def no_hit(outs, B):
        assert (B.host(outs["out"][0], np.uint32)[: B.n] == INV).all()

    def nearest_none(outs, B):
        no_hit(outs, B)
        assert (B.host(outs["dist"][0], outs["dist"][1])[: B.n] == 0).all()

    def flat_empty(outs, B):
        assert outs["len"].value == 0

    return {"traverse": offsets_zero, "traverse_od": offsets_zero, "query": offsets_zero, "nearest_candidates": offsets_zero,
            "traverse_ordered": offsets_zero, "nearest": nearest_none, "closest_hit": no_hit, "any_hit": no_hit, "knn": no_hit,
            "flatten": flat_empty}.get(op)


# The D = 3 host forms that staged the batch before checking n at the parent of this table's commit.
STAGE_FIRST_D3 = {"traverse", "traverse_od", "query", "nearest", "nearest_triangles", "nearest_candidates", "traverse_ordered", "closest_hit"}


def _rows():
    rows = []
    for D in (2, 3, 4):
        for dev in (False, True):
            for op in _ops(D, dev):
                tag = f"{'dev' if dev else 'host'}-{op}"
                batch = op in CSR + PER_ITEM + ("traverse_od", "nearest_triangles")
                if op not in ("tree_nodes", "flatten", "sah_cost"):
                    rows.append((D, tag + "-null_in", Row(op, dev, nulls=("in",), want=INVALID)))
                rows.append((D, tag + "-null_tree", Row(op, dev, tree="null", want=INVALID)))
                if batch and op != "nearest_triangles":
                    rows.append((D, tag + "-null_out", Row(op, dev, nulls=("out",), want=INVALID)))
                if op not in ("tree_nodes", "flatten", "sah_cost", "refit", "optimize"):
                    rows.append((D, tag + "-n0", Row(op, dev, n=0, want=OK)))
                huge_ok = batch or op in ("refit", "optimize", "add_shapes", "remove_shapes")
                if huge_ok:
                    label = "-huge_stage_first" if (D == 3 and not dev and op in STAGE_FIRST_D3) else "-huge"
                    rows.append((D, tag + label, Row(op, dev, n=HUGE, want=INVALID)))
                if op in ("traverse", "traverse_od", "query", "nearest", "nearest_triangles"):
                    # the streamed 3-D host traversal walks every mode other than BVHGPU_TRAVERSE_FLAT as BVHGPU_TRAVERSE_BVH
                    lax = D == 3 and not dev and op in ("traverse", "traverse_od")
                    rows.append((D, tag + "-bad_mode", Row(op, dev, mode=7, want=OK if lax else INVALID)))
                if op == "query":
                    rows.append((D, tag + "-bad_kind0", Row(op, dev, kind=0, want=INVALID)))
                    rows.append((D, tag + "-bad_kind4", Row(op, dev, kind=4, want=INVALID)))
                if op == "knn":
                    rows.append((D, tag + "-bad_k0", Row(op, dev, k=0, want=INVALID)))
                    rows.append((D, tag + "-bad_k_big", Row(op, dev, k=KNN_MAX_K + 1, want=INVALID)))
                if op in ("update", "add_shapes", "optimize"):
                    rows.append((D, tag + "-bad_growth", Row(op, dev, n=1 if op != "optimize" else 8, growth=0.5, want=INVALID)))
                if D == 3 and dev and op in ("closest_hit", "any_hit"):
                    rows.append((D, tag + "-bad_layout", Row(op, dev, layout=5, want=INVALID)))
                # an empty tree
                if op in ("refit", "optimize"):
                    rows.append((D, tag + "-empty_n1", Row(op, dev, tree="empty", want=INVALID)))
                    rows.append((D, tag + "-empty_n0", Row(op, dev, n=0, tree="empty", want=OK)))
                elif op == "remove_shapes":
                    rows.append((D, tag + "-empty", Row(op, dev, tree="empty", want=INVALID)))
                elif op not in ("add_shapes", "nearest_triangles", "sah_cost"):
                    rows.append((D, tag + "-empty", Row(op, dev, tree="empty", want=OK, check=_empty_check(op))))
                # a build that failed on the device (D = 3: bvhgpu_build_dev_* does not wait for the build)
                if D == 3:
                    n_ok = 8 if op in ("refit", "optimize") else 1
                    rows.append((D, tag + "-failed", Row(op, dev, n=n_ok, tree="failed", want=NAN)))
    # n = 0 on a failed tree: the host forms report the build's status, most _dev forms return before they look at the tree
    for op, dev, want in (("traverse", False, NAN), ("traverse", True, OK), ("query", False, NAN), ("query", True, OK),
                          ("closest_hit", False, NAN), ("closest_hit", True, OK), ("any_hit", False, NAN), ("any_hit", True, OK),
                          ("knn", False, NAN), ("knn", True, NAN), ("nearest", False, NAN), ("traverse_ordered", False, NAN)):
        rows.append((3, f"{'dev' if dev else 'host'}-{op}-failed_n0", Row(op, dev, n=0, tree="failed", want=want)))
    out = []
    for D, tag, row in rows:
        for prec in ("f32", "f64"):
            out.append(pytest.param(D, prec, row, id=f"d{D}-{prec}-{tag}"))
    return out


@pytest.fixture(scope="module")
def lib():
    from bvh_b200 import api, capi

    L = capi.lib()
    ctx = api.Context(0)
    yield L, ctx
    for (D, prec, _), h in _TREES.items():
        getattr(L, f"bvhgpu_tree_free_{SFX[(D, prec)]}")(h)
    _TREES.clear()
    del ctx


def _boxes(D, F, n):
    rng = np.random.default_rng(7)
    lo = rng.uniform(-4, 4, size=(n, D))
    return np.concatenate([lo, lo + rng.uniform(0.1, 1, size=(n, D))], axis=1).astype(F)


_TREES = {}


def _tree(L, ctx, D, prec, kind):
    """A healthy tree over 8 boxes or an empty one (cached per module), or a fresh tree whose device build hit a NaN box."""
    s = SFX[(D, prec)]
    F = _F(prec)
    h = C.c_void_p()
    if kind == "failed":
        import torch

        boxes = _boxes(D, F, 8)
        boxes[3, 0] = np.nan
        t = torch.from_numpy(boxes.view(np.uint8).reshape(-1).copy()).to("cuda")
        assert getattr(L, f"bvhgpu_build_dev_{s}")(ctx._h, C.c_void_p(t.data_ptr()), 8, 0, C.byref(h)) == OK
        torch.cuda.synchronize()
        return h, (lambda: getattr(L, f"bvhgpu_tree_free_{s}")(h)), t
    key = (D, prec, kind)
    if key not in _TREES:
        n = 8 if kind == "ok" else 0
        boxes = _boxes(D, F, max(n, 1))
        st = getattr(L, f"bvhgpu_build_{s}")(ctx._h, C.c_void_p(boxes.ctypes.data) if n else None, n, 0, C.byref(h))
        assert st == OK, L.bvhgpu_last_error()
        _TREES[key] = h
    return _TREES[key], None, None


@pytest.mark.parametrize("D,prec,row", _rows())
def test_entry_point_contract(lib, D, prec, row):
    L, ctx = lib
    if row.tree == "null":
        tree, free = None, None
    else:
        tree, free, _keep = _tree(L, ctx, D, prec, row.tree)
    try:
        st, outs, B = _invoke(L, D, prec, tree, row)
        assert st == row.want, f"status {st}, want {row.want}: {L.bvhgpu_last_error()}"
        if row.check is not None:
            row.check(outs, B)
    finally:
        if free is not None:
            free()
