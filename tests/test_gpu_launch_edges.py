"""The batched calls at the batch sizes and launch geometries where their grid arithmetic changes (tests/launch_edges.py reads those
sizes from the CUDA sources), every output written into a buffer with a 4 KB canary guard on both sides.

1. Small sizes: Ray::new and every batched family, host and device forms, f32 and f64, D = 2 / 3 / 4 where it exists, at one item
   either side of the warp, of the 128- and 256-thread blocks, of 1024 and of a scan tile, against the reference each family already
   has: the C++ oracle in 3-D (Ray::new, traverse, query, nearest_to, nearest_triangles, closest_hit in AABB mode),
   tests/dimorder.py / dimref.py in 2-D and 4-D and for the distance-ordered walk, the stated tolerance of tests/prunedcheck.py
   (closest_hit's triangle mode), tests/anyhit.py, multihit.py, knnref.py and knntri.py.  Both guards stay intact, offsets[n] is
   written, CSR outputs get cap == total.
2. Large sizes, only where the arithmetic changes: scan_post_kernel's tile-sum loop (3-D traverse), the streamed host path's
   thresholds and chunk counts, scan_blocks_kernel's loop (a Point query per D, nearest_candidates in 3-D) and walk_top_kernel's
   grid.  The batches tile a base batch, so that the reference is the base's oracle result tiled; CSR and visit counter are exact.
3. Forced geometry: option walk_grid on the persistent walk (host, device and streamed forms), traverse_top on a 2-D tree.
4. The values the library reads once per process (BVHGPU_TOP_REFILL, BVHGPU_CHUNKS, BVHGPU_CHUNK_SCHEDULE), one child process per
   value: the same CSR and visit counter as a child at the defaults.
Run on an H100:  python -m pytest tests/test_gpu_launch_edges.py -m gpu"""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle as O
from tests import anyhit as H
from tests import dimorder, dimref
from tests import knnref as KR
from tests import knntri as KT
from tests import launch_edges as LE
from tests import multihit as MH
from tests import prunedcheck as PC
from tests.scenes import rays_for, scene

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U32_MAX = 0xFFFFFFFF
FT = {"f32": np.float32, "f64": np.float64}
SMALL = LE.edges("small")
NB = SMALL[-1]                   # the references are computed once for NB items; size n compares their first n rows
GUARD, CANARY = 4096, 0xA7
K_MID = 6                        # multi_hit / knn: one k inside a bucket (the K buckets are covered by their own tests)
BASE = 4099                      # large batches tile a base batch of this many items (coprime with the 2048-item scan tile)


@pytest.fixture(scope="module")
def api():
    from bvh_b200 import api as A_

    return A_


# ---- guarded buffers ----------------------------------------------------------------------------------------------------------------
class _Out:
    """An output of `nbytes` between two GUARD-byte canary regions, in device memory (torch) or host memory (numpy)."""

    def __init__(self, nbytes, dev):
        import torch

        self.n, self.dev = int(nbytes), dev
        if dev:
            self.buf = torch.full((2 * GUARD + self.n,), CANARY, dtype=torch.uint8, device="cuda")
            self.ptr = self.buf.data_ptr() + GUARD
        else:
            self.buf = np.full(2 * GUARD + self.n, CANARY, dtype=np.uint8)
            self.ptr = self.buf.ctypes.data + GUARD

    @property
    def vp(self):
        return C.c_void_p(self.ptr)

    def get(self, dtype, what=""):
        raw = self.buf.cpu().numpy() if self.dev else self.buf
        assert np.all(raw[:GUARD] == CANARY), f"{what}: written before the output"
        assert np.all(raw[GUARD + self.n:] == CANARY), f"{what}: written past the output"
        return raw[GUARD:GUARD + self.n].view(dtype).copy()


class _In:
    """Input arrays as pointers: host numpy arrays, or device copies."""

    def __init__(self, dev):
        self.dev, self.keep = dev, []

    def __call__(self, a):
        if a is None:
            return None
        import torch

        a = np.ascontiguousarray(a)
        if self.dev:
            t = torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).cuda()
            self.keep.append(t)
            return C.c_void_p(t.data_ptr())
        self.keep.append(a)
        return C.c_void_p(a.ctypes.data)


def _run(bvh, dev, fn, *args):
    """fn(*args) with the inputs in place; a device form is ordered after the uploads and drained before the outputs are read."""
    from bvh_b200 import capi

    if dev:
        import torch

        torch.cuda.synchronize()
    capi.check(fn(*args))
    if dev:
        bvh.ctx.synchronize()


def _sfx(D, prec):
    return f"{prec}x{D}"


def _lib():
    from bvh_b200 import capi

    return capi.lib()


# ---- scenes of the small sweep -----------------------------------------------------------------------------------------------------
class _Scene:
    """One tree per (D, prec) with NB rays, points and limits; in 3-D the 240 triangles of 20 cubes (most rays miss them)."""

    def __init__(self, api, D, prec):
        from bvh_b200.dtypes import BY_PREC

        F = FT[prec]
        self.D, self.prec, self.F = D, prec, F
        rng = np.random.default_rng(7 * D + (prec == "f64"))
        if D == 3:
            from bvh_b200 import scenes as BS

            self.tris = BS.create_n_cubes_tris(20, prec)
            self.shapes = O.tri_aabbs(self.tris, prec)
            self.bvh = api.Bvh.build(self.shapes, prec=prec)
            self.bvh.set_triangles(self.tris)
            self.nodes = O.build(self.shapes, prec).nodes
            self.flat = O.flatten(self.nodes, prec)
            self.rays = rays_for(self.shapes, NB, prec, seed=3, axis_aligned=NB // 8)
            mn, mx = self.shapes["min"], self.shapes["max"]
            tab = BY_PREC[prec]
        else:
            cls = {2: api.Bvh2, 4: api.Bvh4}[D]
            tab = cls._TABLE[prec]
            mn, mx = dimref.scene("random", 64, D, F, rng)
            self.shapes = np.zeros(len(mn), dtype=tab["aabb"])
            self.shapes["min"], self.shapes["max"] = mn, mx
            self.bvh = cls.build(self.shapes, prec=prec)
            self.nodes = self.bvh.nodes_and_index()[0]
            self.flat = self.bvh.flatten()
            o, d, inv = dimorder.rays(mn, mx, NB, F, rng)
            self.rays = np.zeros(NB, dtype=tab["ray"])
            self.rays["origin"], self.rays["direction"], self.rays["inv_direction"] = o, d, inv
        self.tab, self.mn, self.mx = tab, np.asarray(mn), np.asarray(mx)
        self.o, self.inv = self.rays["origin"], self.rays["inv_direction"]
        self.od = np.ascontiguousarray(np.concatenate([self.rays["origin"], self.rays["direction"]], axis=1), dtype=F)
        self.pts = dimref.points(self.mn, self.mx, NB, F, rng)
        span = float(np.max(self.mx.astype(np.float64) - self.mn.astype(np.float64)))
        self.tmax = rng.uniform(0, 1.5 * max(span, 1.0), NB).astype(F)
        self.radius = rng.uniform(0, 0.3 * max(span, 1.0), NB).astype(F)
        self.tree = dimorder.Tree(self.nodes, self.shapes)

    def free(self):
        self.bvh.free()


# ---- reference rows for NB items ---------------------------------------------------------------------------------------------------
def _csr(lists):
    off = np.zeros(len(lists) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(x) for x in lists])
    flat = np.concatenate([np.asarray(x, dtype=np.uint32) for x in lists]) if lists else np.zeros(0, np.uint32)
    return off, flat.astype(np.uint32)


def _ray_sets(tree, o, inv, flat):
    """Bvh::traverse (flat=False) / FlatBvh::traverse (flat=True) of every ray in 2-D / 4-D over a dimorder.Tree: the candidates in
    DFS order; the flat walk reaches the same leaves and re-tests each shape's own box."""
    out = []
    for i in range(len(o)):
        ray = (list(o[i]), list(inv[i]))
        c = [s for s, _ in tree._candidates(ray)]
        if flat and len(tree.nodes) > 1:
            c = [s for s in c if dimorder.slice(ray, *tree.shapes[s]) is not None]
        out.append(c)
    return _csr(out)


def _traverse_ref(S, flat):
    if S.D == 3:
        r = O.traverse(S.flat if flat else S.nodes, S.shapes, S.rays, O.MODE_FLAT if flat else O.MODE_RECURSIVE, S.prec)
        return r.offsets, r.hits
    return _ray_sets(S.tree, S.o, S.inv, flat)


def _query_ref(S, kind, q, flat):
    if S.D == 3:
        return O.query(kind, q, S.nodes, S.shapes, S.flat if flat else None, S.prec)
    t = dimref.Tree(S.nodes, S.shapes, S.flat)
    return _csr([(t.query_flat if flat else t.query_bvh)(kind, list(r)) for r in q])


def _nearest_ref(S, flat):
    if S.D == 3:
        return O.nearest_to(S.flat if flat else S.nodes, S.shapes, S.pts, S.prec, flat=flat)
    t = dimref.Tree(S.nodes, S.shapes, S.flat)
    rows = [(t.nearest_flat if flat else t.nearest_bvh)(list(p)) for p in S.pts]
    return np.array([r[0] for r in rows], dtype=np.uint32), np.array([r[1] for r in rows], dtype=S.F)


# ---- one call of each family at size n, outputs guarded --------------------------------------------------------------------------
def _call_csr(S, n, dev, name, lead, inputs, cap, ascending=None):
    """A CSR entry point fn(*lead, inputs, n, offsets, hits, cap, &total), or traverse_ordered's fn(tree, rays, n, ascending, offsets,
    hits, dists, cap, &total); returns (offsets, hits, dists or None)."""
    F = S.F
    i = _In(dev)
    off, hits = _Out(4 * (n + 1), dev), _Out(4 * cap, dev)
    dists = _Out(F().itemsize * cap, dev) if ascending is not None else None
    tot = C.c_size_t(U32_MAX)
    outs = [off.vp, hits.vp] + ([dists.vp] if dists else [])
    fn = getattr(_lib(), name)
    if ascending is not None:
        _run(S.bvh, dev, fn, *lead, i(inputs[:n]), n, ascending, *outs, cap, C.byref(tot))
    else:
        _run(S.bvh, dev, fn, *lead, i(inputs[:n]), n, *outs, cap, C.byref(tot))
    assert tot.value == cap, (name, n, tot.value, cap)
    what = f"{name} n={n}"
    return off.get(np.uint32, what), hits.get(np.uint32, what), (dists.get(F, what) if dists else None)


def _check_csr(got, want_off, want_hits, n, what):
    off, hits = got[0], got[1]
    m = int(want_off[n])
    assert np.array_equal(off.astype(np.uint64), want_off[:n + 1]), f"{what} n={n}: offsets"
    assert np.array_equal(hits, want_hits[:m]), f"{what} n={n}: hits"


def _rows(S, n, dev, name, args_before, per_item, outs_spec):
    """A per-item entry point: fn(*args_before(inputs), *outs) with outs_spec = [(bytes per item, dtype), ...]."""
    outs = [_Out(b * n, dev) for b, _ in outs_spec]
    i = _In(dev)
    _run(S.bvh, dev, getattr(_lib(), name), *args_before(i, n), *[o.vp for o in outs])
    return [o.get(dt, f"{name} n={n}").reshape((n,) + per_item[j]) for j, (o, (_, dt)) in enumerate(zip(outs, outs_spec))]


FAMILIES = ["rays_new", "traverse", "query", "nearest", "nearest_triangles", "nearest_candidates", "traverse_ordered", "closest_aabb",
            "closest_triangles", "any_hit", "multi_hit", "knn", "knn_triangles"]
THREE_D_ONLY = {"rays_new", "nearest_triangles", "closest_triangles", "knn_triangles"}


def _sweep(api, family, D, prec):
    from bvh_b200 import capi

    S = _Scene(api, D, prec)
    F, sfx, h = S.F, _sfx(D, prec), S.bvh._h
    isz = F().itemsize
    try:
        if family == "rays_new":                                  # Ray::new on the device: the only form is the _dev one
            org = S.rays["origin"]
            raw = (S.rays["direction"].astype(np.float64) * np.random.default_rng(5).uniform(0.25, 4.0, (NB, 1))).astype(F)
            want = O.ray_new(org, raw, prec)
            rsz = S.tab["ray"].itemsize
            name = f"bvhgpu_rays_new_dev_{sfx}"
            for n in SMALL:
                got, = _rows(S, n, True, name, lambda i, n: (S.bvh.ctx._h, i(org[:n]), i(raw[:n]), n), [(rsz,)], [(rsz, np.uint8)])
                assert got.tobytes() == want[:n].tobytes(), (name, n)
        elif family == "traverse":
            for flat in (False, True):
                mode = capi.TRAVERSE_FLAT if flat else capi.TRAVERSE_BVH
                woff, whits = _traverse_ref(S, flat)
                forms = [(f"bvhgpu_traverse_{sfx}", S.rays, False)]
                if D == 3:
                    forms += [(f"bvhgpu_traverse_od_{sfx}", S.od, False), (f"bvhgpu_traverse_dev_{sfx}", S.rays, True),
                              (f"bvhgpu_traverse_od_dev_{sfx}", S.od, True)]
                if D == 4:
                    forms.append((f"bvhgpu_traverse_dev_{sfx}", S.rays, True))
                for n in SMALL:
                    for name, src, dev in forms:
                        _check_csr(_call_csr(S, n, dev, name, (h, mode), src, int(woff[n])), woff, whits, n, f"{name} flat={flat}")
        elif family == "query":
            rng = np.random.default_rng(D)
            for kind in (capi.QUERY_AABB, capi.QUERY_POINT, capi.QUERY_BALL):
                q = dimref.queries(kind, S.mn, S.mx, NB, F, rng)
                for flat in (False, True):
                    mode = capi.TRAVERSE_FLAT if flat else capi.TRAVERSE_BVH
                    woff, whits = _query_ref(S, kind, q, flat)
                    forms = [(f"bvhgpu_query_{sfx}", False)] + ([(f"bvhgpu_query_dev_{sfx}", True)] if D in (3, 4) else [])
                    for n in SMALL:
                        for name, dev in forms:
                            _check_csr(_call_csr(S, n, dev, name, (h, mode, kind), q, int(woff[n])), woff, whits, n, f"{name} kind={kind} flat={flat}")
        elif family in ("nearest", "nearest_triangles"):
            for flat in (False, True):
                mode = capi.TRAVERSE_FLAT if flat else capi.TRAVERSE_BVH
                if family == "nearest":
                    ws, wd = _nearest_ref(S, flat)
                else:
                    ws, wd = O.nearest_to(S.flat if flat else S.nodes, S.shapes, S.pts, prec, flat=flat, kind=O.DIST_TRIANGLE, tris=S.tris)
                name = f"bvhgpu_{family}_{sfx}"
                for n in SMALL:
                    gs, gd = _rows(S, n, False, name, lambda i, n: (h, mode, i(S.pts[:n]), n), [(), ()], [(4, np.uint32), (isz, F)])
                    assert np.array_equal(gs, ws[:n]) and gd.tobytes() == wd[:n].tobytes(), (name, flat, n)
        elif family == "nearest_candidates":
            if D == 3:
                ws, _ = O.nearest_to(S.nodes, S.shapes, S.pts, prec)
            else:
                ws = np.array([S.tree.nearest_bvh(list(p))[0] for p in S.pts], dtype=np.uint32)
            woff, wc = S.bvh.nearest_candidates(S.pts)
            woff = woff.astype(np.uint64)
            for i in range(NB):
                assert ws[i] in wc[woff[i]:woff[i + 1]], i
            for n in SMALL:                                          # the lists do not depend on the batch they are in
                got = _call_csr(S, n, False, f"bvhgpu_nearest_candidates_{sfx}", (h,), S.pts, int(woff[n]))
                _check_csr(got, woff, wc, n, "nearest_candidates")
        elif family == "traverse_ordered":
            for asc in (1, 0):
                rows = [S.tree.ordered((list(S.o[i]), list(S.inv[i])), bool(asc)) for i in range(NB)]
                woff, whits = _csr([[s for s, _ in r] for r in rows])
                wd = np.array([x[1] for r in rows for x in r], dtype=F)
                for n in SMALL:
                    m = int(woff[n])
                    got = _call_csr(S, n, False, f"bvhgpu_traverse_ordered_{sfx}", (h,), S.rays, m, ascending=asc)
                    _check_csr(got, woff, whits, n, f"traverse_ordered asc={asc}")
                    assert got[2].tobytes() == wd[:m].tobytes(), (asc, n)
        elif family in ("closest_aabb", "closest_triangles"):
            tri = family == "closest_triangles"
            if D == 3:
                ws, wd, wuv = O.closest_hit(S.nodes, S.shapes, S.rays, S.tris if tri else None, prec)
            else:
                rows = [S.tree.closest((list(S.o[i]), list(S.inv[i]))) for i in range(NB)]
                ws = np.array([r[0] for r in rows], dtype=np.uint32)
                wd = np.array([np.inf if r[1] is None else r[1] for r in rows], dtype=F)
            for n in SMALL:
                if D == 3:
                    forms = [(False, f"bvhgpu_closest_hit_{sfx}", lambda i, n: (h, i(S.rays[:n]), n, int(tri)))]
                    for lay, src in ((capi.RAYS_FULL, S.rays), (capi.RAYS_OD, S.od)):
                        forms.append((True, f"bvhgpu_closest_hit_dev_{sfx}", lambda i, n, lay=lay, src=src: (h, i(src[:n]), lay, n, int(tri))))
                    spec, per = [(4, np.uint32), (isz, F), (2 * isz, F)], [(), (), (2,)]
                else:
                    forms = [(False, f"bvhgpu_closest_hit_{sfx}", lambda i, n: (h, i(S.rays[:n]), n))]
                    if D == 4:
                        forms.append((True, f"bvhgpu_closest_hit_dev_{sfx}", lambda i, n: (h, i(S.rays[:n]), n)))
                    spec, per = [(4, np.uint32), (isz, F)], [(), ()]
                for dev, name, args in forms:
                    out = _rows(S, n, dev, name, args, per, spec)
                    if tri:
                        gs, gd, guv = out
                        same = gs == ws[:n]
                        assert np.array_equal(gd[same], wd[:n][same]) and np.array_equal(guv[same], wuv[:n][same]), (name, n)
                        PC.check_closest(gs, gd, guv, ws[:n], wd[:n], S.tris, S.shapes, S.rays[:n], prec)
                    else:
                        assert np.array_equal(out[0], ws[:n]) and out[1].tobytes() == wd[:n].tobytes(), (name, n)
        elif family == "any_hit":
            for tri in ((0, 1) if D == 3 else (0,)):
                want = H.triangles(S.nodes, S.shapes, S.tris, S.rays, S.tmax) if tri else H.aabb_batch(S.nodes, S.shapes, S.o, S.inv, S.tmax)
                for n in SMALL:
                    if D == 3:
                        forms = [(False, f"bvhgpu_any_hit_{sfx}", lambda i, n: (h, i(S.rays[:n]), n, i(S.tmax[:n]), tri))]
                        for lay, src in ((capi.RAYS_FULL, S.rays), (capi.RAYS_OD, S.od)):
                            forms.append((True, f"bvhgpu_any_hit_dev_{sfx}", lambda i, n, lay=lay, src=src: (h, i(src[:n]), lay, n, i(S.tmax[:n]), tri)))
                    else:
                        forms = [(False, f"bvhgpu_any_hit_{sfx}", lambda i, n: (h, i(S.rays[:n]), n, i(S.tmax[:n])))]
                        if D == 4:
                            forms.append((True, f"bvhgpu_any_hit_dev_{sfx}", lambda i, n: (h, i(S.rays[:n]), n, i(S.tmax[:n]))))
                    for dev, name, args in forms:
                        gs, = _rows(S, n, dev, name, args, [()], [(4, np.uint32)])
                        assert np.array_equal(gs, want[:n]), (name, tri, n)
        elif family == "multi_hit":
            k = K_MID
            for tri in ((0, 1) if D == 3 else (0,)):
                if tri:
                    ws, wd, wuv = MH.triangles(S.nodes, S.shapes, S.tris, S.rays, k, S.tmax)
                else:
                    ws, wd, wuv = MH.aabb_batch(S.nodes, S.shapes, S.o, S.inv, k, S.tmax)
                for n in SMALL:
                    if D == 3:
                        spec, per = [(4 * k, np.uint32), (isz * k, F), (2 * isz * k, F)], [(k,), (k,), (k, 2)]
                        forms = [(False, f"bvhgpu_multi_hit_{sfx}", lambda i, n: (h, i(S.rays[:n]), n, k, i(S.tmax[:n]), tri))]
                        for lay, src in ((capi.RAYS_FULL, S.rays), (capi.RAYS_OD, S.od)):
                            forms.append((True, f"bvhgpu_multi_hit_dev_{sfx}", lambda i, n, lay=lay, src=src: (h, i(src[:n]), lay, n, k, i(S.tmax[:n]), tri)))
                    else:
                        spec, per = [(4 * k, np.uint32), (isz * k, F)], [(k,), (k,)]
                        forms = [(False, f"bvhgpu_multi_hit_{sfx}", lambda i, n: (h, i(S.rays[:n]), n, k, i(S.tmax[:n])))]
                        if D == 4:
                            forms.append((True, f"bvhgpu_multi_hit_dev_{sfx}", lambda i, n: (h, i(S.rays[:n]), n, k, i(S.tmax[:n]))))
                    for dev, name, args in forms:
                        out = _rows(S, n, dev, name, args, per, spec)
                        assert np.array_equal(out[0], ws[:n]) and out[1].tobytes() == np.ascontiguousarray(wd[:n]).tobytes(), (name, tri, n)
                        if tri:
                            assert out[2].tobytes() == np.ascontiguousarray(wuv[:n]).tobytes(), (name, n)
        elif family in ("knn", "knn_triangles"):
            k = K_MID
            tri = family == "knn_triangles"
            if tri:
                pts = KT.near_points(S.tris, NB, np.random.default_rng(4))
                ws, wd, wq = KT.brute(S.tris, pts, k, S.radius)
                spec, per = [(4 * k, np.uint32), (isz * k, F), (3 * isz * k, F)], [(k,), (k,), (k, 3)]
            else:
                pts = S.pts
                ws, wd = KR.brute(S.mn, S.mx, pts, k, S.radius)
                spec, per = [(4 * k, np.uint32), (isz * k, F)], [(k,), (k,)]
            forms = [False] + ([True] if D in (3, 4) else [])
            for n in SMALL:
                for dev in forms:
                    name = f"bvhgpu_{family}{'_dev' if dev else ''}_{sfx}"
                    out = _rows(S, n, dev, name, lambda i, n: (h, i(pts[:n]), n, k, i(S.radius[:n])), per, spec)
                    assert np.array_equal(out[0], ws[:n]) and out[1].tobytes() == np.ascontiguousarray(wd[:n]).tobytes(), (name, n)
                    if tri:
                        assert out[2].tobytes() == np.ascontiguousarray(wq[:n]).tobytes(), (name, n)
    finally:
        S.free()


_CASES = [(f, D, p) for f in FAMILIES for D in (2, 3, 4) for p in ("f32", "f64")
          if not (f in THREE_D_ONLY and D != 3)]


@pytest.mark.parametrize("family,D,prec", _CASES, ids=[f"{f}-{D}d-{p}" for f, D, p in _CASES])
def test_small_sizes_with_guarded_outputs(api, family, D, prec):
    """Every size of the small sweep, every form: the first n rows of the reference, both guards intact, offsets[n] written."""
    _sweep(api, family, D, prec)


# ---- large sizes: tiled batches ----------------------------------------------------------------------------------------------------
def _tiled_csr(off, hits, R):
    """The CSR of a batch whose item i is item i % len(base) of the base batch (offsets u64[R+1], hits)."""
    B = len(off) - 1
    cnt = np.diff(off.astype(np.int64))
    idx = np.arange(R) % B
    toff = np.zeros(R + 1, dtype=np.uint64)
    toff[1:] = np.cumsum(cnt[idx])
    reps, rem = divmod(R, B)
    th = np.concatenate([np.tile(hits, reps), hits[:int(off[rem])]])
    return toff, th


def _tile(a, R):
    return np.ascontiguousarray(a[np.arange(R) % len(a)])


def _oracle_visits(nodes, shapes, rays, R, prec):
    """The visit counter of a batch of R rays tiled from `rays`: the device walk visits one record per child box the oracle's
    recursive walk tests (test_gpu_nan_slab.py), in either semantics, so it is the oracle's slab-test count of the base and of the
    remainder."""
    reps, rem = divmod(R, len(rays))
    v = reps * O.traverse(nodes, shapes, rays, O.MODE_RECURSIVE, prec).slab_tests
    if rem:
        v += O.traverse(nodes, shapes, rays[:rem], O.MODE_RECURSIVE, prec).slab_tests
    return v


def _trav_dev(bvh, rays, mode, cap, od=False):
    import torch

    from bvh_b200 import capi

    src = np.ascontiguousarray(np.concatenate([rays["origin"], rays["direction"]], axis=1)) if od else rays
    d_rays = torch.from_numpy(src.view(np.uint8).reshape(-1).copy()).cuda()
    off, hits = _Out(4 * (len(rays) + 1), True), _Out(4 * cap, True)
    tot = C.c_size_t(0)
    fn = getattr(capi.lib(), f"bvhgpu_traverse{'_od' if od else ''}_dev_{bvh.prec}x3")
    torch.cuda.synchronize()
    capi.check(fn(bvh._h, mode, C.c_void_p(d_rays.data_ptr()), len(rays), off.vp, hits.vp, cap, C.byref(tot)))
    bvh.ctx.synchronize()
    assert tot.value == cap
    return off.get(np.uint32, "traverse_dev"), hits.get(np.uint32, "traverse_dev")


def _trav_host(bvh, rays, mode, cap, od=False):
    """bvhgpu_traverse_* / _od_* with guarded host outputs and cap == total."""
    from bvh_b200 import capi

    src = np.ascontiguousarray(np.concatenate([rays["origin"], rays["direction"]], axis=1)) if od else rays
    off, hits = _Out(4 * (len(rays) + 1), False), _Out(4 * cap, False)
    tot = C.c_size_t(0)
    fn = getattr(capi.lib(), f"bvhgpu_traverse{'_od' if od else ''}_{bvh.prec}x3")
    capi.check(fn(bvh._h, mode, C.c_void_p(src.ctypes.data), len(rays), off.vp, hits.vp, cap, C.byref(tot)))
    assert tot.value == cap
    return off.get(np.uint32, "traverse"), hits.get(np.uint32, "traverse")


def _base3(prec="f32"):
    """boxes21 with BASE rays: (shapes, rays, {mode: oracle CSR}, visits(R) = the oracle's visit counter of R tiled rays)."""
    shapes = scene("boxes21", prec)
    nodes = O.build(shapes, prec).nodes
    rays = rays_for(shapes, BASE, prec, seed=11, axis_aligned=300)
    ref = {}
    for mode, tree, om in ((0, nodes, O.MODE_RECURSIVE), (1, O.flatten(nodes, prec), O.MODE_FLAT)):
        r = O.traverse(tree, shapes, rays, om, prec)
        ref[mode] = (r.offsets, r.hits)
    return shapes, rays, ref, lambda R: _oracle_visits(nodes, shapes, rays, R, prec)


def _assert_csr(off, hits, want, what):
    assert np.array_equal(off.astype(np.uint64), want[0]), f"{what}: offsets"
    assert np.array_equal(hits, want[1]), f"{what}: hits"


def test_traverse_across_the_scan_post_tile_loop(api):
    """3-D traverse, BVH and FLAT, host and device forms, at SCAN_TILE * SCAN_THREADS - 1 / + 0 / + 1 rays."""
    shapes, rays, ref, visits_of = _base3()
    bvh = api.Bvh.build(shapes)
    try:
        for R in LE.edges("scan_post"):
            big = _tile(rays, R)
            for mode in (0, 1):
                want = _tiled_csr(*ref[mode], R)
                cap = int(want[0][-1])
                visits = visits_of(R)
                for form in (_trav_dev, _trav_host):
                    _assert_csr(*form(bvh, big, mode, cap), want, f"{form.__name__} R={R} mode={mode}")
                    assert bvh.traverse_stats() == (visits, cap), (form.__name__, R, mode)
    finally:
        bvh.free()


def test_host_path_at_its_thresholds(api):
    """The host path at one ray either side of streaming and of the sliced emit, and at a batch with the largest chunk count and a
    remainder: the CSR and the visit counter of the tiled oracle, streamed exactly from STREAM_MIN rays."""
    shapes, rays, ref, visits_of = _base3()
    bvh = api.Bvh.build(shapes)
    ctx = bvh.ctx
    try:
        ctx.set_option("traverse_stream", 1)
        for R in LE.edges("host"):
            big = _tile(rays, R)
            for mode in (0, 1):
                want = _tiled_csr(*ref[mode], R)
                cap = int(want[0][-1])
                _assert_csr(*_trav_host(bvh, big, mode, cap, od=(mode == 1)), want, f"host R={R} mode={mode}")
                assert ctx.get_metric("host_streamed") == float(R >= LE.CONST["STREAM_MIN"]), R
                assert bvh.traverse_stats() == (visits_of(R), cap), (R, mode)
    finally:
        ctx.set_option("traverse_stream", -1)
        bvh.free()


def test_top_walk_grid_edges(api):
    """walk_top_kernel (traverse_top = 1) at TOP_RAYS_PER_CTA * SMs - 1 / + 0 / + 1 rays: its grid stops growing there."""
    shapes, rays, ref, visits_of = _base3()
    bvh = api.Bvh.build(shapes)
    ctx = bvh.ctx
    try:
        for R in LE.edges("top", LE.sm_count()):
            big = _tile(rays, R)
            for mode in (0, 1):
                want = _tiled_csr(*ref[mode], R)
                cap = int(want[0][-1])
                visits = visits_of(R)
                ctx.set_option("traverse_persistent", 1); ctx.set_option("traverse_top", 1)
                try:
                    _assert_csr(*_trav_dev(bvh, big, mode, cap), want, f"top R={R} mode={mode}")
                    assert bvh.traverse_stats() == (visits, cap), (R, mode)
                finally:
                    ctx.set_option("traverse_persistent", 2); ctx.set_option("traverse_top", -1)
    finally:
        bvh.free()


@pytest.mark.parametrize("D", [2, 3, 4])
def test_csr_queries_across_the_scan_blocks_loop(api, D):
    """A Point query in D dimensions (and nearest_candidates in 3-D) at CSR_SCAN_TILE * 1024 - 1 / + 0 / + 1 items: the tile sums of
    scan_blocks_kernel carry into a second loop step."""
    from bvh_b200 import capi

    F = np.float32
    rng = np.random.default_rng(40 + D)
    mn, mx = dimref.scene("random", 64, D, F, rng)
    q = dimref.queries(capi.QUERY_POINT, mn, mx, BASE, F, rng, nan=False)
    if D == 3:
        shapes = O.make_aabbs(mn, mx, "f32")
        bvh = api.Bvh.build(shapes)
        nodes = O.build(shapes).nodes
        base = O.query(capi.QUERY_POINT, q, nodes, shapes, None, "f32")
        ws, _ = O.nearest_to(nodes, shapes, q)
    else:
        cls = {2: api.Bvh2, 4: api.Bvh4}[D]
        shapes = np.zeros(len(mn), dtype=cls._TABLE["f32"]["aabb"])
        shapes["min"], shapes["max"] = mn, mx
        bvh = cls.build(shapes)
        t = dimref.Tree(bvh.nodes_and_index()[0], shapes)
        base = _csr([t.query_bvh(capi.QUERY_POINT, list(p)) for p in q])
    try:
        if D == 3:
            coff, cand = bvh.nearest_candidates(q)
            for i in range(BASE):
                assert ws[i] in cand[coff[i]:coff[i + 1]], i
        for R in LE.edges("scan_blocks"):
            big = _tile(q, R)
            off, hits = bvh.query_batch(capi.QUERY_POINT, big)
            _assert_csr(off, hits, _tiled_csr(*base, R), f"query D={D} R={R}")
            if D == 3:
                off, c = bvh.nearest_candidates(big)
                _assert_csr(off, c, _tiled_csr(coff.astype(np.uint64), cand, R), f"nearest_candidates R={R}")
    finally:
        bvh.free()


# ---- forced launch geometry ----------------------------------------------------------------------------------------------------------
def test_forced_walk_grid(api):
    """Option walk_grid on the persistent walk (traverse_persistent = 1, traverse_top = 0): 1, 2, 3, SMs - 1, SMs + 1 and 4 SMs + 1
    CTAs give the oracle's CSR and visit counter, f32 and f64, BVH and FLAT, full and OD rays, on the plain walk (host and device
    forms) and on the streamed host path.  The launch caps the grid at one CTA per PERSISTENT_THREADS rays, so every batch is large
    enough for each forced grid to launch as many CTAs as it asks for."""
    sms = LE.sm_count()
    grids = [1, 2, 3, sms - 1, sms + 1, 4 * sms + 1]
    per_cta = LE.CONST["PERSISTENT_THREADS"]
    Rp = per_cta * grids[-1] + 7                             # the plain walk (traverse_stream = 0 keeps the host form off streaming)
    Rs = max(LE.CONST["STREAM_MIN"], Rp) + 7
    for R in (Rp, Rs):
        launched = [min(g, -(-R // per_cta)) for g in grids]
        assert launched == grids, (R, launched)
    for prec in ("f32", "f64"):
        shapes, rays, ref, visits_of = _base3(prec)
        bvh = api.Bvh.build(shapes, prec=prec)
        ctx = bvh.ctx
        try:
            for mode in (0, 1):
                cases = [(_tile(rays, Rp), _tiled_csr(*ref[mode], Rp), False), (_tile(rays, Rs), _tiled_csr(*ref[mode], Rs), True)]
                for batch, want, streamed in cases:
                    cap = int(want[0][-1])
                    visits = visits_of(len(batch))
                    ctx.set_option("traverse_stream", 1 if streamed else 0)
                    ctx.set_option("traverse_persistent", 1); ctx.set_option("traverse_top", 0)
                    try:
                        for g in [0] + grids:
                            ctx.set_option("walk_grid", g)
                            forms = [("host", False), ("host_od", True)] + ([] if streamed else [("dev", False), ("dev_od", True)])
                            for fname, od in forms:
                                form = _trav_host if fname.startswith("host") else _trav_dev
                                _assert_csr(*form(bvh, batch, mode, cap, od=od), want, f"{prec} grid={g} mode={mode} {fname} streamed={streamed}")
                                if fname.startswith("host"):
                                    assert ctx.get_metric("host_streamed") == float(streamed)
                                assert bvh.traverse_stats() == (visits, cap), (prec, g, mode, fname, streamed)
                    finally:
                        ctx.set_option("walk_grid", 0); ctx.set_option("traverse_persistent", 2); ctx.set_option("traverse_top", -1)
                        ctx.set_option("traverse_stream", -1)
        finally:
            bvh.free()


def test_top_walk_on_a_2d_tree(api):
    """A 2-D tree through the 3-D walk with traverse_top = 1, BVH and FLAT, below and above the streaming threshold of 3-D host
    calls with streaming forced on (a 2-D host call uploads its rays, then walks: it never streams): the restated Bvh::traverse /
    FlatBvh::traverse.  The flat walk's leaf re-test reads the 2-D tree's shape boxes lifted to 3-D."""
    F = np.float32
    rng = np.random.default_rng(12)
    mn, mx = dimref.scene("random", 300, 2, F, rng)
    shapes = np.zeros(len(mn), dtype=api.Bvh2._TABLE["f32"]["aabb"])
    shapes["min"], shapes["max"] = mn, mx
    bvh = api.Bvh2.build(shapes)
    o, d, inv = dimorder.rays(mn, mx, BASE, F, rng)
    rays = np.zeros(BASE, dtype=api.Bvh2._TABLE["f32"]["ray"])
    rays["origin"], rays["direction"], rays["inv_direction"] = o, d, inv
    tree = dimorder.Tree(bvh.nodes_and_index()[0], shapes)
    ctx = bvh.ctx
    try:
        for flat in (False, True):
            base = _ray_sets(tree, o, inv, flat)
            for R in (BASE, LE.CONST["STREAM_MIN"] + 7):
                want = _tiled_csr(*base, R)
                ctx.set_option("traverse_persistent", 1); ctx.set_option("traverse_top", 1); ctx.set_option("traverse_stream", 1)
                try:
                    off, hits = bvh.traverse_batch(_tile(rays, R), mode=int(flat))
                finally:
                    ctx.set_option("traverse_persistent", 2); ctx.set_option("traverse_top", -1); ctx.set_option("traverse_stream", -1)
                _assert_csr(off, hits, want, f"2-D flat={flat} R={R}")
    finally:
        bvh.free()


# ---- values read once per process: one child per value --------------------------------------------------------------------------
_CHILD = r"""
import hashlib, json, sys
import numpy as np
sys.path.insert(0, %(root)r)
from bvh_b200 import api, scenes
from oracle import oracle as O
from tests import launch_edges as LE
from tests.scenes import rays_for, scene

def digest(bvh, off, hits):
    return [hashlib.sha256(off.tobytes() + hits.tobytes()).hexdigest(), bvh.traverse_stats()[0]]

out = {}
if %(what)r == "top":
    # walk_top_kernel with 4 visits per vote (records up to TOP_UNROLL_MAX_BYTES), then with 1; both trees exceed the top's budget,
    # so the walk also runs below the top
    for name in ("l2", "beyond_l2"):
        shapes = scene("random5000") if name == "l2" else scenes.create_n_cubes_aabbs(50_000)
        records = LE.trec_bytes(len(shapes))
        assert (records <= LE.CONST["TOP_UNROLL_MAX_BYTES"]) == (name == "l2"), (name, records)
        assert records // LE.CONST["TNODE_F32_BYTES"] > LE.CONST["TOP_BUDGET"], name
        oo, dd = scenes.ray_endpoints(20_000, 3)
        rays = O.ray_new(oo, dd)
        bvh = api.Bvh.build(shapes)
        ctx = bvh.ctx
        ctx.set_option("traverse_persistent", 1); ctx.set_option("traverse_stream", 0)
        launches = []
        for top in (0, 1):                      # the first top walk of a tree builds its top records first: 5 more launches
            ctx.set_option("traverse_top", top)
            before = ctx.launch_count()
            bvh.traverse_batch(rays, mode=0)
            launches.append(ctx.launch_count() - before)
        assert launches[1] > launches[0], (name, launches)
        for mode in (0, 1):
            out[f"{name}/{mode}"] = digest(bvh, *bvh.traverse_batch(rays, mode=mode))
        bvh.free()
else:
    shapes = scene("boxes21")
    base = rays_for(shapes, 4099, seed=11, axis_aligned=300)
    rays = np.ascontiguousarray(base[np.arange(%(R)d) %% len(base)])
    bvh = api.Bvh.build(shapes)
    bvh.ctx.set_option("traverse_stream", 1)
    for mode in (0, 1):
        out[f"stream/{mode}"] = digest(bvh, *bvh.traverse_batch(rays, mode=mode, compact=bool(mode))) + [bvh.ctx.get_metric("host_streamed")]
    bvh.free()
print("RESULT " + json.dumps(out))
"""
_STREAM_R = 1_000_003


def _child(what, env_extra):
    env = {k: v for k, v in os.environ.items() if not k.startswith("BVHGPU_") and k != "CUDA_LAUNCH_BLOCKING"}
    env.update(env_extra)
    r = subprocess.run([sys.executable, "-c", _CHILD % {"root": ROOT, "what": what, "R": _STREAM_R}], capture_output=True, text=True,
                       timeout=600, env=env)
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-1500:]
    return json.loads(r.stdout.split("RESULT ")[-1])


@pytest.fixture(scope="module")
def defaults():
    """The results of a child at the default values."""
    for k in ("BVHGPU_TOP_REFILL", "BVHGPU_CHUNKS", "BVHGPU_CHUNK_SCHEDULE"):
        assert k not in os.environ, k
    return {"top": _child("top", {}), "stream": _child("stream", {})}


@pytest.mark.parametrize("refill", [1, 2, 31, 32])
def test_top_refill_values(defaults, refill):
    """BVHGPU_TOP_REFILL (idle lanes per refill of walk_top_kernel), both visits-per-vote forms: the CSR and the visit counter of
    the default refill."""
    got = _child("top", {"BVHGPU_TOP_REFILL": str(refill)})
    assert got == defaults["top"], refill


@pytest.mark.parametrize("sched", [0, 1])
@pytest.mark.parametrize("chunks", [2, 3, 16, 17])
def test_chunk_count_and_schedule(defaults, chunks, sched):
    """BVHGPU_CHUNKS (17 is clamped to BVH_MAX_CHUNKS) x BVHGPU_CHUNK_SCHEDULE on the streamed host path: streamed, with the CSR and
    the visit counter of the default chunking."""
    got = _child("stream", {"BVHGPU_CHUNKS": str(chunks), "BVHGPU_CHUNK_SCHEDULE": str(sched)})
    for v in got.values():
        assert v[2] == 1.0
    assert got == defaults["stream"], (chunks, sched)
