"""Host-side mirror of the reference crate's interface for the hot path, on top of the C ABI.

Names follow the reference (svenstaro/bvh 0.12.0):

    Bvh.build(shapes) / Bvh.build_par(shapes)     src/bvh/bvh_impl.rs:40-96, src/bounding_hierarchy.rs:158-177
    bvh.nodes, shape node indices                  src/bvh/bvh_impl.rs:27-33, src/bounding_hierarchy.rs:53-65
    bvh.flatten() -> FlatBvh                       src/flat_bvh.rs:312-319
    bvh.traverse(ray, shapes)                      src/bvh/bvh_impl.rs:104-119
    bvh.traverse_iterator(ray, shapes)             src/bvh/bvh_impl.rs:128-134
    flat_bvh.traverse(ray, shapes)                 src/flat_bvh.rs:396-431
    Ray.new(origin, direction)                     src/ray/ray_impl.rs:70-80

plus the batched form the GPU exists for: bvh.traverse_batch(rays) -> CSR (offsets, hits).
"Shapes" are anything with an `.aabb()` method (Bounded, src/aabb/aabb_impl.rs:28-56) and
optionally `set_bh_node_index` (BHShape, src/bounding_hierarchy.rs:53-65); numpy AABB arrays are
accepted directly.  Everything below runs on the GPU through libbvh_b200.so; there is no CPU path.
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, Sequence

import numpy as np

from . import capi
from .dtypes import BY_PREC, BY_PREC_2D, BY_PREC_4D, U32_MAX


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _same_kind(a, b, what: str = "overlap_pairs_with"):
    """The two trees of an overlap_pairs_with / triangle_pairs_with call: the same class (so the same dimension) and the same
    precision."""
    if type(a) is not type(b):
        raise TypeError(f"{what}: {type(a).__name__} against {type(b).__name__}")
    if a.prec != b.prec:
        raise ValueError(f"{what}: {a.prec} tree against a {b.prec} tree")


class Context:
    """One per device (stream + scratch pool)."""

    _default: dict[int, "Context"] = {}

    def __init__(self, device: int = 0):
        self._h = C.c_void_p()
        capi.check(capi.lib().bvhgpu_create(device, C.byref(self._h)))
        self.device = device
        self._host = {}

    @classmethod
    def default(cls, device: int = 0) -> "Context":
        if device not in cls._default:
            cls._default[device] = cls(device)
        return cls._default[device]

    def set_stream(self, cuda_stream_handle: int | None):
        """Enqueue on the given cudaStream_t handle (0 = CUDA's legacy default stream); None = the context's own stream.

        A change of stream keeps the context's calls in order without blocking the host: the new stream waits for
        everything already enqueued on the old one (builds, refits, updates, tree frees), and `synchronize` afterwards
        covers all of it.  The caller still orders the tensors it passes in (and reads back) against the stream it
        installs, e.g. by installing `torch.cuda.current_stream().cuda_stream`."""
        if cuda_stream_handle is None:
            capi.check(capi.lib().bvhgpu_reset_stream(self._h))
        else:
            capi.check(capi.lib().bvhgpu_set_stream(self._h, C.c_void_p(cuda_stream_handle)))

    def synchronize(self):
        capi.check(capi.lib().bvhgpu_synchronize(self._h))

    def launch_count(self) -> int:
        return int(capi.lib().bvhgpu_launch_count(self._h))

    def set_option(self, name: str, value: int):
        capi.check(capi.lib().bvhgpu_set_option(self._h, name.encode(), int(value)))

    def get_metric(self, name: str) -> float:
        out = C.c_double(0.0)
        capi.check(capi.lib().bvhgpu_get_metric(self._h, name.encode(), C.byref(out)))
        return out.value

    def host_alloc(self, nbytes: int, dtype=np.uint8) -> np.ndarray:
        """Pinned host memory on the device's NUMA node (bvhgpu_host_alloc) as a numpy array; release with host_free(arr)."""
        p = C.c_void_p()
        capi.check(capi.lib().bvhgpu_host_alloc(self._h, nbytes, C.byref(p)))
        arr = np.ctypeslib.as_array((C.c_ubyte * nbytes).from_address(p.value)).view(dtype)
        self._host.setdefault(arr.ctypes.data, p)
        return arr

    def host_free(self, arr: np.ndarray):
        p = self._host.pop(arr.ctypes.data)
        capi.check(capi.lib().bvhgpu_host_free(self._h, p))

    def close(self):
        if self._h:
            capi.lib().bvhgpu_destroy(self._h)
            self._h = C.c_void_p()


def _gather_aabbs(shapes, prec):
    d = BY_PREC[prec]
    if isinstance(shapes, np.ndarray):
        return np.ascontiguousarray(shapes, dtype=d["aabb"])
    out = np.zeros(len(shapes), dtype=d["aabb"])
    for i, s in enumerate(shapes):                      # Bounded::aabb(), once per shape
        a = s.aabb()
        out[i]["min"] = a[0]
        out[i]["max"] = a[1]
    return out


class Ray:
    """Ray<T,3> (src/ray/ray_impl.rs:17-29).  Ray.new normalises on the device (bvhgpu_rays_new_dev_*)."""

    @staticmethod
    def new(origins, directions, prec: str = "f32", ctx: Context | None = None) -> np.ndarray:
        import torch

        d = BY_PREC[prec]
        ctx = ctx or Context.default()
        o = np.ascontiguousarray(origins, dtype=d["scalar"]).reshape(-1, 3)
        v = np.ascontiguousarray(directions, dtype=d["scalar"]).reshape(-1, 3)
        n = len(o)
        dev = torch.device("cuda", ctx.device)
        to, tv = torch.from_numpy(o).to(dev), torch.from_numpy(v).to(dev)
        out = torch.empty(n * d["ray"].itemsize, dtype=torch.uint8, device=dev)
        torch.cuda.synchronize(dev)
        capi.check(getattr(capi.lib(), f"bvhgpu_rays_new_dev_{d['suffix']}")(ctx._h, to.data_ptr(), tv.data_ptr(), n, out.data_ptr()))
        ctx.synchronize()
        return out.cpu().numpy().view(d["ray"]).copy()


class FlatBvh:
    """FlatBvh = Vec<FlatNode> (src/flat_bvh.rs:153) produced by Bvh.flatten(); traversal runs on the device tree."""

    def __init__(self, bvh: "Bvh", nodes: np.ndarray):
        self._bvh = bvh
        self.nodes = nodes

    def __len__(self):
        return len(self.nodes)

    def traverse(self, ray, shapes=None):
        return self._bvh._traverse_one(ray, shapes, capi.TRAVERSE_FLAT)

    def traverse_batch(self, rays):
        return self._bvh.traverse_batch(rays, mode=capi.TRAVERSE_FLAT)


class _Tree:
    """What the trees of every dimension share: the handle of one device tree and the calls whose arguments do not depend on D.
    A subclass sets _TABLE (dtypes.BY_PREC*) and _DIM, and defines _num_shapes()."""

    _TABLE: dict
    _DIM: int

    def __init__(self, handle, prec: str, ctx: Context):
        self._h, self.prec, self.ctx, self._d = handle, prec, ctx, self._TABLE[prec]

    def free(self):
        if self._h:
            getattr(capi.lib(), f"bvhgpu_tree_free_{self._d['suffix']}")(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    def _points(self, points) -> np.ndarray:
        return np.ascontiguousarray(points, dtype=self._d["scalar"]).reshape(-1, self._DIM)

    def _limits(self, x, n: int):
        """A per-item limit (tmax, max_dist) as n contiguous scalars of the tree's precision: x is a scalar for all items or one value
        per item.  None stays None, the null pointer that means no limit."""
        return None if x is None else np.ascontiguousarray(np.broadcast_to(np.asarray(x, dtype=self._d["scalar"]), (n,)))

    def _csr(self, fn, n: int, cap: int, *args, dists: bool = False):
        """CSR (offsets u32[n + 1], hits u32[total]) from fn(*args, offsets, hits, cap, &total); with dists=True fn also takes the
        distances after the hits, and they are returned third.  A short capacity (ERR_CAPACITY with a total the u32 offsets can hold)
        is completed as the ABI fixes it: a 3-D tree copies the list its walk retained (bvhgpu_traverse_fetch_*); 2-D and 4-D trees
        retain nothing, and nothing retains distances, so those call again with cap = total."""
        offsets = np.zeros(n + 1, dtype=np.uint32)
        while True:
            out = [np.zeros(cap, dtype=np.uint32)]
            if dists:
                out.append(np.zeros(cap, dtype=self._d["scalar"]))
            total = C.c_size_t(0)
            st = fn(*args, _ptr(offsets), *map(_ptr, out), cap, C.byref(total))
            t = total.value
            if st == capi.ERR_CAPACITY and t <= U32_MAX:
                if self._DIM == 3 and not dists:
                    hits = np.zeros(t, dtype=np.uint32)
                    capi.check(getattr(capi.lib(), f"bvhgpu_traverse_fetch_{self._d['suffix']}")(self._h, _ptr(hits), t))
                    return offsets, hits
                if t > cap:
                    cap = t
                    continue
            capi.check(st)
            return (offsets, *(a[:t] for a in out))

    def flatten(self) -> np.ndarray:
        n = self._num_shapes()
        cap = 0 if n == 0 else (1 if n == 1 else 3 * n - 2)
        out = np.zeros(cap, dtype=self._d["flat"])
        ln = C.c_size_t(0)
        capi.check(getattr(capi.lib(), f"bvhgpu_flatten_{self._d['suffix']}")(self._h, _ptr(out), cap, C.byref(ln)))
        return out[: ln.value]

    def traverse_ordered(self, rays, ascending: bool = True):
        """Batched nearest_traverse_iterator (ascending: by entry distance) / farthest_traverse_iterator (by exit distance,
        descending): (offsets, hits, dists), the set of traverse_batch(..., TRAVERSE_BVH) perfectly sorted per ray, ties in DFS order,
        with the slice distance of the child box the tree stores for each leaf.  A short capacity (default max(8 n, 1024)) is retried
        at the exact total, hits and distances together."""
        rays = np.ascontiguousarray(rays, dtype=self._d["ray"])
        fn = getattr(capi.lib(), f"bvhgpu_traverse_ordered_{self._d['suffix']}")
        return self._csr(fn, len(rays), max(8 * len(rays), 1024), self._h, _ptr(rays), len(rays), 1 if ascending else 0, dists=True)

    def query_batch(self, kind: int, queries, mode: int = capi.TRAVERSE_BVH):
        """Bvh::traverse with Aabb / Point / Ball queries (IntersectsAabb implementors other than Ray): (n, 2D) {min, max} for
        capi.QUERY_AABB, (n, D) points for QUERY_POINT, (n, D+1) {center, radius} for QUERY_BALL.  CSR (offsets, hits), hits of a
        query in the reference's DFS order."""
        D = self._DIM
        stride = {capi.QUERY_AABB: 2 * D, capi.QUERY_POINT: D, capi.QUERY_BALL: D + 1}[kind]
        q = np.ascontiguousarray(queries, dtype=self._d["scalar"]).reshape(-1, stride)
        fn = getattr(capi.lib(), f"bvhgpu_query_{self._d['suffix']}")
        return self._csr(fn, len(q), max(16 * len(q), 1024), self._h, mode, kind, _ptr(q), len(q))

    def overlap_pairs(self, cap: int | None = None):
        """Every pair of shapes whose own current AABBs intersect (touching faces included), each once: CSR (offsets[n + 1], hits)
        indexed by shape, row s = the shapes t with node_index[t] > node_index[s] whose box meets s's, in DFS order.  A short
        capacity (default max(4 n, 1024)) is completed from the retained list in 3-D (bvhgpu_traverse_fetch_*) and retried once at the
        exact total in 2-D and 4-D."""
        n = self._num_shapes()
        fn = getattr(capi.lib(), f"bvhgpu_overlap_pairs_{self._d['suffix']}")
        return self._csr(fn, n, max(4 * n, 1024) if cap is None else int(cap), self._h)

    def overlap_pairs_with(self, other, cap: int | None = None):
        """Every pair (a, b) of a shape of this tree and a shape of `other` whose own current AABBs intersect (touching faces included):
        CSR (offsets[n + 1], hits) indexed by this tree's shapes, row a = other's shapes whose box meets a's, in other's DFS order.
        Both trees must share a context; other may be self.  A short capacity (default max(4 n, 1024)) is completed from this tree's
        retained list in 3-D (bvhgpu_traverse_fetch_*) and retried once at the exact total in 2-D and 4-D."""
        _same_kind(self, other)
        n = self._num_shapes()
        fn = getattr(capi.lib(), f"bvhgpu_overlap_trees_{self._d['suffix']}")
        return self._csr(fn, n, max(4 * n, 1024) if cap is None else int(cap), self._h, other._h)

    def nearest_to_batch(self, points, mode: int = capi.TRAVERSE_BVH):
        """Bvh::nearest_to / FlatBvh::nearest_to (bvh_impl.rs:221-238, flat_bvh.rs:513-562) for shapes whose PointDistance is their AABB
        distance (the reference's UnitBox): (shape index per point, U32_MAX for an empty tree; distance per point).  points: (n, D)."""
        p = self._points(points)
        shape = np.zeros(len(p), dtype=np.uint32)
        dist = np.zeros(len(p), dtype=self._d["scalar"])
        capi.check(getattr(capi.lib(), f"bvhgpu_nearest_{self._d['suffix']}")(self._h, mode, _ptr(p), len(p), _ptr(shape), _ptr(dist)))
        return shape, dist

    def nearest_candidates(self, points):
        """For shapes with their own PointDistance: CSR (offsets, shape indices) of candidate lists that contain the nearest shape of
        every point; evaluate distance_squared on each list and keep the minimum (see `nearest_to`).  points: (n, D)."""
        p = self._points(points)
        fn = getattr(capi.lib(), f"bvhgpu_nearest_candidates_{self._d['suffix']}")
        return self._csr(fn, len(p), max(64 * len(p), 1024), self._h, _ptr(p), len(p))

    def nearest_to(self, point, shapes, distance_squared):
        """BoundingHierarchy::nearest_to for one point and an arbitrary shape distance: `distance_squared(shape, point)` is the shape's
        PointDistance::distance_squared.  Returns (shape, distance) or None for an empty tree."""
        off, cand = self.nearest_candidates([point])
        best = None
        for s in cand[off[0]:off[1]]:
            d = distance_squared(shapes[int(s)], point)
            if best is None or d < best[1]:
                best = (shapes[int(s)], d)
        return None if best is None else (best[0], float(np.sqrt(best[1])))

    def knn(self, points, k: int, max_dist=None):
        """The k nearest shapes of every point (points (n, D)): (shape (n, k) u32, dist (n, k)).  Row i lists the shapes in ascending
        (Aabb::min_distance_squared of the shape's own box, index) order with their distances; with `max_dist` (a scalar for all points,
        one limit per point, or None for no limit) only shapes at squared distance <= fl(r * r) qualify (r < 0 or NaN: none).  Slots
        past the qualifying shapes hold U32_MAX and +inf.  Exact: the head of a stable brute-force sort.  1 <= k <= 64."""
        p = self._points(points)
        n = len(p)
        kk = max(int(k), 0)
        shape = np.zeros((n, kk), dtype=np.uint32)
        dist = np.zeros((n, kk), dtype=self._d["scalar"])
        capi.check(getattr(capi.lib(), f"bvhgpu_knn_{self._d['suffix']}")(self._h, _ptr(p), n, int(k) & 0xFFFFFFFF, _ptr(self._limits(max_dist, n)),
                                                                         _ptr(shape), _ptr(dist)))
        return shape, dist


class Bvh(_Tree):
    """Device-resident Bvh<T,3>."""

    _TABLE = BY_PREC
    _DIM = 3

    def __init__(self, handle, prec: str, ctx: Context):
        super().__init__(handle, prec, ctx)
        self._nodes = None
        self._node_index = None

    # ---- construction ----------------------------------------------------------------------------
    @classmethod
    def build(cls, shapes, prec: str = "f32", ctx: Context | None = None, mode: int = capi.BUILD_EXACT_SAH) -> "Bvh":
        ctx = ctx or Context.default()
        d = BY_PREC[prec]
        aabbs = _gather_aabbs(shapes, prec)
        h = C.c_void_p()
        capi.check(getattr(capi.lib(), f"bvhgpu_build_{d['suffix']}")(ctx._h, _ptr(aabbs), len(aabbs), mode, C.byref(h)))
        bvh = cls(h, prec, ctx)
        if not isinstance(shapes, np.ndarray) and len(shapes) and hasattr(shapes[0], "set_bh_node_index"):
            for s, ni in zip(shapes, bvh.node_index):    # BHShape::set_bh_node_index
                s.set_bh_node_index(int(ni))
        return bvh

    build_par = build          # rayon is off the hot path: same builder (bounding_hierarchy.rs:170-177)

    @classmethod
    def build_dev(cls, dev_ptr: int, n: int, prec: str = "f32", ctx: Context | None = None, mode: int = capi.BUILD_EXACT_SAH) -> "Bvh":
        """AABBs already on the device (C-ABI layout); asynchronous on the context's stream."""
        ctx = ctx or Context.default()
        d = BY_PREC[prec]
        h = C.c_void_p()
        capi.check(getattr(capi.lib(), f"bvhgpu_build_dev_{d['suffix']}")(ctx._h, C.c_void_p(dev_ptr), n, mode, C.byref(h)))
        return cls(h, prec, ctx)

    @classmethod
    def from_nodes(cls, nodes: np.ndarray, shapes, prec: str = "f32", ctx: Context | None = None) -> "Bvh":
        ctx = ctx or Context.default()
        d = BY_PREC[prec]
        nodes = np.ascontiguousarray(nodes, dtype=d["node"])
        aabbs = _gather_aabbs(shapes, prec)
        h = C.c_void_p()
        capi.check(getattr(capi.lib(), f"bvhgpu_tree_from_nodes_{d['suffix']}")(ctx._h, _ptr(nodes), len(nodes), _ptr(aabbs), len(aabbs), C.byref(h)))
        return cls(h, prec, ctx)

    # ---- Bvh.nodes / node indices ------------------------------------------------------------------
    @property
    def num_shapes(self) -> int:
        return int(getattr(capi.lib(), f"bvhgpu_tree_num_shapes_{self._d['suffix']}")(self._h))

    def _num_shapes(self) -> int:
        return self.num_shapes

    def _materialise(self):
        if self._nodes is None:
            n = self.num_shapes
            nodes = np.zeros(max(2 * n - 1, 0), dtype=self._d["node"])
            idx = np.zeros(n, dtype=np.uint32)
            capi.check(getattr(capi.lib(), f"bvhgpu_tree_nodes_{self._d['suffix']}")(self._h, _ptr(nodes), _ptr(idx)))
            self._nodes, self._node_index = nodes, idx

    @property
    def nodes(self) -> np.ndarray:
        self._materialise()
        return self._nodes

    @property
    def node_index(self) -> np.ndarray:
        self._materialise()
        return self._node_index

    # ---- flatten -----------------------------------------------------------------------------------
    def flatten(self) -> FlatBvh:
        return FlatBvh(self, super().flatten())

    def flatten_custom(self, constructor):
        """Bvh::flatten_custom (src/flat_bvh.rs:240-251): `constructor(aabb, entry, exit, shape)` applied to every FlatNode in the
        reference's emission order; aabb = (min[3], max[3])."""
        f = self.flatten().nodes
        return [constructor((f["aabb"]["min"][i], f["aabb"]["max"][i]), int(f["entry_index"][i]), int(f["exit_index"][i]), int(f["shape_index"][i])) for i in range(len(f))]

    def flatten_dev(self) -> int:
        """Build the FlatBvh on the device only (no host copy, asynchronous); returns its length."""
        ln = C.c_size_t(0)
        capi.check(getattr(capi.lib(), f"bvhgpu_flatten_{self._d['suffix']}")(self._h, None, 0, C.byref(ln)))
        return ln.value

    # ---- traversal ---------------------------------------------------------------------------------
    def traverse_batch(self, rays: np.ndarray, mode: int = capi.TRAVERSE_BVH, cap: int | None = None, compact: bool = False):
        """CSR (offsets u32[nrays+1], hits u32[total]); hits of a ray are in the reference's DFS order.
        compact=True ships only origin + direction (BVHGPU_RAYS_OD, 6 scalars per ray); the device recomputes inv_direction with
        the division Ray::new uses, so the result is bit-identical."""
        rays = np.ascontiguousarray(rays, dtype=self._d["ray"])
        nrays = len(rays)
        fn = getattr(capi.lib(), f"bvhgpu_traverse_{self._d['suffix']}")
        if compact:
            od = np.empty((nrays, 6), dtype=self._d["scalar"])
            od[:, :3], od[:, 3:] = rays["origin"], rays["direction"]
            rays, fn = od, getattr(capi.lib(), f"bvhgpu_traverse_od_{self._d['suffix']}")
        return self._csr(fn, nrays, max(4 * nrays, 1024) if cap is None else cap, self._h, mode, _ptr(rays), nrays)

    def set_triangles(self, triangles):
        """Triangle vertices of the shapes (n, 3, 3) or (n, 9): enables closest_hit(..., triangles=True).  Triangle i must lie inside shape i's AABB."""
        t = np.ascontiguousarray(triangles, dtype=self._d["scalar"]).reshape(-1, 9)
        capi.check(getattr(capi.lib(), f"bvhgpu_tree_set_triangles_{self._d['suffix']}")(self._h, _ptr(t), len(t)))

    def closest_hit(self, rays: np.ndarray, triangles: bool = False):
        """Per ray: (shape index or U32_MAX, distance or inf, uv (n, 2)).  triangles=False: the shape whose AABB is entered first (exact);
        triangles=True: Ray::intersects_triangle minimum over the triangles set with set_triangles (front-to-back, distance-pruned)."""
        rays = np.ascontiguousarray(rays, dtype=self._d["ray"])
        n = len(rays)
        shape = np.zeros(n, dtype=np.uint32)
        dist = np.zeros(n, dtype=self._d["scalar"])
        uv = np.zeros((n, 2), dtype=self._d["scalar"])
        capi.check(getattr(capi.lib(), f"bvhgpu_closest_hit_{self._d['suffix']}")(self._h, _ptr(rays), n, 1 if triangles else 0, _ptr(shape), _ptr(dist), _ptr(uv)))
        return shape, dist, uv

    def any_hit(self, rays: np.ndarray, tmax=None, triangles: bool = False) -> np.ndarray:
        """Occlusion: per ray a shape hit at distance < tmax (one limit per ray, a scalar for all, or None for +inf), U32_MAX if none.
        triangles=False: a shape whose own AABB the ray enters before tmax (exact); triangles=True: a triangle (set_triangles) whose
        Ray::intersects_triangle distance is < tmax.  The walk stops at the first such shape; which one is deterministic."""
        rays = np.ascontiguousarray(rays, dtype=self._d["ray"])
        n = len(rays)
        shape = np.zeros(n, dtype=np.uint32)
        capi.check(getattr(capi.lib(), f"bvhgpu_any_hit_{self._d['suffix']}")(self._h, _ptr(rays), n, _ptr(self._limits(tmax, n)),
                                                                             1 if triangles else 0, _ptr(shape)))
        return shape

    def multi_hit(self, rays: np.ndarray, k: int, tmax=None, triangles: bool = False, uv: bool = False):
        """The first k hits along every ray: (shape (n, k) u32, dist (n, k), uv (n, k, 2) with uv=True else None).  Row r is the head
        of a stable sort of the qualifying hits by key; slots past them hold U32_MAX, +inf and uv (0, 0).  tmax: one limit per ray, a
        scalar for all, or None for none; a hit qualifies only at a distance < tmax.  triangles=False: key (entry of the shape's own
        AABB, DFS order), exact; triangles=True: key (Ray::intersects_triangle distance, shape) over the triangles of set_triangles,
        equal to the unpruned sort wherever its triangles are bounded (DESIGN.md 4.18).  k = 1 without tmax is closest_hit."""
        rays = np.ascontiguousarray(rays, dtype=self._d["ray"])
        n = len(rays)
        kk = max(int(k), 0)
        shape = np.zeros((n, kk), dtype=np.uint32)
        dist = np.zeros((n, kk), dtype=self._d["scalar"])
        u = np.zeros((n, kk, 2), dtype=self._d["scalar"]) if uv else None
        capi.check(getattr(capi.lib(), f"bvhgpu_multi_hit_{self._d['suffix']}")(self._h, _ptr(rays), n, int(k) & 0xFFFFFFFF,
                                                                                _ptr(self._limits(tmax, n)), 1 if triangles else 0, _ptr(shape),
                                                                                _ptr(dist), _ptr(u)))
        return shape, dist, u

    def multi_hit_dev(self, rays_ptr: int, nrays: int, k: int, tmax_ptr: int, shape_ptr: int, dist_ptr: int, uv_ptr: int = 0,
                      triangles: bool = False, layout: int = capi.RAYS_FULL):
        """multi_hit from device pointers: nrays rays (layout RAYS_FULL: the Ray structs, RAYS_OD: origin + direction) and nrays
        limits (tmax_ptr = 0: none) in, nrays * k u32 shapes, distances and (uv_ptr != 0) 2 * nrays * k uv out, enqueued on the
        context's stream without host synchronisation."""
        capi.check(getattr(capi.lib(), f"bvhgpu_multi_hit_dev_{self._d['suffix']}")(
            self._h, C.c_void_p(rays_ptr), layout, nrays, k, C.c_void_p(tmax_ptr or None), 1 if triangles else 0, C.c_void_p(shape_ptr),
            C.c_void_p(dist_ptr), C.c_void_p(uv_ptr or None)))

    def knn_dev(self, points_ptr: int, n: int, k: int, max_dist_ptr: int, shape_ptr: int, dist_ptr: int):
        """knn from device pointers: n points (D scalars each) and n limits (max_dist_ptr = 0: no limit) in, n * k u32 shapes and
        distances out, enqueued on the context's stream without host synchronisation."""
        capi.check(getattr(capi.lib(), f"bvhgpu_knn_dev_{self._d['suffix']}")(self._h, C.c_void_p(points_ptr), n, k, C.c_void_p(max_dist_ptr or None),
                                                                             C.c_void_p(shape_ptr), C.c_void_p(dist_ptr)))

    def knn_triangles(self, points, k: int, max_dist=None, closest: bool = False):
        """The k nearest triangles (set_triangles) of every point: (shape (n, k) u32, dist (n, k)), plus closest (n, k, 3) with
        closest=True.  Keys are Triangle::distance_squared (testbase.rs:353-443), the distance of nearest_triangles_batch; NaN keys never
        qualify; `max_dist` as in knn.  Slots past the qualifying triangles hold U32_MAX, +inf and NaN closest points.  Equal to a
        stable brute-force sort wherever every qualifying triangle's key is at least its own box's pruning bound (DESIGN.md 4.17)."""
        p = self._points(points)
        n = len(p)
        kk = max(int(k), 0)
        shape = np.zeros((n, kk), dtype=np.uint32)
        dist = np.zeros((n, kk), dtype=self._d["scalar"])
        q = np.zeros((n, kk, 3), dtype=self._d["scalar"]) if closest else None
        capi.check(getattr(capi.lib(), f"bvhgpu_knn_triangles_{self._d['suffix']}")(self._h, _ptr(p), n, int(k) & 0xFFFFFFFF,
                                                                                   _ptr(self._limits(max_dist, n)), _ptr(shape), _ptr(dist),
                                                                                   _ptr(q)))
        return (shape, dist, q) if closest else (shape, dist)

    def knn_triangles_dev(self, points_ptr: int, n: int, k: int, max_dist_ptr: int, shape_ptr: int, dist_ptr: int, closest_ptr: int = 0):
        """knn_triangles from device pointers: n points and n limits (max_dist_ptr = 0: no limit) in, n * k u32 shapes, distances and
        (closest_ptr != 0) n * k * 3 closest-point coordinates out, enqueued on the context's stream without host synchronisation."""
        capi.check(getattr(capi.lib(), f"bvhgpu_knn_triangles_dev_{self._d['suffix']}")(
            self._h, C.c_void_p(points_ptr), n, k, C.c_void_p(max_dist_ptr or None), C.c_void_p(shape_ptr), C.c_void_p(dist_ptr),
            C.c_void_p(closest_ptr or None)))

    def count_hits(self, rays: np.ndarray, tmax=None):
        """Crossing counts per ray over the triangles of set_triangles: (front (n,) u32, back (n,) u32).  front counts the triangles whose
        Ray::intersects_triangle distance is finite (and < tmax), back the same with the winding reversed (b and c exchanged).  tmax:
        one limit per ray, a scalar for all, or None for none.  Without a limit exactly the loop over Bvh::traverse with both windings
        (DESIGN.md 4.21)."""
        rays = np.ascontiguousarray(rays, dtype=self._d["ray"])
        n = len(rays)
        front = np.zeros(n, dtype=np.uint32)
        back = np.zeros(n, dtype=np.uint32)
        capi.check(getattr(capi.lib(), f"bvhgpu_count_hits_{self._d['suffix']}")(self._h, _ptr(rays), n, _ptr(self._limits(tmax, n)), _ptr(front),
                                                                                _ptr(back)))
        return front, back

    def count_hits_dev(self, rays_ptr: int, nrays: int, tmax_ptr: int, front_ptr: int, back_ptr: int, layout: int = capi.RAYS_FULL):
        """count_hits from device pointers: nrays rays (RAYS_FULL or RAYS_OD) and nrays limits (tmax_ptr = 0: none) in, nrays u32 front
        and back counts out, enqueued on the context's stream without host synchronisation."""
        capi.check(getattr(capi.lib(), f"bvhgpu_count_hits_dev_{self._d['suffix']}")(
            self._h, C.c_void_p(rays_ptr), layout, nrays, C.c_void_p(tmax_ptr or None), C.c_void_p(front_ptr), C.c_void_p(back_ptr)))

    _RULES = {"even_odd": capi.FILL_EVEN_ODD, "nonzero": capi.FILL_NONZERO}

    def contains(self, points, rule: str = "even_odd") -> np.ndarray:
        """Point-in-mesh over the closed triangle mesh of set_triangles: bool (n,).  Three fixed rays per point vote; rule "even_odd"
        (front + back odd, orientation ignored) or "nonzero" (back != front, outward-oriented shells).  Points on the surface are
        undefined; a NaN point is outside (DESIGN.md 4.21)."""
        p = self._points(points)
        out = np.zeros(len(p), dtype=np.uint8)
        capi.check(getattr(capi.lib(), f"bvhgpu_contains_points_{self._d['suffix']}")(self._h, _ptr(p), len(p), self._RULES[rule], _ptr(out)))
        return out.astype(bool)

    def contains_dev(self, points_ptr: int, n: int, inside_ptr: int, rule: str = "even_odd"):
        """contains from device pointers: n points (3 scalars each) in, n bytes (0 / 1) out, on the context's stream without host
        synchronisation."""
        capi.check(getattr(capi.lib(), f"bvhgpu_contains_points_dev_{self._d['suffix']}")(
            self._h, C.c_void_p(points_ptr), n, self._RULES[rule], C.c_void_p(inside_ptr)))

    def signed_distance(self, points, rule: str = "even_odd", closest: bool = False):
        """Signed distance to the closed triangle mesh of set_triangles: (shape (n,) u32, dist (n,)), plus closest (n, 3) with
        closest=True.  shape, |dist| and closest are knn_triangles(points, 1); dist is negated where contains(points, rule) is true."""
        p = self._points(points)
        n = len(p)
        shape = np.zeros(n, dtype=np.uint32)
        dist = np.zeros(n, dtype=self._d["scalar"])
        q = np.zeros((n, 3), dtype=self._d["scalar"]) if closest else None
        capi.check(getattr(capi.lib(), f"bvhgpu_signed_distance_{self._d['suffix']}")(self._h, _ptr(p), n, self._RULES[rule], _ptr(shape),
                                                                                     _ptr(dist), _ptr(q)))
        return (shape, dist, q) if closest else (shape, dist)

    def signed_distance_dev(self, points_ptr: int, n: int, shape_ptr: int, dist_ptr: int, closest_ptr: int = 0, rule: str = "even_odd"):
        """signed_distance from device pointers: n points in, n u32 shapes, distances and (closest_ptr != 0) 3 n coordinates out, on
        the context's stream without host synchronisation."""
        capi.check(getattr(capi.lib(), f"bvhgpu_signed_distance_dev_{self._d['suffix']}")(
            self._h, C.c_void_p(points_ptr), n, self._RULES[rule], C.c_void_p(shape_ptr), C.c_void_p(dist_ptr), C.c_void_p(closest_ptr or None)))

    def overlap_pairs_dev(self, offsets_ptr: int, hits_ptr: int, cap: int, want_total: bool = False):
        """overlap_pairs into device pointers (n + 1 u32 offsets, cap u32 hits), enqueued on the context's stream.  The offsets are
        always complete and hits[0 .. cap) is a prefix of the full list; want_total = False: no host synchronisation."""
        total = C.c_size_t(0)
        capi.check(getattr(capi.lib(), f"bvhgpu_overlap_pairs_dev_{self._d['suffix']}")(self._h, C.c_void_p(offsets_ptr), C.c_void_p(hits_ptr or None),
                                                                                       cap, C.byref(total) if want_total else None))
        return total.value if want_total else None

    def overlap_pairs_with_dev(self, other: "Bvh", offsets_ptr: int, hits_ptr: int, cap: int, want_total: bool = False):
        """overlap_pairs_with into device pointers (n + 1 u32 offsets, cap u32 hits), enqueued on the context's stream.  The offsets
        are always complete and hits[0 .. cap) is a prefix of the full list; want_total = False: no host synchronisation."""
        _same_kind(self, other)
        total = C.c_size_t(0)
        capi.check(getattr(capi.lib(), f"bvhgpu_overlap_trees_dev_{self._d['suffix']}")(self._h, other._h, C.c_void_p(offsets_ptr),
                                                                                       C.c_void_p(hits_ptr or None), cap,
                                                                                       C.byref(total) if want_total else None))
        return total.value if want_total else None

    def triangle_pairs(self, skip_shared: bool = True, cap: int | None = None):
        """Every pair of triangles (set_triangles) of this tree that meet, decided exactly: CSR (offsets[n + 1], hits), row s = row s
        of overlap_pairs keeping the shapes t whose closed triangle has a point in common with s's (touching included).  Excluded
        triangles (a non-finite coordinate, or degenerate) meet nothing; skip_shared drops the pairs that share a vertex (the
        non-adjacent self-intersections); f64 triangles with a nonzero coordinate outside [2^-300, 2^300] keep their box pairs
        (include/bvh_b200.h).  A short capacity (default max(4 n, 1024)) is completed from the retained list."""
        n = self._num_shapes()
        fn = getattr(capi.lib(), f"bvhgpu_triangle_pairs_{self._d['suffix']}")
        return self._csr(fn, n, max(4 * n, 1024) if cap is None else int(cap), self._h, 1 if skip_shared else 0)

    def triangle_pairs_with(self, other: "Bvh", cap: int | None = None):
        """Every pair (a, b) of a triangle of this tree and a triangle of `other` that meet, decided exactly: row a of
        overlap_pairs_with(other) keeping the shapes b whose triangle meets a's (a shared vertex is a contact).  Both trees must share
        a context; other may be self.  A short capacity (default max(4 n, 1024)) is completed from this tree's retained list."""
        _same_kind(self, other, "triangle_pairs_with")
        n = self._num_shapes()
        fn = getattr(capi.lib(), f"bvhgpu_triangle_pairs_trees_{self._d['suffix']}")
        return self._csr(fn, n, max(4 * n, 1024) if cap is None else int(cap), self._h, other._h)

    def triangle_pairs_dev(self, offsets_ptr: int, hits_ptr: int, cap: int, skip_shared: bool = True, want_total: bool = False):
        """triangle_pairs into device pointers (n + 1 u32 offsets, cap u32 hits), enqueued on the context's stream.  The offsets are
        always complete and hits[0 .. cap) is a prefix of the full list; want_total = False: no host synchronisation."""
        total = C.c_size_t(0)
        capi.check(getattr(capi.lib(), f"bvhgpu_triangle_pairs_dev_{self._d['suffix']}")(self._h, 1 if skip_shared else 0, C.c_void_p(offsets_ptr),
                                                                                         C.c_void_p(hits_ptr or None), cap,
                                                                                         C.byref(total) if want_total else None))
        return total.value if want_total else None

    def triangle_pairs_with_dev(self, other: "Bvh", offsets_ptr: int, hits_ptr: int, cap: int, want_total: bool = False):
        """triangle_pairs_with into device pointers (n + 1 u32 offsets, cap u32 hits), enqueued on the context's stream.  The offsets
        are always complete and hits[0 .. cap) is a prefix of the full list; want_total = False: no host synchronisation."""
        _same_kind(self, other, "triangle_pairs_with")
        total = C.c_size_t(0)
        capi.check(getattr(capi.lib(), f"bvhgpu_triangle_pairs_trees_dev_{self._d['suffix']}")(self._h, other._h, C.c_void_p(offsets_ptr),
                                                                                               C.c_void_p(hits_ptr or None), cap,
                                                                                               C.byref(total) if want_total else None))
        return total.value if want_total else None

    def nearest_triangles_batch(self, points, mode: int = capi.TRAVERSE_BVH):
        """Bvh::nearest_to / FlatBvh::nearest_to for triangle shapes (set_triangles first): the reference's walk with
        Triangle::distance_squared (testbase.rs:353-443) at the leaves, on the device: (shape index, distance) per point."""
        p = self._points(points)
        shape = np.zeros(len(p), dtype=np.uint32)
        dist = np.zeros(len(p), dtype=self._d["scalar"])
        capi.check(getattr(capi.lib(), f"bvhgpu_nearest_triangles_{self._d['suffix']}")(self._h, mode, _ptr(p), len(p), _ptr(shape), _ptr(dist)))
        return shape, dist

    def traverse_dev(self, rays_ptr: int, nrays: int, offsets_ptr: int, hits_ptr: int, cap: int, mode: int = capi.TRAVERSE_BVH,
                     want_total: bool = False):
        """Device pointers (e.g. torch tensors' data_ptr()), enqueued on the context's stream.  want_total = False: no host
        synchronisation, hits beyond `cap` are dropped."""
        total = C.c_size_t(0)
        fn = getattr(capi.lib(), f"bvhgpu_traverse_dev_{self._d['suffix']}")
        capi.check(fn(self._h, mode, C.c_void_p(rays_ptr), nrays, C.c_void_p(offsets_ptr), C.c_void_p(hits_ptr), cap,
                      C.byref(total) if want_total else None))
        return total.value if want_total else None

    def traverse_stats(self):
        out = (C.c_uint64 * 2)()
        capi.check(getattr(capi.lib(), f"bvhgpu_traverse_stats_{self._d['suffix']}")(self._h, out))
        return int(out[0]), int(out[1])

    def _traverse_one(self, ray, shapes, mode):
        rays = np.ascontiguousarray(ray, dtype=self._d["ray"]).reshape(1)
        _, hits = self.traverse_batch(rays, mode)
        return [shapes[int(h)] for h in hits] if shapes is not None else hits.tolist()

    def traverse(self, ray, shapes: Sequence | None = None):
        """Bvh::traverse: the shapes (or shape indices) whose AABB the ray hits, reference order."""
        return self._traverse_one(ray, shapes, capi.TRAVERSE_BVH)

    def traverse_iterator(self, ray, shapes: Sequence | None = None) -> Iterable:
        """BvhTraverseIterator (src/bvh/iter.rs): same sequence as traverse, lazily yielded on the host."""
        return iter(self._traverse_one(ray, shapes, capi.TRAVERSE_BVH))

    # ---- extras ------------------------------------------------------------------------------------
    def sah_cost(self):
        out = (C.c_double * 2)()
        capi.check(getattr(capi.lib(), f"bvhgpu_sah_cost_{self._d['suffix']}")(self._h, out))
        return float(out[0]), float(out[1])

    def refit(self, shapes):
        aabbs = _gather_aabbs(shapes, self.prec)
        capi.check(getattr(capi.lib(), f"bvhgpu_refit_{self._d['suffix']}")(self._h, _ptr(aabbs), len(aabbs)))
        self._nodes = self._node_index = None

    def optimize(self, shapes, max_growth: float = 1.5) -> int:
        """Bvh::update_shapes counterpart (src/bvh/optimization.rs:290-302): refit, then rebuild in place the subtrees whose
        surface area grew by more than `max_growth`.  `shapes` = all shapes with their current AABBs.  Returns the number
        of shapes in the rebuilt subtrees; `node_index` must be re-read (set_bh_node_index) afterwards."""
        aabbs = _gather_aabbs(shapes, self.prec)
        rebuilt = C.c_size_t(0)
        capi.check(getattr(capi.lib(), f"bvhgpu_optimize_{self._d['suffix']}")(self._h, _ptr(aabbs), len(aabbs), C.c_double(max_growth),
                                                                              C.byref(rebuilt)))
        self._nodes = self._node_index = None
        return int(rebuilt.value)

    def update_shapes(self, changed, shapes, max_growth: float = 1.5) -> int:
        """Bvh::update_shapes(changed_shape_indices, shapes) (src/bvh/optimization.rs:304-315): only the changed shapes' AABBs are sent.
        `shapes` = all shapes (objects with .aabb(), or an AABB array); max_growth <= 0: refit only.  Returns the number of shapes in
        rebuilt subtrees; node indices must be re-read (set_bh_node_index) when it is non-zero."""
        idx = np.ascontiguousarray(changed, dtype=np.uint32).reshape(-1)
        if isinstance(shapes, np.ndarray):
            fresh = np.ascontiguousarray(shapes[idx], dtype=self._d["aabb"])
        else:
            fresh = _gather_aabbs([shapes[int(i)] for i in idx], self.prec)
        rebuilt = C.c_size_t(0)
        capi.check(getattr(capi.lib(), f"bvhgpu_update_{self._d['suffix']}")(self._h, _ptr(idx), _ptr(fresh), len(idx), C.c_double(max_growth), C.byref(rebuilt)))
        self._nodes = self._node_index = None
        return int(rebuilt.value)

    def add_shapes(self, shapes, max_growth: float = 1.5) -> int:
        """Bvh::add_shape for every new shape (src/bvh/optimization.rs:67-207), batched: `shapes` (objects with .aabb(), or an AABB array)
        get the indices num_shapes .. num_shapes+k-1.  max_growth >= 1: degraded subtrees on the changed paths are rebuilt; <= 0: the
        grafts only (k = 1: the reference's own tree).  Returns the number of shapes in rebuilt subtrees.  The node index of every shape may
        change: re-read node_index (set_bh_node_index) after every call.  Triangles set with set_triangles are discarded."""
        aabbs = _gather_aabbs(shapes, self.prec)
        rebuilt = C.c_size_t(0)
        self._nodes = self._node_index = None
        capi.check(getattr(capi.lib(), f"bvhgpu_add_shapes_{self._d['suffix']}")(self._h, _ptr(aabbs), len(aabbs), C.c_double(max_growth), C.byref(rebuilt)))
        return int(rebuilt.value)

    def remove_shapes(self, indices) -> np.ndarray:
        """Bvh::remove_shape(i, swap_shape=true) for every index (src/bvh/optimization.rs:208-301), batched; indices are distinct, in the
        numbering before the call.  Returns the renumbering as (m, 2) rows (new index, old index): apply it to your shape list, then
        drop its last k entries.  The node index of every shape may change: re-read node_index after every call."""
        idx = np.ascontiguousarray(indices, dtype=np.uint32).reshape(-1)
        n = self.num_shapes
        self._nodes = self._node_index = None
        capi.check(getattr(capi.lib(), f"bvhgpu_remove_shapes_{self._d['suffix']}")(self._h, _ptr(idx), len(idx)))
        return swap_moves(n, idx)


def swap_moves(n: int, indices) -> np.ndarray:
    """The renumbering of Bvh.remove_shapes: (m, 2) rows (new index, old index) of the survivors that move.  Survivors with index
    >= n-k take the vacated indices < n-k, smallest hole first (for k = 1: remove_shape(i, true) followed by pop())."""
    rm = np.zeros(n, dtype=bool)
    rm[np.asarray(indices, dtype=np.int64).reshape(-1)] = True
    m = n - int(rm.sum())
    holes = np.flatnonzero(rm[:m])
    tail = m + np.flatnonzero(~rm[m:])
    return np.stack([holes, tail], axis=1).astype(np.uint32).reshape(-1, 2)


class Bvh2(_Tree):
    """Device-resident Bvh<T,2> (the reference is generic in the dimension): build / nodes / flatten / traverse for 2-D AABBs and rays
    (bvhgpu_*_f32x2 / _f64x2), Aabb / Point / Ball queries, nearest_to, the distance-ordered traversal, the AABB closest hit and any hit,
    and polygons over segments (set_segments: exact contains, knn_segments, signed_distance).  Rays: structured array with 2-component
    origin, direction (normalised), inv_direction."""

    _TABLE = BY_PREC_2D
    _DIM = 2

    def __init__(self, handle, prec: str, ctx: Context, n: int):
        super().__init__(handle, prec, ctx)
        self.n = n

    @classmethod
    def build(cls, aabbs, prec: str = "f32", ctx: Context | None = None, mode: int = capi.BUILD_EXACT_SAH) -> "Bvh2":
        ctx = ctx or Context.default()
        d = cls._TABLE[prec]
        a = np.ascontiguousarray(aabbs, dtype=d["aabb"])
        h = C.c_void_p()
        capi.check(getattr(capi.lib(), f"bvhgpu_build_{d['suffix']}")(ctx._h, _ptr(a), len(a), mode, C.byref(h)))
        return cls(h, prec, ctx, len(a))

    def _num_shapes(self) -> int:
        return self.n

    def nodes_and_index(self):
        nodes = np.zeros(max(2 * self.n - 1, 0), dtype=self._d["node"])
        idx = np.zeros(self.n, dtype=np.uint32)
        capi.check(getattr(capi.lib(), f"bvhgpu_tree_nodes_{self._d['suffix']}")(self._h, _ptr(nodes), _ptr(idx)))
        return nodes, idx

    def traverse_batch(self, rays, mode: int = capi.TRAVERSE_BVH):
        rays = np.ascontiguousarray(rays, dtype=self._d["ray"])
        fn = getattr(capi.lib(), f"bvhgpu_traverse_{self._d['suffix']}")
        return self._csr(fn, len(rays), max(16 * len(rays), 1024), self._h, mode, _ptr(rays), len(rays))

    def closest_hit(self, rays):
        """Per ray: (shape whose own AABB the ray enters first, key (entry distance, DFS order), or U32_MAX; that entry distance or
        +inf).  Exact: the head of traverse_ordered(rays, True) on trees whose stored child boxes are tight."""
        rays = np.ascontiguousarray(rays, dtype=self._d["ray"])
        n = len(rays)
        shape = np.zeros(n, dtype=np.uint32)
        dist = np.zeros(n, dtype=self._d["scalar"])
        capi.check(getattr(capi.lib(), f"bvhgpu_closest_hit_{self._d['suffix']}")(self._h, _ptr(rays), n, _ptr(shape), _ptr(dist)))
        return shape, dist

    def any_hit(self, rays, tmax=None) -> np.ndarray:
        """Occlusion: per ray a shape whose own AABB the ray enters at a distance < tmax (one limit per ray, a scalar for all, or None
        for +inf), U32_MAX if none.  Exact: a shape is reported iff closest_hit's distance is < tmax."""
        rays = np.ascontiguousarray(rays, dtype=self._d["ray"])
        n = len(rays)
        shape = np.zeros(n, dtype=np.uint32)
        capi.check(getattr(capi.lib(), f"bvhgpu_any_hit_{self._d['suffix']}")(self._h, _ptr(rays), n, _ptr(self._limits(tmax, n)), _ptr(shape)))
        return shape

    def multi_hit(self, rays, k: int, tmax=None):
        """The first k hits along every ray in AABB mode, with the contract of Bvh.multi_hit: (shape (n, k) u32, dist (n, k), None).
        Exact: the head of a stable sort by (entry of the shape's own AABB, DFS order) over the hits with distance < tmax."""
        rays = np.ascontiguousarray(rays, dtype=self._d["ray"])
        n = len(rays)
        kk = max(int(k), 0)
        shape = np.zeros((n, kk), dtype=np.uint32)
        dist = np.zeros((n, kk), dtype=self._d["scalar"])
        capi.check(getattr(capi.lib(), f"bvhgpu_multi_hit_{self._d['suffix']}")(self._h, _ptr(rays), n, int(k) & 0xFFFFFFFF,
                                                                                _ptr(self._limits(tmax, n)), _ptr(shape), _ptr(dist)))
        return shape, dist, None

    def refit(self, aabbs):
        """Bvh::update_shapes' refit (fix_aabbs_ascending) for all shapes: `aabbs` = the new boxes of every shape.  Topology is kept."""
        a = np.ascontiguousarray(aabbs, dtype=self._d["aabb"])
        capi.check(getattr(capi.lib(), f"bvhgpu_refit_{self._d['suffix']}")(self._h, _ptr(a), len(a)))

    def update_shapes(self, changed, aabbs, max_growth: float = 1.5) -> int:
        """Bvh::update_shapes(changed_shape_indices, shapes): only the changed shapes' boxes are sent.  `aabbs` = the boxes of all
        shapes (an AABB array); max_growth >= 1: degraded subtrees are rebuilt, <= 0: boxes only.  Returns the number of shapes in
        rebuilt subtrees; node indices must be re-read (nodes_and_index) when it is non-zero."""
        idx = np.ascontiguousarray(changed, dtype=np.uint32).reshape(-1)
        fresh = np.ascontiguousarray(np.asarray(aabbs)[idx], dtype=self._d["aabb"])
        rebuilt = C.c_size_t(0)
        capi.check(getattr(capi.lib(), f"bvhgpu_update_{self._d['suffix']}")(self._h, _ptr(idx), _ptr(fresh), len(idx), C.c_double(max_growth),
                                                                            C.byref(rebuilt)))
        return int(rebuilt.value)

    def _sync_n(self):
        self.n = int(getattr(capi.lib(), f"bvhgpu_tree_num_shapes_{self._d['suffix']}")(self._h))

    def add_shapes(self, aabbs, max_growth: float = 1.5) -> int:
        """Bvh::add_shape for every new box, batched (the contract of Bvh.add_shapes): the k boxes get the indices n .. n+k-1.
        max_growth >= 1: degraded subtrees on the changed paths are rebuilt; <= 0: the grafts only.  Returns the number of shapes in
        subtrees rebuilt by the growth test.  The node index of every shape may change: re-read nodes_and_index after every call."""
        a = np.ascontiguousarray(aabbs, dtype=self._d["aabb"]).reshape(-1)
        rebuilt = C.c_size_t(0)
        try:
            capi.check(getattr(capi.lib(), f"bvhgpu_add_shapes_{self._d['suffix']}")(self._h, _ptr(a), len(a), C.c_double(max_growth),
                                                                                    C.byref(rebuilt)))
        finally:
            self._sync_n()
        return int(rebuilt.value)

    def remove_shapes(self, indices) -> np.ndarray:
        """Bvh::remove_shape(i, swap_shape=true) for every index, batched (the contract of Bvh.remove_shapes): indices are distinct, in
        the numbering before the call.  Returns the renumbering as (m, 2) rows (new index, old index)."""
        idx = np.ascontiguousarray(indices, dtype=np.uint32).reshape(-1)
        n = self.n
        try:
            capi.check(getattr(capi.lib(), f"bvhgpu_remove_shapes_{self._d['suffix']}")(self._h, _ptr(idx), len(idx)))
        finally:
            self._sync_n()
        return swap_moves(n, idx)

    # ---- polygons: the segments of set_segments (D = 2 only; include/bvh_b200.h, DESIGN.md 4.23) ----
    _POLY_RULES = {"even_odd": capi.FILL_EVEN_ODD, "nonzero": capi.FILL_NONZERO}

    def set_segments(self, segs):
        """Segment s = (a, b) for every shape s: segs of shape (n, 2, 2) (or (n, 4): ax, ay, bx, by), n = num shapes.  Shape s's box
        must contain segment s (not checked).  remove_shapes permutes them, add_shapes drops them, refit / update_shapes keep them."""
        sg = np.ascontiguousarray(segs, dtype=self._d["scalar"]).reshape(-1, 4)
        capi.check(getattr(capi.lib(), f"bvhgpu_tree_set_segments_{self._d['suffix']}")(self._h, _ptr(sg), len(sg)))

    @classmethod
    def from_segments(cls, segs, prec: str = "f32", ctx: Context | None = None, mode: int = capi.BUILD_EXACT_SAH) -> "Bvh2":
        """A tree over the exact end-point boxes of the segments ((n, 2, 2)), with the segments set.  A NaN coordinate takes the other
        end point's value in the box (the segment is excluded by every query anyway)."""
        d = cls._TABLE[prec]
        sg = np.ascontiguousarray(segs, dtype=d["scalar"]).reshape(-1, 2, 2)
        a = np.zeros(len(sg), dtype=d["aabb"])
        a["min"] = np.fmin(sg[:, 0], sg[:, 1])
        a["max"] = np.fmax(sg[:, 0], sg[:, 1])
        bvh = cls.build(a, prec, ctx, mode)
        bvh.set_segments(sg)
        return bvh

    def contains(self, points, rule: str = "even_odd", winding: bool = False):
        """Exact point-in-polygon over the segments: class (n,) u8 (0 outside, 1 inside, 2 boundary, 3 undecided: f64 coordinates
        outside [2^-300, 2^300]), plus the winding number (n,) i32 with winding=True."""
        p = self._points(points)
        n = len(p)
        cls_ = np.zeros(n, dtype=np.uint8)
        w = np.zeros(n, dtype=np.int32) if winding else None
        capi.check(getattr(capi.lib(), f"bvhgpu_contains_points_{self._d['suffix']}")(self._h, _ptr(p), n, self._POLY_RULES[rule], _ptr(cls_),
                                                                                     _ptr(w)))
        return (cls_, w) if winding else cls_

    def knn_segments(self, points, k: int, max_dist=None, closest: bool = False):
        """The k nearest segments of every point: (shape (n, k) u32, dist (n, k)), plus closest (n, k, 2) with closest=True; the
        contract of Bvh.knn_triangles with the segment key (include/bvh_b200.h)."""
        p = self._points(points)
        n = len(p)
        kk = max(int(k), 0)
        shape = np.zeros((n, kk), dtype=np.uint32)
        dist = np.zeros((n, kk), dtype=self._d["scalar"])
        q = np.zeros((n, kk, 2), dtype=self._d["scalar"]) if closest else None
        capi.check(getattr(capi.lib(), f"bvhgpu_knn_segments_{self._d['suffix']}")(self._h, _ptr(p), n, int(k) & 0xFFFFFFFF,
                                                                                  _ptr(self._limits(max_dist, n)), _ptr(shape), _ptr(dist), _ptr(q)))
        return (shape, dist, q) if closest else (shape, dist)

    def signed_distance(self, points, rule: str = "even_odd", closest: bool = False):
        """Signed distance to the segments: (shape (n,) u32, dist (n,)), plus closest (n, 2) with closest=True.  shape, |dist| and
        closest are knn_segments(points, 1); dist is negated where contains(points, rule) gives 1 (inside)."""
        p = self._points(points)
        n = len(p)
        shape = np.zeros(n, dtype=np.uint32)
        dist = np.zeros(n, dtype=self._d["scalar"])
        q = np.zeros((n, 2), dtype=self._d["scalar"]) if closest else None
        capi.check(getattr(capi.lib(), f"bvhgpu_signed_distance_{self._d['suffix']}")(self._h, _ptr(p), n, self._POLY_RULES[rule], _ptr(shape),
                                                                                     _ptr(dist), _ptr(q)))
        return (shape, dist, q) if closest else (shape, dist)


class Bvh4(Bvh2):
    """Device-resident Bvh<T,4> (bvhgpu_*_f32x4 / _f64x4): the exact SAH build (the only mode for D = 4), nodes, flatten, batched
    ray traversal of 4-D AABBs and rays (4-component origin, direction (normalised), inv_direction), and the queries and nearest_to
    of Bvh2 with 4 components (refit, update_shapes, add_shapes and remove_shapes included), plus query_dev, refit_dev, update_dev,
    add_shapes_dev, remove_shapes_dev, closest_hit_dev and any_hit_dev."""

    _TABLE = BY_PREC_4D
    _DIM = 4

    def _segments_are_2d(self, *args, **kwargs):
        raise TypeError("Bvh4 has no segments: polygons (set_segments, contains, knn_segments, signed_distance) are 2-D only")

    set_segments = contains = knn_segments = signed_distance = _segments_are_2d
    from_segments = classmethod(_segments_are_2d)

    # The device-pointer forms the 3-D tree has too (Bvh2 has no C entry point for them).
    traverse_dev, overlap_pairs_dev, overlap_pairs_with_dev, knn_dev = (Bvh.traverse_dev, Bvh.overlap_pairs_dev, Bvh.overlap_pairs_with_dev,
                                                                        Bvh.knn_dev)

    def query_dev(self, kind: int, queries_ptr: int, n: int, offsets_ptr: int, hits_ptr: int, cap: int, mode: int = capi.TRAVERSE_BVH,
                  want_total: bool = False):
        """Aabb / Point / Ball queries from device pointers (records of 8 / 4 / 5 scalars), enqueued on the context's stream.  The
        offsets are always complete and hits[0 .. cap) is a prefix of the full list; want_total = False: no host synchronisation."""
        total = C.c_size_t(0)
        fn = getattr(capi.lib(), f"bvhgpu_query_dev_{self._d['suffix']}")
        capi.check(fn(self._h, mode, kind, C.c_void_p(queries_ptr), n, C.c_void_p(offsets_ptr), C.c_void_p(hits_ptr), cap,
                      C.byref(total) if want_total else None))
        return total.value if want_total else None

    def closest_hit_dev(self, rays_ptr: int, nrays: int, shape_ptr: int, dist_ptr: int):
        """closest_hit from device pointers: nrays full 4-D rays (12 scalars each) in, u32 shapes and distances out, enqueued on the
        context's stream without host synchronisation."""
        capi.check(getattr(capi.lib(), f"bvhgpu_closest_hit_dev_{self._d['suffix']}")(self._h, C.c_void_p(rays_ptr), nrays, C.c_void_p(shape_ptr),
                                                                                     C.c_void_p(dist_ptr)))

    def any_hit_dev(self, rays_ptr: int, nrays: int, tmax_ptr: int, shape_ptr: int):
        """any_hit from device pointers: nrays full 4-D rays (12 scalars each) and nrays limits (tmax_ptr = 0: +inf for every ray) in,
        u32 shapes out, enqueued on the context's stream without host synchronisation."""
        capi.check(getattr(capi.lib(), f"bvhgpu_any_hit_dev_{self._d['suffix']}")(self._h, C.c_void_p(rays_ptr), nrays, C.c_void_p(tmax_ptr or None),
                                                                                 C.c_void_p(shape_ptr)))

    def multi_hit_dev(self, rays_ptr: int, nrays: int, k: int, tmax_ptr: int, shape_ptr: int, dist_ptr: int):
        """multi_hit from device pointers: nrays full 4-D rays (12 scalars each) and nrays limits (tmax_ptr = 0: none) in, nrays * k
        u32 shapes and distances out, enqueued on the context's stream without host synchronisation."""
        capi.check(getattr(capi.lib(), f"bvhgpu_multi_hit_dev_{self._d['suffix']}")(self._h, C.c_void_p(rays_ptr), nrays, k,
                                                                                    C.c_void_p(tmax_ptr or None), C.c_void_p(shape_ptr),
                                                                                    C.c_void_p(dist_ptr)))

    def refit_dev(self, aabbs_ptr: int, n: int):
        """refit from the new boxes of all n shapes on the device (C-ABI layout), enqueued on the context's stream."""
        capi.check(getattr(capi.lib(), f"bvhgpu_refit_dev_{self._d['suffix']}")(self._h, C.c_void_p(aabbs_ptr), n))

    def update_dev(self, changed_ptr: int, aabbs_ptr: int, m: int, max_growth: float = 1.5, want_rebuilt: bool = True):
        """update_shapes from device pointers: m u32 shape indices and their m new boxes (C-ABI layout), on the context's stream.
        Returns the number of shapes in rebuilt subtrees (None with want_rebuilt = False)."""
        rebuilt = C.c_size_t(0)
        capi.check(getattr(capi.lib(), f"bvhgpu_update_dev_{self._d['suffix']}")(self._h, C.c_void_p(changed_ptr), C.c_void_p(aabbs_ptr), m,
                                                                                C.c_double(max_growth), C.byref(rebuilt) if want_rebuilt else None))
        return int(rebuilt.value) if want_rebuilt else None

    def add_shapes_dev(self, aabbs_ptr: int, k: int, max_growth: float = 1.5) -> int:
        """add_shapes from k new boxes on the device (C-ABI layout).  Returns the number of shapes in subtrees rebuilt by the growth
        test."""
        rebuilt = C.c_size_t(0)
        try:
            capi.check(getattr(capi.lib(), f"bvhgpu_add_shapes_dev_{self._d['suffix']}")(self._h, C.c_void_p(aabbs_ptr), k,
                                                                                        C.c_double(max_growth), C.byref(rebuilt)))
        finally:
            self._sync_n()
        return int(rebuilt.value)

    def remove_shapes_dev(self, indices_ptr: int, k: int, indices=None) -> np.ndarray | None:
        """remove_shapes from k u32 shape indices on the device.  Returns the renumbering when the same indices are also given on the
        host (`indices`), else None."""
        n = self.n
        try:
            capi.check(getattr(capi.lib(), f"bvhgpu_remove_shapes_dev_{self._d['suffix']}")(self._h, C.c_void_p(indices_ptr), k))
        finally:
            self._sync_n()
        return None if indices is None else swap_moves(n, indices)
