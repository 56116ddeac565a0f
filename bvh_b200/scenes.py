"""Synthetic inputs of the reference's benches (src/testbase.rs), vectorised with numpy so that the
bench can generate millions of shapes / rays quickly: splitmix64 has a closed-form state
(state_k = k * GOLDEN mod 2^64), so the "seed chain" is a plain arange.

    create_n_cubes_aabbs(n)   create_n_cubes(n, default_bounds())  -> the 12n triangle AABBs  (:490-615)
    ray_endpoints(n, ...)     the (origin, direction) pairs create_ray draws                   (:687-691)

All float arithmetic is done in the target dtype with the reference's operation order; the CPU test
tests/test_scenes_cpu.py checks these against the scalar restatement in oracle/ bit for bit.
"""
from __future__ import annotations

import numpy as np

from .dtypes import BY_PREC

_GOLDEN = np.uint64(0x9E3779B97F4A7C15)
_M1 = np.uint64(0xBF58476D1CE4E5B9)
_M2 = np.uint64(0x94D049BB133111EB)


def _splitmix_outputs(first_index: int, count: int) -> np.ndarray:
    """Outputs of calls first_index .. first_index+count-1 (0-based) of splitmix64 started from seed 0."""
    with np.errstate(over="ignore"):
        k = np.arange(first_index + 1, first_index + count + 1, dtype=np.uint64)
        z = k * _GOLDEN
        z = (z ^ (z >> np.uint64(30))) * _M1
        z = (z ^ (z >> np.uint64(27))) * _M2
        return z ^ (z >> np.uint64(31))


def _next_point3(u: np.ndarray, bounds_min, bounds_max, F) -> np.ndarray:
    """next_point3 (testbase.rs:569-597) for an array of splitmix outputs."""
    a = ((u >> np.uint64(32)) & np.uint64(0xFFFFFFFF)).astype(np.int64) - np.int64(0x80000000)
    b = (u & np.uint64(0xFFFFFFFF)).astype(np.int64) - np.int64(0x80000000)
    ub = b.view(np.uint64)
    rot = ((ub << np.uint64(6)) | (ub >> np.uint64(58))).view(np.int64)
    c = a ^ rot
    raw = np.stack([a.astype(np.int32), b.astype(np.int32), c.astype(np.int32)], axis=1)      # `as i32` truncates
    imax = F(2147483647)                                                                       # i32::MAX as T
    fv = ((raw.astype(F) / imax) + F(1)) * F(0.5)
    bmin, bmax = np.asarray(bounds_min, dtype=F), np.asarray(bounds_max, dtype=F)
    size = bmax - bmin
    return (bmin + fv * size).astype(F)


def default_bounds(prec: str = "f32"):
    F = BY_PREC[prec]["scalar"]
    return np.full(3, -100000.0, dtype=F), np.full(3, 100000.0, dtype=F)


def create_n_cubes_aabbs(n_cubes: int, prec: str = "f32", bounds=None) -> np.ndarray:
    d = BY_PREC[prec]
    F = d["scalar"]
    bmin, bmax = bounds if bounds is not None else default_bounds(prec)
    pos = _next_point3(_splitmix_outputs(0, n_cubes), bmin, bmax, F)      # one splitmix call per cube
    lo, hi = (pos + F(-0.5)).astype(F), (pos + F(0.5)).astype(F)           # push_cube vertices (:490-498)
    out = np.zeros((n_cubes, 12), dtype=d["aabb"])
    # Every triangle of a face spans the whole face rectangle: faces in push_cube order are
    # top(y+), bottom(y-), left(x-), right(x+), front(z-), back(z+), two triangles each (:500-555).
    for face, (axis, side) in enumerate([(1, 1), (1, 0), (0, 0), (0, 1), (2, 0), (2, 1)]):
        mn, mx = lo.copy(), hi.copy()
        plane = hi[:, axis] if side else lo[:, axis]
        mn[:, axis] = plane
        mx[:, axis] = plane
        for t in (2 * face, 2 * face + 1):
            out["min"][:, t, :] = mn
            out["max"][:, t, :] = mx
    return out.reshape(-1)


_TFR, _TBR, _TBL, _TFL = (1, 1, 0), (1, 1, 1), (0, 1, 1), (0, 1, 0)       # push_cube's corners: 1 = pos + 0.5, 0 = pos - 0.5 per axis
_BFR, _BBR, _BBL, _BFL = (1, 0, 0), (1, 0, 1), (0, 0, 1), (0, 0, 0)
_CUBE_TRIS = [(_TBR, _TFR, _TFL), (_TFL, _TBL, _TBR), (_BFL, _BFR, _BBR), (_BBR, _BBL, _BFL), (_TBL, _TFL, _BFL), (_BFL, _BBL, _TBL),
              (_BFR, _TFR, _TBR), (_TBR, _BBR, _BFR), (_TFL, _TFR, _BFR), (_BFR, _BFL, _TFL), (_BBR, _TBR, _TBL), (_TBL, _BBL, _BBR)]


def create_n_cubes_tris(n_cubes: int, prec: str = "f32", bounds=None) -> np.ndarray:
    """The (12n, 3, 3) triangle vertices of create_n_cubes (push_cube, :490-555), in the order of create_n_cubes_aabbs."""
    F = BY_PREC[prec]["scalar"]
    bmin, bmax = bounds if bounds is not None else default_bounds(prec)
    pos = _next_point3(_splitmix_outputs(0, n_cubes), bmin, bmax, F)
    side = np.stack([(pos + F(-0.5)).astype(F), (pos + F(0.5)).astype(F)])                # [0 / 1, cube, axis]
    sel = np.array(_CUBE_TRIS)                                                           # (12, 3 vertices, 3 axes) of 0 / 1
    ax = np.arange(3)
    out = side[sel[None, :, :, :], np.arange(n_cubes)[:, None, None, None], ax[None, None, None, :]]
    return np.ascontiguousarray(out.reshape(-1, 3, 3), dtype=F)


def ray_endpoints(n: int, first_ray: int = 0, prec: str = "f32", bounds=None):
    """Origins and (un-normalised) directions of rays first_ray .. first_ray+n-1 of the create_ray chain
    started from seed 0 (two splitmix calls per ray); Ray::new normalises them (on the device)."""
    F = BY_PREC[prec]["scalar"]
    bmin, bmax = bounds if bounds is not None else default_bounds(prec)
    u = _splitmix_outputs(2 * first_ray, 2 * n)
    pts = _next_point3(u, bmin, bmax, F)
    return np.ascontiguousarray(pts[0::2]), np.ascontiguousarray(pts[1::2])


def pinhole_rays(width: int = 2048, height: int = 2048, prec: str = "f32"):
    """The coherent primary-ray batch of BASELINE.json configs[2] (SURVEY.md 8d): pinhole camera at
    (-15, 2, 0) looking down +x, up = +y, right = +z, 60 degree vertical field of view, row-major pixels.
    Returns (origins, directions) for Ray::new; all arithmetic in T."""
    F = BY_PREC[prec]["scalar"]
    tan_half = F(np.tan(np.deg2rad(30.0)))
    j, i = np.meshgrid(np.arange(height, dtype=F), np.arange(width, dtype=F), indexing="ij")
    u = ((i + F(0.5)) / F(width) * F(2) - F(1)) * tan_half * F(width / height)
    v = (F(1) - (j + F(0.5)) / F(height) * F(2)) * tan_half
    d = np.stack([np.ones_like(u), v, u], axis=-1).reshape(-1, 3).astype(F)
    o = np.broadcast_to(np.array([-15.0, 2.0, 0.0], dtype=F), d.shape).copy()
    return o, d
