"""The restatement of tests/crossings.py without a GPU:
- mt in both windings equals the C++ oracle's Ray::intersects_triangle bit for bit (the back winding on the triangle with b and c
  exchanged) on random, grazing, degenerate, |det|-near-eps and f32 overflow-scale triangles;
- the three-ray vote gives the true answer away from the surface on the cube scene (parity of the cubes holding the point), an icosphere
  and a torus, and on the icosphere with flipped triangles for EVEN_ODD; NONZERO is wrong there, as documented; single-ray errors are
  counted;
- the directions of the header meet their stated conditions, and every new entry point is declared in the header and typed from it by
  capi.py."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import crossings as X

FT = {"f32": np.float32, "f64": np.float64}
NEW = [f"bvhgpu_{f}_{p}x3" for f in ("count_hits", "count_hits_dev", "contains_points", "contains_points_dev", "signed_distance",
                                     "signed_distance_dev") for p in ("f32", "f64")]


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def _families(F, rng):
    """(tris (m, 3, 3), origins (m, 3), dirs (m, 3)) per family."""
    m = 400
    out = {}
    a = rng.uniform(-1, 1, (m, 3, 3))
    o = rng.uniform(-3, 3, (m, 3))
    out["random"] = (a, o, a.mean(axis=1) - o + rng.normal(0, 0.2, (m, 3)))
    # grazing: rays in (or next to) the triangle's plane, aimed at an edge
    t = rng.uniform(-1, 1, (m, 3, 3))
    t[:, :, 2] = 0
    e = (t[:, 0] + t[:, 1]) / 2
    o = e + np.stack([rng.uniform(-2, 2, m), rng.uniform(-2, 2, m), rng.choice([0.0, 1e-7, -1e-7], m)], axis=1)
    out["grazing"] = (t, o, e - o)
    # degenerate: repeated vertices and collinear triangles
    d = rng.uniform(-1, 1, (m, 3, 3))
    d[: m // 2, 2] = d[: m // 2, 1]
    d[m // 2:, 2] = 2 * d[m // 2:, 1] - d[m // 2:, 0]
    o = rng.uniform(-3, 3, (m, 3))
    out["degenerate"] = (d, o, d.mean(axis=1) - o)
    # |det| near eps: right triangles with legs L around sqrt(eps), rays along z
    eps = np.finfo(F).eps
    L = np.sqrt(eps) * rng.uniform(0.5, 2.0, m)
    tri = np.zeros((m, 3, 3))
    tri[:, 1, 0], tri[:, 2, 1] = L, L
    o = np.stack([L / 4, L / 4, np.full(m, 1.0)], axis=1)
    dz = np.stack([rng.normal(0, 0.02, m) * L, rng.normal(0, 0.02, m) * L, -np.ones(m)], axis=1)
    out["det_eps"] = (tri, o, dz)
    # overflow scale (f32): coordinates near 1e38
    big = rng.uniform(-3e38, 3e38, (m, 3, 3)) if F == np.float32 else rng.uniform(-1e300, 1e300, (m, 3, 3))
    o = rng.uniform(-1, 1, (m, 3)) * (1e38 if F == np.float32 else 1e300)
    out["overflow"] = (big, o, big.mean(axis=1) - o)
    return out


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_mt_both_windings_equal_the_oracle(prec):
    F = FT[prec]
    rng = np.random.default_rng(3)
    hits = {}
    for name, (tris, o, d) in _families(F, rng).items():
        with np.errstate(all="ignore"):
            rays = O.ray_new(np.asarray(o, dtype=F), np.asarray(d, dtype=F), prec)
        tris = np.asarray(tris, dtype=F)
        ro, rd = rays["origin"], rays["direction"]
        front = X.mt(ro, rd, tris[:, 0], tris[:, 1], tris[:, 2])
        back = X.mt(ro, rd, tris[:, 0], tris[:, 2], tris[:, 1])
        flipped = tris[:, [0, 2, 1]]
        for i in range(len(tris)):
            assert _bits(front[i]) == _bits(O.ray_triangle(rays[i], tris[i].reshape(9), prec)[0]), (name, i)
            assert _bits(back[i]) == _bits(O.ray_triangle(rays[i], flipped[i].reshape(9), prec)[0]), (name, i)
        hits[name] = int(np.isfinite(front).sum() + np.isfinite(back).sum())
    # the families exercise hits as well as misses
    assert hits["random"] > 50 and hits["det_eps"] > 20 and hits["grazing"] > 0, hits


def test_det_eps_hides_tiny_triangles_in_f32():
    """The header's statement: in f32 a triangle with legs well below sqrt(eps) ~ 3.5e-4 never counts, well above it does."""
    F = np.float32
    for L, want in ((1e-4, False), (1e-3, True)):
        tri = np.array([[[0, 0, 0], [L, 0, 0], [0, L, 0]]], dtype=F)
        rays = X.point_rays(np.array([[L / 4, L / 4, -1.0]]), F)[:1]
        rays["direction"] = np.array([[0, 0, 1]], dtype=F)
        f, b = X.counts_brute(rays, tri), X.counts_brute(rays, tri[:, [0, 2, 1]])
        assert bool(f[0][0] + b[0][0]) == want, L


def test_directions_meet_their_conditions():
    D = X.directions()
    u = D / np.linalg.norm(D, axis=1, keepdims=True)
    assert np.all(np.abs(D) > 0.1)                                         # not axis-aligned, not in a coordinate plane
    diags = [np.array(v) / np.sqrt(2) for v in ((1, 1, 0), (1, -1, 0), (1, 0, 1), (1, 0, -1), (0, 1, 1), (0, 1, -1))]
    for a in u:
        assert all(abs(abs(a @ g) - 1) > 0.05 for g in diags)              # not parallel to a face diagonal
    for i in range(3):
        for j in range(i + 1, 3):
            assert abs(abs(u[i] @ u[j]) - 1) > 0.05                       # not parallel to each other


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_point_rays_equal_ray_new(prec):
    F = FT[prec]
    p = np.random.default_rng(1).uniform(-10, 10, (50, 3))
    rays = X.point_rays(p, F)
    want = O.ray_new(rays["origin"], np.tile(X.directions().astype(F), (50, 1)), prec)
    for f in ("origin", "direction", "inv_direction"):
        assert np.array_equal(_bits(rays[f]), _bits(want[f])), f


def _vote_brute(tris, points, F, rule):
    rays = X.point_rays(points, F)
    f, b = X.counts_brute(rays, tris)
    return X.vote(f, b, rule), X.ray_votes(f, b, rule).reshape(-1, 3)


def cube_points(tris, F, rng, m):
    """Points near the cubes of create_n_cubes_tris, at least 0.05 from every face, and the parity of the cubes holding them."""
    t = np.asarray(tris, dtype=F).reshape(-1, 12, 3, 3)
    lo, hi = t.min(axis=(1, 2)).astype(np.float64), t.max(axis=(1, 2)).astype(np.float64)
    c = rng.integers(0, len(lo), 4 * m)
    p = ((lo[c] + hi[c]) / 2 + rng.uniform(-0.8, 0.8, (4 * m, 3))).astype(F).astype(np.float64)
    from scipy.spatial import cKDTree

    near = cKDTree((lo + hi) / 2).query_ball_point(p, r=1.0, p=np.inf)
    keep, inside = [], []
    for i, cs in enumerate(near):
        cs = np.asarray(cs, dtype=np.int64)
        gap = np.minimum(p[i] - lo[cs], hi[cs] - p[i]).min(axis=1) if len(cs) else np.zeros(0)
        if np.all(np.abs(gap) > 0.05):
            keep.append(i)
            inside.append(int((gap > 0).sum()) % 2 == 1)
    keep = keep[:m]
    return p[keep].astype(F), np.array(inside[:m])


def sphere_points(rng, m, margin=0.05):
    p = rng.uniform(-1.5, 1.5, (4 * m, 3))
    r = np.linalg.norm(p, axis=1)
    p = p[np.abs(r - 1) > margin][:m]
    return p, np.linalg.norm(p, axis=1) < 1


def torus_points(rng, m, R=1.0, r=0.4, margin=0.03):
    p = rng.uniform([-1.6, -1.6, -0.6], [1.6, 1.6, 0.6], (4 * m, 3))
    q = (np.hypot(p[:, 0], p[:, 1]) - R) ** 2 + p[:, 2] ** 2
    p = p[np.abs(np.sqrt(q) - r) > margin][:m]
    return p, (np.hypot(p[:, 0], p[:, 1]) - R) ** 2 + p[:, 2] ** 2 < r * r


def flip_some(tris, rng, frac):
    t = np.array(tris, copy=True)
    f = rng.random(len(t)) < frac
    t[f] = t[f][:, [0, 2, 1]]
    return t, f


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_vote_is_the_truth_away_from_the_surface(prec):
    from bvh_b200 import scenes

    F = FT[prec]
    rng = np.random.default_rng(11)
    ico = X.icosphere(3, F)
    assert X.outward(ico) == 1.0
    cubes = scenes.create_n_cubes_tris(40, prec)
    pc, tc = cube_points(cubes, F, rng, 600)
    ps, ts = sphere_points(rng, 600)
    pt, tt = torus_points(rng, 600)
    single = {}
    for name, tris, p, truth, rules in (("cubes", cubes, pc, tc, (X.EVEN_ODD,)), ("icosphere", ico, ps, ts, (X.EVEN_ODD, X.NONZERO)),
                                        ("torus", X.torus(F=F), pt, tt, (X.EVEN_ODD, X.NONZERO))):
        assert truth.sum() > 50 and (~truth).sum() > 50, name
        for rule in rules:
            inside, per_ray = _vote_brute(tris, p, F, rule)
            assert np.array_equal(inside, truth), (name, rule, int((inside != truth).sum()))
            single[(name, rule)] = int((per_ray != truth[:, None]).sum())
    print("single-ray errors:", single)
    # flipped triangles: EVEN_ODD ignores orientation; NONZERO counts an outside ray through a flipped triangle as inside
    flipped, f = flip_some(ico, rng, 0.5)
    assert f.sum() > 50
    inside, _ = _vote_brute(flipped, ps, F, X.EVEN_ODD)
    assert np.array_equal(inside, ts)
    inside_nz, _ = _vote_brute(flipped, ps, F, X.NONZERO)
    wrong = inside_nz != ts
    assert wrong.sum() > 0 and np.all(ts[wrong] == False)                 # noqa: E712  only outside points go wrong
    print("NONZERO on the flipped icosphere: wrong on", int(wrong.sum()), "of", len(ts))


def test_signed_composition():
    shape = np.array([0, 1, X.U32_MAX, 2], dtype=np.uint32)
    dist = np.array([1.5, 0.0, np.inf, 2.0], dtype=np.float32)
    got = X.signed(shape, dist, np.array([True, True, True, False]))
    assert _bits(got).tolist() == _bits(np.array([-1.5, -0.0, np.inf, 2.0], dtype=np.float32)).tolist()


def test_every_new_entry_point_is_declared_and_typed_from_the_header():
    """The library's argtypes / restype of the six crossing families in both precisions are set and equal the header's prototypes."""
    import ctypes as C

    from bvh_b200 import capi

    declared = capi.declared_symbols()
    for name in NEW:
        assert name in declared, name
    vp, sz, i32 = C.c_void_p, C.c_size_t, C.c_int
    want = {"count_hits": [vp, vp, sz, vp, vp, vp], "count_hits_dev": [vp, vp, i32, sz, vp, vp, vp],
            "contains_points": [vp, vp, sz, i32, vp], "contains_points_dev": [vp, vp, sz, i32, vp],
            "signed_distance": [vp, vp, sz, i32, vp, vp, vp], "signed_distance_dev": [vp, vp, sz, i32, vp, vp, vp]}
    sigs, L = capi.signatures(), capi.lib()
    for name in NEW:
        fn, argtypes = getattr(L, name), want[name[len("bvhgpu_"):-len("_f32x3")]]
        assert sigs[name] == (C.c_int, argtypes), name
        assert fn.argtypes is not None and list(fn.argtypes) == argtypes and fn.restype is C.c_int, name
