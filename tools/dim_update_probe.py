#!/usr/bin/env python
"""Cost of refit and update_shapes for 4-D and 2-D trees (DESIGN.md section 5): 1.2 M random 4-D boxes, f32 and f64, with 1 % and
10 % of the shapes moved by small offsets (0.5, inside their subtrees) and by large ones (300: across the scene), max_growth = 1.5.
Times the host-pointer update (indices and boxes uploaded), the device-pointer update, refit_dev of all boxes and a full
bvhgpu_build_*x4 of the same moved boxes; and the 2-D update of 1.2 M random 2-D boxes at 1 %.  Every timed update starts from a
fresh build of the unmoved boxes (not timed).  CUDA events on the context's stream, median of 3 after one warm-up call.  `rebuilt`
is the number of shapes in the rebuilt subtrees.  Prints one JSON line with the card name and its power limit, read in the same call.

    python tools/dim_update_probe.py
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bvh_b200 import api  # noqa: E402
from bvh_b200.dtypes import BY_PREC_2D, BY_PREC_4D  # noqa: E402
from tools.dim_query_probe import card  # noqa: E402

N = 1_200_000


def timed(setup, fn, stream, reps=3):
    """fn(state) timed with events after setup() (not timed); the warm-up call is not counted.  Returns (median ms, last result)."""
    import torch

    fn(setup())
    out, res = [], None
    for _ in range(reps):
        st = setup()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        res = fn(st)
        b.record(stream)
        b.synchronize()
        out.append(a.elapsed_time(b))
        if isinstance(st, tuple) and hasattr(st[0], "free"):
            st[0].free()
    return round(float(np.median(out)), 3), res


def scene(D, prec, rng):
    table = (BY_PREC_2D if D == 2 else BY_PREC_4D)[prec]
    a = np.zeros(N, dtype=table["aabb"])
    mn = rng.uniform(-1000, 1000, (N, D))
    a["min"], a["max"] = mn, mn + rng.uniform(0, 3 if D == 2 else 60, (N, D))
    return a


def moved(a, frac, scale, rng):
    n, D = a["min"].shape
    changed = np.sort(rng.choice(n, int(n * frac), replace=False)).astype(np.uint32)
    b = a.copy()
    off = rng.uniform(-scale, scale, (len(changed), D))
    b["min"][changed] = b["min"][changed] + off
    b["max"][changed] = b["max"][changed] + off
    return changed, b


def probe4(prec, ctx, stream):
    import torch

    rng = np.random.default_rng(4)
    a = scene(4, prec, rng)
    out = {"shapes": N}
    ms, _ = timed(lambda: None, lambda _: api.Bvh4.build(a, prec=prec, ctx=ctx).free(), stream)
    out["build_ms"] = ms
    for frac in (0.01, 0.10):
        for scale in (0.5, 300.0):
            changed, b = moved(a, frac, scale, rng)
            fresh = np.ascontiguousarray(b[changed])
            d_idx = torch.from_numpy(changed.view(np.int32)).cuda()
            d_box = torch.from_numpy(fresh.view(np.uint8).copy()).cuda()
            d_all = torch.from_numpy(b.view(np.uint8).copy()).cuda()
            setup = lambda: (api.Bvh4.build(a, prec=prec, ctx=ctx),)
            host_ms, rebuilt = timed(setup, lambda s: s[0].update_shapes(changed, b), stream)
            dev_ms, _ = timed(setup, lambda s: s[0].update_dev(d_idx.data_ptr(), d_box.data_ptr(), len(changed)), stream)
            refit_ms, _ = timed(setup, lambda s: s[0].refit_dev(d_all.data_ptr(), N), stream)
            build_ms, _ = timed(lambda: None, lambda _: api.Bvh4.build(b, prec=prec, ctx=ctx).free(), stream)
            out[f"moved_{int(frac * 100)}pct_offset_{scale:g}"] = {
                "update_ms": host_ms, "update_dev_ms": dev_ms, "refit_dev_ms": refit_ms, "build_ms": build_ms, "rebuilt": rebuilt,
                "update_dev_over_build": round(dev_ms / build_ms, 3)}
    return out


def probe2(prec, ctx, stream):
    rng = np.random.default_rng(2)
    a = scene(2, prec, rng)
    out = {"shapes": N}
    for scale in (0.5, 300.0):
        changed, b = moved(a, 0.01, scale, rng)
        setup = lambda: (api.Bvh2.build(a, prec=prec, ctx=ctx),)
        ms, rebuilt = timed(setup, lambda s: s[0].update_shapes(changed, b), stream)
        bms, _ = timed(lambda: None, lambda _: api.Bvh2.build(b, prec=prec, ctx=ctx).free(), stream)
        out[f"moved_1pct_offset_{scale:g}"] = {"update_ms": ms, "build_ms": bms, "rebuilt": rebuilt}
    return out


def main():
    import torch

    ctx = api.Context(0)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    name, power = card()
    res = {"card": name, "power_limit": power, "what": "CUDA events on the context's stream, median of 3 after one warm-up call; "
           "every update starts from a fresh build of the unmoved boxes; host forms include the host -> device copies"}
    try:
        for prec in ("f32", "f64"):
            res[f"d4_{prec}"] = probe4(prec, ctx, stream)
        res["d2_f32"] = probe2("f32", ctx, stream)
    finally:
        ctx.set_stream(None)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
