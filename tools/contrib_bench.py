"""What the blending-weight statistics cost (DGR_RASTER_CONTRIB) and what prune_unseen removes.

  * cfg2 (100k Gaussians, 800 x 800, degree 3) through GaussianRasterizer: forward only (no_grad) and forward + backward, without
    and with contributions=, alternating on the same seeded inputs, the L2 flushed before every call, medians;
  * in profiled calls of their own: render_fwd against render_fwd_contrib and contrib_finalize, per-kernel microseconds;
  * cfg3-sized batch (500k Gaussians, 8 views of 512 x 512, one batched forward), without and with the statistics, medians;
  * prune_unseen at the end of a 500-iteration stage-1 run: seconds, Gaussians before and removed.
Prints the card and its power limit, then one JSON line per part.

    python tools/contrib_bench.py [--steps 30] [--profile-steps 10] [--iters 500]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from det_bench import card  # noqa: E402


def _settings(cams, res, dev):
    import torch
    from dreamgaussian_b200.rasterizer import GaussianRasterizationSettings
    t = lambda x: torch.tensor(np.asarray(x, np.float32), device=dev)
    bg = t(np.ones(3, np.float32))
    return [GaussianRasterizationSettings(image_height=res, image_width=res, tanfovx=c.tanfovx, tanfovy=c.tanfovy, bg=bg, scale_modifier=1.0,
                                          viewmatrix=t(c.world_view_transform), projmatrix=t(c.full_proj_transform), sh_degree=3,
                                          campos=t(c.camera_center), prefiltered=False, debug=False) for c in cams]


def cfg2(dev, steps, profile_steps):
    import torch
    import bench
    from dreamgaussian_b200 import _lib
    from dreamgaussian_b200.rasterizer import ContributionStats, GaussianRasterizer
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
    a = argparse.Namespace(sh_degree=3, opacity="trained", seed=0, workload="cfg2",
                           **{k: bench.WORKLOADS["cfg2"][k] for k in ("points", "res", "views_per_gpu", "views")})
    cloud, cams, ups = bench.build_scene(a)
    t = lambda x: torch.tensor(np.asarray(x, np.float32), device=dev)
    inp = {k: t(cloud[k]).requires_grad_(True) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    settings = _settings(cams, a.res, dev)
    upc = [t(u[0]) for u in ups]
    P = a.points
    stats = ContributionStats(P, dev)

    def call(i, on, backward):
        for p in inp.values():
            p.grad = None
        with torch.set_grad_enabled(backward):
            means2D = torch.zeros_like(inp["means3D"], requires_grad=backward)
            c, _, _, _ = GaussianRasterizer(settings[i % len(settings)], contributions=stats if on else None)(
                means3D=inp["means3D"], means2D=means2D, opacities=inp["opacities"], shs=inp["shs"], scales=inp["scales"], rotations=inp["rotations"])
            if backward:
                (c * upc[i % len(upc)]).sum().backward()

    out = {"workload": bench.workload_name(a)}
    for backward in (False, True):
        for i in range(4):
            call(i, bool(i & 1), backward)
        torch.cuda.synchronize(dev)
        times = {False: [], True: []}
        for i in range(2 * steps):
            on = bool(i & 1)
            flush.zero_()
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            call(i // 2, on, backward)
            torch.cuda.synchronize(dev)
            times[on].append((time.perf_counter() - t0) * 1000.0)
        m0, m1 = float(np.median(times[False])), float(np.median(times[True]))
        key = "fwd_bwd" if backward else "fwd"
        out[key] = {"plain_ms": round(m0, 4), "contrib_ms": round(m1, 4), "ratio": round(m1 / m0, 3)}
    lib = _lib.load()
    kern = {}
    for i in range(2 * profile_steps):
        flush.zero_()
        torch.cuda.synchronize(dev)
        lib.dgr_profile_enable(1)
        call(i // 2, bool(i & 1), False)
        torch.cuda.synchronize(dev)
        for n, ms in _lib.profile_collect():
            if n.startswith(("render_fwd", "contrib_finalize")):
                kern.setdefault(n, []).append(ms * 1000.0)
        lib.dgr_profile_enable(0)
    out["kernel_us_median"] = {n: round(float(np.median(v)), 2) for n, v in kern.items()}
    return out


def cfg3(dev, steps):
    import torch
    from dreamgaussian_b200 import scene
    from dreamgaussian_b200.rasterizer import ContributionStats, rasterize_views
    P, res, V = 500000, 512, 8
    cloud = scene.make_cloud(P, 3, seed=0)
    cams = scene.bench_views(V, res, res)
    t = lambda x: torch.tensor(np.asarray(x, np.float32), device=dev)
    inp = {k: t(cloud[k]) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    settings = _settings(cams, res, dev)
    stats = ContributionStats(P, dev)
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)

    def call(on):
        with torch.no_grad():
            rasterize_views(settings, inp["means3D"], None, inp["opacities"], inp["shs"], inp["scales"], inp["rotations"],
                            contributions=stats if on else None)
    for i in range(4):
        call(bool(i & 1))
    times = {False: [], True: []}
    for i in range(2 * steps):
        on = bool(i & 1)
        flush.zero_()
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        call(on)
        torch.cuda.synchronize(dev)
        times[on].append((time.perf_counter() - t0) * 1000.0)
    m0, m1 = float(np.median(times[False])), float(np.median(times[True]))
    return {"points": P, "views": V, "res": res, "fwd_plain_ms": round(m0, 4), "fwd_contrib_ms": round(m1, 4), "ratio": round(m1 / m0, 3)}


def stage1_prune(iters):
    import torch
    from dreamgaussian_b200 import stage1
    tr = stage1.Stage1Trainer(stage1.Stage1Config(iters=iters))
    tr.train()
    n0 = tr.gaussians.num_points
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    removed = tr.prune_unseen(1e-3)
    torch.cuda.synchronize()
    return {"iters": iters, "points": n0, "removed_weight_max_below_1e-3": removed, "seconds": round(time.perf_counter() - t0, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30, help="timed calls per arm")
    ap.add_argument("--profile-steps", type=int, default=10, help="profiled cfg2 forwards per arm for the per-kernel times")
    ap.add_argument("--iters", type=int, default=500, help="stage-1 iterations before prune_unseen")
    a = ap.parse_args()
    import torch
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name = card()
    print("card, power limit:", name, flush=True)
    print(json.dumps({"card": name, "cfg2": cfg2(dev, a.steps, a.profile_steps)}), flush=True)
    print(json.dumps({"card": name, "cfg3": cfg3(dev, a.steps)}), flush=True)
    print(json.dumps({"card": name, "stage1_prune_unseen": stage1_prune(a.iters)}), flush=True)


if __name__ == "__main__":
    main()
