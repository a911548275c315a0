"""What the absolute-gradient statistic costs (DGR_RASTER_ABS_GRAD) and what it does to stage 1.

  * cfg2 (100k Gaussians, 800 x 800, degree 3) through the fused raw-parameter rasterizer with densification statistics: steps
    without and with the absolute statistic alternate on the same seeded inputs, the L2 is flushed before every step, medians;
  * in profiled steps of their own: render_bwd against render_bwd_abs, and absgrad_stats, per-kernel microseconds;
  * 500 stage-1 iterations without and with densify_abs_grad_threshold: seconds, final point count, final known-view MSE
    (reported, not asserted: the guidance is a stub, so this says nothing about quality).
Prints the card and its power limit, then one JSON line per part.

    python tools/absgrad_bench.py [--steps 30] [--profile-steps 10] [--iters 500] [--threshold 0.02]
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


def cfg2(dev, steps, profile_steps):
    import torch
    import bench
    from dreamgaussian_b200 import _lib, scene
    from dreamgaussian_b200 import rasterizer as R
    from dreamgaussian_b200.fused import DensifyStats, FusedGaussianRasterizer
    from dreamgaussian_b200.rasterizer import GaussianRasterizationSettings
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
    a = argparse.Namespace(sh_degree=3, opacity="trained", seed=0, workload="cfg2",
                           **{k: bench.WORKLOADS["cfg2"][k] for k in ("points", "res", "views_per_gpu", "views")})
    cloud, cams, ups = bench.build_scene(a)
    raw = scene.to_raw_parameters(cloud, seed=0)
    t = lambda x: torch.tensor(np.asarray(x, np.float32), device=dev)
    params = {k: t(v).requires_grad_(True) for k, v in raw.items()}
    bg = t(np.ones(3, np.float32))
    settings = [GaussianRasterizationSettings(image_height=a.res, image_width=a.res, tanfovx=c.tanfovx, tanfovy=c.tanfovy, bg=bg,
                                              scale_modifier=1.0, viewmatrix=t(c.world_view_transform), projmatrix=t(c.full_proj_transform),
                                              sh_degree=3, campos=t(c.camera_center), prefiltered=False, debug=False) for c in cams]
    upc, upa = [t(u[0]) for u in ups], [t(u[2]) for u in ups]
    P = a.points
    stats = {False: DensifyStats(P, dev), True: DensifyStats(P, dev, absgrad=True)}

    def step(i, ab, profile=False):
        for p in params.values():
            p.grad = None
        means2D = torch.zeros((P, 3), device=dev, requires_grad=True)
        st = stats[ab]
        c, _, _, al = FusedGaussianRasterizer(settings[i % len(settings)])(params["xyz"], params["features_dc"], params["features_rest"],
                                                                           params["opacity"], params["scaling"], params["rotation"],
                                                                           means2D=means2D, stats=st)
        if profile:              # on this thread: dgr_profile_* records the launches of the calling host thread
            e = lambda *shape: torch.empty(shape, device=dev)
            R.backward_impl(c.grad_fn.state, upc[i % len(upc)], None, upa[i % len(upa)], e(P, 3), e(P, 3), e(P, 1, 3), None, e(P, 1),
                            e(P, 3), e(P, 4), None, d_sh_rest=e(*params["features_rest"].shape), densify=st.as_tuple(),
                            absgrad=st.xyz_gradient_accum_abs)
            return
        ((c * upc[i % len(upc)]).sum() + (al * upa[i % len(upa)]).sum()).backward()

    for i in range(4):
        step(i, bool(i & 1))
    torch.cuda.synchronize(dev)
    times = {False: [], True: []}
    for i in range(2 * steps):
        ab = bool(i & 1)
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); step(i // 2, ab); e1.record()
        torch.cuda.synchronize(dev)
        times[ab].append(e0.elapsed_time(e1))
    lib = _lib.load()
    kern = {}
    for i in range(2 * profile_steps):
        flush.zero_()
        torch.cuda.synchronize(dev)
        lib.dgr_profile_enable(1)
        step(i // 2, bool(i & 1), profile=True)
        torch.cuda.synchronize(dev)
        for n, ms in _lib.profile_collect():
            if n.startswith(("render_bwd", "absgrad_stats", "preprocess_bwd")):
                kern.setdefault(n, []).append(ms * 1000.0)
        lib.dgr_profile_enable(0)
    md, ma = float(np.median(times[False])), float(np.median(times[True]))
    return {"workload": bench.workload_name(a), "steps_per_arm": steps, "stats_ms": round(md, 4), "stats_and_abs_ms": round(ma, 4),
            "ratio": round(ma / md, 3), "kernel_us_median": {n: round(float(np.median(v)), 2) for n, v in kern.items()}}


def stage1_runs(iters, threshold):
    import torch
    from dreamgaussian_b200 import stage1
    rows = {}
    for thr in (None, threshold):
        cfg = stage1.Stage1Config(iters=iters, densify_abs_grad_threshold=thr)
        tr = stage1.Stage1Trainer(cfg)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        tr.train()
        torch.cuda.synchronize()
        sec = time.perf_counter() - t0
        with torch.no_grad():
            out = tr.render(tr.fixed_cam, track_stats=False)
            mse = float(torch.nn.functional.mse_loss(out["image"].unsqueeze(0), tr.input_img))
        rows["default" if thr is None else "abs_threshold_%g" % thr] = {"seconds": round(sec, 3), "points": tr.gaussians.num_points,
                                                                         "known_view_mse": round(mse, 6)}
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30, help="timed cfg2 steps per arm")
    ap.add_argument("--profile-steps", type=int, default=10, help="profiled cfg2 steps per arm for the per-kernel times")
    ap.add_argument("--iters", type=int, default=500, help="stage-1 iterations per run")
    ap.add_argument("--threshold", type=float, default=0.02, help="densify_abs_grad_threshold of the second stage-1 run")
    a = ap.parse_args()
    import torch
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name = card()
    print("card, power limit:", name, flush=True)
    print(json.dumps({"card": name, "cfg2": cfg2(dev, a.steps, a.profile_steps)}), flush=True)
    print(json.dumps({"card": name, "stage1": stage1_runs(a.iters, a.threshold)}), flush=True)


if __name__ == "__main__":
    main()
