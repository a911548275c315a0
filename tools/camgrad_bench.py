"""What camera gradients cost (DGR_RASTER_CAMERA_GRADS): on the same seeded inputs, default forward+backward steps and steps whose
viewmatrix / projmatrix / campos require grad alternate, the L2 is flushed before every step, and the median step time of each
arm is reported for cfg2 (100k Gaussians, 800 x 800, degree 3) and cfg3 (8 views in one same-size batched call); then, in
separate profiled steps, the per-kernel times of the two new kernels (camera_bwd, camera_reduce) from dgr_profile_*.
Prints the card and its power limit, then one JSON line.

    python tools/camgrad_bench.py [--steps 30] [--profile-steps 10]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from det_bench import card  # noqa: E402


def shape_rows(dev, steps, profile_steps):
    import torch
    import bench
    from dreamgaussian_b200 import _lib
    from dreamgaussian_b200 import rasterizer as R
    from dreamgaussian_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer, rasterize_views
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
    rows = {}
    for key, wl, views in (("cfg2", "cfg2", 1), ("cfg3_8_views_batched", "cfg3", 8)):
        a = argparse.Namespace(sh_degree=3, opacity="trained", seed=0, workload=wl,
                               **{k: bench.WORKLOADS[wl][k] for k in ("points", "res", "views_per_gpu", "views")})
        cloud, cams, ups = bench.build_scene(a)
        t = lambda x: torch.tensor(np.asarray(x, np.float32), device=dev)
        params = {k: t(v).requires_grad_(True) for k, v in cloud.items()}
        bg = t(np.ones(3, np.float32))
        settings = {}
        for cg in (False, True):
            settings[cg] = [GaussianRasterizationSettings(
                image_height=a.res, image_width=a.res, tanfovx=c.tanfovx, tanfovy=c.tanfovy, bg=bg, scale_modifier=1.0,
                viewmatrix=t(c.world_view_transform).requires_grad_(cg), projmatrix=t(c.full_proj_transform).requires_grad_(cg), sh_degree=3,
                campos=t(c.camera_center).requires_grad_(cg), prefiltered=False, debug=False) for c in cams]
        upc, upa = [t(u[0]) for u in ups], [t(u[2]) for u in ups]
        P = a.points

        def step(i, cg, profile=False):
            """One forward+backward; profile=True: the backward runs through backward_impl on this thread (dgr_profile_* records the
            launches of the calling host thread; loss.backward() would run it in autograd's device thread)."""
            for p in params.values():
                p.grad = None
            ss = settings[cg]
            if views == 1:
                means2D = torch.zeros((P, 3), device=dev, requires_grad=True)
                c, _, _, al = GaussianRasterizer(ss[i % len(ss)])(
                    means3D=params["means3D"], means2D=means2D, opacities=params["opacities"], shs=params["shs"],
                    scales=params["scales"], rotations=params["rotations"])
                loss = (c * upc[i % len(upc)]).sum() + (al * upa[i % len(upa)]).sum()
                if profile:
                    e = lambda *shape: torch.empty(shape, device=dev)
                    R.backward_impl(c.grad_fn.state, upc[i % len(upc)], None, upa[i % len(upa)], e(P, 3), e(P, 3), e(*params["shs"].shape),
                                    None, e(P, 1), e(P, 3), e(P, 4), None, camera=R._camera_outputs(0, dev))
                    return
            else:
                vs = [(i * views + k) % len(ss) for k in range(views)]
                means2D = torch.zeros((views, P, 3), device=dev, requires_grad=True)
                c, _, _, al = rasterize_views([ss[v] for v in vs], params["means3D"], means2D, params["opacities"], params["shs"],
                                              params["scales"], params["rotations"])
                loss = sum((c[k] * upc[v % len(upc)]).sum() + (al[k] * upa[v % len(upa)]).sum() for k, v in enumerate(vs))
                if profile:
                    e = lambda *shape: torch.empty(shape, device=dev)
                    R.views_backward_impl(c.grad_fn.state, torch.stack([upc[v % len(upc)] for v in vs]), None,
                                          torch.stack([upa[v % len(upa)] for v in vs]), e(P, 3), e(views, P, 3), e(*params["shs"].shape),
                                          e(P, 1), e(P, 3), e(P, 4), camera=R._camera_outputs(views, dev))
                    return
            loss.backward()

        for i in range(4):
            step(i, bool(i & 1))
        torch.cuda.synchronize(dev)
        times = {False: [], True: []}
        for i in range(2 * steps):
            cg = bool(i & 1)
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); step(i // 2, cg); e1.record()
            torch.cuda.synchronize(dev)
            times[cg].append(e0.elapsed_time(e1))
        # per-kernel times of the new kernels, in profiled steps of their own (the event pairs slow the host)
        lib = _lib.load()
        kern = {}
        for i in range(profile_steps):
            flush.zero_()
            torch.cuda.synchronize(dev)
            lib.dgr_profile_enable(1)
            step(i, True, profile=True)
            torch.cuda.synchronize(dev)
            for n, ms in _lib.profile_collect():
                if n.startswith(("camera_", "preprocess_bwd", "preprocess_views_bwd")):
                    kern.setdefault(n, []).append(ms * 1000.0)
            lib.dgr_profile_enable(0)
        md, mc = float(np.median(times[False])), float(np.median(times[True]))
        rows[key] = {"workload": bench.workload_name(a), "views_per_call": views, "steps_per_arm": steps, "default_ms": round(md, 4),
                     "camera_grads_ms": round(mc, 4), "ratio": round(mc / md, 3),
                     "kernel_us_median": {n: round(float(np.median(v)), 2) for n, v in kern.items()}}
        print(json.dumps({key: rows[key]}), flush=True)
        del params, settings, upc, upa
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30, help="timed steps per arm and shape")
    ap.add_argument("--profile-steps", type=int, default=10, help="profiled steps per shape for the per-kernel times")
    a = ap.parse_args()
    import torch
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name = card()
    print("card, power limit:", name, flush=True)
    print(json.dumps({"card": name, "shapes": shape_rows(dev, a.steps, a.profile_steps)}), flush=True)


if __name__ == "__main__":
    main()
