"""What the deterministic backward costs: on the same seeded inputs, default and deterministic forward+backward steps alternate
(torch.use_deterministic_algorithms off / on), the L2 is flushed before every step, and the median step time of each arm and the
per-kernel times of the library's CUDA events (forward and backward kernels in microseconds per step, driven on the calling thread;
"det_memset" is the instance-scratch memset) are reported for cfg2, cfg2 at opacity 0.1, cfg3 (8 views in one same-size batched
call) and cfg5; then 500 iterations of the stage-1 loop in both arms.  Prints the card and its power limit, then one JSON line.

    python tools/det_bench.py [--steps 30] [--stage1-iters 500]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                             stderr=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:  # noqa: BLE001
        return "unknown"


def shape_rows(dev, steps):
    import torch
    import bench
    from dreamgaussian_b200 import _lib
    from dreamgaussian_b200 import rasterizer as R
    from dreamgaussian_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer, rasterize_views
    lib = _lib.load()
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
    rows = {}
    for key, wl, over, views in (("cfg2", "cfg2", {}, 1), ("cfg2_opacity_0.1", "cfg2", dict(opacity="init"), 1),
                                 ("cfg3_8_views_batched", "cfg3", {}, 8), ("cfg5", "cfg5", {}, 1)):
        a = argparse.Namespace(sh_degree=3, opacity="trained", seed=0, workload=wl,
                               **{k: bench.WORKLOADS[wl][k] for k in ("points", "res", "views_per_gpu", "views")})
        for k, v in over.items():
            setattr(a, k, v)
        cloud, cams, ups = bench.build_scene(a)
        t = lambda x: torch.tensor(np.asarray(x, np.float32), device=dev)
        params = {k: t(v).requires_grad_(True) for k, v in cloud.items()}
        bg = t(np.ones(3, np.float32))
        settings = [GaussianRasterizationSettings(
            image_height=a.res, image_width=a.res, tanfovx=c.tanfovx, tanfovy=c.tanfovy, bg=bg, scale_modifier=1.0,
            viewmatrix=t(c.world_view_transform), projmatrix=t(c.full_proj_transform), sh_degree=3, campos=t(c.camera_center),
            prefiltered=False, debug=False) for c in cams]
        upc = [t(u[0]) for u in ups]
        upa = [t(u[2]) for u in ups]
        P = a.points

        def step(i):
            for p in params.values():
                p.grad = None
            if views == 1:
                means2D = torch.zeros((P, 3), device=dev, requires_grad=True)
                c, _, _, al = GaussianRasterizer(settings[i % len(settings)])(
                    means3D=params["means3D"], means2D=means2D, opacities=params["opacities"], shs=params["shs"],
                    scales=params["scales"], rotations=params["rotations"])
                loss = (c * upc[i % len(upc)]).sum() + (al * upa[i % len(upa)]).sum()
            else:
                vs = [(i * views + k) % len(settings) for k in range(views)]
                means2D = torch.zeros((views, P, 3), device=dev, requires_grad=True)
                c, _, _, al = rasterize_views([settings[v] for v in vs], params["means3D"], means2D, params["opacities"], params["shs"],
                                              params["scales"], params["rotations"])
                loss = sum((c[k] * upc[v % len(upc)]).sum() + (al[k] * upa[v % len(upa)]).sum() for k, v in enumerate(vs))
            loss.backward()

        times = {False: [], True: []}
        for i in range(4):
            torch.use_deterministic_algorithms(bool(i & 1)); step(i)
        torch.cuda.synchronize(dev)
        for i in range(2 * steps):
            det = bool(i & 1)
            torch.use_deterministic_algorithms(det)
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); step(i); e1.record()
            torch.cuda.synchronize(dev)
            times[det].append(e0.elapsed_time(e1))
        # per-kernel times: the library records its CUDA events per host thread and the autograd engine runs a backward on its own
        # thread, so this pass drives forward_impl / backward_impl (views_*_impl) directly on this thread, on the same inputs
        det_p = {k: v.detach() for k, v in params.items()}
        grads = {k: torch.empty_like(v) for k, v in det_p.items()}
        d_m2d = torch.empty((views, P, 3) if views > 1 else (P, 3), device=dev)

        def step_direct(i):
            m3, sh, op, sc, rot = det_p["means3D"], det_p["shs"], det_p["opacities"], det_p["scales"], det_p["rotations"]
            if views == 1:
                j = i % len(settings)
                st = R.forward_impl(settings[j], m3, sh, None, op, sc, rot, None)[4]
                R.backward_impl(st, upc[j % len(upc)], None, upa[j % len(upa)], grads["means3D"], d_m2d, grads["shs"], None,
                                grads["opacities"], grads["scales"], grads["rotations"], None)
            else:
                vs = [(i * views + k) % len(settings) for k in range(views)]
                st = R.views_forward_impl([settings[v] for v in vs], m3, sh, op, sc, rot)[4]
                gC = torch.stack([upc[v % len(upc)] for v in vs]).contiguous()
                gA = torch.stack([upa[v % len(upa)] for v in vs]).contiguous()
                R.views_backward_impl(st, gC, None, gA, grads["means3D"], d_m2d, grads["shs"], grads["opacities"], grads["scales"],
                                      grads["rotations"])

        kern = {}
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            step_direct(0)
            torch.cuda.synchronize(dev)
            lib.dgr_profile_enable(1)
            for i in range(3):
                flush.zero_(); step_direct(i)
            torch.cuda.synchronize(dev)
            per = {}
            for name, v in _lib.profile_collect():
                per.setdefault(name, []).append(v)
            lib.dgr_profile_enable(0)
            kern["det" if det else "default"] = {k: round(float(np.sum(v)) / 3 * 1e3, 1) for k, v in per.items()}
        torch.use_deterministic_algorithms(False)
        md, mt = float(np.median(times[False])), float(np.median(times[True]))
        rows[key] = {"workload": bench.workload_name(a), "views_per_call": views, "steps_per_arm": steps, "default_ms": round(md, 4),
                     "det_ms": round(mt, 4), "ratio": round(mt / md, 3), "kernels_us_per_step": kern}
        print(json.dumps({key: rows[key]}), flush=True)
        del params, settings, upc, upa, det_p, grads, d_m2d
        torch.cuda.empty_cache()
    return rows


def stage1_rows(iters):
    import torch
    from dreamgaussian_b200 import stage1
    rows = {}
    for fused in (True, False):
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            tr = stage1.Stage1Trainer(stage1.Stage1Config(iters=iters, seed=0), fused=fused)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tr.train(iters)
            torch.cuda.synchronize()
            rows["%s_%s" % ("fused" if fused else "reference", "det" if det else "default")] = {
                "s_total": round(time.perf_counter() - t0, 3), "points_end": int(tr.gaussians.num_points)}
            torch.use_deterministic_algorithms(False)
            del tr
            torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30, help="timed steps per arm and shape")
    ap.add_argument("--stage1-iters", type=int, default=500)
    a = ap.parse_args()
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")      # cuBLAS under torch.use_deterministic_algorithms(True)
    import torch
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name = card()
    print("card, power limit:", name, flush=True)
    out = {"card": name, "shapes": shape_rows(dev, a.steps)}
    if a.stage1_iters > 0:
        out["stage1_%d_iters" % a.stage1_iters] = stage1_rows(a.stage1_iters)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
