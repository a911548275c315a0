"""What the anti-aliased mode costs: on the same seeded inputs, default and anti-aliased forward+backward steps alternate, the L2 is
flushed before every step, and the median step time and tile-instance count of each arm are reported for cfg2 (100k Gaussians,
800 x 800, degree 3) and cfg3 (8 views in one same-size batched call); then 500 iterations of the stage-1 loop at the
configs/image.yaml shape in both arms.  Prints the card and its power limit, then one JSON line.

    python tools/aa_bench.py [--steps 30] [--stage1-iters 500]
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


def shape_rows(dev, steps):
    import torch
    import bench
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
        settings = [GaussianRasterizationSettings(
            image_height=a.res, image_width=a.res, tanfovx=c.tanfovx, tanfovy=c.tanfovy, bg=bg, scale_modifier=1.0,
            viewmatrix=t(c.world_view_transform), projmatrix=t(c.full_proj_transform), sh_degree=3, campos=t(c.camera_center),
            prefiltered=False, debug=False) for c in cams]
        upc, upa = [t(u[0]) for u in ups], [t(u[2]) for u in ups]
        P = a.points
        inst = {False: [], True: []}

        def step(i, aa):
            for p in params.values():
                p.grad = None
            if views == 1:
                means2D = torch.zeros((P, 3), device=dev, requires_grad=True)
                c, _, _, al = GaussianRasterizer(settings[i % len(settings)], antialiasing=aa)(
                    means3D=params["means3D"], means2D=means2D, opacities=params["opacities"], shs=params["shs"],
                    scales=params["scales"], rotations=params["rotations"])
                loss = (c * upc[i % len(upc)]).sum() + (al * upa[i % len(upa)]).sum()
                node = c.grad_fn
            else:
                vs = [(i * views + k) % len(settings) for k in range(views)]
                means2D = torch.zeros((views, P, 3), device=dev, requires_grad=True)
                c, _, _, al = rasterize_views([settings[v] for v in vs], params["means3D"], means2D, params["opacities"], params["shs"],
                                              params["scales"], params["rotations"], antialiasing=aa)
                loss = sum((c[k] * upc[v % len(upc)]).sum() + (al[k] * upa[v % len(upa)]).sum() for k, v in enumerate(vs))
                node = c.grad_fn
            inst[aa].append(int(node.state.num_rendered))
            loss.backward()

        for i in range(4):
            step(i, bool(i & 1))
        torch.cuda.synchronize(dev)
        times = {False: [], True: []}
        for k in inst:
            inst[k].clear()
        for i in range(2 * steps):
            aa = bool(i & 1)
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); step(i // 2, aa); e1.record()
            torch.cuda.synchronize(dev)
            times[aa].append(e0.elapsed_time(e1))
        md, ma = float(np.median(times[False])), float(np.median(times[True]))
        rows[key] = {"workload": bench.workload_name(a), "views_per_call": views, "steps_per_arm": steps, "default_ms": round(md, 4),
                     "aa_ms": round(ma, 4), "ratio": round(ma / md, 3), "instances_default": int(np.mean(inst[False])),
                     "instances_aa": int(np.mean(inst[True]))}
        print(json.dumps({key: rows[key]}), flush=True)
        del params, settings, upc, upa
        torch.cuda.empty_cache()
    return rows


def stage1_rows(iters):
    import torch
    from dreamgaussian_b200 import stage1
    rows = {}
    for aa in (False, True, False, True):
        tr = stage1.Stage1Trainer(stage1.Stage1Config(iters=iters, seed=0, antialiasing=aa), fused=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        tr.train(iters)
        torch.cuda.synchronize()
        r = rows.setdefault("aa" if aa else "default", {"s_total": [], "points_end": int(tr.gaussians.num_points)})
        r["s_total"].append(round(time.perf_counter() - t0, 3))
        del tr
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30, help="timed steps per arm and shape")
    ap.add_argument("--stage1-iters", type=int, default=500)
    a = ap.parse_args()
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
