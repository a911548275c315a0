"""Batched cameras against a loop of single-view calls, on the GPU, in one run.

For each shape it times, alternating the two paths step by step with an L2 flush before every step and CUDA events around
it:
  loop     V single-view forward+backward calls accumulating into one gradient (what multiview.render_views does);
  batched  one dgr_views forward+backward (rasterize_views' host path);
for the mixed-size shapes (stage1_mixed: the stage-1 step's known view at 256^2 and novel view at 512^2) the batched path is
one dgr_views_mixed forward+backward (rasterize_views_mixed's host path).
It then compares the two paths' outputs on the timed inputs: images per view and the summed gradients.  Prints one JSON line
per shape plus the card's name and power limit, read in the same run.

    python tools/views_bench.py [--steps 20] [--warmup 3] [--shapes cfg3,mvdream,stage1,bake,stage1_mixed]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dreamgaussian_b200 import rasterizer as R  # noqa: E402
from dreamgaussian_b200 import scene  # noqa: E402

SHAPES = {                     # name: (P, resolution, views, sh degree, backward)
    "cfg3": (500_000, 512, 8, 3, True),
    "mvdream": (50_000, 256, 4, 0, True),
    "stage1": (5_000, 128, 4, 0, True),
    "bake": (50_000, 512, 26, 0, False),
}
MIXED_SHAPES = {               # name: (P, resolution per view, sh degree, backward)
    "stage1_mixed": (5_000, (256, 512), 0, True),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return dict(name=name, power_limit=power)
    except Exception as e:  # noqa: BLE001
        return dict(name=torch.cuda.get_device_name(0), power_limit="unknown (%s)" % e)


def make(shape):
    if shape in MIXED_SHAPES:
        P, sizes, deg, bwd = MIXED_SHAPES[shape]
    else:
        P, res, V, deg, bwd = SHAPES[shape]
        sizes = (res,) * V
    V = len(sizes)
    cloud = scene.make_cloud(P, deg, seed=1)
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda")
    inputs = {k: t(cloud[k]) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    settings = []
    for v, res in enumerate(sizes):
        cam = scene.orbit_camera(-15.0 + 10.0 * (v % 4), 360.0 * v / V, 2.0, res, res)
        settings.append(R.GaussianRasterizationSettings(res, res, cam.tanfovx, cam.tanfovy, t([1.0, 1.0, 1.0]), 1.0,
                                                        t(cam.world_view_transform), t(cam.full_proj_transform), deg,
                                                        t(cam.camera_center), False, False))
    g = torch.Generator(device="cuda").manual_seed(5)
    if shape in MIXED_SHAPES:           # per view (gC [3,H,W], gD, gA), and the flat layout the mixed call takes
        per_view = [[torch.randn((c, res, res), device="cuda", generator=g) for c in (3, 1, 1)] for res in sizes]
        up = [[pv[k] for pv in per_view] for k in range(3)]
        up.append([torch.cat([x.reshape(-1) for x in up[k]]) for k in range(3)])
    else:
        up = [torch.randn((V, c, res, res), device="cuda", generator=g) for c in (3, 1, 1)]
    return inputs, settings, up, bwd


def grads_like(inputs, V=None):
    P, M = inputs["means3D"].shape[0], inputs["shs"].shape[1]
    e = lambda *s: torch.zeros(s, device="cuda")
    return [e(P, 3), e(V, P, 3) if V else e(P, 3), e(P, M, 3), e(P, 1), e(P, 3), e(P, 4)]


def run_loop(inputs, settings, up, bwd):
    i = inputs
    d = grads_like(i)
    imgs = []
    for v, rs in enumerate(settings):
        color, radii, depth, alpha, st = R.forward_impl(rs, i["means3D"], i["shs"], None, i["opacities"], i["scales"], i["rotations"], None)
        imgs.append(color)
        if bwd:
            R.backward_impl(st, up[0][v], up[1][v], up[2][v], d[0], d[1], d[2], None, d[3], d[4], d[5], None, accumulate=v > 0)
    return imgs, d


def run_batched(inputs, settings, up, bwd):
    i = inputs
    d = grads_like(i, len(settings))
    color, radii, depth, alpha, st = R.views_forward_impl(settings, i["means3D"], i["shs"], i["opacities"], i["scales"], i["rotations"])
    if bwd:
        R.views_backward_impl(st, up[0], up[1], up[2], d[0], d[1], d[2], d[3], d[4], d[5])
    return list(color), d


def run_mixed(inputs, settings, up, bwd):
    i = inputs
    d = grads_like(i, len(settings))
    color, radii, depth, alpha, st = R.views_forward_impl(settings, i["means3D"], i["shs"], i["opacities"], i["scales"], i["rotations"],
                                                          mixed=True)
    if bwd:
        R.views_backward_impl(st, *up[3], d[0], d[1], d[2], d[3], d[4], d[5])
    return R.split_views(settings, color, depth, alpha)[0], d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--shapes", default="cfg3,mvdream,stage1,bake,stage1_mixed")
    a = ap.parse_args()
    info = card()
    print(json.dumps(dict(card=info)), flush=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")       # > L2 (50 MB)
    for shape in a.shapes.split(","):
        inputs, settings, up, bwd = make(shape)
        batched = run_mixed if shape in MIXED_SHAPES else run_batched
        paths = dict(loop=run_loop, batched=batched)
        for _ in range(a.warmup):
            for fn in paths.values():
                fn(inputs, settings, up, bwd)
        torch.cuda.synchronize()
        ms = {k: [] for k in paths}
        for _ in range(a.steps):
            for k, fn in paths.items():                  # alternating
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn(inputs, settings, up, bwd)
                e1.record()
                e1.synchronize()
                ms[k].append(e0.elapsed_time(e1))
        # outputs of the two paths on the timed inputs
        il, dl = run_loop(inputs, settings, up, bwd)
        ib, db = batched(inputs, settings, up, bwd)
        img_diff = max(float((x - y).abs().max()) for x, y in zip(il, ib))
        rel = lambda x, y: float((x - y).abs().max() / max(float(y.abs().max()), 1e-30))
        grad_rel = max(rel(db[k], dl[k]) for k in (0, 2, 3, 4, 5)) if bwd else None
        res = [int(s.image_height) for s in settings]
        rec = dict(shape=shape, P=inputs["means3D"].shape[0], res=res[0] if len(set(res)) == 1 else res, views=len(settings),
                   deg=int(settings[0].sh_degree), backward=bwd, loop_ms=round(statistics.median(ms["loop"]), 4), batched_ms=round(statistics.median(ms["batched"]), 4),
                   loop_ms_min=round(min(ms["loop"]), 4), batched_ms_min=round(min(ms["batched"]), 4),
                   speedup=round(statistics.median(ms["loop"]) / statistics.median(ms["batched"]), 3),
                   max_image_abs_diff=img_diff, max_grad_rel_diff=grad_rel,
                   outputs_match=bool(img_diff <= 1e-2 and (grad_rel is None or grad_rel <= 2e-4)), card=info["name"],
                   power_limit=info["power_limit"], steps=a.steps)
        print(json.dumps(rec), flush=True)
        del inputs, settings, up
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
