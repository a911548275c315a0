"""What MCMC densification costs (dgr_mcmc_refine / dgr_mcmc_inject_noise) and what it does to stage 1.

  * one refinement (relocation of the dead rows, growth by 5 %) and one noise call at P = 5k, 50k, 500k and 2M Gaussians (degree 3,
    about 3 % of them dead), CUDA events around the call, medians over --reps calls on the same inputs;
  * 500 stage-1 iterations at the configs/image.yaml shape, default densification against densify_strategy="mcmc": seconds (host
    clock ending in a synchronise), final point count, and the CUDA kernels per step counted by torch.profiler over --profile-steps
    further steps of each run (no refinement among them) and over one refinement call.
Prints the card and its power limit, then one JSON line per part.

    python tools/mcmc_bench.py [--reps 20] [--iters 500] [--profile-steps 20] [--sizes 5000,50000,500000,2000000]
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


def _model(P, dev, seed=0):
    import torch
    from dreamgaussian_b200 import stage1
    rng = np.random.default_rng(seed)
    f = lambda *s: torch.tensor(rng.normal(size=s).astype(np.float32), device=dev)
    g = stage1.GaussianModelB200(3)
    g._set(dict(xyz=f(P, 3) * 0.3, f_dc=f(P, 1, 3), f_rest=f(P, 15, 3) * 0.1, opacity=f(P, 1) * 2.0 - 1.5, scaling=f(P, 3) * 0.5 - 4.0,
                rotation=f(P, 4)))
    g.training_setup()
    g.fused_adam = g.fused_densify = True
    return g


def _kernels(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith(("Memset", "Memcpy")))


def calls(dev, sizes, reps):
    import torch
    from dreamgaussian_b200 import stage1
    for P in sizes:
        g = _model(P, dev)
        saved = ({k: v.detach().clone() for k, v in g.p.items()}, {k: v.clone() for k, v in g.exp_avg.items()},
                 {k: v.clone() for k, v in g.exp_avg_sq.items()})
        n_add = stage1.mcmc_add_count(P, 10 ** 9)
        u, ua = torch.rand((P,), device=dev), torch.rand((n_add,), device=dev)
        zn = torch.randn((P + n_add, 3), device=dev)
        t_ref, t_noise = [], []
        for r in range(reps + 2):
            g._set(saved[0])
            g.exp_avg = {k: v.clone() for k, v in saved[1].items()}
            g.exp_avg_sq = {k: v.clone() for k, v in saved[2].items()}
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            n = g.relocate_and_grow_mcmc(10 ** 9, u_relocate=u, u_add=ua)
            b.record()
            c, d = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            c.record()
            g.inject_noise_mcmc(100.0, normals=zn)
            d.record()
            torch.cuda.synchronize()
            if r >= 2:                                  # warm-up: module load, allocator
                t_ref.append(a.elapsed_time(b)); t_noise.append(c.elapsed_time(d))
        g._set(saved[0])
        g.exp_avg = {k: v.clone() for k, v in saved[1].items()}
        g.exp_avg_sq = {k: v.clone() for k, v in saved[2].items()}
        launches = _kernels(lambda: g.relocate_and_grow_mcmc(10 ** 9, u_relocate=u, u_add=ua))
        print(json.dumps(dict(part="calls", P=P, n_add=n_add, relocated=int(n), refine_ms=float(np.median(t_ref)),
                              noise_ms=float(np.median(t_noise)), refine_kernels=launches)), flush=True)
        del g, saved


def stage1_runs(iters, profile_steps):
    import torch
    from dreamgaussian_b200 import stage1
    for strategy in ("default", "mcmc"):
        tr = stage1.Stage1Trainer(stage1.Stage1Config(iters=iters, densify_strategy=strategy))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        losses = tr.train(iters)
        torch.cuda.synchronize()
        sec = time.perf_counter() - t0
        n = tr.gaussians.num_points
        per_step = _kernels(lambda: tr.train(profile_steps)) / profile_steps
        print(json.dumps(dict(part="stage1", strategy=strategy, iters=iters, seconds=sec, final_points=n, final_loss=float(losses[-1]),
                              kernels_per_step=per_step)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--iters", type=int, default=500)
    ap.add_argument("--profile-steps", type=int, default=20)
    ap.add_argument("--sizes", default="5000,50000,500000,2000000")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("mcmc_bench.py needs a CUDA device")
    print(json.dumps(dict(part="card", card=card())), flush=True)
    calls(torch.device("cuda"), [int(s) for s in a.sizes.split(",")], a.reps)
    stage1_runs(a.iters, a.profile_steps)


if __name__ == "__main__":
    main()
