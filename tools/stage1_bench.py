"""BASELINE.json configs[3] / SURVEY §8 row f2 measurement: the DreamGaussian stage-1 loop (configs/image.yaml, synthetic
RGBA input, guidance stubbed), 500 iterations on one B200 — fused path (FusedGaussianRasterizer + one-launch Adam +
in-kernel densification statistics + own distCUDA2) against the reference's formulation of the same loop running on this
library's plain op (torch activations + cat, torch statistic updates, per-tensor Adam ops).  Wall clock around a device
synchronise.  Writes gpurun_out/stage1_bench.json."""
import json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np, torch
from dreamgaussian_b200 import stage1

out = {"config": "configs/image.yaml: 5000 initial points, sh_degree 0, 256^2 known view + 128/256/512^2 novel view per iteration, 500 iterations, densify every 100 from 100"}
# the arms alternate; fused_batched = the fused path with both renders of a step in one mixed-size batched call
# (Stage1Trainer(batched=True))
ARMS = (("reference_formulation", False, False), ("fused", True, False), ("fused_batched", True, True),
        ("reference_formulation_again", False, False), ("fused_again", True, False), ("fused_batched_again", True, True))
for name, fused, batched in ARMS:
    tr = stage1.Stage1Trainer(stage1.Stage1Config(), fused=fused, batched=batched)
    tr.train(10); torch.cuda.synchronize()                      # warm-up (allocator, capacity hints)
    tr = stage1.Stage1Trainer(stage1.Stage1Config(), fused=fused, batched=batched)
    torch.cuda.synchronize(); t0 = time.perf_counter()
    losses = tr.train(500)
    torch.cuda.synchronize(); dt = time.perf_counter() - t0
    out[name] = {"seconds": dt, "iters_per_s": 500 / dt, "final_points": tr.gaussians.num_points, "loss_first": float(losses[0]), "loss_last": float(losses[-1])}
    print(name, json.dumps(out[name]), flush=True)
out["speedup"] = out["reference_formulation_again"]["seconds"] / out["fused_again"]["seconds"]
out["batched_speedup"] = out["fused_again"]["seconds"] / out["fused_batched_again"]["seconds"]       # fused -> fused_batched
print(json.dumps({"speedup": out["speedup"], "batched_speedup": out["batched_speedup"]}))
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
json.dump(out, open(os.path.join(ROOT, "gpurun_out", "stage1_bench.json"), "w"), indent=1)
