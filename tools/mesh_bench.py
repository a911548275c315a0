"""Cost of the device mesh export (include/dgr_mesh.h) on two models at resolutions 128 / 256 / 512: a 500-iteration Stage1Trainer
model and a 100k model-like cloud (built as tests/test_fields_gpu.py builds it).

    python tools/mesh_bench.py [--out results.json] [--reps 20]

Per model and resolution: CUDA-event medians over --reps calls after a warm-up of extract_fields, marching cubes (count + read-back +
emit) and component removal; the per-kernel times of one separate torch.profiler run; bytes each kernel needs, computed from shapes
and counts, against 3.35 TB/s (the H100 SXM data-sheet HBM3 rate); and the CPU time of the numpy oracle (tests/mesh_oracle.py,
labelled as the oracle) where it fits.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from dreamgaussian_b200 import fields, meshing, scene, stage1  # noqa: E402

HBM = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=60).stdout.strip()
    except Exception as e:  # noqa: BLE001
        out = "nvidia-smi unavailable: %s" % e
    return dict(nvidia_smi=out, torch_name=torch.cuda.get_device_name(0))


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(np.min(ts))


class Cloud:
    pass


def cloud_model():
    raw = scene.to_raw_parameters(scene.make_cloud(100000, 0, seed=4, sigma=0.0128))
    g = Cloud()
    g._xyz, g._opacity, g._scaling, g._rotation = (torch.tensor(raw[k], device="cuda") for k in ("xyz", "opacity", "scaling", "rotation"))
    return g


def kernel_times(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "mesh_" in e.name:
            name = e.name.split("(")[0].replace("void ", "").replace("dgr::", "")
            out[name] = out.get(name, 0.0) + e.device_time / 1000.0        # ms
    return out


def model_bytes(res, nv, nf, kv, kf):
    """Bytes each kernel must move at least (inputs read once, outputs written once)."""
    N = res ** 3
    tiles = -(-N // 1024)
    E = max(nv, nf)
    return {
        "mesh_classify_kernel": 4 * N + N + 8 * tiles,                      # occ once, one code byte per point, tile counts
        "mesh_vertices_kernel": 12 * nv + 4 * nv,                           # positions (+ first ids); codes of active tiles only
        "mesh_faces_kernel": 12 * nf,
        "mesh_cc_link_kernel": 12 * nf + 4 * nv,
        "mesh_cc_stats_kernel": 12 * nv + 4 * nf + 24 * nv,
        "mesh_cc_count_kernel": 4 * nv + 4 * nf + E,
        "mesh_cc_vertices_kernel": 12 * kv + E,
        "mesh_cc_faces_kernel": 12 * kf + E,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the whole result as JSON to this path")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--resolutions", default="128,256,512")
    ap.add_argument("--iters", type=int, default=500)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_bench needs a CUDA device")
    import mesh_oracle as O
    result = dict(card=card(), reps=args.reps, models={})
    tr = stage1.Stage1Trainer(stage1.Stage1Config(iters=args.iters))
    tr.train(args.iters)
    models = {"stage1_%d" % args.iters: tr.gaussians, "cloud_100k": cloud_model()}
    result["card_after_training"] = card()
    for mname, g in models.items():
        for res in (int(r) for r in args.resolutions.split(",")):
            nb = max(16, res // 16)                      # extract_fields takes at most 16^3 voxels per block
            occ = fields.extract_fields_of_model(g, res, num_blocks=nb)
            peak = float(occ.max())
            for thr in (1.0, 0.3 * peak):
                v, f = meshing.marching_cubes(occ, thr)
                w = meshing.to_world(v, res, g.center, g.scale)
                vk, fk = meshing.remove_small_components(w, f)
                row = dict(res=res, num_blocks=nb, thr=thr, occ_max=peak, Nv=len(v), Nf=len(f), kept_Nv=len(vk), kept_Nf=len(fk))
                row["extract_fields_ms"] = timed(lambda: fields.extract_fields_of_model(g, res, num_blocks=nb), args.reps)
                row["marching_cubes_ms"] = timed(lambda: meshing.marching_cubes(occ, thr), args.reps)
                row["remove_components_ms"] = timed(lambda: meshing.remove_small_components(w, f), args.reps)
                kt = kernel_times(lambda: (meshing.marching_cubes(occ, thr), meshing.remove_small_components(w, f)))
                need = model_bytes(res, len(v), len(f), len(vk), len(fk))
                row["kernels_ms"] = kt
                row["kernel_bytes"] = need
                row["kernel_share_of_hbm_rate"] = {k: need[k] / HBM / (kt[k] / 1e3) for k in need if kt.get(k)}
                if res <= 256:
                    o = occ.cpu().numpy()
                    t0 = time.perf_counter()
                    O.marching_cubes(o, thr)
                    row["numpy_oracle_marching_cubes_cpu_s"] = time.perf_counter() - t0
                result["models"].setdefault(mname, []).append(row)
                print(mname, json.dumps(row), flush=True)
    if args.out:
        d = os.path.dirname(os.path.abspath(args.out))
        os.makedirs(d, exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
