"""Golden vectors for the two GPU tests that compare with the reference's own code, made by RUNNING that code on a GPU:

  * reference_knn.npz: the reference's simple_knn.cu (oracle/_ref/libsimple_knn_ref.so, compiled unmodified by
    `make -C oracle ref`) on the clouds of tests/test_knn_gpu.py -- a fixed, seeded sample of every output plus its float64
    sum over all points;
  * reference_caller.npz: the reference's own caller (gs_renderer.Renderer.initialize / render, loaded by oracle/ref_caller.py)
    on this repository's drop-in packages for the cases of tests/test_reference_caller_gpu.py -- the camera it built, seeded
    samples and float64 sums of the parameters it handed to the rasterizer, and of everything it got back.

Needs a CUDA device and oracle/_ref (built by __graft_entry__.build() where the reference sources exist).
Usage: python tests/golden/make_golden_reference_gpu.py [OUT_DIR]   (default: tests/golden)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]

import helpers as h  # noqa: E402
import test_knn_gpu as tk  # noqa: E402
import test_reference_caller_gpu as tc  # noqa: E402
from oracle import knn_oracle, ref_caller  # noqa: E402


def knn(out_dir):
    out = {}
    for kind, P in tk.REF_CASES:
        p = tk._cloud(kind, P)
        ref = knn_oracle.reference_dist_cuda2(torch.tensor(p, device="cuda")).cpu().numpy()
        idx = tk.sample_index(P)
        out["%s_%d_idx" % (kind, P)] = idx
        out["%s_%d_val" % (kind, P)] = ref[idx]
        out["%s_%d_sum" % (kind, P)] = np.float64(ref.astype(np.float64).sum())
    np.savez_compressed(os.path.join(out_dir, "reference_knn.npz"), **out)


def caller(out_dir):
    cam_utils, gs, _sh = ref_caller.load()
    out = {}
    for name, c in tc.CASES.items():
        np.random.seed(7)
        torch.manual_seed(7)
        r = gs.Renderer(sh_degree=c["sh_degree"])
        r.initialize(num_pts=c["num_pts"])
        gm = r.gaussians
        gm.training_setup(tc._training_args())
        for _ in range(c["ups"]):
            gm.oneupSHdegree()
        if c["ups"]:
            tc.perturb(gm._features_rest, gm._scaling, gm._rotation, gm._opacity)
        oc = cam_utils.OrbitCamera(c["W"], c["H"], r=2, fovy=49.1)
        cam = gs.MiniCam(cam_utils.orbit_camera(c["elev"], c["azim"], 2), c["W"], c["H"], oc.fovy, oc.fovx, oc.near, oc.far)
        bg = None if c["bg"] is None else torch.tensor(c["bg"], dtype=torch.float32, device="cuda")
        res = r.render(cam, scaling_modifier=c["scaling_modifier"], bg_color=bg)
        gC, gD, gA = h.upstream_grads(c["H"], c["W"], seed=5, depth=False)
        t = lambda a: torch.tensor(a, device="cuda")
        ((res["image"] * t(gC)).sum() + (res["alpha"] * t(gA)).sum()).backward()
        gm.add_densification_stats(res["viewspace_points"], res["visibility_filter"])
        rec = dict(
            # the camera as the caller built it: MiniCam's world-to-camera matrix (world_view_transform is its transpose)
            w2c=cam.world_view_transform.transpose(0, 1).cpu().numpy(), full_proj=cam.full_proj_transform.cpu().numpy(),
            campos=cam.camera_center.cpu().numpy(), fov=np.array([cam.FoVx, cam.FoVy]),
            bg=(r.bg_color if bg is None else bg).cpu().numpy(), active_sh_degree=np.int32(gm.active_sh_degree))
        tensors = dict(xyz=gm._xyz, features_dc=gm._features_dc, features_rest=gm._features_rest, opacity=gm._opacity,
                       scaling=gm._scaling, rotation=gm._rotation)
        for k, v in tensors.items():
            rec["in_" + k] = v.detach()
            rec["grad_" + k] = v.grad if v.grad is not None else torch.zeros_like(v)
        rec.update(out_image=res["image"].detach(), out_alpha=res["alpha"].detach(), out_depth=res["depth"].detach(),
                   out_radii=res["radii"], grad_means2D=res["viewspace_points"].grad,
                   stat_xyz_gradient_accum=gm.xyz_gradient_accum, stat_denom=gm.denom)
        for k, v in rec.items():
            if isinstance(v, torch.Tensor):
                out.update({"%s/%s/%s" % (name, k, s): a for s, a in tc.summarize(v).items()})
            else:
                out["%s/%s" % (name, k)] = v
    np.savez_compressed(os.path.join(out_dir, "reference_caller.npz"), **out)


if __name__ == "__main__":
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    os.makedirs(out_dir, exist_ok=True)
    knn(out_dir)
    caller(out_dir)
    print("wrote", out_dir)
