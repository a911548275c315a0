"""The reference's OWN caller on the drop-in packages of this repo (SURVEY.md §8 row A0), replayed from a recording.

`gs_renderer.Renderer.initialize` -> `GaussianModel.create_from_pcd` -> `simple_knn._C.distCUDA2` (gs_renderer.py:689-715,
331-354) and `Renderer.render` (gs_renderer.py:717-822: transposed float64 `viewmatrix` of MiniCam :662, the retain_grad dummy
`means2D` :727-739, `clamp(0, 1)` :811) were run as they are, with `diff_gaussian_rasterization` / `simple_knn._C` resolving to
THIS repo, by tests/golden/make_golden_reference_gpu.py; tests/golden/reference_caller.npz holds the camera that caller built and
seeded samples + sums of the parameters it handed to the op and of everything it got back.  Here the same call is made again:
the parameters are regenerated from the caller's seed and must equal the recorded ones exactly, the results must match the
recorded ones, and everything is compared with the CPU oracle fed the same tensors.
"""
import math
import os
import types

import numpy as np
import pytest
import torch

import helpers as h

pytestmark = pytest.mark.gpu
SH_C0 = 0.28209479177387814


def _training_args():
    # configs/image.yaml:67-75 of the reference
    return types.SimpleNamespace(position_lr_init=0.001, position_lr_final=0.00002, position_lr_delay_mult=0.02,
                                 position_lr_max_steps=500, feature_lr=0.01, opacity_lr=0.05, scaling_lr=0.005,
                                 rotation_lr=0.005, percent_dense=0.01)


CASES = {
    # BASELINE.json configs[0]: what `python main.py --config configs/image.yaml` renders first (image.yaml:65-66, 12, 41-44)
    "image_yaml_init": dict(sh_degree=0, num_pts=5000, W=256, H=256, elev=0.0, azim=0.0, scaling_modifier=1.0, bg=None, ups=0),
    # SH degree 3 active, non-square image, scaling modifier, explicit background, perturbed parameters
    "deg3_perturbed": dict(sh_degree=3, num_pts=20000, W=320, H=200, elev=-20.0, azim=130.0, scaling_modifier=1.15,
                           bg=(0.1, 0.4, 0.7), ups=3),
}


def perturb(features_rest, scaling, rotation, opacity):
    """Leave the symmetric initial state: anisotropy, rotations, colour detail (torch's CUDA generator, seed 7)."""
    with torch.no_grad():
        features_rest.normal_(0.0, 0.1)
        scaling.add_(0.3 * torch.randn_like(scaling))
        rotation.copy_(torch.randn_like(rotation))
        opacity.copy_(torch.logit(torch.rand_like(opacity) * 0.9 + 0.05))


def summarize(t, n=4096, stride=8):
    """What the recording keeps of a tensor: a fixed, seeded sample of its elements, their sum and the sum of magnitudes."""
    a = t.detach().reshape(-1).cpu().numpy()
    idx = np.sort(np.random.default_rng(a.size).choice(a.size, size=min(n, a.size), replace=False))[::stride]
    a64 = a.astype(np.float64)
    return {"sample": a[idx], "sum": a64.sum(), "abs": np.abs(a64).sum()}


def _gold(name):
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_caller.npz"))
    return {k[len(name) + 1:]: g[k] for k in g.files if k.startswith(name + "/")}


def _replay(c, gold):
    """The caller's call, made again: the initial cloud from numpy's legacy generator with its seed (a uniform ball of radius
    0.5, colours SH2RGB(U/255)), create_from_pcd's parameters, the test's perturbation, the recorded camera, render()."""
    import diff_gaussian_rasterization as ours
    from simple_knn._C import distCUDA2
    np.random.seed(7)
    torch.manual_seed(7)
    n = c["num_pts"]
    phis = np.random.random((n,)) * 2 * np.pi
    thetas = np.arccos(np.random.random((n,)) * 2 - 1)
    radius = 0.5 * np.cbrt(np.random.random((n,)))
    xyz = np.stack((radius * np.sin(thetas) * np.cos(phis), radius * np.sin(thetas) * np.sin(phis), radius * np.cos(thetas)), axis=1)
    colors = np.random.random((n, 3)) / 255.0 * SH_C0 + 0.5
    M = (c["sh_degree"] + 1) ** 2
    pts = torch.tensor(xyz).float().cuda()
    feats = torch.zeros((n, 3, M), device="cuda")
    feats[:, :3, 0] = (torch.tensor(colors).float().cuda() - 0.5) / SH_C0
    dist2 = torch.clamp_min(distCUDA2(pts), 0.0000001)
    op0 = 0.1 * torch.ones((n, 1), dtype=torch.float, device="cuda")
    rot = torch.zeros((n, 4), device="cuda")
    rot[:, 0] = 1
    p = dict(xyz=pts, features_dc=feats[:, :, 0:1].transpose(1, 2).contiguous(), features_rest=feats[:, :, 1:].transpose(1, 2).contiguous(),
             opacity=torch.log(op0 / (1 - op0)), scaling=torch.log(torch.sqrt(dist2))[..., None].repeat(1, 3), rotation=rot)
    p = {k: v.requires_grad_(True) for k, v in p.items()}
    if c["ups"]:
        perturb(p["features_rest"], p["scaling"], p["rotation"], p["opacity"])

    H, W = c["H"], c["W"]
    view = torch.tensor(gold["w2c"]).transpose(0, 1).cuda()
    proj, campos, bg = (torch.tensor(gold[k]).cuda() for k in ("full_proj", "campos", "bg"))
    fovx, fovy = (float(v) for v in gold["fov"])
    screen = torch.zeros_like(p["xyz"], requires_grad=True) + 0
    screen.retain_grad()
    rs = ours.GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=math.tan(fovx * 0.5), tanfovy=math.tan(fovy * 0.5),
                                            bg=bg, scale_modifier=c["scaling_modifier"], viewmatrix=view, projmatrix=proj,
                                            sh_degree=int(gold["active_sh_degree"]), campos=campos, prefiltered=False, debug=False)
    img, radii, depth, alpha = ours.GaussianRasterizer(raster_settings=rs)(
        means3D=p["xyz"], means2D=screen, shs=torch.cat((p["features_dc"], p["features_rest"]), dim=1), colors_precomp=None,
        opacities=torch.sigmoid(p["opacity"]), scales=torch.exp(p["scaling"]), rotations=torch.nn.functional.normalize(p["rotation"]),
        cov3D_precomp=None)
    image = img.clamp(0, 1)
    gC, gD, gA = h.upstream_grads(H, W, seed=5, depth=False)
    t = lambda a: torch.tensor(a, device="cuda")
    ((image * t(gC)).sum() + (alpha * t(gA)).sum()).backward()
    vis = radii > 0
    accum, denom = torch.zeros((n, 1), device="cuda"), torch.zeros((n, 1), device="cuda")
    accum[vis] += torch.norm(screen.grad[vis, :2], dim=-1, keepdim=True)
    denom[vis] += 1
    rec = {"in_" + k: v.detach() for k, v in p.items()}
    rec.update({"grad_" + k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in p.items()})
    rec.update(out_image=image.detach(), out_alpha=alpha.detach(), out_depth=depth.detach(), out_radii=radii, grad_means2D=screen.grad,
               stat_xyz_gradient_accum=accum, stat_denom=denom)
    return p, rs, img.detach(), rec, (gC, gA)


@pytest.mark.parametrize("name", list(CASES))
def test_recorded_reference_call_on_the_drop_in(name):
    c = CASES[name]
    gold = _gold(name)
    p, rs, pre, rec, (gC, gA) = _replay(c, gold)
    H, W = c["H"], c["W"]
    assert rec["out_image"].shape == (3, H, W) and rec["out_alpha"].shape == (1, H, W) and rec["out_depth"].shape == (1, H, W)
    assert rec["out_radii"].dtype == torch.int32

    # ---- the recording: the same parameters exactly, the same results.  The backward adds its float32 terms in a different
    # order each run, so a gradient differs by rounding relative to the largest gradient of the case (the rotation gradient of
    # the isotropic initial cloud is zero up to exactly that noise)
    gscale = max(float(np.abs(gold[k]).max(initial=0.0)) for k in gold if k.startswith(("grad_", "stat_")) and k.endswith("/sample"))
    for k, v in rec.items():
        s = summarize(v)
        want = {q: gold["%s/%s" % (k, q)] for q in s}
        if k.startswith("in_"):
            assert np.array_equal(s["sample"], want["sample"]) and s["sum"] == want["sum"], k
            continue
        scale = max(float(np.abs(want["sample"]).max(initial=0.0)), gscale if k.startswith(("grad_", "stat_")) else 0.0, 1e-30)
        np.testing.assert_allclose(s["sample"], want["sample"], rtol=1e-4, atol=1e-5 * scale, err_msg=k)
        # a sum of n such roundings grows like sqrt(n) times one of them
        np.testing.assert_allclose(s["sum"], want["sum"], rtol=1e-4, atol=1e-5 * (float(want["abs"]) + scale * math.sqrt(v.numel())),
                                   err_msg=k)

    # ---- the oracle on the very tensors the caller handed to the op
    f64 = lambda x: x.detach().double().cpu().numpy()
    settings = dict(image_height=H, image_width=W, tanfovx=rs.tanfovx, tanfovy=rs.tanfovy, bg=f64(rs.bg), scale_modifier=c["scaling_modifier"],
                    viewmatrix=f64(rs.viewmatrix), projmatrix=f64(rs.projmatrix), sh_degree=rs.sh_degree, campos=f64(rs.campos))
    raw = {k: f64(v) for k, v in p.items()}
    # clamp(0, 1) of the caller: gradient passes where the un-clamped colour lies in [0, 1] (torch's rule)
    passes = ((pre >= 0) & (pre <= 1)).cpu().numpy()
    ref = h.run_oracle_raw(settings, raw, (gC * passes, None, gA))
    cu = dict(color=pre.cpu().numpy(), depth=rec["out_depth"].cpu().numpy(), alpha=rec["out_alpha"].cpu().numpy(),
              radii=rec["out_radii"].cpu().numpy(), grads={k: rec["grad_" + k].cpu().numpy() for k in p})
    cu["grads"]["means2D"] = rec["grad_means2D"].cpu().numpy()
    ok, rep = h.compare(cu, ref, max_ambig_frac=0.10)
    assert ok, rep
    assert int((rec["out_radii"] > 0).sum()) > c["num_pts"] // 2

    # densification statistics as the caller's add_densification_stats computes them from OUR viewspace gradient
    vis = ref["radii"] > 0
    want = np.linalg.norm(ref["grads"]["means2D"][:, :2], axis=-1)
    got = rec["stat_xyz_gradient_accum"][:, 0].cpu().numpy()
    clean = (ref["ambig_g"] == 0) & vis
    assert np.abs(got[clean] - want[clean]).max() <= 1e-3 * max(want.max(), 1e-12)
    assert np.array_equal(rec["stat_denom"][:, 0].cpu().numpy()[ref["ambig_g"] == 0], vis[ref["ambig_g"] == 0].astype(np.float32))
