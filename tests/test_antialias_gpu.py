"""The anti-aliased mode on the GPU: parity of every single-view input combination with the mode's oracles (tests/aa_oracle.py)
under the suite's rule (helpers.both_oracles), the known answer and the resolution property on the product, batched and mixed-size
calls against per-view single-view calls, the *_ex calls with flags 0 against the existing entry points, both host layers, the
deterministic backward, and seeded stage-1 runs."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import aa_oracle
import helpers as h
import test_antialias_cpu as cpu
import trained_scenes as ts

pytestmark = pytest.mark.gpu


def _rs(s, device="cuda"):
    from dreamgaussian_b200.rasterizer import GaussianRasterizationSettings
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device=device)
    return GaussianRasterizationSettings(
        image_height=s["image_height"], image_width=s["image_width"], tanfovx=s["tanfovx"], tanfovy=s["tanfovy"], bg=t(s["bg"]),
        scale_modifier=s["scale_modifier"], viewmatrix=t(s["viewmatrix"]), projmatrix=t(s["projmatrix"]), sh_degree=s["sh_degree"],
        campos=t(s["campos"]), prefiltered=False, debug=False)


def run_cuda(s, i, grads=None, antialiasing=True):
    """helpers.run_cuda with GaussianRasterizer(raster_settings, antialiasing=...)."""
    from diff_gaussian_rasterization import GaussianRasterizer
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda")
    tin = {k: t(v).requires_grad_(grads is not None) for k, v in i.items()}
    means2D = torch.zeros_like(tin["means3D"], requires_grad=grads is not None)
    color, radii, depth, alpha = GaussianRasterizer(_rs(s), antialiasing=antialiasing)(means2D=means2D, **tin)
    out = dict(color=color.detach().cpu().numpy(), depth=depth.detach().cpu().numpy(), alpha=alpha.detach().cpu().numpy(),
               radii=radii.cpu().numpy())
    if grads is not None:
        gC, gD, gA = (t(x) for x in grads)
        ((color * gC).sum() + (alpha * gA).sum() + (depth * gD).sum()).backward()
        out["grads"] = {k: v.grad.detach().cpu().numpy() for k, v in tin.items()} | dict(means2D=means2D.grad.detach().cpu().numpy())
    return out


def run_cuda_raw(s, raw, grads):
    from dreamgaussian_b200.fused import FusedGaussianRasterizer
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda")
    tin = {k: t(raw[k]).requires_grad_(True) for k in h.RAW_KEYS}
    means2D = torch.zeros_like(tin["xyz"], requires_grad=True)
    color, radii, depth, alpha = FusedGaussianRasterizer(_rs(s), antialiasing=True)(
        tin["xyz"], tin["features_dc"], tin["features_rest"], tin["opacity"], tin["scaling"], tin["rotation"], means2D=means2D)
    gC, gD, gA = (t(x) for x in grads)
    ((color * gC).sum() + (alpha * gA).sum() + (depth * gD).sum()).backward()
    g = {k: v.grad.detach().cpu().numpy() for k, v in tin.items()} | dict(means2D=means2D.grad.detach().cpu().numpy())
    return dict(color=color.detach().cpu().numpy(), depth=depth.detach().cpu().numpy(), alpha=alpha.detach().cpu().numpy(),
                radii=radii.cpu().numpy(), grads=g)


def _parity(name, s, i, raw=False, f64=True):
    g = h.upstream_grads(s["image_height"], s["image_width"])
    refs = aa_oracle.oracles(s, i, g, f64=f64, raw=raw)
    if f64:
        # The kernel rounds o_eff in float32 from its own float32 geometry; the float32 oracle is given o_eff rounded from float64.
        # So unlike the default mode the float32 oracle cannot take the kernel's exact alpha >= 1/255 and 0.99 decisions: a pixel
        # within rounding of one (the 128 x 128 cases below have one) is set aside in the float32
        # comparison when the float64 oracle flags it, as its tie pixels are; the float64 comparison still bounds it.
        r32, r64 = refs["f32"], refs["f64"]
        r32["ambig_px"] = r32["ambig_px"] | np.where(r64["ambig_px"] != 0, 4, 0).astype(r32["ambig_px"].dtype)
        r32["ambig_g"] = r32["ambig_g"] | np.where(r64["ambig_g"] != 0, 2, 0).astype(r32["ambig_g"].dtype)
    cu = run_cuda_raw(s, i, g) if raw else run_cuda(s, i, g)
    return h.both_oracles(name, s, i, g, refs=refs, cu=cu)


@pytest.mark.parametrize("deg", [0, 3])
def test_parity_sh_scale_rotation(deg):
    s, i = h.make_case(P=3000, res=128, deg=deg, sigma=0.02, elev=10.0, azim=30.0)
    _parity("aa_deg%d" % deg, s, i)


def test_parity_raw_parameters():
    s, i = h.make_case(P=3000, res=128, deg=3, sigma=0.02, elev=-15.0, azim=80.0)
    _parity("aa_raw", s, ts.raw_of(i), raw=True)


def test_parity_colors_precomp_and_cov3d_precomp():
    s, i = h.make_case(P=3000, res=128, deg=0, sigma=0.02, azim=140.0)
    rng = np.random.default_rng(4)
    col = dict(i, colors_precomp=rng.uniform(0, 1, (3000, 3)).astype(np.float32))
    del col["shs"]
    _parity("aa_colors", s, col)
    q = i["rotations"] / np.linalg.norm(i["rotations"], axis=1, keepdims=True)
    R = aa_oracle.T._quat_to_R(torch.tensor(q, dtype=torch.float64)).numpy()
    M = R * (s["scale_modifier"] * i["scales"].astype(np.float64))[:, None, :]
    S = M @ M.transpose(0, 2, 1)
    cov = dict(means3D=i["means3D"], opacities=i["opacities"], shs=i["shs"],
               cov3D_precomp=np.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1).astype(np.float32))
    _parity("aa_cov3D", s, cov)


def test_parity_scale_modifier_of_the_gui_slider():
    s, i = h.make_case(P=3000, res=256, deg=1, sigma=0.02, scale_modifier=0.3, elev=20.0)
    _parity("aa_scale_modifier_0.3", s, i)


# det0 is formed in float32 from the entries of the 2D covariance before the low-pass, as upstream diff-gaussian-rasterization
# forms it: its relative error is about 3e-8 r^2 for a footprint of aspect ratio r (a0 c0 / det0 ~ r^2 / 4), so the compensation
# of a needle beyond ~100:1 carries a float32 error of 1e-4 and more against the float64 oracle, and that of the constructed
# needles of trained_scenes (1e-3 px across, up to 400 px long) is rounding noise.  The needle case here is the random needles
# and discs up to 30:1 (3e-5); include/dgr_b200.h states the limit.
@pytest.mark.parametrize("regime, kw", [("saturated", {}), ("needles", dict(max_ratio=30.0, constructed=0)), ("frustum_edge", {})])
def test_parity_trained_regimes(regime, kw):
    s, i = getattr(ts, regime)(**kw)
    _parity("aa_" + regime, s, i)


def test_parity_800x800_view():
    s, i = h.make_case(P=20000, res=800, deg=3, sigma=0.01, elev=15.0, azim=40.0)
    _parity("aa_800", s, i, f64=False)


# ---- the known answer and the property the mode exists for, on the product --------------------------------------------------------
def test_known_answer_on_the_product():
    s, i, want, comp, _ = cpu.known_answer_case()
    got = run_cuda(s, i)["alpha"][0, 399, 399]
    assert abs(got - want) < 2e-6 * max(1.0, want) + 1e-6, (got, want)


def test_antialiased_coverage_does_not_depend_on_resolution_on_the_product():
    run = lambda s, i, aa: run_cuda(s, i, antialiasing=aa)
    aa, plain = cpu.mean_alpha(run, True), cpu.mean_alpha(run, False)
    print("mean alpha, anti-aliased:", aa, "default:", plain)
    assert aa.max() / aa.min() - 1 < cpu.AA_SPREAD, aa
    assert plain.max() / plain.min() - 1 > cpu.DEFAULT_SPREAD, plain
    assert np.allclose(aa, cpu.mean_alpha(cpu._oracle_run, True), rtol=1e-4)


# ---- batched calls = per-view single-view calls ------------------------------------------------------------------------------------
def _views_case(sizes, P=4000, deg=3):
    s0, i = h.make_case(P=P, res=sizes[0][0], deg=deg, sigma=0.02)
    from dreamgaussian_b200 import scene
    ss = []
    for v, (H, W) in enumerate(sizes):
        cam = scene.orbit_camera(10.0 * v - 10.0, 35.0 * v, 2.0, W, H)
        ss.append(dict(image_height=H, image_width=W, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=np.array([0.2 * v, 0.5, 1.0], np.float32),
                       scale_modifier=1.0, viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform, sh_degree=deg,
                       campos=cam.camera_center))
    return ss, i


def _close(a, b, what, rtol=1e-5, atol=1e-5):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    scale = max(1.0, float(np.abs(b).max()))
    assert np.abs(a - b).max() <= atol * scale + rtol * np.abs(b).max(), (what, float(np.abs(a - b).max()), scale)


@pytest.mark.parametrize("mixed", [False, True])
def test_batched_antialiased_call_equals_single_view_calls(mixed):
    from dreamgaussian_b200 import rasterizer as R
    from dreamgaussian_b200.fused import DensifyStats, rasterize_views_mixed_raw, FusedGaussianRasterizer
    sizes = [(128, 128), (96, 160), (128, 128)] if mixed else [(128, 128)] * 3
    ss, i = _views_case(sizes)
    raw = ts.raw_of(i)
    V, P = len(ss), len(i["means3D"])
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda")
    gens = [h.upstream_grads(H, W, seed=10 + v) for v, (H, W) in enumerate(sizes)]
    # per view, single-view fused calls; gradients summed, statistics of views 1 and 2 in view order
    sums, m2d, stats1 = None, [], DensifyStats(P, "cuda")
    imgs = []
    for v, s in enumerate(ss):
        tin = {k: t(raw[k]).requires_grad_(True) for k in h.RAW_KEYS}
        means2D = torch.zeros((P, 3), device="cuda", requires_grad=True)
        c, r, d, a = FusedGaussianRasterizer(_rs(s), antialiasing=True)(tin["xyz"], tin["features_dc"], tin["features_rest"], tin["opacity"],
                                                                         tin["scaling"], tin["rotation"], means2D=means2D,
                                                                         stats=stats1 if (mixed and v > 0) else None)
        gC, gD, gA = (t(x) for x in gens[v])
        ((c * gC).sum() + (d * gD).sum() + (a * gA).sum()).backward()
        imgs.append((c.detach().cpu().numpy(), r.cpu().numpy()))
        gv = {k: tin[k].grad.cpu().numpy() for k in h.RAW_KEYS}
        sums = gv if sums is None else {k: sums[k] + gv[k] for k in gv}
        m2d.append(means2D.grad.cpu().numpy())
    tin = {k: t(raw[k]).requires_grad_(True) for k in h.RAW_KEYS}
    means2D = torch.zeros((V, P, 3), device="cuda", requires_grad=True)
    settings = [_rs(s) for s in ss]
    stats2 = DensifyStats(P, "cuda")
    if mixed:
        colors, radii, depths, alphas = rasterize_views_mixed_raw(settings, tin["xyz"], means2D, tin["features_dc"], tin["features_rest"],
                                                                  tin["opacity"], tin["scaling"], tin["rotation"], stats=stats2,
                                                                  stats_views=(1, 2), antialiasing=True)
    else:
        from dreamgaussian_b200.fused import rasterize_views_raw
        c, radii, d, a = rasterize_views_raw(settings, tin["xyz"], means2D, tin["features_dc"], tin["features_rest"], tin["opacity"],
                                             tin["scaling"], tin["rotation"], antialiasing=True)
        colors, depths, alphas = list(c), list(d), list(a)
    loss = 0
    for v in range(V):
        gC, gD, gA = (t(x) for x in gens[v])
        loss = loss + (colors[v] * gC).sum() + (depths[v].reshape(gD.shape) * gD).sum() + (alphas[v].reshape(gA.shape) * gA).sum()
    loss.backward()
    for v in range(V):
        _close(colors[v].detach().cpu().numpy(), imgs[v][0], "color %d" % v)
        assert np.array_equal(radii[v].cpu().numpy(), imgs[v][1])
        _close(means2D.grad[v].cpu().numpy(), m2d[v], "means2D %d" % v, rtol=1e-4, atol=1e-6)
    for k in h.RAW_KEYS:
        _close(tin[k].grad.cpu().numpy(), sums[k], k, rtol=1e-4, atol=1e-6)
    if mixed:
        for a_, b_ in zip(stats2.as_tuple(), stats1.as_tuple()):
            _close(a_.cpu().numpy(), b_.cpu().numpy(), "stats", rtol=1e-4, atol=1e-6)


# ---- flags 0 = the existing entry points; both host layers; the deterministic backward -----------------------------------------------
def test_ex_with_flags_0_is_bit_identical_to_the_existing_preprocess():
    from dreamgaussian_b200 import _lib
    lib = _lib.load()
    s, i = h.make_case(P=5000, res=128, deg=3, sigma=0.02)
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda").contiguous()
    tin = {k: t(v) for k, v in i.items()}
    cam = {k: t(s[k]) for k in ("bg", "viewmatrix", "projmatrix", "campos")}
    p = lambda x: ctypes.c_void_p(x.data_ptr())
    st = _lib.DgrSettings(128, 128, s["tanfovx"], s["tanfovy"], 1.0, 3, 0, 0, p(cam["bg"]), p(cam["viewmatrix"]), p(cam["projmatrix"]), p(cam["campos"]))
    g = _lib.DgrGaussians(5000, 16, p(tin["means3D"]), p(tin["shs"]), None, p(tin["opacities"]), p(tin["scales"]), p(tin["rotations"]), None, None, 0)
    outs = []
    for opt in (None, "null", 0):
        geom = torch.zeros(lib.dgr_geom_bytes(5000, 128, 128), dtype=torch.uint8, device="cuda")
        image = torch.zeros(lib.dgr_image_bytes(128, 128), dtype=torch.uint8, device="cuda")
        radii = torch.zeros(5000, dtype=torch.int32, device="cuda")
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        if opt is None:
            _lib.check(lib.dgr_forward_preprocess(ctypes.byref(st), ctypes.byref(g), p(geom), p(image), p(radii), stream))
        else:
            o = None if opt == "null" else ctypes.byref(_lib.DgrRasterOptions(0))
            _lib.check(lib.dgr_forward_preprocess_ex(ctypes.byref(st), ctypes.byref(g), p(geom), p(image), p(radii), o, stream))
        torch.cuda.synchronize()
        L = 256 + 5000 * 48                                        # header + records (the run matrix holds atomics' order)
        outs.append((geom[:L].cpu().numpy(), radii.cpu().numpy()))
    for o in outs[1:]:
        assert np.array_equal(o[0], outs[0][0]) and np.array_equal(o[1], outs[0][1])


def test_ex_with_flags_0_is_bit_identical_to_the_existing_calls_end_to_end():
    """The default mode through the public API (which calls the *_ex entries with flags 0) against a forward + backward through
    the existing entry points: images, radii and, under the deterministic flag, gradients bit-identical."""
    from dreamgaussian_b200 import _lib, rasterizer as R
    s, i = h.make_case(P=5000, res=128, deg=3, sigma=0.02, elev=5.0)
    g = h.upstream_grads(128, 128)
    torch.use_deterministic_algorithms(True)
    try:
        new = h.run_tuned(h.DEFAULT_TUNING, lambda: run_cuda(s, i, g, antialiasing=False), fast_host=False)
        lib = _lib.load()
        names = ("dgr_forward_preprocess_ex", "dgr_backward_det_ex")
        saved = {n: getattr(lib, n) for n in names}
        # the ctypes layer with its *_ex calls routed to the existing entry points (the options argument dropped)
        lib.dgr_forward_preprocess_ex = lambda *a: saved_old["pre"](*a[:-2], a[-1])
        lib.dgr_backward_det_ex = lambda *a: saved_old["det"](*a[:-2], a[-1])
        saved_old = {"pre": lib.dgr_forward_preprocess, "det": lib.dgr_backward_det}
        try:
            old = h.run_tuned(h.DEFAULT_TUNING, lambda: run_cuda(s, i, g, antialiasing=False), fast_host=False)
        finally:
            for n, f in saved.items():
                setattr(lib, n, f)
    finally:
        torch.use_deterministic_algorithms(False)
    for k in ("color", "depth", "alpha", "radii"):
        assert np.array_equal(new[k], old[k]), k
    for k in new["grads"]:
        assert np.array_equal(new["grads"][k], old["grads"][k]), k


def test_both_host_layers_agree():
    s, i = h.make_case(P=4000, res=128, deg=3, sigma=0.02, azim=60.0)
    g = h.upstream_grads(128, 128)
    torch.use_deterministic_algorithms(True)
    try:
        fast = h.run_tuned(h.DEFAULT_TUNING, lambda: run_cuda(s, i, g), fast_host=True)
        slow = h.run_tuned(h.DEFAULT_TUNING, lambda: run_cuda(s, i, g), fast_host=False)
    finally:
        torch.use_deterministic_algorithms(False)
    for k in ("color", "depth", "alpha", "radii"):
        assert np.array_equal(fast[k], slow[k]), k
    for k in fast["grads"]:
        assert np.array_equal(fast["grads"][k], slow["grads"][k]), k
    plain = run_cuda(s, i, g, antialiasing=False)
    assert not np.array_equal(plain["color"], fast["color"])           # the switch does reach the kernels


def test_deterministic_antialiased_backward_is_bit_identical_and_matches_the_default_one():
    s, i = h.make_case(P=6000, res=192, deg=3, sigma=0.02, elev=-5.0)
    g = h.upstream_grads(192, 192)
    ref = run_cuda(s, i, g)
    torch.use_deterministic_algorithms(True)
    try:
        runs = [run_cuda(s, i, g) for _ in range(3)]
        runs.append(h.run_tuned((1, 2, 1 | (1 << 21)), lambda: run_cuda(s, i, g)))
    finally:
        torch.use_deterministic_algorithms(False)
    for r in runs[1:]:
        for k in r["grads"]:
            assert np.array_equal(r["grads"][k], runs[0]["grads"][k]), k
    for k in ref["grads"]:
        _close(runs[0]["grads"][k], ref["grads"][k], k, rtol=1e-4, atol=1e-6)


def test_debug_backward_refuses_a_forward_of_the_other_mode():
    from dreamgaussian_b200 import rasterizer as R
    s, i = h.make_case(P=500, res=64, deg=0, sigma=0.03)
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda")
    rs = _rs(s)._replace(debug=True)
    tin = {k: t(v) for k, v in i.items()}
    for fast in (True, False):
        R.set_fast_host(fast)
        try:
            color, radii, depth, alpha, state = R.forward_impl(rs, tin["means3D"], tin["shs"], None, tin["opacities"], tin["scales"],
                                                               tin["rotations"], None, antialiasing=True)
            if state.fast is None:
                state.antialiasing = False                                # the backward of the other mode
                outs = [torch.empty((500, 3), device="cuda") for _ in range(2)]
                with pytest.raises(RuntimeError, match="differ from those of the forward"):
                    R.backward_impl(state, t(np.ones((3, 64, 64))), None, None, outs[0], outs[1], None, None,
                                    torch.empty((500, 1), device="cuda"), None, None, None)
        finally:
            R.set_fast_host(True)


# ---- stage 1 -----------------------------------------------------------------------------------------------------------------------
STAGE1 = r"""
import sys, numpy as np, torch
if sys.argv[3] == "det":
    torch.use_deterministic_algorithms(True)
from dreamgaussian_b200 import stage1
cfg = stage1.Stage1Config(iters=120, num_pts=1500, ref_size=96, density_start_iter=20, densification_interval=50, seed=5,
                          antialiasing=sys.argv[2] == "aa")
t = stage1.Stage1Trainer(cfg, fused=True)
t.train(120)
m = t.gaussians
out = {"n": np.array([m.num_points]), "losses": np.array([float(x) for x in t.losses])}
for k in stage1.GROUPS:
    out["p_" + k] = m.p[k].detach().cpu().numpy()
np.savez(sys.argv[1], **out)
"""


def _stage1(tmp_path, tag, mode, det):
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8", PYTHONPATH=h.ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    path = str(tmp_path / (tag + ".npz"))
    p = subprocess.run([sys.executable, "-c", STAGE1, path, mode, "det" if det else "-"], env=env, cwd=h.ROOT, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=1200)
    assert p.returncode == 0, p.stdout[-4000:]
    return dict(np.load(path))


def test_seeded_antialiased_stage1_runs(tmp_path):
    a1 = _stage1(tmp_path, "aa1", "aa", det=True)
    a2 = _stage1(tmp_path, "aa2", "aa", det=True)
    d = _stage1(tmp_path, "default", "default", det=True)
    assert np.isfinite(a1["losses"]).all() and int(a1["n"][0]) != 1500            # finite, and the densifications ran
    for k in a1:
        assert np.array_equal(a1[k], a2[k]), k                                   # bit-identical under the deterministic flag
    assert not np.array_equal(a1["losses"], d["losses"])                         # the mode changes the run
