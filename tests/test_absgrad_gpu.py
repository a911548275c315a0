"""The absolute-gradient densification statistic (DGR_RASTER_ABS_GRAD; AbsGS) on the GPU: parity with both builds of the C oracle,
the triangle inequality, gradient collision, what the bit leaves unchanged, bit-reproducibility under the deterministic flag, and
the stage-1 densification rule."""
import numpy as np
import pytest
import torch

import absgrad_oracle as AO
import aa_oracle
import helpers
import trained_scenes as TS
from dreamgaussian_b200 import _lib, stage1
from dreamgaussian_b200 import rasterizer as R
from dreamgaussian_b200.fused import DensifyStats, FusedGaussianRasterizer, rasterize_views_mixed_raw
from dreamgaussian_b200.rasterizer import GaussianRasterizationSettings
from oracle import c_oracle

pytestmark = pytest.mark.gpu
KEYS = helpers.RAW_KEYS


def _rs(settings):
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda")
    return GaussianRasterizationSettings(
        image_height=settings["image_height"], image_width=settings["image_width"], tanfovx=settings["tanfovx"],
        tanfovy=settings["tanfovy"], bg=t(settings["bg"]), scale_modifier=settings["scale_modifier"],
        viewmatrix=t(settings["viewmatrix"]), projmatrix=t(settings["projmatrix"]), sh_degree=settings["sh_degree"],
        campos=t(settings["campos"]), prefiltered=False, debug=False)


def render(settings, raw, grads, absgrad=True, antialiasing=False, camera=False):
    """One fused render + backward with fresh statistics -> dict of numpy: stats, grads (and camera grads); launches of the backward."""
    rs = _rs(settings)
    if camera:
        rs = rs._replace(viewmatrix=rs.viewmatrix.clone().requires_grad_(True))
    tin = {k: torch.tensor(np.asarray(raw[k], np.float32), device="cuda").requires_grad_(True) for k in KEYS}
    P = tin["xyz"].shape[0]
    st = DensifyStats(P, "cuda", absgrad=absgrad)
    means2D = torch.zeros_like(tin["xyz"], requires_grad=True)
    color, radii, depth, alpha = FusedGaussianRasterizer(rs, antialiasing)(tin["xyz"], tin["features_dc"], tin["features_rest"], tin["opacity"],
                                                                           tin["scaling"], tin["rotation"], means2D=means2D, stats=st)
    gC, gD, gA = (torch.tensor(np.asarray(x, np.float32), device="cuda") if x is not None else None for x in grads)
    loss = (color * gC).sum() + (alpha * gA).sum() + ((depth * gD).sum() if gD is not None else 0.0)
    loss.backward()
    torch.cuda.synchronize()
    out = dict(radii=radii.cpu().numpy(), stats={k: (v.cpu().numpy() if v is not None else None) for k, v in vars(st).items()},
               grads={k: v.grad.cpu().numpy() for k, v in tin.items() if v.grad is not None})
    out["grads"]["means2D"] = means2D.grad.cpu().numpy()
    if camera:
        out["camera"] = rs.viewmatrix.grad.cpu().numpy()
    return out


def activated(raw, settings=None, antialiasing=False):
    """The activated inputs of the C oracle (float64), with the anti-aliased mode's o_eff when asked."""
    t = {k: torch.tensor(np.asarray(raw[k], np.float64)) for k in KEYS}
    act = dict(means3D=t["xyz"], shs=torch.cat((t["features_dc"], t["features_rest"]), dim=1), opacities=torch.sigmoid(t["opacity"]),
               scales=torch.exp(t["scaling"]), rotations=torch.nn.functional.normalize(t["rotation"]))
    if antialiasing:
        act["opacities"] = act["opacities"] * aa_oracle.comp(settings, act["means3D"], act["scales"], act["rotations"]).reshape(-1, 1)
    return {k: v.numpy() for k, v in act.items()}


def oracle_stat(settings, act, grads, dtype):
    """-> (abs statistic [P], default statistic [P], decision-ambiguity flags [P], radii) of the C oracle's build `dtype`."""
    r = c_oracle.forward(**settings, **act, dtype=dtype)
    a, d = AO.stat(AO.c_terms(r, *grads), r.radii, r.H, r.W)
    _, ag, _ = r.flags()
    radii = r.radii.copy()
    r.close()
    return a, d, ag, radii


def check_rule(cu, ref, flags, name, f32=False):
    """The gradient rule of helpers.compare (f64) / compare_f32 (f32), applied to one per-Gaussian statistic."""
    clean = (flags == 0) if not f32 else ((flags & (2 | 16)) == 0)
    scale = max(float(np.abs(ref).max()), 1e-30)
    e = (np.abs(cu.astype(np.float64) - ref) - helpers.GRAD_RTOL * np.abs(ref)) / scale
    e = e[clean]
    worst, p999 = float(e.max()), float(np.percentile(e, 99.9))
    helpers.report(name, abs_stat=dict(worst=worst, p999=p999, clean=int(clean.sum())))
    if f32:
        assert p999 <= helpers.F32_GRAD_ATOL and worst <= helpers.F32_GRAD_OUTLIER_ATOL, (name, worst, p999)
    else:
        assert p999 <= helpers.GRAD_ATOL and worst <= helpers.GRAD_ATOL_MAX, (name, worst, p999)


def parity(name, settings, inputs, grads=None, antialiasing=False, f64=True, det=False, f32=True):
    raw = TS.raw_of(inputs)
    H, W = settings["image_height"], settings["image_width"]
    grads = grads or helpers.upstream_grads(H, W)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        cu = render(settings, raw, grads, antialiasing=antialiasing)
    finally:
        torch.use_deterministic_algorithms(prev)
    act = activated(raw, settings, antialiasing)
    a_cu, d_cu = cu["stats"]["xyz_gradient_accum_abs"], cu["stats"]["xyz_gradient_accum"]
    # the triangle inequality, per Gaussian; where the summed gradient cancels to float32 noise (needles: the moments' cancellation in
    # preprocess_bwd), the default statistic is held to the gradient rule's 1e-3 of its scale instead
    below = a_cu < d_cu * (1 - 1e-5)
    helpers.report(name + " triangle", below=dict(n=int(below.sum()), worst=float((d_cu - a_cu)[below].max() / d_cu.max()) if below.any() else 0.0))
    assert np.all((d_cu - a_cu)[below] <= helpers.GRAD_ATOL_MAX * d_cu.max()), name
    for dt in (np.float32,) * f32 + (np.float64,) * f64:
        a, d, flags, radii = oracle_stat(settings, act, grads, dt)
        assert (radii > 0).sum() > 10
        check_rule(a_cu, a, flags, "%s abs %s" % (name, np.dtype(dt).name), f32=dt is np.float32)
    return cu


@pytest.mark.parametrize("deg", [0, 3])
def test_parity_single_view(deg):
    s, i = helpers.make_case(P=3000, res=128, deg=deg, sigma=0.03, elev=15.0, azim=40.0)
    parity("deg%d" % deg, s, i)


@pytest.mark.parametrize("regime", ["saturated", "needles", "faint", "subpixel"])
def test_parity_trained_regimes(regime):
    # needles: the statistic is a sum of |A dx + B dy| per pixel, whose float32 cancellation grows with the square of the aspect ratio;
    # the float32 oracle forms each conic with its own rounding, so needles are held to the float64 build (unflagged Gaussians) only
    s, i = getattr(TS, regime)()
    parity(regime, s, i, f32=regime != "needles")


def test_parity_large_view():
    s, i = helpers.make_case(P=100000, res=800, deg=3, sigma=0.02)
    parity("100k/800", s, i, f64=False)


def test_parity_antialiased():
    s, i = helpers.make_case(P=3000, res=128, deg=1, sigma=0.02, elev=10.0)
    parity("aa", s, i, antialiasing=True)


def test_parity_deterministic():
    s, i = helpers.make_case(P=3000, res=128, deg=1, sigma=0.03, elev=-20.0, azim=100.0)
    parity("det", s, i, det=True)


def test_mixed_three_views_two_selected():
    sizes = [(96, 128), (64, 64), (128, 80)]
    base, inputs = helpers.make_case(P=2000, res=64, deg=1, sigma=0.03)
    raw = TS.raw_of(inputs)
    settings = [helpers.make_case(P=1, res=64, deg=1, elev=10.0 * v, azim=50.0 * v, width=w, height=h)[0] for v, (h, w) in enumerate(sizes)]
    grads = [helpers.upstream_grads(h, w, seed=7 + v) for v, (h, w) in enumerate(sizes)]
    tin = {k: torch.tensor(np.asarray(raw[k], np.float32), device="cuda").requires_grad_(True) for k in KEYS}
    P = tin["xyz"].shape[0]
    st = DensifyStats(P, "cuda", absgrad=True)
    colors, radii, depths, alphas = rasterize_views_mixed_raw([_rs(x) for x in settings], tin["xyz"], None, tin["features_dc"], tin["features_rest"],
                                                              tin["opacity"], tin["scaling"], tin["rotation"], stats=st, stats_views=(0, 2))
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda")
    loss = sum((colors[v] * t(g[0])).sum() + (depths[v] * t(g[1])).sum() + (alphas[v] * t(g[2])).sum() for v, g in enumerate(grads))
    loss.backward()
    a_cu = st.xyz_gradient_accum_abs.cpu().numpy()
    act = activated(raw)
    for dt in (np.float32, np.float64):
        total, flags = np.zeros(P), np.zeros(P, np.uint8)
        for v in (0, 2):
            a, _, f, _ = oracle_stat(settings[v], act, grads[v], dt)
            total += a
            flags |= f
        check_rule(a_cu, total, flags, "mixed %s" % np.dtype(dt).name, f32=dt is np.float32)
    assert np.all(a_cu >= st.xyz_gradient_accum.cpu().numpy() * (1 - 1e-5))


# ---- constructed scenes: one-pixel Gaussians and gradient collision ----------------------------------------------------------
H = W = 64
TAN = 0.5


def _axis_settings():
    PM = np.zeros((4, 4), np.float32)
    PM[0, 0], PM[1, 1] = 1 / TAN, 1 / TAN
    PM[2, 2], PM[3, 2], PM[2, 3] = 100.0 / 99.99, -100.0 * 0.01 / 99.99, 1.0
    return dict(image_height=H, image_width=W, tanfovx=TAN, tanfovy=TAN, bg=np.zeros(3, np.float32), scale_modifier=1.0,
                viewmatrix=np.eye(4, dtype=np.float32), projmatrix=PM, sh_degree=0, campos=np.zeros(3, np.float32))


def _at_pixel(x, y, z=3.0):
    return [((2 * x + 1) / W - 1) * z * TAN, ((2 * y + 1) / H - 1) * z * TAN, z]


def _raw(xyz, log_scale, logit, rgb):
    n = len(xyz)
    return dict(xyz=np.asarray(xyz, np.float32), features_dc=((np.asarray(rgb, np.float32) - 0.5) / 0.28209479177387814).reshape(n, 1, 3),
                features_rest=np.zeros((n, 0, 3), np.float32), opacity=np.full((n, 1), logit, np.float32),
                scaling=np.full((n, 3), log_scale, np.float32), rotation=np.tile(np.float32([1, 0, 0, 0]), (n, 1)))


def test_one_pixel_gaussians_have_equal_statistics():
    """Opacity 0.008 and a point-like scale (2D variance 0.3 px^2), a quarter pixel off a pixel centre (so its one term is not zero):
    that pixel's alpha is 0.008 exp(-0.25) = 0.0062, the nearest other pixel's 0.008 exp(-1.09) = 0.0027, below 1/255."""
    xyz = [_at_pixel(x + 0.25, y + 0.3) for y in range(4, 64, 8) for x in range(4, 64, 8)]
    raw = _raw(xyz, np.log(1e-4), np.log(0.008 / 0.992), np.full((len(xyz), 3), 0.7))
    grads = helpers.upstream_grads(H, W, seed=5)
    cu = render(_axis_settings(), raw, grads)
    a, d = cu["stats"]["xyz_gradient_accum_abs"], cu["stats"]["xyz_gradient_accum"]
    assert (cu["radii"] > 0).all() and (d > 0).all()
    assert np.allclose(a, d, rtol=1e-5, atol=0), np.abs(a / d - 1).max()


def _collision_model():
    """One large Gaussian at the image centre, its parameters as a stage-1 model.  Opacity 0.18: its alpha >= 1/255 footprint
    (14.8 px) stays inside its 3-sigma tile rectangle, which would otherwise clip one side and break the mirror symmetry."""
    m = stage1.GaussianModelB200(0)
    m.absgrad = True
    raw = _raw([_at_pixel(31.5, 31.5)], np.log(0.25), -1.5, [[0.5, 0.5, 0.5]])
    names = dict(xyz="xyz", features_dc="f_dc", features_rest="f_rest", opacity="opacity", scaling="scaling", rotation="rotation")
    m._set({names[k]: torch.tensor(v, device="cuda") for k, v in raw.items()})
    m.training_setup()
    return m


def _collision_step(m):
    """MSE to a target of two bright blobs left and right of the Gaussian: its left half is pulled left, its right half right."""
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float32)
    blob = lambda cx: np.exp(-((xs - cx) ** 2 + (ys - 31.5) ** 2) / (2 * 6.0 ** 2))
    target = torch.tensor(np.stack([blob(12.0) + blob(51.0)] * 3), device="cuda")
    color, radii, _, _ = FusedGaussianRasterizer(_rs(_axis_settings()))(m._xyz, m._features_dc, m._features_rest, m._opacity, m._scaling,
                                                                        m._rotation, stats=m.stats)
    ((color - target) ** 2).mean().backward()
    return radii


def test_gradient_collision_splits_with_the_absolute_rule_only():
    m = _collision_model()
    _collision_step(m)
    a, d = float(m.stats.xyz_gradient_accum_abs[0]), float(m.stats.xyz_gradient_accum[0])
    helpers.report("collision", stats=dict(abs=a, default=d))
    assert a > 0 and d < 1e-3 * a
    thr = 0.5 * a
    for use_abs, n in ((False, 1), (True, 2)):
        m = _collision_model()
        _collision_step(m)
        m.densify_and_prune(thr, min_opacity=0.005, extent=4, max_screen_size=0, max_abs_grad=thr if use_abs else None)
        assert m.num_points == n, (use_abs, m.num_points)


# ---- what the bit changes and what it does not ---------------------------------------------------------------------------------
def _close(a, b, what):
    scale = max(float(np.abs(b).max()), 1e-30)
    err = float(np.abs(a.astype(np.float64) - b).max()) / scale
    assert err <= 2e-5, (what, err)
    return bool(np.array_equal(a, b))


@pytest.mark.parametrize("camera", [False, True])
def test_the_bit_adds_one_kernel_and_leaves_gradients_and_statistics(camera):
    s, i = helpers.make_case(P=5000, res=160, deg=1, sigma=0.03, elev=20.0)
    raw = TS.raw_of(i)
    grads = helpers.upstream_grads(160, 160)
    off0, on = render(s, raw, grads, absgrad=False, camera=camera), render(s, raw, grads, absgrad=True, camera=camera)
    # launches of the backward on this host thread (the launch counter is per thread; autograd runs its backward on its own)
    tin = {k: torch.tensor(np.asarray(raw[k], np.float32), device="cuda").requires_grad_(True) for k in KEYS}
    P = tin["xyz"].shape[0]
    gC, gA = torch.tensor(grads[0], device="cuda"), torch.tensor(grads[2], device="cuda")
    lib, n = _lib.load(), {}
    for absgrad in (False, True, False):
        st = DensifyStats(P, "cuda", absgrad=absgrad)
        c = FusedGaussianRasterizer(_rs(s))(tin["xyz"], tin["features_dc"], tin["features_rest"], tin["opacity"], tin["scaling"],
                                            tin["rotation"], stats=st)[0]
        e = lambda *shape: torch.empty(shape, device="cuda")
        torch.cuda.synchronize()
        lib.dgr_reset_launch_count()
        R.backward_impl(c.grad_fn.state, gC, None, gA, e(P, 3), e(P, 3), e(P, 1, 3), None, e(P, 1), e(P, 3), e(P, 4), None,
                        d_sh_rest=e(*tin["features_rest"].shape), densify=st.as_tuple(), absgrad=st.xyz_gradient_accum_abs)
        n.setdefault(absgrad, []).append(int(lib.dgr_launch_count()))
    assert n[False][0] == n[False][1] > 0 and n[True][0] == n[False][0] + 1, n
    ident = {}
    for k, v in off0["grads"].items():
        ident[k] = _close(on["grads"][k], v, k)
    for k in ("xyz_gradient_accum", "denom", "max_radii2D"):
        ident[k] = _close(on["stats"][k], off0["stats"][k], k)
    if camera:
        ident["viewmatrix"] = _close(on["camera"], off0["camera"], "viewmatrix")
    helpers.report("bit on vs off", bit_identical=ident)


def test_deterministic_statistic_is_bit_identical_across_runs_knobs_staging_and_host_layers():
    s, i = helpers.make_case(P=4000, res=128, deg=1, sigma=0.03, elev=5.0, azim=70.0)
    raw = TS.raw_of(i)
    grads = helpers.upstream_grads(128, 128)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        runs = []
        for word in (helpers.DEFAULT_TUNING, helpers.DEFAULT_TUNING, (2, 2, 1 | (2 << 8) | (1 << 21)), (1, 1, 1 | (2 << 22)), (1, 1, 1 | (1 << 22)),
                     (4, 1, 1 | (3 << 16))):
            for fast in (True, False):
                runs.append(helpers.run_tuned(word, lambda: render(s, raw, grads), fast_host=fast))
    finally:
        torch.use_deterministic_algorithms(prev)
    ref = runs[0]["stats"]["xyz_gradient_accum_abs"]
    assert (ref > 0).sum() > 100
    for r in runs[1:]:
        assert np.array_equal(r["stats"]["xyz_gradient_accum_abs"], ref)
        assert np.array_equal(r["stats"]["xyz_gradient_accum"], runs[0]["stats"]["xyz_gradient_accum"])


# ---- stage 1 -------------------------------------------------------------------------------------------------------------------
def test_fused_and_torch_densify_agree_with_the_absolute_rule():
    rng = np.random.default_rng(9)
    P = 20000
    init = dict(xyz=rng.normal(0, 0.3, (P, 3)), f_dc=rng.normal(0, 1, (P, 1, 3)), f_rest=rng.normal(0, 0.1, (P, 3, 3)),
                opacity=rng.normal(-1.0, 2.5, (P, 1)), scaling=rng.normal(-3.4, 0.6, (P, 3)), rotation=rng.normal(0, 1, (P, 4)))
    acc = torch.tensor(np.abs(rng.normal(0, 0.02, (P,))).astype(np.float32) * 3, device="cuda")
    acc_abs = acc * torch.tensor(rng.uniform(1.0, 4.0, (P,)).astype(np.float32), device="cuda")
    den = torch.tensor(rng.integers(0, 4, (P,)).astype(np.float32), device="cuda")
    draws = torch.randn((2 * P, 3), device="cuda")

    class Noise:
        def to(self, stds):
            return draws[: stds.shape[0]].to(stds)
    models = []
    for fused in (True, False):
        m = stage1.GaussianModelB200(1)
        m.fused_adam, m.fused_densify, m.absgrad = True, fused, True
        m._set({k: torch.tensor(v, dtype=torch.float32, device="cuda") for k, v in init.items()})
        m.training_setup()
        m.stats.xyz_gradient_accum, m.stats.xyz_gradient_accum_abs, m.stats.denom = acc.clone(), acc_abs.clone(), den.clone()
        m.densify_and_prune(0.01, min_opacity=0.01, extent=4, max_screen_size=1, noise=Noise(), max_abs_grad=0.03)
        models.append(m)
    a, b = models
    assert a.num_points == b.num_points and a.num_points != P
    for k in stage1.GROUPS:
        scale = max(1.0, float(b.p[k].abs().max()))
        assert float((a.p[k] - b.p[k]).abs().max()) <= 3e-6 * scale, k
        assert torch.equal(a.exp_avg[k], b.exp_avg[k]), k


@pytest.mark.parametrize("batched", [False, True])
def test_seeded_stage1_runs_with_the_threshold_are_bit_identical(batched):
    cfg = stage1.Stage1Config(iters=200, densify_abs_grad_threshold=0.02, densification_interval=50, density_start_iter=50)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        out = []
        for _ in range(2):
            t = stage1.Stage1Trainer(cfg, batched=batched)
            losses = t.train()
            out.append((losses, {k: v.detach().cpu().numpy() for k, v in t.gaussians.p.items()}))
    finally:
        torch.use_deterministic_algorithms(prev)
    (la, pa), (lb, pb) = out
    helpers.report("stage1 abs", run=dict(batched=batched, points=int(pa["xyz"].shape[0])))
    assert pa["xyz"].shape[0] != stage1.Stage1Config().num_pts
    assert np.array_equal(la, lb) and all(np.array_equal(pa[k], pb[k]) for k in pa)
