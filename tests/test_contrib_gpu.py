"""The blending-weight statistics (DGR_RASTER_CONTRIB) on the GPU: parity with both builds of the C oracle, the alpha identity, what the
bit leaves unchanged, bit-reproducibility (runs, knobs, staging, host layers, batched against single-view calls, a forced stage-2
re-run), accumulation, pruning of occluded Gaussians, and prune_unseen after a stage-1 run."""
import numpy as np
import pytest
import torch

import aa_oracle
import contrib_oracle as CO
import helpers
import trained_scenes as TS
from dreamgaussian_b200 import _lib, stage1
from dreamgaussian_b200 import rasterizer as R
from dreamgaussian_b200.rasterizer import ContributionStats, GaussianRasterizationSettings, GaussianRasterizer
from oracle import c_oracle

pytestmark = pytest.mark.gpu
ACT = ("means3D", "shs", "opacities", "scales", "rotations")


def _rs(settings):
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda")
    return GaussianRasterizationSettings(
        image_height=settings["image_height"], image_width=settings["image_width"], tanfovx=settings["tanfovx"],
        tanfovy=settings["tanfovy"], bg=t(settings["bg"]), scale_modifier=settings["scale_modifier"],
        viewmatrix=t(settings["viewmatrix"]), projmatrix=t(settings["projmatrix"]), sh_degree=settings["sh_degree"],
        campos=t(settings["campos"]), prefiltered=False, debug=False)


def _tin(inputs, grad=False):
    return {k: torch.tensor(np.asarray(inputs[k], np.float32), device="cuda").requires_grad_(grad) for k in ACT}


def render(settings, inputs, contrib=True, antialiasing=False, grads=None):
    """One render (and a backward with `grads`) -> dict of numpy: images, radii, statistics (None without contrib), gradients."""
    tin = _tin(inputs, grad=grads is not None)
    P = tin["means3D"].shape[0]
    st = ContributionStats(P, "cuda") if contrib else None
    means2D = torch.zeros_like(tin["means3D"], requires_grad=grads is not None)
    color, radii, depth, alpha = GaussianRasterizer(_rs(settings), antialiasing, st)(
        means3D=tin["means3D"], means2D=means2D, opacities=tin["opacities"], shs=tin["shs"], scales=tin["scales"], rotations=tin["rotations"])
    out = dict(color=color.detach().cpu().numpy(), depth=depth.detach().cpu().numpy(), alpha=alpha.detach().cpu().numpy(),
               radii=radii.cpu().numpy())
    if st is not None:
        assert st.renders == 1
        out["wsum"], out["wmax"] = st.weight_sum.cpu().numpy(), st.weight_max.cpu().numpy()
    if grads is not None:
        gC, gD, gA = (torch.tensor(np.asarray(x, np.float32), device="cuda") if x is not None else None for x in grads)
        loss = (color * gC).sum() + (alpha * gA).sum() + ((depth * gD).sum() if gD is not None else 0.0)
        loss.backward()
        out["grads"] = {k: v.grad.cpu().numpy() for k, v in tin.items()}
        out["grads"]["means2D"] = means2D.grad.cpu().numpy()
    torch.cuda.synchronize()
    return out


def check_rule(cu, ref, flags, name, f32=False):
    """The gradient rule of helpers.compare (f64) / compare_f32 (f32), applied to one per-Gaussian statistic."""
    clean = (flags == 0) if not f32 else ((flags & (2 | 16)) == 0)
    scale = max(float(np.abs(ref).max()), 1e-30)
    e = (np.abs(cu.astype(np.float64) - ref) - helpers.GRAD_RTOL * np.abs(ref)) / scale
    e = e[clean]
    worst, p999 = float(e.max()), float(np.percentile(e, 99.9))
    helpers.report(name, contrib=dict(worst=worst, p999=p999, clean=int(clean.sum())))
    if f32:
        assert p999 <= helpers.F32_GRAD_ATOL and worst <= helpers.F32_GRAD_OUTLIER_ATOL, (name, worst, p999)
    else:
        assert p999 <= helpers.GRAD_ATOL and worst <= helpers.GRAD_ATOL_MAX, (name, worst, p999)


def parity(name, settings, inputs, antialiasing=False, f32=True, f64=True):
    cu = render(settings, inputs, antialiasing=antialiasing)
    act = {k: np.asarray(inputs[k], np.float64) for k in ACT}
    if antialiasing:
        t = {k: torch.tensor(act[k]) for k in ("means3D", "scales", "rotations")}
        act["opacities"] = act["opacities"] * aa_oracle.comp(settings, t["means3D"], t["scales"], t["rotations"]).numpy().reshape(-1, 1)
    rest = {k: v for k, v in inputs.items() if k not in ACT}
    for dt in (np.float32,) * f32 + (np.float64,) * f64:
        r = c_oracle.forward(**settings, **act, **rest, dtype=dt)
        ws, wm = CO.c_stats(r)
        _, flags, _ = r.flags()
        assert (wm > 0).sum() > 10
        tag = "%s %s" % (name, np.dtype(dt).name)
        check_rule(cu["wsum"], ws, flags, tag + " sum", f32=dt is np.float32)
        check_rule(cu["wmax"], wm, flags, tag + " max", f32=dt is np.float32)
        r.close()
    # the alpha identity: sum over Gaussians of weight_sum = sum of the alpha image (float64 on the host)
    a = float(cu["alpha"].astype(np.float64).sum())
    rel = abs(float(cu["wsum"].astype(np.float64).sum()) - a) / a
    helpers.report(name + " identity", alpha=dict(rel=rel))
    assert rel <= 1e-5, (name, rel)
    return cu


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_parity_seeded(deg):
    s, i = helpers.make_case(P=3000, res=128, deg=deg, sigma=0.03, elev=15.0, azim=40.0)
    parity("deg%d" % deg, s, i)


@pytest.mark.parametrize("regime", ["saturated", "dark", "needles", "faint", "subpixel", "frustum_edge"])
def test_parity_trained_regimes(regime):
    s, i = getattr(TS, regime)()
    parity(regime, s, i, f32=regime != "needles")


def test_parity_antialiased():
    s, i = helpers.make_case(P=3000, res=128, deg=1, sigma=0.02, elev=10.0)
    parity("aa", s, i, antialiasing=True)


@pytest.mark.parametrize("staging", [1, 2])
def test_parity_both_record_stagings(staging):
    s, i = helpers.make_case(P=3000, res=128, deg=1, sigma=0.03, elev=5.0, azim=20.0)
    helpers.run_tuned((1, 1, 1 | (staging << 22)), lambda: parity("staging%d" % staging, s, i))


def test_the_bit_changes_nothing_else():
    s, i = helpers.make_case(P=4000, res=128, deg=2, sigma=0.03, elev=5.0, azim=70.0)
    grads = helpers.upstream_grads(128, 128)
    lib = _lib.load()
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for fast in (True, False):
            def both():
                return render(s, i, contrib=False, grads=grads), render(s, i, contrib=True, grads=grads)
            off, on = helpers.run_tuned(helpers.DEFAULT_TUNING, both, fast_host=fast)
            for k in ("color", "depth", "alpha", "radii"):
                assert np.array_equal(off[k], on[k]), k
            for k in off["grads"]:
                assert np.array_equal(off["grads"][k], on["grads"][k]), k
    finally:
        torch.use_deterministic_algorithms(prev)

    # the forward's launches (this host thread's; the backward runs on autograd's): the same without the bit, and with it
    # render_fwd_contrib in render_fwd's place followed by contrib_finalize
    def launches(contrib):
        lib.dgr_reset_launch_count()
        lib.dgr_profile_enable(1)
        render(s, i, contrib=contrib)
        names = [n for n, _ in _lib.profile_collect()]
        lib.dgr_profile_enable(0)
        return int(lib.dgr_launch_count()), names
    n0, names0 = launches(False)
    n1, names1 = launches(False)
    n2, names2 = launches(True)
    assert n0 == n1 == len(names0) and names0 == names1 and not any("contrib" in n for n in names0)
    assert n2 == n0 + 1
    assert names2 == [("render_fwd_contrib" if n == "render_fwd" else n) for n in names0] + ["contrib_finalize"]


def test_bit_reproducible_across_runs_knobs_staging_and_host_layers():
    s, i = helpers.make_case(P=6000, res=160, deg=1, sigma=0.03, elev=5.0, azim=70.0)
    runs = []
    for word in (helpers.DEFAULT_TUNING, helpers.DEFAULT_TUNING, (2, 2, 1 | (2 << 4)), (4, 1, 1 | (3 << 12)), (1, 1, 1 | (4 << 4)),
                 (1, 1, 1 | (2 << 22)), (1, 1, 1 | (1 << 22)), (1, 1, 1 | (1 << 20))):
        for fast in (True, False):
            runs.append(helpers.run_tuned(word, lambda: render(s, i), fast_host=fast))
    ref = runs[0]
    assert (ref["wmax"] > 0).sum() > 1000
    for r in runs[1:]:
        assert np.array_equal(r["wsum"], ref["wsum"]) and np.array_equal(r["wmax"], ref["wmax"])


def _views(n=3, res=96, seed=4):
    out = []
    for v in range(n):
        s, i = helpers.make_case(P=3000, res=res, deg=1, sigma=0.03, elev=10.0 * v - 5, azim=35.0 * v, seed=seed)
        out.append((s, i))
    return out


@pytest.mark.parametrize("mixed", [False, True])
def test_batched_views_equal_single_view_calls(mixed):
    cases = _views()
    i = cases[0][1]
    settings = [c[0] for c in cases]
    if mixed:
        for k, (h, w) in enumerate([(96, 96), (64, 128), (112, 80)]):
            settings[k] = dict(settings[k], image_height=h, image_width=w)
    single = [render(sk, i) for sk in settings]
    tin = _tin(i)
    P = tin["means3D"].shape[0]
    runs = []
    for fast in (True, False):
        def batched():
            st = ContributionStats(P, "cuda")
            f = R.rasterize_views_mixed if mixed else R.rasterize_views
            with torch.no_grad():
                f([_rs(sk) for sk in settings], tin["means3D"], None, tin["opacities"], tin["shs"], tin["scales"], tin["rotations"],
                  contributions=st)
            return st
        st = helpers.run_tuned(helpers.DEFAULT_TUNING, batched, fast_host=fast)
        assert st.renders == 3
        runs.append((st.weight_sum.cpu().numpy(), st.weight_max.cpu().numpy()))
    # both host layers: bit-identical
    assert np.array_equal(runs[0][0], runs[1][0]) and np.array_equal(runs[0][1], runs[1][1])
    # every view against the single-view call of its camera.  The batched per-Gaussian kernel is a different kernel, whose fused
    # multiply-adds ptxas chooses on its own (include/dgr_b200.h): the records, and so the weights, agree up to that rounding
    state = R.views_forward_impl([_rs(sk) for sk in settings], *(tin[k] for k in ("means3D", "shs", "opacities", "scales", "rotations")),
                                 mixed=mixed, contrib=True)[4]
    ws, wm = np.zeros(P), np.zeros(P)
    for v, r in enumerate(single):
        bs, bm = state.contrib[0][v].cpu().numpy(), state.contrib[1][v].cpu().numpy()
        ident = np.array_equal(bs, r["wsum"]) and np.array_equal(bm, r["wmax"])
        es, em = np.abs(bs - r["wsum"]).max() / r["wsum"].max(), np.abs(bm - r["wmax"]).max() / r["wmax"].max()
        helpers.report("batched view %d" % v, contrib=dict(mixed=mixed, bit_identical=bool(ident), sum_err=float(es), max_err=float(em)))
        assert es <= 1e-4 and em <= 1e-4
        ws, wm = ws + bs, np.maximum(wm, bm)
    assert np.allclose(runs[0][0], ws, rtol=1e-5, atol=1e-6 * ws.max()) and np.array_equal(runs[0][1], wm.astype(np.float32))


@pytest.mark.parametrize("fast", [True, False])
def test_forced_rerun_is_not_doubled(fast):
    s, i = helpers.make_case(P=5000, res=128, deg=1, sigma=0.03)

    def run(cap):
        if cap is not None:
            R.set_capacity_hint(0, 5000, 128, 128, cap, False)
        return render(s, i)
    ref = helpers.run_tuned(helpers.DEFAULT_TUNING, lambda: run(None), fast_host=fast)
    rerun = helpers.run_tuned(helpers.DEFAULT_TUNING, lambda: run(16), fast_host=fast)
    assert np.array_equal(rerun["wsum"], ref["wsum"]) and np.array_equal(rerun["wmax"], ref["wmax"])
    assert np.array_equal(rerun["color"], ref["color"])


def test_accumulation_over_renders_and_under_no_grad():
    (s1, i), (s2, _) = _views(2)[:2]
    tin = _tin(i, grad=True)
    P = tin["means3D"].shape[0]

    def go(st, settings):
        means2D = torch.zeros_like(tin["means3D"], requires_grad=True)
        return GaussianRasterizer(_rs(settings), contributions=st)(means3D=tin["means3D"], means2D=means2D, opacities=tin["opacities"],
                                                                    shs=tin["shs"], scales=tin["scales"], rotations=tin["rotations"])
    a, b, both = ContributionStats(P, "cuda"), ContributionStats(P, "cuda"), ContributionStats(P, "cuda")
    go(a, s1)
    with torch.no_grad():
        go(b, s2)
    color, *_ = go(both, s1)
    with torch.no_grad():
        go(both, s2)
    color.sum().backward()                   # the backward does not touch the statistics
    assert both.renders == 2
    assert torch.equal(both.weight_sum, a.weight_sum + b.weight_sum)
    assert torch.equal(both.weight_max, torch.maximum(a.weight_max, b.weight_max))


def test_occluded_gaussians_are_pruned_and_the_images_do_not_change():
    """Three large opaque layers in front of the camera and 300 small Gaussians far behind them, inside the view: the layers stop
    every pixel the small ones reach (T < 1e-4), so those have radii > 0 but weight_max == 0, while each layer is composited
    somewhere (the third at the image corners, where the layers are thinner).  Pruning with a tiny threshold removes exactly the 300,
    and the view renders bit-identically."""
    rng = np.random.default_rng(5)
    cam = TS.camera(128, 128)
    s = TS.settings_of(cam, 0)
    layers = np.array([[0.0, 0.0, 1.5], [0.0, 0.0, 1.6], [0.0, 0.0, 1.7]])
    layer_o = np.array([0.9997, 0.985, 0.9997])
    hidden = np.stack([rng.uniform(-0.3, 0.3, 300), rng.uniform(-0.3, 0.3, 300), np.full(300, 4.0)], 1)
    world = TS.view_to_world(cam, np.concatenate([layers, hidden]))
    P = world.shape[0]
    o = np.concatenate([layer_o, np.full(300, 0.9)])
    sc = np.concatenate([np.full(3, 1.0), np.full(300, 0.06)])
    from dreamgaussian_b200.stage1 import GaussianModelB200
    f32 = dict(dtype=torch.float32, device="cuda")
    m = GaussianModelB200(0)
    m._set(dict(xyz=torch.tensor(world, **f32), f_dc=torch.tensor(rng.normal(0, 1, (P, 1, 3)), **f32), f_rest=torch.zeros(P, 0, 3, **f32),
                opacity=torch.tensor(np.log(o / (1 - o))[:, None], **f32), scaling=torch.tensor(np.log(sc)[:, None].repeat(3, 1), **f32),
                rotation=torch.tensor([[1.0, 0, 0, 0]], **f32).repeat(P, 1)))
    m.training_setup()
    rs = _rs(s)
    st = ContributionStats(P, "cuda")
    from dreamgaussian_b200.fused import render_gaussian_model
    with torch.no_grad():
        out = render_gaussian_model(m, rs, contributions=st)
    radii = out["radii"].cpu().numpy()
    wmax = st.weight_max.cpu().numpy()
    helpers.report("occlusion", layers=dict(wmax=wmax[:3].tolist(), wsum=st.weight_sum[:3].tolist()))
    assert np.all(radii > 0) and np.all(wmax[3:] == 0) and np.all(wmax[:3] > 0)
    before = out["image"].clone()
    keep_rows = {k: v.detach()[:3].clone() for k, v in m.p.items()}
    assert m.prune_by_contribution(st, 1e-12) == 300
    assert all(torch.equal(m.p[k].detach(), keep_rows[k]) for k in m.p)
    with torch.no_grad():
        after = render_gaussian_model(m, rs)["image"]
    assert torch.equal(before, after)


def test_stage1_prune_unseen():
    t = stage1.Stage1Trainer(stage1.Stage1Config(iters=500))
    t.train()
    g = t.gaussians
    before = ({k: v.detach().clone() for k, v in g.p.items()}, {k: v.clone() for k, v in g.exp_avg.items()},
              {k: v.clone() for k, v in g.exp_avg_sq.items()})
    n0 = g.num_points
    settings = t.export_settings(512)
    from dreamgaussian_b200.fused import rasterize_views_raw
    stats = ContributionStats(n0, "cuda")
    with torch.no_grad():
        imgs0 = rasterize_views_raw(settings, g._xyz, None, g._features_dc, g._features_rest, g._opacity, g._scaling, g._rotation,
                                    contributions=stats)[0]
    keep = (stats.weight_max >= 1e-3)
    removed = t.prune_unseen(1e-3)
    assert removed == int((~keep).sum()) and g.num_points == n0 - removed
    for k in g.p:
        assert torch.equal(g.p[k].detach(), before[0][k][keep]) and torch.equal(g.exp_avg[k], before[1][k][keep])
        assert torch.equal(g.exp_avg_sq[k], before[2][k][keep])
    with torch.no_grad():
        imgs1 = rasterize_views_raw(t.export_settings(512), g._xyz, None, g._features_dc, g._features_rest, g._opacity, g._scaling,
                                    g._rotation)[0]
    from dreamgaussian_b200.fields import extract_fields_of_model
    extract_fields_of_model(g)
    helpers.report("stage1 prune_unseen", run=dict(points=n0, removed=removed,
                                                  max_image_change=float((imgs1 - imgs0).abs().max()),
                                                  mean_image_change=float((imgs1 - imgs0).abs().mean())))
