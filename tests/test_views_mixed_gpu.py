"""The batched call with a size per view (rasterize_views_mixed, rasterize_views_mixed_raw, dgr_views_mixed_*) on the GPU: every
view against both CPU oracles, against the single-view op and the same-size call, its densification statistics, its host
protocol, its limits and the batched stage-1 step."""
import numpy as np
import pytest

import helpers
import test_views_gpu as tv
from dreamgaussian_b200 import scene

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

# sizes (height, width): non-multiples of 16, a view smaller than one tile, a wide and a tall view
SIZES = [(9, 17), (72, 96), (40, 150), (130, 50)]


def _cams(P, sizes, deg, views, seed=0):
    """tv._cams with a size per view."""
    cloud = scene.make_cloud(P, deg, seed=seed, opacity="trained")
    settings = []
    for (H, W), (elev, azim, fovy, bg) in zip(sizes, views):
        cam = scene.orbit_camera(elev, azim, 2.0, W, H, fovy_deg=fovy)
        settings.append(dict(image_height=H, image_width=W, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=np.asarray(bg, np.float32),
                             scale_modifier=1.0, viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform,
                             sh_degree=deg, campos=cam.camera_center))
    inputs = dict(means3D=cloud["means3D"], opacities=cloud["opacities"], shs=cloud["shs"], scales=cloud["scales"],
                  rotations=cloud["rotations"])
    return settings, inputs


def run_mixed(settings, inputs, grads=None, raw=False, retain=False, stats=None, stats_views=(), means2D=True):
    """The mixed-size product path; outputs per view.  stats: a DensifyStats (raw only)."""
    from dreamgaussian_b200.fused import rasterize_views_mixed_raw
    from dreamgaussian_b200.rasterizer import rasterize_views_mixed
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda")
    V = len(settings)
    want = grads is not None
    rs = [tv._rs(s) for s in settings]
    keys = helpers.RAW_KEYS if raw else ("means3D", "opacities", "shs", "scales", "rotations")
    tin = {k: t(inputs[k]).requires_grad_(want) for k in keys}
    P = tin[keys[0]].shape[0]
    m2d = torch.zeros((V, P, 3), device="cuda", requires_grad=want) if means2D else None
    if raw:
        colors, radii, depths, alphas = rasterize_views_mixed_raw(rs, tin["xyz"], m2d, tin["features_dc"], tin["features_rest"], tin["opacity"],
                                                                  tin["scaling"], tin["rotation"], stats=stats, stats_views=stats_views)
    else:
        colors, radii, depths, alphas = rasterize_views_mixed(rs, tin["means3D"], m2d, tin["opacities"], tin["shs"], tin["scales"],
                                                              tin["rotations"])
    out = dict(color=[c.detach().cpu().numpy() for c in colors], depth=[d.detach().cpu().numpy() for d in depths],
               alpha=[a.detach().cpu().numpy() for a in alphas], radii=radii.cpu().numpy())
    if want:
        loss = sum(tv._loss(colors[v], depths[v], alphas[v], grads[v], t) for v in range(V) if grads[v] is not None)
        loss.backward(retain_graph=retain)
        g = {k: (v.grad.detach().cpu().numpy() if v.grad is not None else np.zeros(v.shape, np.float32)) for k, v in tin.items()}
        if m2d is not None:
            g["means2D"] = m2d.grad.detach().cpu().numpy()
        out["grads"] = g
        if retain:
            for v in tin.values():
                v.grad = None
            loss.backward()
            out["grads2"] = {k: (v.grad.detach().cpu().numpy() if v.grad is not None else np.zeros(v.shape, np.float32)) for k, v in tin.items()}
    return out


def _view(out, v):
    return dict(color=out["color"][v], depth=out["depth"][v], alpha=out["alpha"][v], radii=out["radii"][v])


# ---- every view against both oracles -------------------------------------------------------------------------------------
@pytest.mark.parametrize("deg", [0, 3])
def test_each_view_passes_both_oracles(deg):
    settings, inputs = _cams(2001, SIZES, deg, tv.VIEWS4, seed=deg)
    for v in range(len(settings)):
        H, W = SIZES[v]
        g = helpers.upstream_grads(H, W, seed=40 + v)
        cu = run_mixed(settings, inputs, [g if u == v else None for u in range(len(settings))])
        cv = _view(cu, v)
        cv["grads"] = dict(cu["grads"], means2D=cu["grads"]["means2D"][v])
        helpers.both_oracles("mixed deg%d v%d %dx%d" % (deg, v, H, W), settings[v], inputs, g, cu=cv, max_ambig_frac=0.06)


@pytest.mark.parametrize("deg", [0, 3])
def test_each_view_passes_the_oracle_with_raw_parameters(deg):
    settings, _ = _cams(1501, SIZES, deg, tv.VIEWS4, seed=7)
    raw = scene.to_raw_parameters(scene.make_cloud(1501, deg, seed=7), seed=7)
    for v in range(len(settings)):
        H, W = SIZES[v]
        g = helpers.upstream_grads(H, W, seed=60 + v)
        cu = run_mixed(settings, raw, [g if u == v else None for u in range(len(settings))], raw=True)
        ref = helpers.run_oracle_raw(settings[v], raw, g)
        cv = _view(cu, v)
        cv["grads"] = dict(cu["grads"], means2D=cu["grads"]["means2D"][v])
        ok, rep = helpers.compare(cv, ref)
        helpers.report("mixed raw deg%d v%d" % (deg, v), vs_f64=rep)
        assert ok, rep


# ---- against the single-view op and the same-size call -------------------------------------------------------------------
def test_batch_matches_the_single_view_op():
    settings, inputs = _cams(5003, SIZES, 3, tv.VIEWS4, seed=11)
    grads = [helpers.upstream_grads(H, W, seed=80 + v) for v, (H, W) in enumerate(SIZES)]
    cu = run_mixed(settings, inputs, grads)
    total = None
    for v in range(len(settings)):
        one = helpers.run_cuda(settings[v], inputs, grads[v])
        tv._forward_rule(_view(cu, v), one, "view %d" % v)
        scale = float(np.abs(one["grads"]["means2D"]).max())
        assert np.abs(cu["grads"]["means2D"][v] - one["grads"]["means2D"]).max() <= 2e-5 * scale, v
        g = {k: one["grads"][k] for k in ("means3D", "opacities", "shs", "scales", "rotations")}
        total = g if total is None else {k: total[k] + g[k] for k in g}
    tv._grads_close({k: cu["grads"][k] for k in total}, total, "sum over views")


def test_equal_sizes_are_bit_identical_to_the_same_size_call():
    W, H = 96, 80
    settings, inputs = tv._cams(3001, W, H, 2, tv.VIEWS4, seed=3)
    same = tv.run_views(settings, inputs)
    mixed = run_mixed(settings, inputs)
    for v in range(4):
        for k in ("color", "depth", "alpha", "radii"):
            assert np.array_equal(mixed[k][v], same[k][v]), (v, k)


def test_permuting_the_batch_permutes_its_images():
    settings, inputs = _cams(4000, SIZES, 2, tv.VIEWS4, seed=5)
    base = run_mixed(settings, inputs)
    perm = [2, 0, 3, 1]
    shuf = run_mixed([settings[i] for i in perm], inputs)
    for j, i in enumerate(perm):
        for k in ("color", "depth", "alpha", "radii"):
            assert np.array_equal(shuf[k][j], base[k][i]), (j, k)


# ---- densification statistics --------------------------------------------------------------------------------------------
# views 0, 1 and 3 see the middle of the cloud only (12 degree field of view), view 2 all of it
STATS_VIEWS = [(0.0, 0.0, 12.0, (1.0, 1.0, 1.0)), (-20.0, 90.0, 12.0, (0.0, 0.0, 0.0)), (15.0, 180.0, 55.0, (0.2, 0.5, 0.9)),
               (-35.0, 270.0, 12.0, (1.0, 0.0, 0.3))]


def _raw_case(P=3001, deg=0, seed=13):
    settings, _ = _cams(P, SIZES, deg, STATS_VIEWS, seed=seed)
    raw = scene.to_raw_parameters(scene.make_cloud(P, deg, seed=seed), seed=seed)
    grads = [helpers.upstream_grads(H, W, seed=100 + v) for v, (H, W) in enumerate(SIZES)]
    return settings, raw, grads


def _stats(P, prefill=False):
    from dreamgaussian_b200.fused import DensifyStats
    st = DensifyStats(P, "cuda")
    if prefill:
        g = torch.Generator(device="cpu").manual_seed(3)
        for t in st.as_tuple():
            t.copy_((torch.rand((P,), generator=g) * 4).round())
    return st


def _rule(stats0, out, selected):
    """The single-view rule applied in view order to the call's own means2D gradient and radii."""
    acc, den, mx = (np.asarray(x, np.float32).copy() for x in stats0)
    m2d, radii = out["grads"]["means2D"], out["radii"]
    for v in selected:
        vis = radii[v] > 0
        gx, gy = m2d[v, :, 0], m2d[v, :, 1]
        acc[vis] += np.sqrt(gx * gx + gy * gy)[vis]
        den[vis] += np.float32(1.0)
        mx[vis] = np.maximum(mx[vis], radii[v][vis].astype(np.float32))
    return acc, den, mx


@pytest.mark.parametrize("prefill", [False, True])
@pytest.mark.parametrize("selected", [(1,), (0, 3), (0, 1, 2, 3)])
def test_statistics_follow_the_single_view_rule_on_the_selected_views(selected, prefill):
    settings, raw, grads = _raw_case()
    P = raw["xyz"].shape[0]
    st = _stats(P, prefill)
    before = [t.cpu().numpy() for t in st.as_tuple()]
    out = run_mixed(settings, raw, grads, raw=True, stats=st, stats_views=selected)
    acc, den, mx = _rule(before, out, selected)
    got = [t.cpu().numpy() for t in st.as_tuple()]
    assert np.array_equal(got[2], mx) and np.array_equal(got[1], den)
    assert np.allclose(got[0], acc, rtol=1e-6, atol=0.0)
    # a Gaussian visible only in views that are not selected is untouched
    radii = out["radii"]
    others = [v for v in range(4) if v not in selected]
    if not others:
        return
    only_other = (radii[others] > 0).any(0) & ~(radii[list(selected)] > 0).any(0)
    assert only_other.any()
    for a, b in zip(got, before):
        assert np.array_equal(a[only_other], b[only_other])


def test_a_retained_double_backward_counts_the_views_once():
    settings, raw, grads = _raw_case()
    P = raw["xyz"].shape[0]
    once, twice = _stats(P), _stats(P)
    a = run_mixed(settings, raw, grads, raw=True, stats=once, stats_views=(1, 2))
    b = run_mixed(settings, raw, grads, raw=True, stats=twice, stats_views=(1, 2), retain=True)
    assert np.array_equal(twice.denom.cpu().numpy(), once.denom.cpu().numpy())
    assert np.array_equal(twice.max_radii2D.cpu().numpy(), once.max_radii2D.cpu().numpy())
    assert np.allclose(twice.xyz_gradient_accum.cpu().numpy(), once.xyz_gradient_accum.cpu().numpy(), rtol=2e-5, atol=1e-7)
    tv._grads_close(b["grads2"], {k: b["grads"][k] for k in b["grads2"]}, "retain_graph", rtol=2e-5)
    assert a["radii"].shape == b["radii"].shape


def test_statistics_match_a_loop_of_fused_single_view_calls():
    from dreamgaussian_b200.fused import FusedGaussianRasterizer
    settings, raw, grads = _raw_case(deg=1)
    P = raw["xyz"].shape[0]
    selected = (0, 2, 3)
    batched = _stats(P)
    run_mixed(settings, raw, grads, raw=True, stats=batched, stats_views=selected)
    loop = _stats(P)
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda")
    for v in selected:
        tin = {k: t(raw[k]).requires_grad_(True) for k in helpers.RAW_KEYS}
        m2d = torch.zeros((P, 3), device="cuda", requires_grad=True)
        color, radii, depth, alpha = FusedGaussianRasterizer(tv._rs(settings[v]))(
            tin["xyz"], tin["features_dc"], tin["features_rest"], tin["opacity"], tin["scaling"], tin["rotation"], means2D=m2d, stats=loop)
        tv._loss(color, depth, alpha, grads[v], t).backward()
    assert np.array_equal(batched.denom.cpu().numpy(), loop.denom.cpu().numpy())
    assert np.array_equal(batched.max_radii2D.cpu().numpy(), loop.max_radii2D.cpu().numpy())
    tv._grads_close({"acc": batched.xyz_gradient_accum.cpu().numpy()}, {"acc": loop.xyz_gradient_accum.cpu().numpy()}, "accum")


# ---- protocol and edges --------------------------------------------------------------------------------------------------
_restore = tv._restore


@pytest.mark.parametrize("raw", [False, True])
def test_compiled_and_ctypes_host_layers_agree(raw, _restore):
    from dreamgaussian_b200 import rasterizer as R
    settings, inputs = _cams(3001, SIZES[:3], 3, tv.VIEWS4[:3], seed=9)
    if raw:
        inputs = scene.to_raw_parameters(scene.make_cloud(3001, 3, seed=9), seed=9)
    grads = [helpers.upstream_grads(H, W, seed=90 + v) for v, (H, W) in enumerate(SIZES[:3])]
    kw = dict(stats_views=(0, 2)) if raw else {}
    stats = [_stats(3001), _stats(3001)] if raw else [None, None]
    assert R.set_fast_host(True)
    fast = run_mixed(settings, inputs, grads, raw=raw, stats=stats[0], **kw)
    assert not R.set_fast_host(False)
    slow = run_mixed(settings, inputs, grads, raw=raw, stats=stats[1], **kw)
    for v in range(3):
        for k in ("color", "depth", "alpha", "radii"):
            assert np.array_equal(fast[k][v], slow[k][v]), (v, k)
    tv._grads_close(fast["grads"], slow["grads"], "host layers", rtol=2e-5)
    if raw:
        assert np.array_equal(stats[0].denom.cpu().numpy(), stats[1].denom.cpu().numpy())
        assert np.array_equal(stats[0].max_radii2D.cpu().numpy(), stats[1].max_radii2D.cpu().numpy())


@pytest.mark.parametrize("fast_host", [True, False])
def test_small_capacity_hint_is_repaired(fast_host, _restore):
    from dreamgaussian_b200 import rasterizer as R
    settings, inputs = _cams(3001, SIZES[:3], 3, tv.VIEWS4[:3], seed=9)
    grads = [helpers.upstream_grads(H, W, seed=90 + v) for v, (H, W) in enumerate(SIZES[:3])]
    base = run_mixed(settings, inputs, grads)
    assert R.set_fast_host(fast_host) == fast_host
    R.set_views_mixed_capacity_hint(0, 3001, SIZES[:3], 16, False)
    got = run_mixed(settings, inputs, grads)
    for v in range(3):
        for k in ("color", "depth", "alpha", "radii"):
            assert np.array_equal(got[k][v], base[k][v]), (v, k)
    tv._grads_close(got["grads"], base["grads"], "repaired", rtol=2e-5)
    assert R.get_views_mixed_capacity_hint(0, 3001, SIZES[:3])[0] > 16


def test_a_view_looking_away_renders_the_background():
    settings, inputs = _cams(2000, [(48, 64), (33, 70)], 0, tv.VIEWS4[:2], seed=4)
    away = dict(settings[1])
    V = np.asarray(away["viewmatrix"], np.float32).copy()
    F = np.diag([1.0, 1.0, -1.0, 1.0]).astype(np.float32)          # mirror z: the cloud is now behind the camera
    away["viewmatrix"] = V @ F
    away["projmatrix"] = away["viewmatrix"] @ (np.linalg.inv(V) @ np.asarray(settings[1]["projmatrix"], np.float32))
    out = run_mixed([settings[0], away], inputs)
    assert (out["radii"][1] == 0).all()
    assert np.array_equal(out["color"][1], np.broadcast_to(np.asarray(away["bg"], np.float32)[:, None, None], (3, 33, 70)))
    assert (out["alpha"][1] == 0).all() and (out["radii"][0] > 0).any()


def test_empty_cloud():
    settings, inputs = _cams(64, SIZES[:2], 1, tv.VIEWS4[:2], seed=4)
    empty = {k: v[:0] for k, v in inputs.items()}
    out = run_mixed(settings, empty, [helpers.upstream_grads(H, W) for H, W in SIZES[:2]])
    assert out["radii"].shape == (2, 0)
    for v in range(2):
        assert np.allclose(out["color"][v], np.asarray(settings[v]["bg"])[:, None, None])


def test_batch_at_the_tile_limit_and_one_tile_beyond():
    sizes = [(512, 512)] * 49 + [(512, 496), (16, 512)]                  # 49 x 1024 + 992 + 32 = 51,200 tiles
    views = [(-30.0 + v, 7.2 * v, 49.1, (0.5, 0.5, 0.5)) for v in range(len(sizes))]
    settings, inputs = _cams(3000, sizes, 0, views, seed=6)
    v = 49
    g = helpers.upstream_grads(512, 496, seed=5)
    cu = run_mixed(settings, inputs, [g if u == v else None for u in range(len(sizes))])
    cv = _view(cu, v)
    cv["grads"] = dict(cu["grads"], means2D=cu["grads"]["means2D"][v])
    helpers.both_oracles("mixed 51200 tiles v%d" % v, settings[v], inputs, g, cu=cv)
    over = list(settings)
    over[-1] = dict(over[-1], image_width=528)                           # one tile more
    with pytest.raises(RuntimeError, match="51200"):
        run_mixed(over, inputs)


def test_launch_count_equals_the_same_size_batch():
    settings, inputs = _cams(3000, SIZES, 1, tv.VIEWS4, seed=8)
    grads = [helpers.upstream_grads(H, W) for H, W in SIZES]
    same_settings, _ = tv._cams(3000, 96, 80, 1, tv.VIEWS4, seed=8)
    g = helpers.upstream_grads(80, 96)
    mixed = tv._launches(lambda: run_mixed(settings, inputs, grads))
    same = tv._launches(lambda: tv.run_views(same_settings, inputs, [g] * 4))
    assert mixed == same, (mixed, same)


# ---- the batched stage-1 step --------------------------------------------------------------------------------------------
def test_batched_stage1_tracks_the_fused_loop():
    from dreamgaussian_b200.stage1 import Stage1Config, Stage1Trainer
    # 30 iterations: the novel view is 128^2 for steps 1-8, 256^2 for 9-17 and 512^2 after; densification every 4 steps from 6
    cfg = Stage1Config(iters=30, num_pts=3000, density_start_iter=6, densification_interval=4)
    fused, batched = Stage1Trainer(cfg, device="cuda", fused=True), Stage1Trainer(cfg, device="cuda", fused=True, batched=True)
    for _ in range(5):
        a, b = float(fused.train_step()), float(batched.train_step())
        assert np.isclose(b, a, rtol=2e-3), (fused.step, a, b)
    sizes = []
    for _ in range(25):
        batched.train_step()
        g = batched.gaussians
        P = g._xyz.shape[0]
        assert all(t.shape[0] == P for t in (g._features_dc, g._features_rest, g._opacity, g._scaling, g._rotation))
        assert all(t.shape[0] == P for t in g.stats.as_tuple())
        sizes.append(P)
    losses = torch.stack(batched.losses).cpu().numpy()
    assert np.isfinite(losses).all()
    assert len(set(sizes)) > 1                                           # densification changed the cloud
    per_ratio = losses / (np.arange(1, 31) / 30.0)                       # the reconstruction terms grow with step_ratio
    assert per_ratio[-5:].mean() < per_ratio[:5].mean()
