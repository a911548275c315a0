"""The batched-camera call (rasterize_views, dgr_views_*) on the GPU: every view against both CPU oracles, against the
single-view op, its determinism, its host protocol and its limits."""
import numpy as np
import pytest

import helpers
from dreamgaussian_b200 import scene

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def _cams(P, W, H, deg, views, seed=0, opacity="trained"):
    """One cloud and one settings dict per (elev, azim, fovy_deg, bg) of `views`."""
    cloud = scene.make_cloud(P, deg, seed=seed, opacity=opacity)
    settings = []
    for elev, azim, fovy, bg in views:
        cam = scene.orbit_camera(elev, azim, 2.0, W, H, fovy_deg=fovy)
        settings.append(dict(image_height=H, image_width=W, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=np.asarray(bg, np.float32),
                             scale_modifier=1.0, viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform,
                             sh_degree=deg, campos=cam.camera_center))
    inputs = dict(means3D=cloud["means3D"], opacities=cloud["opacities"], shs=cloud["shs"], scales=cloud["scales"],
                  rotations=cloud["rotations"])
    return settings, inputs


VIEWS4 = [(0.0, 0.0, 49.1, (1.0, 1.0, 1.0)), (-20.0, 90.0, 40.0, (0.0, 0.0, 0.0)), (15.0, 180.0, 55.0, (0.2, 0.5, 0.9)),
          (-35.0, 270.0, 49.1, (1.0, 0.0, 0.3))]


ORACLE_VIEWS = [(0.0, 0.0, 49.1, (1.0, 1.0, 1.0)), (15.0, 120.0, 40.0, (0.0, 0.0, 0.0)), (25.0, 240.0, 55.0, (0.2, 0.5, 0.9))]


def _rs(s, device="cuda"):
    from dreamgaussian_b200.rasterizer import GaussianRasterizationSettings
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device=device)
    return GaussianRasterizationSettings(
        image_height=s["image_height"], image_width=s["image_width"], tanfovx=s["tanfovx"], tanfovy=s["tanfovy"], bg=t(s["bg"]),
        scale_modifier=s["scale_modifier"], viewmatrix=t(s["viewmatrix"]), projmatrix=t(s["projmatrix"]), sh_degree=s["sh_degree"],
        campos=t(s["campos"]), prefiltered=False, debug=False)


def _loss(color, depth, alpha, grads, t):
    gC, gD, gA = grads
    loss = (color * t(gC)).sum() + (alpha * t(gA)).sum()
    if gD is not None:
        loss = loss + (depth * t(gD)).sum()
    return loss


def run_views(settings, inputs, grads=None, raw=False, retain=False):
    """The batched product path.  grads: one (gC, gD, gA) or None per view (None: no upstream gradient on that view)."""
    from dreamgaussian_b200.fused import rasterize_views_raw
    from dreamgaussian_b200.rasterizer import rasterize_views
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda")
    V = len(settings)
    want = grads is not None
    rs = [_rs(s) for s in settings]
    keys = helpers.RAW_KEYS if raw else ("means3D", "opacities", "shs", "scales", "rotations")
    tin = {k: t(inputs[k]).requires_grad_(want) for k in keys}
    P = tin[keys[0]].shape[0]
    means2D = torch.zeros((V, P, 3), device="cuda", requires_grad=want)
    if raw:
        color, radii, depth, alpha = rasterize_views_raw(rs, tin["xyz"], means2D, tin["features_dc"], tin["features_rest"], tin["opacity"],
                                                         tin["scaling"], tin["rotation"])
    else:
        color, radii, depth, alpha = rasterize_views(rs, tin["means3D"], means2D, tin["opacities"], tin["shs"], tin["scales"], tin["rotations"])
    out = dict(color=color.detach().cpu().numpy(), depth=depth.detach().cpu().numpy(), alpha=alpha.detach().cpu().numpy(),
               radii=radii.cpu().numpy())
    if want:
        loss = sum(_loss(color[v], depth[v], alpha[v], grads[v], t) for v in range(V) if grads[v] is not None)
        loss.backward(retain_graph=retain)
        g = {k: (v.grad.detach().cpu().numpy() if v.grad is not None else np.zeros(v.shape, np.float32)) for k, v in tin.items()}
        g["means2D"] = means2D.grad.detach().cpu().numpy()
        out["grads"] = g
        if retain:
            for v in list(tin.values()) + [means2D]:
                v.grad = None
            loss.backward()
            out["grads2"] = {k: v.grad.detach().cpu().numpy() for k, v in tin.items()}
    return out


def _view(out, v):
    return dict(color=out["color"][v], depth=out["depth"][v], alpha=out["alpha"][v], radii=out["radii"][v])


def _forward_rule(a, b, name):
    """Images within 2e-6 relative except <= 1e-4 of the pixels (each <= 1e-2); at most 2 radii differ (ptxas fuses
    multiply-adds per kernel instantiation, which moves a few alpha >= 1/255 decisions)."""
    for k in ("color", "depth", "alpha"):
        x, y = a[k].astype(np.float64), b[k].astype(np.float64)
        d = np.abs(x - y)
        off = d > 2e-6 * np.maximum(1.0, np.abs(y))
        assert off.sum() <= max(1, int(1e-4 * d.size)) and (d.max() if d.size else 0.0) <= 1e-2, (name, k, int(off.sum()), float(d.max()))
    assert int((a["radii"] != b["radii"]).sum()) <= 2, (name, int((a["radii"] != b["radii"]).sum()))


def _grads_close(a, b, name, rtol=2e-4):
    for k in b:
        x, y = np.asarray(a[k], np.float64), np.asarray(b[k], np.float64).reshape(np.shape(a[k]))
        scale = float(np.abs(y).max()) if y.size else 0.0
        assert np.abs(x - y).max(initial=0.0) <= rtol * scale + 1e-6, (name, k, float(np.abs(x - y).max(initial=0.0)), scale)


# ---- every view against both oracles -------------------------------------------------------------------------------------
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_each_view_passes_both_oracles(deg):
    W, H = 96, 72
    settings, inputs = _cams(2001, W, H, deg, ORACLE_VIEWS, seed=deg)        # P = 2001: staged warps + a per-thread partial warp
    for v in range(len(settings)):
        g = helpers.upstream_grads(H, W, seed=40 + v)
        cu = run_views(settings, inputs, [g if u == v else None for u in range(len(settings))])
        cv = _view(cu, v)
        cv["grads"] = dict(cu["grads"], means2D=cu["grads"]["means2D"][v])
        # (views seen from below the cloud's equator have more depth-key ties: the float32 oracle sets those aside, the float64
        #  one flags a few more pixels than the suite's usual 4%)
        helpers.both_oracles("views deg%d v%d" % (deg, v), settings[v], inputs, g, cu=cv, max_ambig_frac=0.06)


@pytest.mark.parametrize("deg", [0, 3])
def test_each_view_passes_the_oracle_with_raw_parameters(deg):
    W, H = 80, 64
    settings, _ = _cams(1501, W, H, deg, VIEWS4[1:4], seed=7)
    raw = scene.to_raw_parameters(scene.make_cloud(1501, deg, seed=7), seed=7)
    for v in range(len(settings)):
        g = helpers.upstream_grads(H, W, seed=60 + v)
        cu = run_views(settings, raw, [g if u == v else None for u in range(len(settings))], raw=True)
        ref = helpers.run_oracle_raw(settings[v], raw, g)
        cv = _view(cu, v)
        cv["grads"] = dict(cu["grads"], means2D=cu["grads"]["means2D"][v])
        ok, rep = helpers.compare(cv, ref)
        helpers.report("views raw deg%d v%d" % (deg, v), vs_f64=rep)
        assert ok, rep


# ---- against the single-view op ------------------------------------------------------------------------------------------
def test_batch_matches_the_single_view_op():
    W, H = 128, 96
    settings, inputs = _cams(5003, W, H, 3, VIEWS4, seed=11)
    grads = [helpers.upstream_grads(H, W, seed=80 + v) for v in range(4)]
    cu = run_views(settings, inputs, grads)
    total = None
    for v in range(4):
        one = helpers.run_cuda(settings[v], inputs, grads[v])
        _forward_rule(_view(cu, v), one, "view %d" % v)
        scale = float(np.abs(one["grads"]["means2D"]).max())
        assert np.abs(cu["grads"]["means2D"][v] - one["grads"]["means2D"]).max() <= 2e-5 * scale, v
        g = {k: one["grads"][k] for k in ("means3D", "opacities", "shs", "scales", "rotations")}
        total = g if total is None else {k: total[k] + g[k] for k in g}
    _grads_close({k: cu["grads"][k] for k in total}, total, "sum over views")


def test_one_view_equals_the_single_view_op():
    settings, inputs = _cams(3000, 112, 80, 1, VIEWS4[2:3], seed=2)
    _forward_rule(_view(run_views(settings, inputs), 0), helpers.run_cuda(settings[0], inputs), "V = 1")


# ---- determinism inside the batched path ---------------------------------------------------------------------------------
def test_identical_and_permuted_cameras_give_bit_identical_views():
    settings, inputs = _cams(4000, 96, 96, 2, VIEWS4, seed=5)
    same = run_views([settings[1]] * 5, inputs)
    for v in range(1, 5):
        for k in ("color", "depth", "alpha", "radii"):
            assert np.array_equal(same[k][v], same[k][0]), (v, k)
    base = run_views(settings, inputs)
    perm = [2, 0, 3, 1]
    shuf = run_views([settings[i] for i in perm], inputs)
    for j, i in enumerate(perm):
        for k in ("color", "depth", "alpha", "radii"):
            assert np.array_equal(shuf[k][j], base[k][i]), (j, k)


# ---- protocol ------------------------------------------------------------------------------------------------------------
@pytest.fixture
def _restore():
    from dreamgaussian_b200 import rasterizer as R
    hints = dict(R._CAPACITY_HINT)
    yield
    helpers.set_tuning(helpers.DEFAULT_TUNING)
    R.set_fast_host(True)
    R._CAPACITY_HINT.clear()
    R._CAPACITY_HINT.update(hints)


def _case3():
    W, H = 96, 80
    settings, inputs = _cams(3001, W, H, 3, VIEWS4[:3], seed=9)
    return settings, inputs, [helpers.upstream_grads(H, W, seed=90 + v) for v in range(3)]


@pytest.mark.parametrize("staging", [1, 2])
def test_forced_record_staging_matches_the_default(staging, _restore):
    settings, inputs, grads = _case3()
    base = run_views(settings, inputs, grads)
    helpers.set_tuning((1, 1, staging << 22))
    got = run_views(settings, inputs, grads)
    for k in ("color", "depth", "alpha", "radii"):
        assert np.array_equal(got[k], base[k]), k
    _grads_close(got["grads"], base["grads"], "staging %d" % staging, rtol=2e-5)


def test_knobs_changed_between_forward_and_backward(_restore):
    from dreamgaussian_b200.rasterizer import rasterize_views
    settings, inputs, grads = _case3()
    base = run_views(settings, inputs, grads)
    for before, after in (((1, 1, 2 << 22), (1, 1, 1 << 22)), ((1, 1, 1 << 22), (1, 1, 2 << 22)), ((1, 1, 0), (2, 2, (1 << 21) | (1 << 25)))):
        helpers.set_tuning(before)
        t = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda")
        tin = {k: t(inputs[k]).requires_grad_(True) for k in ("means3D", "opacities", "shs", "scales", "rotations")}
        m2d = torch.zeros((3, inputs["means3D"].shape[0], 3), device="cuda", requires_grad=True)
        color, radii, depth, alpha = rasterize_views([_rs(s) for s in settings], tin["means3D"], m2d, tin["opacities"], tin["shs"],
                                                     tin["scales"], tin["rotations"])
        loss = sum(_loss(color[v], depth[v], alpha[v], grads[v], t) for v in range(3))
        helpers.set_tuning(after)
        loss.backward()
        _grads_close({k: v.grad.cpu().numpy() for k, v in tin.items()}, {k: base["grads"][k] for k in tin}, str((before, after)), rtol=2e-5)
        helpers.set_tuning(helpers.DEFAULT_TUNING)


@pytest.mark.parametrize("fast_host", [True, False])
def test_small_capacity_hint_is_repaired(fast_host, _restore):
    from dreamgaussian_b200 import rasterizer as R
    settings, inputs, grads = _case3()
    base = run_views(settings, inputs, grads)
    assert R.set_fast_host(fast_host) == fast_host
    R.set_views_capacity_hint(0, inputs["means3D"].shape[0], 80, 96, 3, 16, False)
    got = run_views(settings, inputs, grads)
    for k in ("color", "depth", "alpha", "radii"):
        assert np.array_equal(got[k], base[k]), k
    _grads_close(got["grads"], base["grads"], "repaired", rtol=2e-5)
    assert R.get_views_capacity_hint(0, inputs["means3D"].shape[0], 80, 96, 3)[0] > 16


@pytest.mark.parametrize("raw", [False, True])
def test_compiled_and_ctypes_host_layers_agree(raw, _restore):
    from dreamgaussian_b200 import rasterizer as R
    W, H = 96, 80
    settings, inputs = _cams(3001, W, H, 3, VIEWS4[:3], seed=9)
    if raw:
        inputs = scene.to_raw_parameters(scene.make_cloud(3001, 3, seed=9), seed=9)
    grads = [helpers.upstream_grads(H, W, seed=90 + v) for v in range(3)]
    assert R.set_fast_host(True)
    fast = run_views(settings, inputs, grads, raw=raw)
    assert not R.set_fast_host(False)
    slow = run_views(settings, inputs, grads, raw=raw)
    for k in ("color", "depth", "alpha", "radii"):
        assert np.array_equal(fast[k], slow[k]), k
    _grads_close(fast["grads"], slow["grads"], "host layers", rtol=2e-5)


def test_means2D_may_be_None():
    from dreamgaussian_b200.rasterizer import rasterize_views
    settings, inputs, grads = _case3()
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda")
    tin = {k: t(inputs[k]).requires_grad_(True) for k in ("means3D", "opacities", "shs", "scales", "rotations")}
    color, radii, depth, alpha = rasterize_views([_rs(s) for s in settings], tin["means3D"], None, tin["opacities"], tin["shs"],
                                                 tin["scales"], tin["rotations"])
    sum(_loss(color[v], depth[v], alpha[v], grads[v], t) for v in range(3)).backward()
    base = run_views(settings, inputs, grads)
    _grads_close({k: v.grad.cpu().numpy() for k, v in tin.items()}, {k: base["grads"][k] for k in tin}, "means2D None", rtol=2e-5)


def test_accumulate_adds_onto_a_prefilled_buffer():
    from dreamgaussian_b200 import rasterizer as R
    settings, inputs, grads = _case3()
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda")
    tin = {k: t(inputs[k]) for k in ("means3D", "opacities", "shs", "scales", "rotations")}
    color, radii, depth, alpha, state = R.views_forward_impl([_rs(s) for s in settings], tin["means3D"], tin["shs"], tin["opacities"],
                                                             tin["scales"], tin["rotations"])
    gC = torch.stack([t(g[0]) for g in grads]); gD = torch.stack([t(g[1]) for g in grads]); gA = torch.stack([t(g[2]) for g in grads])
    P = tin["means3D"].shape[0]
    shapes = dict(m3=(P, 3), m2=(3, P, 3), sh=tuple(tin["shs"].shape), op=(P, 1), sc=(P, 3), rot=(P, 4))
    fresh = {k: torch.empty(s, device="cuda") for k, s in shapes.items()}
    R.views_backward_impl(state, gC, gD, gA, fresh["m3"], fresh["m2"], fresh["sh"], fresh["op"], fresh["sc"], fresh["rot"])
    pre = {k: torch.randn(s, device="cuda") for k, s in shapes.items()}
    acc = {k: v.clone() for k, v in pre.items()}
    R.views_backward_impl(state, gC, gD, gA, acc["m3"], acc["m2"], acc["sh"], acc["op"], acc["sc"], acc["rot"], accumulate=True)
    for k in shapes:            # (the moment reductions of the backward render are float atomics: last-bit differences between runs)
        scale = float(fresh[k].abs().max())
        assert float((acc[k] - (pre[k] + fresh[k])).abs().max()) <= 2e-5 * scale + 1e-6, k


def test_retained_double_backward():
    settings, inputs, grads = _case3()
    out = run_views(settings, inputs, grads, retain=True)
    _grads_close(out["grads2"], {k: out["grads"][k] for k in out["grads2"]}, "retain_graph", rtol=2e-5)


# ---- edges ---------------------------------------------------------------------------------------------------------------
def test_a_view_looking_away_renders_the_background():
    settings, inputs = _cams(2000, 64, 48, 0, VIEWS4[:2], seed=4)
    away = dict(settings[1])
    V = np.asarray(away["viewmatrix"], np.float32).copy()
    F = np.diag([1.0, 1.0, -1.0, 1.0]).astype(np.float32)          # mirror z: the cloud is now behind the camera
    away["viewmatrix"] = V @ F
    away["projmatrix"] = away["viewmatrix"] @ (np.linalg.inv(V) @ np.asarray(settings[1]["projmatrix"], np.float32))
    out = run_views([settings[0], away], inputs)
    assert (out["radii"][1] == 0).all()
    assert np.array_equal(out["color"][1], np.broadcast_to(np.asarray(away["bg"], np.float32)[:, None, None], (3, 48, 64)))
    assert (out["alpha"][1] == 0).all() and (out["radii"][0] > 0).any()


def test_empty_cloud():
    settings, inputs = _cams(64, 64, 48, 1, VIEWS4[:2], seed=4)
    empty = {k: v[:0] for k, v in inputs.items()}
    out = run_views(settings, empty, [helpers.upstream_grads(48, 64)] * 2)
    assert out["radii"].shape == (2, 0)
    for v in range(2):
        assert np.allclose(out["color"][v], np.asarray(settings[v]["bg"])[:, None, None])


def test_batch_at_the_tile_limit_and_one_view_beyond():
    views = [(-30.0 + v, 7.2 * v, 49.1, (0.5, 0.5, 0.5)) for v in range(51)]
    settings, inputs = _cams(3000, 512, 512, 0, views, seed=6)
    g = helpers.upstream_grads(512, 512, seed=5)
    v = 37
    cu = run_views(settings[:50], inputs, [g if u == v else None for u in range(50)])      # 50 x 1024 = 51,200 tiles
    cv = _view(cu, v)
    cv["grads"] = dict(cu["grads"], means2D=cu["grads"]["means2D"][v])
    helpers.both_oracles("views 50 x 512^2 v%d" % v, settings[v], inputs, g, cu=cv)
    with pytest.raises(RuntimeError, match="51200"):
        run_views(settings, inputs)                                                          # 51 x 1024 = 52,224 tiles


# ---- launches ------------------------------------------------------------------------------------------------------------
def _launches(fn):
    from dreamgaussian_b200 import _lib
    lib = _lib.load()
    fn()                                   # settles the capacity hint
    torch.cuda.synchronize()
    lib.dgr_reset_launch_count()
    fn()
    torch.cuda.synchronize()
    return int(lib.dgr_launch_count())


def test_launch_count_does_not_grow_with_the_views():
    W, H = 96, 80
    settings, inputs = _cams(3000, W, H, 1, VIEWS4 * 2, seed=8)
    g = helpers.upstream_grads(H, W)
    counts = {V: _launches(lambda: run_views(settings[:V], inputs, [g] * V)) for V in (1, 2, 8)}
    single = _launches(lambda: helpers.run_cuda(settings[0], inputs, g))
    assert counts[1] == counts[2] == counts[8], counts
    assert counts[1] <= single, (counts, single)
