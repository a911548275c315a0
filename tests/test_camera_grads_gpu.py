"""Camera gradients on the GPU (DGR_RASTER_CAMERA_GRADS): dL/dviewmatrix, dL/dprojmatrix and dL/dcampos of every render call.

1. the translation identity (shifting the world and the camera together changes nothing), independent of any oracle;
2. parity with the float64 torch oracle on a coherent loss;
3. the entries the forward never reads are zero;
4. batched and mixed-size calls agree per view with single-view calls;
5. bit-reproducible under torch.use_deterministic_algorithms(True), across knobs, record staging and both host layers;
6. nothing changes when no camera tensor requires grad;
7. pose recovery: a perturbed camera converges back to the target pose by Adam on a 6-DoF pose."""
import math

import numpy as np
import pytest
import torch

import camgrad_helpers as C
import helpers as h
import trained_scenes as ts
from dreamgaussian_b200 import _lib, fused, scene
from dreamgaussian_b200 import rasterizer as R

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _settings(s, requires_grad=True, dtype=torch.float32):
    t = lambda a: torch.tensor(np.asarray(a, np.float64), dtype=dtype, device=DEV)
    cam = [t(s[k]).requires_grad_(requires_grad) for k in ("viewmatrix", "projmatrix", "campos")]
    rs = R.GaussianRasterizationSettings(
        image_height=s["image_height"], image_width=s["image_width"], tanfovx=s["tanfovx"], tanfovy=s["tanfovy"], bg=t(s["bg"]).float(),
        scale_modifier=s["scale_modifier"], viewmatrix=cam[0], projmatrix=cam[1], sh_degree=s["sh_degree"], campos=cam[2],
        prefiltered=False, debug=False)
    return rs, cam


def _upstream(color, depth, alpha, seed=123):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return ((color * torch.randn(color.shape, generator=gen, device=DEV)).sum() + (depth * torch.randn(depth.shape, generator=gen, device=DEV)).sum()
            + (alpha * torch.randn(alpha.shape, generator=gen, device=DEV)).sum())


def _inputs(i, kind):
    """kind: sh | colors_cov | sh_cov | colors"""
    i = dict(i)
    if kind in ("colors_cov", "sh_cov"):
        q = torch.tensor(i.pop("rotations"), dtype=torch.float64)
        Mx = C.T._quat_to_R(q / q.norm(dim=1, keepdim=True)) * torch.tensor(i.pop("scales"), dtype=torch.float64)[:, None, :]
        S = (Mx @ Mx.transpose(1, 2)).numpy()
        i["cov3D_precomp"] = np.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1).astype(np.float32)
    if kind in ("colors_cov", "colors"):
        i.pop("shs")
        i["colors_precomp"] = np.random.default_rng(5).uniform(0.05, 0.95, (len(i["means3D"]), 3)).astype(np.float32)
    return {k: torch.tensor(v, device=DEV, requires_grad=True) for k, v in i.items()}


def _single(s, tin, aa=False, cam_grad=True, loss=_upstream):
    rs, cam = _settings(s, cam_grad)
    means2D = torch.zeros_like(tin["means3D"], requires_grad=True)
    color, radii, depth, alpha = R.GaussianRasterizer(rs, antialiasing=aa)(means2D=means2D, **tin)
    loss(color, depth, alpha).backward()
    return cam, tin


def _identity_residual(Vm, PMm, dV, dPM, dc, dmean):
    """Sum_g dL/dmeans3D_g - (V[:3,:] dL/dV[3,:] + PM[:3,:] dL/dPM[3,:] - dL/dcampos), and the scale sum_g |dL/dmeans3D_g|."""
    Vm, PMm, dV, dPM, dc, dmean = (x.detach().double().cpu() for x in (Vm, PMm, dV, dPM, dc, dmean))
    rhs = Vm[:3, :] @ dV[3, :] + PMm[:3, :] @ dPM[3, :] - dc
    return (dmean.sum(0) - rhs).abs().max().item(), dmean.abs().sum().item()


# ---- 1. translation identity ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("kind,deg", [("sh", 0), ("sh", 3), ("colors_cov", 0), ("sh_cov", 2), ("colors", 0)])
def test_translation_identity_single_view(kind, deg, aa):
    s, i = h.make_case(P=3000, res=96, deg=deg, sigma=0.04, elev=20, azim=40)
    cam, tin = _single(s, _inputs(i, kind), aa=aa)
    res, scale = _identity_residual(cam[0], cam[1], cam[0].grad, cam[1].grad, cam[2].grad, tin["means3D"].grad)
    print(kind, deg, aa, "residual", res, "scale", scale)
    assert res <= 1e-5 * scale, (res, scale)


@pytest.mark.parametrize("aa", [False, True])
def test_translation_identity_raw_parameters(aa):
    s, i = h.make_case(P=3000, res=96, deg=2, sigma=0.04, elev=-15, azim=120)
    raw = {k: torch.tensor(v, device=DEV, requires_grad=True) for k, v in ts.raw_of(i).items()}
    rs, cam = _settings(s)
    color, radii, depth, alpha = fused.FusedGaussianRasterizer(rs, antialiasing=aa)(
        raw["xyz"], raw["features_dc"], raw["features_rest"], raw["opacity"], raw["scaling"], raw["rotation"])
    _upstream(color, depth, alpha).backward()
    res, scale = _identity_residual(cam[0], cam[1], cam[0].grad, cam[1].grad, cam[2].grad, raw["xyz"].grad)
    assert res <= 1e-5 * scale, (res, scale)


def _views_settings(sizes, deg, seed=0):
    out = []
    for v, (H, W) in enumerate(sizes):
        c = scene.orbit_camera(10.0 * v - 15.0, 35.0 * v, 2.0 + 0.1 * v, W, H)
        out.append(dict(image_height=H, image_width=W, tanfovx=c.tanfovx, tanfovy=c.tanfovy, bg=np.ones(3, np.float32), scale_modifier=1.0,
                        viewmatrix=c.world_view_transform, projmatrix=c.full_proj_transform, sh_degree=deg, campos=c.camera_center))
    return out


def _batched(slist, i, mixed, aa=False, raw=False, seed=7):
    """(per-view camera tensors with .grad, Gaussian tensors with .grad) of one batched call with per-view upstream gradients."""
    rss, cams = zip(*(_settings(s) for s in slist))
    V = len(slist)
    if raw:
        tin = {k: torch.tensor(v, device=DEV, requires_grad=True) for k, v in ts.raw_of(i).items()}
        args = (tin["xyz"], None, tin["features_dc"], tin["features_rest"], tin["opacity"], tin["scaling"], tin["rotation"])
        out = (fused.rasterize_views_mixed_raw if mixed else fused.rasterize_views_raw)(list(rss), *args, antialiasing=aa)
    else:
        tin = {k: torch.tensor(v, device=DEV, requires_grad=True) for k, v in i.items()}
        out = (R.rasterize_views_mixed if mixed else R.rasterize_views)(list(rss), tin["means3D"], None, tin["opacities"], tin["shs"],
                                                                        tin["scales"], tin["rotations"], antialiasing=aa)
    color, _, depth, alpha = out
    if not mixed:
        color, depth, alpha = list(color), list(depth), list(alpha)
    sum(_upstream(color[v], depth[v], alpha[v], seed=seed + v) for v in range(V)).backward()
    return cams, tin


@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("mixed", [False, True])
def test_translation_identity_batched(mixed, aa):
    sizes = [(9, 17), (64, 64), (130, 50), (33, 47)] if mixed else [(64, 80)] * 4
    s, i = h.make_case(P=3000, res=64, deg=1, sigma=0.04)
    slist = _views_settings(sizes, 1)
    cams, tin = _batched(slist, i, mixed, aa)
    rhs = sum(c[0].detach().double()[:3, :] @ c[0].grad.double()[3, :] + c[1].detach().double()[:3, :] @ c[1].grad.double()[3, :]
              - c[2].grad.double() for c in cams)
    dmean = tin["means3D"].grad.double()
    res, scale = (dmean.sum(0) - rhs).abs().max().item(), dmean.abs().sum().item()
    assert res <= 1e-5 * scale, (res, scale)


def test_rotation_identity_with_precomputed_colour_and_covariance():
    """Rotating the world by exp(eps K) and the camera with it leaves the image unchanged:
    sum_g (dmean_g x p_g + the Sigma term) + the camera's rotation terms = 0, per generator K (colors_precomp, cov3D_precomp)."""
    s, i = h.make_case(P=2000, res=96, deg=0, sigma=0.04, elev=10, azim=60)
    cam, tin = _single(s, _inputs(i, "colors_cov"))
    Vm, PM = cam[0].detach().double(), cam[1].detach().double()
    dV, dPM = cam[0].grad.double(), cam[1].grad.double()
    p, dp = tin["means3D"].detach().double(), tin["means3D"].grad.double()
    c6, dc6 = tin["cov3D_precomp"].detach().double(), tin["cov3D_precomp"].grad.double()
    sym = lambda c: torch.stack([c[:, 0], c[:, 1], c[:, 2], c[:, 1], c[:, 3], c[:, 4], c[:, 2], c[:, 4], c[:, 5]], 1).reshape(-1, 3, 3)
    S = sym(c6)
    dS = sym(dc6 * torch.tensor([1, 0.5, 0.5, 1, 0.5, 1], dtype=torch.float64, device=DEV))   # off-diagonals count twice in the packed layout
    worst, scale = 0.0, (dp.abs() * p.abs()).sum().item() + (dS.abs() * S.abs()).sum().item()
    for a in range(3):
        K = torch.zeros(3, 3, dtype=torch.float64, device=DEV)
        K[(a + 1) % 3, (a + 2) % 3], K[(a + 2) % 3, (a + 1) % 3] = -1.0, 1.0
        # world: p -> (I + eps K) p, Sigma -> Sigma + eps (K Sigma - Sigma K); the camera follows, [p',1] M' = [p,1] M:
        # M[:3,:] -> (I + eps K) M[:3,:] for M = viewmatrix and projmatrix
        world = (dp * (p @ K.t())).sum() + (dS * (K @ S - S @ K)).sum()
        camera = (dV[:3, :] * (K @ Vm[:3, :])).sum() + (dPM[:3, :] * (K @ PM[:3, :])).sum()
        worst = max(worst, abs((world + camera).item()))
    print("rotation identity residual", worst, "scale", scale)
    assert worst <= 1e-5 * scale, (worst, scale)


# ---- 2 + 3. parity with the float64 torch oracle, zero entries ----------------------------------------------------------------
PARITY = {
    "tiny_deg0": lambda: h.make_case(P=64, res=32, deg=0, sigma=0.08),
    "small_deg3": lambda: h.make_case(P=300, res=64, deg=3, sigma=0.05, elev=10, azim=30),
    "odd_size_deg1": lambda: h.make_case(P=500, res=0, width=100, height=70, deg=1, sigma=0.04, elev=-20, azim=200),
    "saturated": lambda: ts.saturated(W=64, H=64, n=400),
    "frustum_edge": lambda: ts.frustum_edge(W=64, H=48, n_near=120, n_edge=20),
}


@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("name", list(PARITY))
def test_parity_with_the_float64_oracle(name, aa):
    s, i = PARITY[name]()
    # target: the oracle's render from the camera turned by 3 degrees about its own y axis (p_view' = Ry p_view)
    th = math.radians(3.0)
    Ry = np.array([[math.cos(th), 0, -math.sin(th), 0], [0, 1, 0, 0], [math.sin(th), 0, math.cos(th), 0], [0, 0, 0, 1]])
    V0 = np.asarray(s["viewmatrix"], np.float64)
    s_t = dict(s, viewmatrix=V0 @ Ry)
    s_t["projmatrix"] = s_t["viewmatrix"] @ np.linalg.solve(V0, np.asarray(s["projmatrix"], np.float64))
    tin64 = {k: torch.tensor(np.asarray(v, np.float64)) for k, v in i.items()}
    with torch.no_grad():
        target = C.oracle_render(s_t, tin64, *(torch.tensor(np.asarray(s_t[k], np.float64)) for k in ("viewmatrix", "projmatrix", "campos")),
                                 antialiased=aa)[0]

    def loss(color, depth, alpha):
        tg = target.to(color.device, color.dtype)
        return ((color - tg) ** 2).mean() + 0.1 * alpha.mean()

    g64 = [g.numpy() if g is not None else np.zeros(3) for g in C.oracle_camera_grads(s, i, loss, antialiased=aa)]
    g32 = [g.numpy() if g is not None else np.zeros(3) for g in C.oracle_camera_grads(s, i, loss, antialiased=aa, dtype=torch.float32)]
    cam, _ = _single(s, {k: torch.tensor(v, device=DEV, requires_grad=True) for k, v in i.items()}, aa=aa, loss=loss)
    gcu = [c.grad.cpu().numpy() for c in cam]
    for n, a, b, f in zip(("viewmatrix", "projmatrix", "campos"), gcu, g64, g32):
        scale = max(np.abs(b).max(), 1e-12)
        d, d32 = np.abs(a - b).max() / scale, np.abs(f - b).max() / scale
        print("%s aa=%d %s: |cuda - f64| / max|f64| = %.2e, float32 oracle: %.2e" % (name, aa, n, d, d32))
        assert d <= max(1e-3, 3 * d32), (n, d, d32)
    # 3. entries the forward never reads
    assert (gcu[0].reshape(4, 4)[:, 3] == 0).all() and (gcu[1].reshape(4, 4)[:, 2] == 0).all()
    if s["sh_degree"] == 0:
        assert (gcu[2] == 0).all()


def test_zero_campos_gradient_with_precomputed_colours():
    s, i = h.make_case(P=500, res=64, deg=2, sigma=0.05)
    cam, _ = _single(s, _inputs(i, "colors"))
    assert (cam[2].grad == 0).all() and (cam[0].grad[:, 3] == 0).all() and (cam[1].grad[:, 2] == 0).all()
    assert cam[0].grad.abs().max() > 0 and cam[1].grad.abs().max() > 0


# ---- 4. batched calls agree with single-view calls ------------------------------------------------------------------------------
@pytest.mark.parametrize("raw", [False, True])
@pytest.mark.parametrize("mixed", [False, True])
def test_batched_calls_agree_with_single_views(mixed, raw):
    sizes = [(9, 17), (64, 64), (130, 50), (40, 72)] if mixed else [(64, 80)] * 3
    s, i = h.make_case(P=2000, res=64, deg=2, sigma=0.04)
    slist = _views_settings(sizes, 2)
    cams, _ = _batched(slist, i, mixed, raw=raw)
    for v, sv in enumerate(slist):
        if raw:
            rawi = {k: torch.tensor(x, device=DEV, requires_grad=True) for k, x in ts.raw_of(i).items()}
            rs, cam = _settings(sv)
            color, _, depth, alpha = fused.FusedGaussianRasterizer(rs)(rawi["xyz"], rawi["features_dc"], rawi["features_rest"], rawi["opacity"],
                                                                       rawi["scaling"], rawi["rotation"])
            _upstream(color, depth, alpha, seed=7 + v).backward()
        else:
            cam, _ = _single(dict(sv), {k: torch.tensor(x, device=DEV, requires_grad=True) for k, x in i.items()},
                             loss=lambda c, d, a, v=v: _upstream(c, d, a, seed=7 + v))
        for a, b in zip(cams[v], cam):
            scale = b.grad.abs().max().item()
            assert (a.grad - b.grad).abs().max().item() <= 2e-4 * scale + 1e-6, (v, (a.grad - b.grad).abs().max().item(), scale)


def test_transposed_view_and_float64_cameras_get_their_own_gradients():
    """The reference builds viewmatrix as a transposed view; autograd must route the gradient back through it."""
    s, i = h.make_case(P=1000, res=64, deg=1, sigma=0.04)
    w2c = torch.tensor(np.asarray(s["viewmatrix"], np.float64).T, device=DEV, requires_grad=True)
    rs, cam = _settings(s)
    rs = rs._replace(viewmatrix=w2c.transpose(0, 1))
    tin = {k: torch.tensor(v, device=DEV, requires_grad=True) for k, v in i.items()}
    color, _, depth, alpha = R.GaussianRasterizer(rs)(means2D=torch.zeros_like(tin["means3D"]), **tin)
    _upstream(color, depth, alpha).backward()
    ref, _ = _single(s, {k: torch.tensor(v, device=DEV, requires_grad=True) for k, v in i.items()})
    assert w2c.grad.dtype == torch.float64 and w2c.grad.shape == (4, 4)
    assert (w2c.grad.t().float() - ref[0].grad).abs().max() <= 2e-5 * ref[0].grad.abs().max()       # float atomics: not bit-exact


# ---- 5. determinism ------------------------------------------------------------------------------------------------------------
@pytest.fixture
def deterministic():
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(False)
        h.set_tuning(h.DEFAULT_TUNING)
        R.set_fast_host(True)


def _cam_grads_single(s, i, aa):
    cam, _ = _single(s, {k: torch.tensor(v, device=DEV, requires_grad=True) for k, v in i.items()}, aa=aa)
    return [c.grad.clone() for c in cam]


@pytest.mark.parametrize("aa", [False, True])
def test_deterministic_camera_grads_are_bit_identical(deterministic, aa):
    s, i = h.make_case(P=20000, res=128, deg=3, sigma=0.02)
    base = _cam_grads_single(s, i, aa)
    words = [h.DEFAULT_TUNING, (2, 2, 1), (1, 1, 1 | (1 << 22)), (1, 1, 1 | (2 << 22)), (1, 1, 1 | (1 << 25))]
    for word in words:
        for fast in (True, False):
            got = h.run_tuned(word, lambda: _cam_grads_single(s, i, aa), fast_host=fast)
            for a, b in zip(got, base):
                assert torch.equal(a, b), (word, fast)
    slist = _views_settings([(64, 64), (48, 96), (130, 50)], 3)
    first = [[c.grad.clone() for c in cv] for cv in _batched(slist, i, True, aa)[0]]
    for fast in (True, False):
        R.set_fast_host(fast)
        again = [[c.grad.clone() for c in cv] for cv in _batched(slist, i, True, aa)[0]]
        assert all(torch.equal(a, b) for x, y in zip(first, again) for a, b in zip(x, y)), fast


# ---- 6. nothing changes when nothing asks ---------------------------------------------------------------------------------------
def _profiled_backward(s, i, cam_grad):
    """The kernels one backward launches (profiling is per host thread: the backward runs here, not in autograd's device thread)."""
    lib = _lib.load()
    rs, cam = _settings(s, cam_grad)
    tin = {k: torch.tensor(v, device=DEV, requires_grad=True) for k, v in i.items()}
    color, _, depth, alpha = R.GaussianRasterizer(rs)(means2D=torch.zeros_like(tin["means3D"], requires_grad=True), **tin)
    gen = torch.Generator(device=DEV).manual_seed(5)
    gC, gD, gA = (torch.randn(x.shape, generator=gen, device=DEV) for x in (color, depth, alpha))
    P = tin["means3D"].shape[0]
    e = lambda *shape: torch.empty(shape, device=DEV)
    outs = [e(P, 3), e(P, 3), e(*tin["shs"].shape), None, e(P, 1), e(P, 3), e(P, 4), None]
    camera = R._camera_outputs(0, DEV) if cam_grad else None
    torch.cuda.synchronize()
    lib.dgr_profile_enable(1)
    R.backward_impl(color.grad_fn.state, gC, gD, gA, *outs, camera=camera)
    torch.cuda.synchronize()
    names = [n for n, _ in _lib.profile_collect()]
    lib.dgr_profile_enable(0)
    return names, [o for o in outs if o is not None]


def test_without_camera_grads_the_backward_is_unchanged(deterministic):
    s, i = h.make_case(P=20000, res=128, deg=3, sigma=0.02)
    for fast in (True, False):
        R.set_fast_host(fast)
        names0, g0 = _profiled_backward(s, i, False)
        names1, g1 = _profiled_backward(s, i, True)
        assert not any(n.startswith("camera_") for n in names0), names0
        assert names1 == names0 + ["camera_bwd", "camera_reduce"], (names0, names1)
        for a, b in zip(g0, g1):
            assert torch.equal(a, b)                    # asking for camera gradients changes no Gaussian gradient
    # no gradient is asked for under no_grad-built settings either: the autograd function gets no extra inputs
    rs, cam = _settings(s, True)
    with torch.no_grad():
        assert R._camera_tensors([rs]) == ()
    assert len(R._camera_tensors([rs])) == 3 and R._camera_tensors([_settings(s, False)[0]]) == ()


# ---- 7. pose recovery -----------------------------------------------------------------------------------------------------------
POSE_FRACTION = 0.05          # final rotation / translation error below this fraction of the initial one


def _pose_recovery(aa, fast, steps=300):
    R.set_fast_host(fast)
    W = H = 256
    cloud = scene.make_cloud(20000, 0, seed=3, sigma=0.012)
    tin = {k: torch.tensor(cloud[k], device=DEV) for k in ("means3D", "opacities", "shs", "scales", "rotations")}
    bg = torch.ones(3, device=DEV)
    target_c2w = torch.tensor(scene.orbit_pose(-10.0, 20.0, 2.0), dtype=torch.float32, device=DEV)
    start_c2w = torch.tensor(scene.orbit_pose(-4.0, 26.0, 2.1), dtype=torch.float32, device=DEV)

    def render(c2w):
        V, PM, campos, tx, ty = C.minicam(c2w, W, H)
        rs = R.GaussianRasterizationSettings(H, W, tx, ty, bg, 1.0, V, PM, 0, campos, False, False)
        color, _, _, alpha = R.GaussianRasterizer(rs, antialiasing=aa)(means3D=tin["means3D"], means2D=torch.zeros_like(tin["means3D"]),
                                                                      opacities=tin["opacities"],
                                                                      shs=tin["shs"], scales=tin["scales"], rotations=tin["rotations"])
        return color, alpha

    with torch.no_grad():
        tc, ta = render(target_c2w)
    delta = torch.zeros(6, device=DEV, requires_grad=True)
    opt = torch.optim.Adam([delta], lr=4e-3)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, steps, eta_min=2e-4)
    err = lambda c2w: (C.rotation_angle(c2w[:3, :3].double().cpu(), target_c2w[:3, :3].double().cpu()),
                       float((c2w[:3, 3] - target_c2w[:3, 3]).norm()))
    e0 = err(start_c2w)
    for _ in range(steps):
        opt.zero_grad()
        c, a = render(C.pose_of(start_c2w, delta))
        loss = (c - tc).abs().mean() + (a - ta).abs().mean()
        loss.backward()
        opt.step()
        sched.step()
    e1 = err(C.pose_of(start_c2w, delta).detach())
    return e0, e1


@pytest.mark.parametrize("aa,fast", [(False, True), (False, False), (True, True)])
def test_pose_recovery(aa, fast):
    try:
        (r0, t0), (r1, t1) = _pose_recovery(aa, fast)
    finally:
        R.set_fast_host(True)
    print("pose recovery aa=%d fast=%d: rotation %.4f -> %.5f rad, translation %.4f -> %.5f" % (aa, fast, r0, r1, t0, t1))
    assert r1 <= POSE_FRACTION * r0 and t1 <= POSE_FRACTION * t0, (r0, r1, t0, t1)
