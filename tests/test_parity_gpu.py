"""GPU parity tests: the CUDA path (public API -> C ABI -> sm_90a kernels) against the float64 CPU oracle on the same
seeded inputs, plus size-independent properties at BASELINE.json's full sizes.  Tolerances: tests/helpers.py."""
import ctypes

import numpy as np
import pytest
import torch

import helpers as h
from dreamgaussian_b200 import _lib, multiview, scene
from dreamgaussian_b200 import rasterizer as R

pytestmark = pytest.mark.gpu

CASES = {
    "tiny_deg0": dict(P=64, res=32, deg=0, sigma=0.08),
    "small_deg3": dict(P=300, res=64, deg=3, sigma=0.05, elev=10, azim=30),
    "odd_size_deg1": dict(P=500, res=0, width=100, height=70, deg=1, sigma=0.04, elev=-20, azim=200),
    "cfg1_5k_256_init": dict(P=5000, res=256, deg=0, opacity="init", anisotropic=False),      # BASELINE.json configs[0]
    "big_gaussians_deg2": dict(P=500, res=80, deg=2, sigma=0.2, elev=25, azim=-100),          # J clamp, near cull, huge radii
    "mid_20k_400_deg3": dict(P=20000, res=400, deg=3),
    "scale_modifier": dict(P=400, res=64, deg=1, sigma=0.04, scale_modifier=1.6, bg=(0.2, 0.7, 0.1)),
    "big_tiles": dict(P=20000, res=32, deg=0, sigma=0.02),             # ~5k instances per tile: big-tile sorter
    "huge_tiles": dict(P=60000, res=32, deg=0, sigma=0.01),            # > 12288 per tile: in-place global sort path
}


both_oracles = h.both_oracles          # the rule of the suite (tests/helpers.py)


@pytest.mark.parametrize("name", list(CASES))
def test_forward_backward_parity(name):
    s, i = h.make_case(**CASES[name])
    both_oracles(name, s, i, h.upstream_grads(s["image_height"], s["image_width"]))


def test_cfg2_full_size_parity():
    """BASELINE.json configs[1]: 100k Gaussians, 800x800, SH degree 3, forward + backward."""
    s, i = h.make_case(P=100000, res=800, deg=3)
    both_oracles("cfg2_100k_800", s, i, h.upstream_grads(800, 800))


def test_cfg2_at_the_reference_initial_opacity_full_size_parity():
    """configs[1] with every opacity at the reference's initial 0.1 (gs_renderer.py:346): no early termination, every list is
    walked to its end.  8 % of the pixels sit within float32 reach of the alpha >= 1/255 contour of some Gaussian (each
    Gaussian's footprint ends on that contour at o = 0.1), hence the larger allowance for flagged pixels against float64."""
    s, i = h.make_case(P=100000, res=800, deg=3, opacity="init")
    both_oracles("cfg2_100k_800_init", s, i, h.upstream_grads(800, 800), max_ambig_frac=0.12)


def test_cfg3_view_full_size_parity():
    """One view of BASELINE.json configs[2] (500k Gaussians, 512x512, SH degree 3; ~2000-entry pixel lists, big-tile sorter).
    Float32 depth keys tie between consecutive contributors here: the float64 comparison allows a tied pixel the colour shift
    of its ties (oracle tie_slack) and sets aside the Gaussians compositing in front of a material tie (flag bit 16)."""
    s, i = h.make_case(P=500000, res=512, deg=3, sigma=0.0075, elev=-12, azim=75)
    both_oracles("cfg3_view_500k_512", s, i, h.upstream_grads(512, 512, depth=False))


def test_cfg5_full_size_parity_against_the_float32_oracle():
    """BASELINE.json configs[4]: 2M Gaussians, 1600x1600, SH degree 3 (14 M tile instances, big-tile sorter on most tiles),
    forward + backward against the float32 oracle (the float64 one adds nothing here: the deviations between the two CPU
    builds at this depth complexity are float32 depth-key ties, DESIGN.md §2)."""
    s, i = h.make_case(P=2000000, res=1600, deg=3, sigma=0.595 * 2000000 ** (-1.0 / 3.0), elev=10, azim=30)
    both_oracles("cfg5_2M_1600", s, i, h.upstream_grads(1600, 1600, depth=False), f64=False)


def test_equal_depths_resolve_by_index_like_the_reference():
    """All Gaussians at the same view depth: the (tile, depth) sort must fall back to Gaussian-index order."""
    s, i = h.make_case(P=3000, res=64, deg=1, sigma=0.03)
    i["means3D"] = i["means3D"].copy(); i["means3D"][:, 2] = 0.0
    g = h.upstream_grads(64, 64)
    ref = h.run_oracle(s, i, g)
    cu = h.run_cuda(s, i, g)
    for k in ("color", "depth", "alpha"):          # every pixel is "ambiguous" for float32 here, but the order is pinned
        assert np.abs(cu[k] - ref[k]).max() < 1e-4, k
    assert (cu["radii"] == ref["radii"]).all()
    for k, v in ref["grads"].items():
        if k in cu["grads"]:
            assert np.abs(cu["grads"][k].reshape(v.shape) - v).max() <= 2e-3 * max(np.abs(v).max(), 1e-6), k


def _torch_inputs(i, dev="cuda"):
    return {k: torch.tensor(v, device=dev) for k, v in i.items()}


def _settings(s, dev="cuda"):
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device=dev)
    return R.GaussianRasterizationSettings(
        image_height=s["image_height"], image_width=s["image_width"], tanfovx=s["tanfovx"], tanfovy=s["tanfovy"], bg=t(s["bg"]),
        scale_modifier=s["scale_modifier"], viewmatrix=t(s["viewmatrix"]), projmatrix=t(s["projmatrix"]), sh_degree=s["sh_degree"],
        campos=t(s["campos"]), prefiltered=False, debug=False)


def test_precomputed_colour_and_covariance_paths():
    s, i = h.make_case(P=600, res=64, deg=0, sigma=0.05, elev=5, azim=140)
    rng = np.random.default_rng(3)
    q, sc = i["rotations"].astype(np.float64), i["scales"].astype(np.float64)
    Rm = np.stack([
        1 - 2 * (q[:, 2] ** 2 + q[:, 3] ** 2), 2 * (q[:, 1] * q[:, 2] - q[:, 0] * q[:, 3]), 2 * (q[:, 1] * q[:, 3] + q[:, 0] * q[:, 2]),
        2 * (q[:, 1] * q[:, 2] + q[:, 0] * q[:, 3]), 1 - 2 * (q[:, 1] ** 2 + q[:, 3] ** 2), 2 * (q[:, 2] * q[:, 3] - q[:, 0] * q[:, 1]),
        2 * (q[:, 1] * q[:, 3] - q[:, 0] * q[:, 2]), 2 * (q[:, 2] * q[:, 3] + q[:, 0] * q[:, 1]), 1 - 2 * (q[:, 1] ** 2 + q[:, 2] ** 2)],
        1).reshape(-1, 3, 3)
    Mx = Rm * sc[:, None, :]
    S = Mx @ Mx.transpose(0, 2, 1)
    cov6 = np.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1).astype(np.float32)
    inp = dict(means3D=i["means3D"], opacities=i["opacities"], colors_precomp=rng.random((600, 3)).astype(np.float32), cov3D_precomp=cov6)
    g = h.upstream_grads(64, 64)
    ok, rep = h.compare(h.run_cuda(s, inp, g), h.run_oracle(s, inp, g))
    assert ok, rep


def test_empty_cloud_and_offscreen_cloud():
    s, i = h.make_case(P=50, res=40, deg=0, sigma=0.05, bg=(0.3, 0.6, 0.9))
    rs = _settings(s)
    z = lambda *shape: torch.zeros(*shape, device="cuda")
    color, radii, depth, alpha = R.GaussianRasterizer(rs)(means3D=z(0, 3), means2D=z(0, 3), opacities=z(0, 1), shs=z(0, 1, 3),
                                                          scales=z(0, 3), rotations=z(0, 4))
    assert radii.numel() == 0 and float(alpha.abs().max()) == 0.0
    assert torch.allclose(color, torch.tensor([0.3, 0.6, 0.9], device="cuda")[:, None, None].expand_as(color))
    ti = _torch_inputs(i)
    ti["means3D"] = ti["means3D"] + torch.tensor([0.0, 0.0, 10.0], device="cuda")         # behind the eye: everything culled
    for v in ti.values():
        v.requires_grad_(True)
    color, radii, depth, alpha = R.GaussianRasterizer(rs)(means2D=torch.zeros_like(ti["means3D"]), **ti)
    assert int(radii.max()) == 0 and float(alpha.max()) == 0.0
    (color.sum() + alpha.sum()).backward()
    assert all(float(v.grad.abs().max()) == 0.0 for v in ti.values())


def test_mark_visible_and_input_validation():
    s, i = h.make_case(P=200, res=32, deg=0, sigma=0.05)
    rs = _settings(s)
    pos = torch.tensor(i["means3D"], device="cuda")
    pos[:7, 2] += 10.0
    vis = R.GaussianRasterizer(rs).markVisible(pos)
    V = np.asarray(s["viewmatrix"], np.float64)
    tz = np.concatenate([pos.cpu().numpy().astype(np.float64), np.ones((200, 1))], 1) @ V[:, 2]
    assert vis.dtype == torch.bool and (vis.cpu().numpy() == (tz > 0.2)).all() and not vis[:7].any()
    ti = _torch_inputs(i)
    with pytest.raises(ValueError):
        R.GaussianRasterizer(rs)(means3D=ti["means3D"][:, :2], means2D=ti["means3D"], opacities=ti["opacities"], shs=ti["shs"],
                                 scales=ti["scales"], rotations=ti["rotations"])
    # a non-contiguous viewmatrix (the reference passes a transposed view, gs_renderer.py:662) is accepted
    rs2 = rs._replace(viewmatrix=rs.viewmatrix.t().contiguous().t())
    a = R.GaussianRasterizer(rs)(means2D=torch.zeros_like(ti["means3D"]), **ti)[0]
    b = R.GaussianRasterizer(rs2)(means2D=torch.zeros_like(ti["means3D"]), **ti)[0]
    assert torch.equal(a, b)


@pytest.mark.parametrize("case", ["plain", "raw"])
def test_staged_and_per_thread_input_paths_and_both_step2_forms_agree(case):
    """dgr_set_tuning bits 24 / 25: the per-Gaussian kernels read their inputs through bulk-TMA staging (full warps) or with
    per-thread loads — same registers, same expressions.  Bit 26: step 2 of the backward render in its per-row or per-pixel
    form — same sums in a different association: float32 round-off only.  P is not a multiple of 32, so the staged
    runs mix both input paths in one launch."""
    lib = _lib.load()
    if case == "plain":
        s, i = h.make_case(P=20011, res=400, deg=3)
        run = lambda: h.run_cuda(s, i, g)
    else:
        s, i = h.make_case(P=9007, res=200, deg=2)
        raw = scene.to_raw_parameters(i)
        run = lambda: h.run_cuda_raw(s, raw, g)
    g = h.upstream_grads(s["image_height"], s["image_width"])
    try:
        base = run()                                                  # defaults: staged inputs, per-row step 2
        # (gradients: the backward render accumulates the moments with red.global.add in whatever order the warps arrive, so two
        #  runs of the SAME variant already differ in the last bits; the images and radii are deterministic)
        for bits in (1 << 24, 1 << 25, (1 << 24) | (1 << 25), 1 << 26, 7 << 24):
            _lib.check(lib.dgr_set_tuning(1, 1, 1 | bits))
            other = run()
            # the forward: the two instantiations of a kernel hold the same expressions, but ptxas decides per instantiation which
            # multiply-add pairs it fuses, so their float32 results may differ in the last bits (both equally valid): images to
            # 2e-6 except a handful of pixels next to a decision threshold, radii equal except where ceil(3 sigma) sits on an integer
            for k in ("color", "depth", "alpha"):
                d = np.abs(base[k] - other[k]) / max(1.0, float(np.abs(base[k]).max()))
                assert float((d > 2e-6).mean()) <= 1e-4 and float(d.max()) <= 1e-2, (bits, k, float(d.max()), float((d > 2e-6).mean()))
            assert int((base["radii"] != other["radii"]).sum()) <= 2, bits
            for k, v in base["grads"].items():
                scale = float(np.abs(v).max())
                if scale > 0:
                    assert float(np.abs(v - other["grads"][k]).max()) <= 2e-5 * scale, (bits, k)
    finally:
        _lib.check(lib.dgr_set_tuning(1, 1, 1))


def test_input_views_that_start_off_a_16_byte_boundary_are_accepted():
    """Contiguous views into a larger buffer (``flat[1:].view(P, K)``: 4-byte aligned only) give the same result as fresh tensors:
    the host layer re-allocates them (the kernels use 128-bit loads and bulk-TMA staging, include/dgr_b200.h)."""
    s, i = h.make_case(P=1500, res=96, deg=3, sigma=0.04, elev=10, azim=50)
    ti, rs = _torch_inputs(i), _settings(s)
    off = {}
    for k, v in ti.items():
        flat = torch.empty(v.numel() + 1, dtype=torch.float32, device=v.device)
        flat[1:] = v.reshape(-1)
        off[k] = flat[1:].view(v.shape)
        assert off[k].data_ptr() % 16 != 0 and off[k].is_contiguous()
    a = R.GaussianRasterizer(rs)(means2D=torch.zeros_like(ti["means3D"]), **ti)
    b = R.GaussianRasterizer(rs)(means2D=torch.zeros_like(ti["means3D"]), **off)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_padded_sh_storage_with_lower_active_degree():
    """gs_renderer.py:806 passes get_features ([P, (max_sh_degree+1)^2, 3]) with sh_degree=active_sh_degree: the storage can
    hold more coefficients than the active degree reads.  Unused coefficients change nothing and get zero gradient."""
    s, i = h.make_case(P=600, res=72, deg=1, sigma=0.05, elev=15, azim=70)
    rng = np.random.default_rng(3)
    padded = dict(i)
    padded["shs"] = np.concatenate([i["shs"], rng.normal(size=(600, 12, 3)).astype(np.float32)], axis=1)      # M = 16, 4 in use
    g = h.upstream_grads(72, 72)
    ref = h.run_oracle(s, padded, g)
    cu = h.run_cuda(s, padded, g)
    ok, rep = h.compare(cu, ref)
    assert ok, rep
    assert cu["grads"]["shs"].shape == (600, 16, 3)
    assert not cu["grads"]["shs"][:, 4:].any()
    small = h.run_cuda(s, i, g)
    assert np.array_equal(cu["color"], small["color"])
    assert np.array_equal(cu["grads"]["shs"][:, :4], small["grads"]["shs"]) or \
        np.abs(cu["grads"]["shs"][:, :4] - small["grads"]["shs"]).max() <= 2e-5 * np.abs(small["grads"]["shs"]).max()


RAW_CASES = {
    "raw_deg0": dict(P=300, res=64, deg=0, sigma=0.06, elev=5, azim=20),                 # _features_rest is [P,0,3]
    "raw_deg1": dict(P=400, res=64, deg=1, sigma=0.05, elev=-10, azim=120),
    "raw_deg2_scale_modifier": dict(P=500, res=80, deg=2, sigma=0.05, elev=25, azim=-100, scale_modifier=1.4),
    "raw_deg3_20k_400": dict(P=20000, res=400, deg=3),
}


@pytest.mark.parametrize("name", list(RAW_CASES))
def test_fused_activation_path_parity(name):
    """SURVEY §8 f1: raw GaussianModel parameters in, activations + their chain rule inside the kernels."""
    s, i = h.make_case(**RAW_CASES[name])
    raw = scene.to_raw_parameters(i)
    g = h.upstream_grads(s["image_height"], s["image_width"])
    ok, rep = h.compare(h.run_cuda_raw(s, raw, g), h.run_oracle_raw(s, raw, g))
    assert ok, rep


def test_fused_path_matches_torch_activations_plus_plain_op_and_updates_densify_stats():
    from dreamgaussian_b200.fused import DensifyStats, FusedGaussianRasterizer
    s, i = h.make_case(P=3000, res=128, deg=3, sigma=0.03)
    raw = {k: torch.tensor(v, device="cuda") for k, v in scene.to_raw_parameters(i).items()}
    rs = _settings(s)
    # reference formulation (gs_renderer.py:196-216, 762-806): torch activations + cat, then the plain op
    lv = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
    m2d = torch.zeros_like(lv["xyz"], requires_grad=True)
    img, radii, depth, alpha = R.GaussianRasterizer(rs)(
        means3D=lv["xyz"], means2D=m2d, shs=torch.cat((lv["features_dc"], lv["features_rest"]), dim=1),
        opacities=torch.sigmoid(lv["opacity"]), scales=torch.exp(lv["scaling"]), rotations=torch.nn.functional.normalize(lv["rotation"]))
    gen = torch.Generator(device="cuda").manual_seed(11)
    up, upa = torch.randn(img.shape, device="cuda", generator=gen), torch.randn(alpha.shape, device="cuda", generator=gen)
    ((img * up).sum() + (alpha * upa).sum()).backward()
    # fused
    lf = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
    m2f = torch.zeros_like(lf["xyz"], requires_grad=True)
    stats = DensifyStats(3000, "cuda")
    stats.max_radii2D.fill_(3.0)
    out = FusedGaussianRasterizer(rs)(lf["xyz"], lf["features_dc"], lf["features_rest"], lf["opacity"], lf["scaling"], lf["rotation"],
                                      means2D=m2f, stats=stats)
    ((out[0] * up).sum() + (out[3] * upa).sum()).backward()
    assert torch.equal(out[1], radii)
    assert float((out[0] - img).abs().max()) <= 2e-5 and float((out[3] - alpha).abs().max()) <= 2e-5
    for k in lv:
        a, b = lf[k].grad, lv[k].grad
        assert float((a - b).abs().max()) <= 2e-4 * float(b.abs().max()) + 1e-12, k
    vis = radii > 0
    norm = m2f.grad[:, :2].norm(dim=-1)
    assert torch.allclose(stats.xyz_gradient_accum[vis], norm[vis], rtol=1e-5, atol=1e-12) and not stats.xyz_gradient_accum[~vis].any()
    assert torch.equal(stats.denom, vis.float())
    want = torch.where(vis, torch.maximum(torch.full_like(stats.max_radii2D, 3.0), radii.float()), torch.full_like(stats.max_radii2D, 3.0))
    assert torch.equal(stats.max_radii2D, want)
    # a second render accumulates
    lf2 = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
    out2 = FusedGaussianRasterizer(rs)(lf2["xyz"], lf2["features_dc"], lf2["features_rest"], lf2["opacity"], lf2["scaling"], lf2["rotation"],
                                       stats=stats)
    ((out2[0] * up).sum() + (out2[3] * upa).sum()).backward()
    assert torch.equal(stats.denom, 2 * vis.float())
    assert torch.allclose(stats.xyz_gradient_accum[vis], 2 * norm[vis], rtol=1e-4, atol=1e-12)


def test_backward_twice_of_one_forward_gives_the_same_gradients():
    """retain_graph: a second backward through the same forward runs from the same geometry / binning / image buffers and
    must not see the first one's per-Gaussian moment accumulators."""
    s, i = h.make_case(P=5000, res=160, deg=2)
    ti, rs = _torch_inputs(i), _settings(s)
    leaves = {k: v.clone().requires_grad_(True) for k, v in ti.items()}
    m2d = torch.zeros_like(ti["means3D"], requires_grad=True)
    img, radii, depth, alpha = R.GaussianRasterizer(rs)(means2D=m2d, **leaves)
    g = torch.Generator(device="cuda").manual_seed(5)
    up = torch.randn(img.shape, device="cuda", generator=g)
    loss = (img * up).sum() + alpha.sum()
    names = list(leaves)
    first = torch.autograd.grad(loss, [leaves[k] for k in names] + [m2d], retain_graph=True)
    second = torch.autograd.grad(loss, [leaves[k] for k in names] + [m2d])
    for a, b, k in zip(first, second, names + ["means2D"]):
        scale = float(a.abs().max()) + 1e-20
        assert float((a - b).abs().max()) <= 2e-5 * scale, k      # float atomics: order differs, values do not


def test_compiled_host_layer_and_ctypes_layer_give_identical_results():
    """csrc/dgr_torch.cpp (compiled binding) and the ctypes binding issue the same C-ABI calls: bit-identical images, and
    gradients equal up to the order of the float atomics."""
    if not R.set_fast_host(True):
        pytest.skip("dgr_torch_host.so not built")
    s, i = h.make_case(P=6000, res=160, deg=3)
    g = h.upstream_grads(160, 160)
    try:
        fast = h.run_cuda(s, i, g)
        assert R.set_fast_host(False) is False
        slow = h.run_cuda(s, i, g)
    finally:
        R.set_fast_host(True)
    for k in ("color", "depth", "alpha", "radii"):
        assert np.array_equal(fast[k], slow[k]), k
    for k, v in slow["grads"].items():
        assert np.abs(fast["grads"][k] - v).max() <= 2e-5 * (np.abs(v).max() + 1e-20), k


def test_capacity_guess_too_small_is_repaired():
    s, i = h.make_case(P=3000, res=128, deg=1, sigma=0.05)
    ti, rs = _torch_inputs(i), _settings(s)
    ref = [o.clone() for o in R.GaussianRasterizer(rs)(means2D=torch.zeros_like(ti["means3D"]), **ti)]
    key = (torch.cuda.current_device(), 3000, 128, 128)
    assert R.get_capacity_hint(*key) is not None
    R.set_capacity_hint(*key, 64, False)                     # absurdly small instance buffer, no big-tile sorter
    out = R.GaussianRasterizer(rs)(means2D=torch.zeros_like(ti["means3D"]), **ti)
    for a, b in zip(ref, out):
        assert torch.equal(a, b)
    assert R.get_capacity_hint(*key)[0] > 64


def test_view_accumulation_equals_sum_of_views():
    """DgrGaussianGrads.accumulate: two views into one flat buffer == sum of the per-view autograd gradients."""
    P, deg, res = 4000, 2, 160
    cloud = scene.make_cloud(P, deg, seed=1)
    dev = torch.device("cuda")
    params = {k: torch.tensor(v, device=dev) for k, v in cloud.items()}
    cams = scene.bench_views(2, res, res)
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device=dev)
    sets = [R.GaussianRasterizationSettings(image_height=res, image_width=res, tanfovx=c.tanfovx, tanfovy=c.tanfovy, bg=t(np.ones(3)),
                                            scale_modifier=1.0, viewmatrix=t(c.world_view_transform), projmatrix=t(c.full_proj_transform),
                                            sh_degree=deg, campos=t(c.camera_center), prefiltered=False, debug=False) for c in cams]
    ups = [(t(g[0]), None, t(g[2])) for g in (h.upstream_grads(res, res, seed=7), h.upstream_grads(res, res, seed=8))]
    vsr = multiview.ViewShardedRasterizer(P, (deg + 1) ** 2, dev)
    vsr.render_views(params, sets, ups)
    total = {k: torch.zeros_like(v) for k, v in params.items()}
    for rs, up in zip(sets, ups):
        pin = {k: v.clone().requires_grad_(True) for k, v in params.items()}
        color, radii, depth, alpha = R.GaussianRasterizer(rs)(means3D=pin["means3D"], means2D=torch.zeros_like(pin["means3D"]),
                                                              opacities=pin["opacities"], shs=pin["shs"], scales=pin["scales"],
                                                              rotations=pin["rotations"])
        ((color * up[0]).sum() + (alpha * up[2]).sum()).backward()
        for k in total:
            total[k] += pin[k].grad
    for k in total:
        got = vsr.grads.views[k]
        scale = float(total[k].abs().max())
        assert float((got - total[k]).abs().max()) <= 2e-4 * scale + 1e-6, k     # atomics: summation order differs


def test_full_size_properties_cfg5_like():
    """Size-independent checks at a bandwidth-stress size (1M Gaussians, 1600x1600): alpha in [0,1], colour bounded by the
    convex combination, gradients linear in the upstream gradient."""
    P, deg, res = 1000000, 3, 1600
    cloud = scene.make_cloud(P, deg, seed=2, sigma=0.006)
    dev = torch.device("cuda")
    params = {k: torch.tensor(v, device=dev) for k, v in cloud.items()}
    cam = scene.orbit_camera(10, 30, 2.0, res, res)
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device=dev)
    rs = R.GaussianRasterizationSettings(image_height=res, image_width=res, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=t(np.zeros(3)),
                                         scale_modifier=1.0, viewmatrix=t(cam.world_view_transform), projmatrix=t(cam.full_proj_transform),
                                         sh_degree=deg, campos=t(cam.camera_center), prefiltered=False, debug=False)
    g1 = torch.randn(3, res, res, device=dev); g2 = torch.randn(3, res, res, device=dev)

    def grads(gc):
        pin = {k: v.clone().requires_grad_(True) for k, v in params.items()}
        color, radii, depth, alpha = R.GaussianRasterizer(rs)(means3D=pin["means3D"], means2D=torch.zeros_like(pin["means3D"]),
                                                              opacities=pin["opacities"], shs=pin["shs"], scales=pin["scales"],
                                                              rotations=pin["rotations"])
        (color * gc).sum().backward()
        return color.detach(), alpha.detach(), depth.detach(), radii, {k: v.grad for k, v in pin.items()}

    c1, a1, d1, r1, ga = grads(g1)
    assert float(a1.min()) >= 0.0 and float(a1.max()) <= 1.0 + 1e-6 and float(c1.min()) >= 0.0
    assert int((r1 > 0).sum()) > P // 2
    assert float((d1 - 0.2 * a1).min()) >= -1e-5                     # every contributing depth exceeds the near cull
    _, _, _, _, gb = grads(g2)
    _, _, _, _, gab = grads(g1 + g2)
    for k in ga:
        scale = float(gab[k].abs().max())
        assert float((ga[k] + gb[k] - gab[k]).abs().max()) <= 5e-4 * scale, k


def _allreduce_worker(rank, world, port, out):
    import os
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        dev = torch.device("cuda", rank)
        ok, how = True, []
        for env in ({}, {"DGR_INKERNEL_BARRIERS": "0"}, {"DGR_NO_MULTIMEM": "1"}, {"DGR_PUSH": "1"}):     # default first
            for k in ("DGR_PUSH", "DGR_INKERNEL_BARRIERS", "DGR_NO_MULTIMEM"):
                os.environ.pop(k, None)
            os.environ.update(env)
            vsr = multiview.ViewShardedRasterizer(5000, 16, dev)
            g = torch.Generator(device=dev); g.manual_seed(77 + rank)
            src = torch.randn(vsr.grads.flat.numel(), device=dev, generator=g)
            ref = src.clone(); dist.all_reduce(ref)
            for rep in range(3):
                vsr.grads.flat.copy_(src)
                got = vsr.all_reduce()
                ok = ok and bool(torch.allclose(got, ref, rtol=1e-6, atol=1e-6))
            how.append(vsr.collective)
            del vsr
        for k in ("DGR_PUSH", "DGR_INKERNEL_BARRIERS", "DGR_NO_MULTIMEM"):
            os.environ.pop(k, None)
        okt = torch.tensor([int(ok)], device=dev); dist.all_reduce(okt, op=dist.ReduceOp.MIN)
        if rank == 0:
            open(out, "w").write("%s|%s" % (bool(int(okt)), " / ".join(how)))
    finally:
        dist.destroy_process_group()


def _push_worker(rank, world, port, out):
    """The reduce-scatter half fused into the backward (DgrPeerPush) + dgr_peer_reduce_staged against NCCL on the same
    per-rank gradients: several views per rank, a rank without a view, Gaussian counts that leave the last owner short or
    misalign the flat segments (scalar path), and the stand-alone push (dgr_peer_push_flat) bit for bit."""
    import os
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    os.environ["DGR_PUSH"] = "1"                                     # the opt-in path under test
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    msgs = []
    try:
        dev = torch.device("cuda", rank)
        t = lambda a: torch.tensor(np.asarray(a, np.float32), device=dev)
        res, deg = 96, 2
        for P, nviews in ((5000, (2, 1)), (4999, (1, 3)), (300, (1, 1)), (5000, (2, 0))):
            cloud = scene.make_cloud(P, deg, seed=3, sigma=0.02)
            params = {k: t(v) for k, v in cloud.items()}
            cams = [scene.orbit_camera(5.0 * i, 40.0 * i + 100.0 * rank, 2.0, res, res) for i in range(nviews[rank])]
            rs = [R.GaussianRasterizationSettings(image_height=res, image_width=res, tanfovx=c.tanfovx, tanfovy=c.tanfovy, bg=t(np.zeros(3)),
                                                  scale_modifier=1.0, viewmatrix=t(c.world_view_transform), projmatrix=t(c.full_proj_transform),
                                                  sh_degree=deg, campos=t(c.camera_center), prefiltered=False, debug=False) for c in cams]
            g = torch.Generator(device=dev); g.manual_seed(5 + rank)
            ups = [(torch.randn(3, res, res, device=dev, generator=g), None, torch.randn(1, res, res, device=dev, generator=g)) for _ in cams]
            ref = multiview.ViewShardedRasterizer(P, (deg + 1) ** 2, dev, peer_allreduce=False)
            ref.render_views(params, rs, ups)
            want = ref.all_reduce().clone()                          # NCCL
            vsr = multiview.ViewShardedRasterizer(P, (deg + 1) ** 2, dev)
            if not vsr._use_push:
                msgs.append("push path not active: %s" % getattr(vsr, "_why_nccl", vsr.collective))
                break
            for rep in range(2):                                     # twice: the staging area and the flags are reused
                vsr.render_views(params, rs, ups)
                got = vsr.all_reduce().clone()
                scale = float(want.abs().max())
                err = float((got - want).abs().max())
                if not err <= 2e-5 * scale:                          # atomics order inside a view differs run to run
                    msgs.append("P=%d views=%s rep %d: fused push err %.3e of %.3e" % (P, nviews, rep, err, scale))
            # stand-alone push of a hand-filled buffer: bit-identical to NCCL at two ranks
            gen = torch.Generator(device=dev); gen.manual_seed(99 + rank)
            src = torch.randn(vsr.grads.flat.numel(), device=dev, generator=gen)
            exact = src.clone(); dist.all_reduce(exact)
            vsr.grads.flat.copy_(src)
            got = vsr.all_reduce()
            if not torch.equal(got, exact):
                msgs.append("P=%d: stand-alone push differs from NCCL by %.3e" % (P, float((got - exact).abs().max())))
            del vsr, ref
        every = [None] * world
        dist.all_gather_object(every, msgs)
        if rank == 0:
            flat = ["rank %d: %s" % (r, m) for r, ms in enumerate(every) for m in ms]
            open(out, "w").write("%s|%s" % (not flat, "; ".join(flat) or "ok"))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_push_fused_into_the_backward_matches_nccl(tmp_path):
    import socket
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    out = str(tmp_path / "r.txt")
    mp.spawn(_push_worker, args=(2, port, out), nprocs=2, join=True)
    ok, how = open(out).read().split("|")
    assert ok == "True", how


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_own_nvlink_allreduce_matches_nccl(tmp_path):
    import socket
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    out = str(tmp_path / "r.txt")
    mp.spawn(_allreduce_worker, args=(2, port, out), nprocs=2, join=True)
    ok, how = open(out).read().split("|")
    assert ok == "True", how
