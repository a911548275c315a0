"""The absolute-gradient densification statistic (DGR_RASTER_ABS_GRAD, include/dgr_b200.h; AbsGS) without a GPU: the exports and
refusals of the C ABI, the two float64 oracles against each other and a known answer, the stage-1 densification rule on a hand-built
statistics snapshot, and the SASS of the new kernels."""
import ctypes
import os
import shutil

import numpy as np
import pytest
import torch

import absgrad_oracle as AO
import helpers
from dreamgaussian_b200 import _lib
from oracle import c_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_exports_and_layout():
    lib = _lib.load()
    assert lib.dgr_abi_version() == 5 == _lib.ABI_VERSION
    assert "dgr_densify_plan_ex" in _lib.EXPORTS and hasattr(lib, "dgr_densify_plan_ex")
    assert _lib.RASTER_ABS_GRAD == 16
    assert _lib.RASTER_ABS_GRAD & (_lib.RASTER_ANTIALIAS | 2 | _lib.RASTER_CAMERA_GRADS | 8) == 0
    assert _lib.DgrRasterOptionsFull.camera.offset == 8 and _lib.DgrRasterOptionsFull.xyz_gradient_accum_abs.offset == 16
    with open(os.path.join(ROOT, "include", "dgr_b200.h")) as f:
        hdr = f.read()
    assert "#define DGR_RASTER_ABS_GRAD 16u" in hdr and "float *xyz_gradient_accum_abs;" in hdr


# ---- refusals before any device work (no pointer here is ever dereferenced by a kernel) ---------------------------------------
def _refuse(call, want):
    lib = _lib.load()
    assert call() != 0, want
    assert want.encode() in lib.dgr_last_error(), (want, lib.dgr_last_error())


def _opts(flags, absbuf, camera=None):
    o = _lib.DgrRasterOptionsFull(flags, ctypes.pointer(camera) if camera is not None else None, absbuf)
    return o, ctypes.cast(ctypes.pointer(o), ctypes.POINTER(_lib.DgrRasterOptions))


def test_refusals():
    import test_camera_grads_cpu as cg
    lib = _lib.load()
    keep, p = cg._buf()
    P = 3
    k2, calls, _ = cg._calls(lib, p, P)
    s = _lib.DgrSettings(16, 16, 0.5, 0.5, 1.0, 0, 0, 0, p, p, p, p)
    g = _lib.DgrGaussians(P, 1, p, p, None, p, p, p, None, None, 0)
    vs = _lib.DgrViews(2, 16, 16, 1.0, 0, 0, p, p, p, p, p)
    hw = (ctypes.c_int32 * 4)(16, 16, 24, 8)
    # the bit on a forward call
    o, op = _opts(_lib.RASTER_ABS_GRAD, p)
    want = "DGR_RASTER_ABS_GRAD is backward-only"
    _refuse(lambda: lib.dgr_forward_preprocess_ex(ctypes.byref(s), ctypes.byref(g), p, p, p, op, None), want)
    _refuse(lambda: lib.dgr_views_forward_preprocess_ex(ctypes.byref(vs), ctypes.byref(g), p, p, p, op, None), want)
    _refuse(lambda: lib.dgr_views_mixed_forward_preprocess_ex(ctypes.byref(vs), hw, ctypes.byref(g), p, p, p, op, None), want)
    # the bit with a NULL buffer, on every backward *_ex call (alone and with the other bits)
    for flags in (_lib.RASTER_ABS_GRAD, _lib.RASTER_ABS_GRAD | _lib.RASTER_ANTIALIAS):
        o, op = _opts(flags, None)
        for name, call in calls.items():
            _refuse(lambda: call(op), "DGR_RASTER_ABS_GRAD with xyz_gradient_accum_abs == NULL")
    # the bit on the same-size batched call, which has no statistics
    o, op = _opts(_lib.RASTER_ABS_GRAD, p)
    for name in ("dgr_views_backward_ex", "dgr_views_backward_det_ex"):
        _refuse(lambda: calls[name](op), "DGR_RASTER_ABS_GRAD is not supported by the same-size batched call")
    # the bit on a mixed call with stats_views == 0 (the _calls helpers pass 0)
    for name in ("dgr_views_mixed_backward_ex", "dgr_views_mixed_backward_det_ex"):
        _refuse(lambda: calls[name](op), "DGR_RASTER_ABS_GRAD with stats_views == 0")
    # bits 2 and 8 stay unknown, with or without the new bit
    for flags in (2, 8, 2 | _lib.RASTER_ABS_GRAD, 8 | _lib.RASTER_ABS_GRAD):
        o, op = _opts(flags, p)
        _refuse(lambda: calls["dgr_backward_ex"](op), "unknown flag bits")
    # dgr_densify_plan_ex without the absolute statistic
    _refuse(lambda: lib.dgr_densify_plan_ex(P, p, None, p, p, p, 0.01, 0.02, 0.04, 0.005, 0.4, 0, p, None, None), "NULL argument")


# ---- the two float64 oracles ----------------------------------------------------------------------------------------------------
def _case(P=80, res=48, seed=3, deg=1):
    s, i = helpers.make_case(P=P, res=res, deg=deg, sigma=0.05, seed=seed)
    return s, i, helpers.upstream_grads(res, res)


@pytest.mark.parametrize("seed", [3, 11])
def test_hand_derived_and_autograd_oracles_agree(seed):
    s, i, g = _case(seed=seed)
    r = c_oracle.forward(**s, **i, dtype=np.float64)
    ct, at = AO.c_terms(r, *g), AO.autograd_terms(r, i["opacities"], s["bg"], *g)
    for k in ("abs_x", "abs_y", "sum_x", "sum_y"):
        scale = max(np.abs(ct[k]).max(), 1e-30)
        assert np.abs(ct[k] - at[k]).max() <= 1e-9 * scale, k
    a64, d64 = AO.stat(ct, r.radii, r.H, r.W)
    assert (r.radii > 0).sum() > 40 and np.all(a64 >= d64 * (1 - 1e-12))       # the triangle inequality, per Gaussian
    # the float32 build of the hand-derived oracle follows it (loosely: it is the large-case fallback, not a reference)
    r32 = c_oracle.forward(**s, **i, dtype=np.float32)
    a32, _ = AO.stat(AO.c_terms(r32, *g), r32.radii, r32.H, r32.W)
    assert np.abs(a32 - a64).max() <= 1e-3 * a64.max()
    r.close(); r32.close()


def test_per_pixel_terms_sum_to_the_mean_gradient():
    s, i, g = _case(seed=5)
    r = c_oracle.forward(**s, **i, dtype=np.float64)
    m2 = r.backward(*g)["means2D"]
    at = AO.autograd_terms(r, i["opacities"], s["bg"], *g, per_pixel=True)
    assert len(at["pixels"]) > 40
    for gi, (tx, ty) in at["pixels"].items():
        scale = max(np.abs(m2[gi, :2]).max(), 1e-12)
        assert abs(tx.sum() * 0.5 * r.W - m2[gi, 0]) <= 1e-9 * scale and abs(ty.sum() * 0.5 * r.H - m2[gi, 1]) <= 1e-9 * scale
        assert abs(np.abs(tx).sum() - at["abs_x"][gi]) <= 1e-12 * max(np.abs(tx).sum(), 1e-300)
    # the default statistic of the same oracle is |dL/dmeans2D[:2]|
    _, d = AO.stat(at, r.radii, r.H, r.W)
    assert np.allclose(d, np.linalg.norm(m2[:, :2], axis=1), rtol=1e-9, atol=1e-12)
    r.close()


def test_known_answer_centred_isotropic_gaussian():
    """One isotropic Gaussian centred at ((W-1)/2, (H-1)/2) on a 64x64 image, constant colour, dL/dcolor = 1: the per-pixel terms
    cancel in pairs, so the summed gradient vanishes while the absolute statistic is a direct float64 sum over the pixels."""
    H = W = 64
    tan = 0.5
    V = np.eye(4, dtype=np.float64)
    z, f, n = 3.0, 100.0, 0.01
    PM = np.zeros((4, 4))
    PM[0, 0], PM[1, 1] = 1 / tan, 1 / tan
    PM[2, 2], PM[3, 2], PM[2, 3] = f / (f - n), -f * n / (f - n), 1.0
    sig = 0.15
    col, bg, o = np.array([0.8, 0.3, 0.1]), np.array([0.0, 0.0, 0.0]), 0.7
    r = c_oracle.forward(image_height=H, image_width=W, tanfovx=tan, tanfovy=tan, bg=bg, scale_modifier=1.0, viewmatrix=V,
                         projmatrix=PM, sh_degree=0, campos=np.zeros(3), means3D=np.array([[0.0, 0.0, z]]), opacities=np.array([[o]]),
                         colors_precomp=col[None], cov3D_precomp=np.array([[sig * sig, 0, 0, sig * sig, 0, sig * sig]]), dtype=np.float64)
    st = r.state()
    assert st["px"][0] == (W - 1) / 2 and st["py"][0] == (H - 1) / 2 and st["conic"][0, 1] == 0.0
    gC = np.ones((3, H, W))
    ct = AO.c_terms(r, gC)
    at = AO.autograd_terms(r, [o], bg, gC)
    a, d = AO.stat(ct, r.radii, H, W)
    # direct float64 sum: one Gaussian in front of a black background, dL/dalpha = sum(colour - bg), u = o G dL/dalpha
    A, C = st["conic"][0, 0], st["conic"][0, 2]
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    dx, dy = st["px"][0] - xs, st["py"][0] - ys
    power = -0.5 * (A * dx * dx + C * dy * dy)
    G = np.exp(power)
    alpha = np.minimum(0.99, o * G)
    on = (power <= 0) & (alpha >= np.float32(1.0) / np.float32(255.0))
    u = np.where(on, o * G * (col - bg).sum(), 0.0)
    ax, ay = np.abs(u * A * dx).sum() * 0.5 * W, np.abs(u * C * dy).sum() * 0.5 * H
    direct = np.sqrt(ax * ax + ay * ay)
    assert on.sum() > 100 and a[0] > 0
    assert abs(a[0] - direct) <= 1e-9 * direct
    assert d[0] <= 1e-9 * a[0]
    a2, d2 = AO.stat(at, r.radii, H, W)
    assert abs(a2[0] - direct) <= 1e-9 * direct and d2[0] <= 1e-9 * a2[0]
    r.close()


# ---- stage 1: the densification rule on a hand-built snapshot -------------------------------------------------------------------
def _model(stats_abs):
    from dreamgaussian_b200.stage1 import GaussianModelB200
    m = GaussianModelB200(0)
    m.absgrad = stats_abs
    small, large = np.log(0.01), np.log(0.1)           # percent_dense 0.01 x extent 4 = 0.04: clone at or below, split above
    sc = torch.tensor([small, small, large, large, large], dtype=torch.float64)[:, None].repeat(1, 3)
    xyz = torch.arange(5, dtype=torch.float32)[:, None].repeat(1, 3)
    m._set(dict(xyz=xyz, f_dc=torch.zeros(5, 1, 3), f_rest=torch.zeros(5, 0, 3), opacity=torch.zeros(5, 1), scaling=sc,
                rotation=torch.tensor([[1.0, 0, 0, 0]]).repeat(5, 1)))
    m.fused_adam = False
    m.training_setup()
    st = m.stats
    st.denom.copy_(torch.tensor([2.0, 2.0, 2.0, 2.0, 0.0]))
    st.xyz_gradient_accum.copy_(2 * torch.tensor([0.02, 0.005, 0.005, 0.05, 0.0]))
    if stats_abs:
        st.xyz_gradient_accum_abs.copy_(2 * torch.tensor([0.03, 0.5, 0.03, 0.015, 0.0]))
    return m


def test_torch_densify_rule_selects_what_the_rule_says():
    noise = torch.zeros(2, 3)
    # default rule: clone point 0 (small, grad 0.02 >= 0.01), split point 3 (large, grad 0.05)
    m = _model(False)
    assert m.stats.xyz_gradient_accum_abs is None
    m.densify_and_prune(0.01, 0.005, 4, 0, noise=noise)
    assert m.p["xyz"][:, 0].tolist() == [0.0, 1.0, 2.0, 4.0, 0.0, 3.0, 3.0]
    # AbsGS rule: clone still by the default statistic (point 0; point 1's large absolute value does not clone it), split by the
    # absolute one: point 2 (0.03 >= 0.02) instead of point 3 (0.015 < 0.02); point 4 (denom 0 -> NaN -> 0) never
    m = _model(True)
    m.densify_and_prune(0.01, 0.005, 4, 0, noise=noise, max_abs_grad=0.02)
    assert m.p["xyz"][:, 0].tolist() == [0.0, 1.0, 3.0, 4.0, 0.0, 2.0, 2.0]
    assert torch.allclose(torch.exp(m.p["scaling"][5:]), torch.full((2, 3), 0.1 / 1.6))
    assert m.stats.xyz_gradient_accum_abs is not None and m.stats.xyz_gradient_accum_abs.shape == (7,)
    # the statistic follows a prune (_select)
    m.stats.xyz_gradient_accum_abs.copy_(torch.arange(7.0))
    m.prune_points(torch.tensor([True, False, False, False, False, False, True]))
    assert m.stats.xyz_gradient_accum_abs.tolist() == [1.0, 2.0, 3.0, 4.0, 5.0]
    # asking for the rule without the statistic is an error
    with pytest.raises(ValueError, match="max_abs_grad"):
        _model(False).densify_and_prune(0.01, 0.005, 4, 0, noise=noise, max_abs_grad=0.02)


def test_stage1_threshold_needs_the_fused_trainer():
    from dreamgaussian_b200.stage1 import Stage1Config, Stage1Trainer
    assert Stage1Config().densify_abs_grad_threshold is None
    with pytest.raises(ValueError, match="densify_abs_grad_threshold needs fused=True"):
        Stage1Trainer(Stage1Config(densify_abs_grad_threshold=0.02), device="cpu", fused=False)


# ---- SASS of the new kernels ---------------------------------------------------------------------------------------------------
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
NEW = {"render_bwd_abs_kernelILb0E": 96, "render_bwd_abs_kernelILb1E": 96, "render_views_bwd_abs_kernelILb0E": 96,
       "render_views_bwd_abs_kernelILb1E": 96, "render_bwd_det_abs_kernelILb0E": 128, "render_bwd_det_abs_kernelILb1E": 128,
       "render_views_bwd_det_abs_kernelILb0E": 128, "render_views_bwd_det_abs_kernelILb1E": 128,
       "det_moments_gather_abs_kernel": 48, "absgrad_stats_kernel": 32, "densify_classify_abs_kernel": 32}


def test_new_kernels_registers_no_local_memory_and_reductions():
    """Registers (ptxas's choice; DESIGN.md §4 has the CTAs per SM they allow next to the default render_bwd's 80) and no stack."""
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not found")
    import test_deterministic_cpu as dc
    import test_sass_contract as sc
    path, res = dc._resources()
    for part, limit in NEW.items():
        name = sc._one(res, part)
        r = res[name]
        assert r["stack"] == 0 and r["reg"] <= limit, (part, r)
        ops = sc._sass(path, name)
        assert not any(op.startswith("STL") or op.startswith("LDL") for op in ops), part
        if part.startswith(("render_bwd_abs", "render_views_bwd_abs")):       # 12 moments leave as reductions, no returning atomics
            assert sum(op.startswith("REDG.E.ADD.F32") for op in ops) >= 12 and not any(op.startswith("ATOMG.E.ADD.F32") for op in ops)
        if "det" in part or part == "absgrad_stats_kernel":                   # no float atomics: bit-reproducible
            assert not any(op.startswith(("RED", "ATOMG.E.ADD.F")) for op in ops), part
