"""The blending-weight statistics (DGR_RASTER_CONTRIB, include/dgr_b200.h) without a GPU: the exports and refusals of the C ABI, the
C oracle against the float64 torch restatement, a known answer, the alpha identity, the SASS of the new kernels, and the host logic
of ContributionStats and prune_by_contribution."""
import ctypes
import os
import shutil

import numpy as np
import pytest
import torch

import contrib_oracle as CO
import helpers
from dreamgaussian_b200 import _lib
from oracle import c_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_exports_and_layout():
    lib = _lib.load()
    assert lib.dgr_abi_version() == 5 == _lib.ABI_VERSION
    for sym in ("dgr_contrib_scratch_bytes", "dgr_forward_render_ex", "dgr_views_forward_render_ex", "dgr_views_mixed_forward_render_ex"):
        assert sym in _lib.EXPORTS and hasattr(lib, sym)
    assert _lib.RASTER_CONTRIB == 32
    assert _lib.RASTER_CONTRIB & (_lib.RASTER_ANTIALIAS | 2 | _lib.RASTER_CAMERA_GRADS | 8 | _lib.RASTER_ABS_GRAD) == 0
    O = _lib.DgrRasterOptionsContrib
    assert O.camera.offset == 8 and O.xyz_gradient_accum_abs.offset == 16 and O.contrib.offset == 24
    assert lib.dgr_contrib_scratch_bytes(0) == 0 and lib.dgr_contrib_scratch_bytes(1) >= 8
    assert lib.dgr_contrib_scratch_bytes(1000) >= 8000 and lib.dgr_contrib_scratch_bytes(1000) % 256 == 0
    with open(os.path.join(ROOT, "include", "dgr_b200.h")) as f:
        hdr = f.read()
    assert "#define DGR_RASTER_CONTRIB 32u" in hdr and "const DgrContrib *contrib;" in hdr and "2^38" in hdr


# ---- refusals before any device work (no pointer here is ever dereferenced by a kernel) ---------------------------------------
def _refuse(call, want):
    lib = _lib.load()
    assert call() != 0, want
    assert want.encode() in lib.dgr_last_error(), (want, lib.dgr_last_error())


def _opts(flags, contrib=None):
    o = _lib.DgrRasterOptionsContrib(flags, None, None, ctypes.pointer(contrib) if contrib is not None else None)
    return o, ctypes.cast(ctypes.pointer(o), ctypes.POINTER(_lib.DgrRasterOptions))


def test_refusals():
    import test_camera_grads_cpu as cg
    lib = _lib.load()
    keep, p = cg._buf()
    P = 3
    k2, bwd_calls, _ = cg._calls(lib, p, P)
    s = _lib.DgrSettings(16, 16, 0.5, 0.5, 1.0, 0, 0, 0, p, p, p, p)
    g = _lib.DgrGaussians(P, 1, p, p, None, p, p, p, None, None, 0)
    vs = _lib.DgrViews(2, 16, 16, 1.0, 0, 0, p, p, p, p, p)
    hw = (ctypes.c_int32 * 4)(16, 16, 24, 8)
    out = _lib.DgrImages(p, p, p, p)
    tail = (ctypes.c_uint64(1024), p, ctypes.byref(out), 0, p, ctypes.c_uint64(0), None)
    render = {
        "dgr_forward_render_ex": (lambda op: lib.dgr_forward_render_ex(ctypes.byref(s), ctypes.byref(g), p, p, *tail, op, None), P),
        "dgr_views_forward_render_ex": (lambda op: lib.dgr_views_forward_render_ex(ctypes.byref(vs), ctypes.byref(g), p, p, *tail, op, None), 2 * P),
        "dgr_views_mixed_forward_render_ex": (lambda op: lib.dgr_views_mixed_forward_render_ex(ctypes.byref(vs), hw, ctypes.byref(g), p, p, *tail,
                                                                                             op, None), 2 * P),
    }
    for name, (call, records) in render.items():
        # any other bit
        for flags in (_lib.RASTER_ANTIALIAS, 2, _lib.RASTER_CAMERA_GRADS, 8, _lib.RASTER_ABS_GRAD, _lib.RASTER_CONTRIB | _lib.RASTER_ANTIALIAS):
            o, op = _opts(flags)
            _refuse(lambda: call(op), "accepts DGR_RASTER_CONTRIB only")
        # the bit without its struct, with NULL outputs, NULL scratch or a short scratch
        o, op = _opts(_lib.RASTER_CONTRIB)
        _refuse(lambda: call(op), "DGR_RASTER_CONTRIB with contrib == NULL")
        need = lib.dgr_contrib_scratch_bytes(records)
        for c, want in ((_lib.DgrContrib(None, p, p, need), "weight_sum / weight_max is NULL"),
                        (_lib.DgrContrib(p, None, p, need), "weight_sum / weight_max is NULL"),
                        (_lib.DgrContrib(p, p, None, need), "scratch is NULL"),
                        (_lib.DgrContrib(p, p, p, need - 1), "scratch is smaller than dgr_contrib_scratch_bytes")):
            o, op = _opts(_lib.RASTER_CONTRIB, c)
            _refuse(lambda: call(op), want)
    # the bit on the preprocess and backward *_ex calls
    c = _lib.DgrContrib(p, p, p, 1 << 20)
    o, op = _opts(_lib.RASTER_CONTRIB, c)
    want = "DGR_RASTER_CONTRIB belongs to the stage-2 render calls"
    _refuse(lambda: lib.dgr_forward_preprocess_ex(ctypes.byref(s), ctypes.byref(g), p, p, p, op, None), want)
    _refuse(lambda: lib.dgr_views_forward_preprocess_ex(ctypes.byref(vs), ctypes.byref(g), p, p, p, op, None), want)
    _refuse(lambda: lib.dgr_views_mixed_forward_preprocess_ex(ctypes.byref(vs), hw, ctypes.byref(g), p, p, p, op, None), want)
    for name, call in bwd_calls.items():
        _refuse(lambda: call(op), want)


# ---- the oracles ------------------------------------------------------------------------------------------------------------------
def _case(P=80, res=48, seed=3, deg=1):
    return helpers.make_case(P=P, res=res, deg=deg, sigma=0.05, seed=seed)


@pytest.mark.parametrize("seed", [3, 11])
def test_c_oracle_and_torch_restatement_agree(seed):
    s, i = _case(seed=seed)
    r = c_oracle.forward(**s, **i, dtype=np.float64)
    cs, cm = CO.c_stats(r)
    ts, tm = CO.torch_stats(r, i["opacities"])
    assert (cm > 0).sum() > 40
    assert np.abs(cs - ts).max() <= 1e-9 * cs.max() and np.abs(cm - tm).max() <= 1e-9 * cm.max()
    assert np.all(cs >= cm) and np.all(cm <= 0.99 + 1e-12)
    assert np.all(cm[np.asarray(r.radii) == 0] == 0)
    # the float32 build follows it (it is the large-case fallback, not a reference)
    r32 = c_oracle.forward(**s, **i, dtype=np.float32)
    s32, m32 = CO.c_stats(r32)
    assert np.abs(s32 - cs).max() <= 1e-3 * cs.max() and np.abs(m32 - cm).max() <= 1e-3
    r.close(); r32.close()


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_weights_sum_to_the_alpha_image(dtype):
    s, i = _case(P=200, res=64, seed=7)
    r = c_oracle.forward(**s, **i, dtype=dtype)
    ws, _ = CO.c_stats(r)
    a = float(np.asarray(r.alpha, np.float64).sum())
    assert a > 10
    assert abs(ws.sum() - a) <= (1e-12 if dtype == np.float64 else 1e-5) * a
    r.close()


def test_known_answer_centred_isotropic_gaussian():
    """One isotropic Gaussian centred on a pixel centre of a 64x64 image: weight_max = min(0.99, o) (G = 1 at that pixel, T = 1), and
    weight_sum is the direct float64 sum of alpha over its alpha >= 1/255 pixels (nothing in front of it: w = alpha)."""
    H = W = 64
    tan = 0.5
    V = np.eye(4, dtype=np.float64)
    z, f, n = 3.0, 100.0, 0.01
    PM = np.zeros((4, 4))
    PM[0, 0], PM[1, 1] = 1 / tan, 1 / tan
    PM[2, 2], PM[3, 2], PM[2, 3] = f / (f - n), -f * n / (f - n), 1.0
    sig = 0.15
    for o in (0.7, 1.0):
        r = c_oracle.forward(image_height=H, image_width=W, tanfovx=tan, tanfovy=tan, bg=np.zeros(3), scale_modifier=1.0, viewmatrix=V,
                             projmatrix=PM, sh_degree=0, campos=np.zeros(3), means3D=np.array([[0.0, 0.0, z]]), opacities=np.array([[o]]),
                             colors_precomp=np.array([[0.8, 0.3, 0.1]]), cov3D_precomp=np.array([[sig * sig, 0, 0, sig * sig, 0, sig * sig]]),
                             dtype=np.float64)
        st = r.state()
        assert st["px"][0] == (W - 1) / 2 and st["py"][0] == (H - 1) / 2 and st["conic"][0, 1] == 0.0
        # (W-1)/2 is not a pixel centre for even W: the centre pixel has G < 1.  Read weight_max off the exact G at the nearest pixel.
        A, C = st["conic"][0, 0], st["conic"][0, 2]
        ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
        dx, dy = st["px"][0] - xs, st["py"][0] - ys
        power = -0.5 * (A * dx * dx + C * dy * dy)
        alpha = np.minimum(0.99, o * np.exp(power))
        on = (power <= 0) & (alpha >= np.float32(1.0) / np.float32(255.0))
        ws, wm = CO.c_stats(r)
        ts, tm = CO.torch_stats(r, [o])
        assert on.sum() > 100
        assert abs(ws[0] - alpha[on].sum()) <= 1e-12 * ws[0] and abs(ts[0] - ws[0]) <= 1e-12 * ws[0]
        assert abs(wm[0] - alpha[on].max()) <= 1e-12 * wm[0] and abs(tm[0] - wm[0]) <= 1e-12 * wm[0]
        r.close()
    # and on an odd image the centre IS a pixel centre: weight_max = min(0.99, o) exactly
    H = W = 63
    for o in (0.7, 1.0):
        r = c_oracle.forward(image_height=H, image_width=W, tanfovx=tan, tanfovy=tan, bg=np.zeros(3), scale_modifier=1.0, viewmatrix=V,
                             projmatrix=PM, sh_degree=0, campos=np.zeros(3), means3D=np.array([[0.0, 0.0, z]]), opacities=np.array([[o]]),
                             colors_precomp=np.array([[0.8, 0.3, 0.1]]), cov3D_precomp=np.array([[sig * sig, 0, 0, sig * sig, 0, sig * sig]]),
                             dtype=np.float64)
        assert r.state()["px"][0] == 31.0
        ws, wm = CO.c_stats(r)
        assert wm[0] == min(float(np.float32(0.99)), o)          # DGR_ALPHA_MAX is the float32 0.99
        r.close()


# ---- SASS of the new kernels ---------------------------------------------------------------------------------------------------
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
NEW = {"render_fwd_contrib_kernelILb0E": 64, "render_fwd_contrib_kernelILb1E": 64, "render_views_fwd_contrib_kernelILb0E": 64,
       "render_views_fwd_contrib_kernelILb1E": 64, "contrib_finalize_kernel": 32}


def test_new_kernels_no_float_atomics_no_local_memory():
    """8 CTAs of 4 warps per SM (<= 64 registers), no stack, no spills; the cross-warp sums are 64-bit integer reductions and the max
    an integer max: no float atomic, so the statistics are bit-reproducible.  The default render_fwd keeps its budget."""
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not found")
    import test_deterministic_cpu as dc
    import test_sass_contract as sc
    path, res = dc._resources()
    for part, limit in NEW.items():
        name = sc._one(res, part)
        r = res[name]
        assert r["stack"] == 0 and r["reg"] <= limit, (part, r)
        ops = dc._sass(path, name)
        assert not any(op.startswith(("STL", "LDL")) for op in ops), part
        assert not any(op.startswith(("RED", "ATOM")) and ".F32" in op for op in ops), part
        assert not any(op.startswith(("RED", "ATOM")) and ".F" in op.split(".E.", 1)[-1][:3] for op in ops), part
        if part.startswith("render"):
            assert any(op.startswith(("REDG.E.ADD.64", "ATOMG.E.ADD.64")) for op in ops), part
            assert any(op.startswith(("REDG.E.MAX", "ATOMG.E.MAX")) for op in ops), part
    r = res[sc._one(res, "render_fwd_kernelILi1ELi1ELb0E")]
    assert r["stack"] == 0 and r["reg"] <= 64


# ---- host logic ---------------------------------------------------------------------------------------------------------------
def test_contribution_stats_accumulate_sum_and_max_in_view_order():
    from dreamgaussian_b200.rasterizer import ContributionStats
    st = ContributionStats(4, "cpu")
    assert st.renders == 0 and st.weight_sum.dtype == torch.float32 and st.weight_sum.tolist() == [0.0] * 4
    st.add(torch.tensor([0.5, 0.0, 0.25, 1.0]), torch.tensor([0.25, 0.0, 0.125, 0.5]))
    st.add(torch.tensor([[0.5, 0.0, 0.0, 2.0], [1.0, 0.0, 0.5, 0.0]]), torch.tensor([[0.5, 0.0, 0.0, 0.25], [0.125, 0.0, 0.5, 0.0]]))
    assert st.renders == 3
    assert st.weight_sum.tolist() == [2.0, 0.0, 0.75, 3.0] and st.weight_max.tolist() == [0.5, 0.0, 0.5, 0.5]
    # in view order: float sums are not associative, the stats add view by view
    a = ContributionStats(1, "cpu")
    a.add(torch.tensor([[1.0], [2.0 ** -24], [2.0 ** -24]]), torch.zeros(3, 1))
    assert a.weight_sum.item() == 1.0
    with pytest.raises(ValueError):
        st.add(torch.zeros(5), torch.zeros(5))


def _model(P=6):
    from dreamgaussian_b200.stage1 import GaussianModelB200
    m = GaussianModelB200(0)
    xyz = torch.arange(P, dtype=torch.float32)[:, None].repeat(1, 3)
    m._set(dict(xyz=xyz, f_dc=torch.zeros(P, 1, 3), f_rest=torch.zeros(P, 0, 3), opacity=torch.zeros(P, 1), scaling=torch.zeros(P, 3),
                rotation=torch.tensor([[1.0, 0, 0, 0]]).repeat(P, 1)))
    m.fused_adam = False
    m.training_setup()
    for k in m.exp_avg:
        m.exp_avg[k].copy_(torch.arange(m.exp_avg[k].numel(), dtype=torch.float32).view_as(m.exp_avg[k]))
        m.exp_avg_sq[k].copy_(2 * torch.arange(m.exp_avg_sq[k].numel(), dtype=torch.float32).view_as(m.exp_avg_sq[k]))
    m.stats.denom.copy_(torch.arange(P, dtype=torch.float32))
    return m


def test_prune_by_contribution_keeps_rows_and_moments():
    from dreamgaussian_b200.rasterizer import ContributionStats
    m = _model()
    before = ({k: v.detach().clone() for k, v in m.p.items()}, {k: v.clone() for k, v in m.exp_avg.items()},
              {k: v.clone() for k, v in m.exp_avg_sq.items()})
    st = ContributionStats(6, "cpu")
    st.add(torch.ones(6), torch.tensor([0.0, 0.3, 1e-13, 0.01, 0.0, 0.5]))
    assert m.prune_by_contribution(st, 1e-12) == 3
    keep = torch.tensor([False, True, False, True, False, True])
    assert m.num_points == 3 and m.p["xyz"][:, 0].tolist() == [1.0, 3.0, 5.0]
    for k in m.p:
        assert torch.equal(m.p[k].detach(), before[0][k][keep]) and m.p[k].requires_grad
        assert torch.equal(m.exp_avg[k], before[1][k][keep]) and torch.equal(m.exp_avg_sq[k], before[2][k][keep])
    assert m.stats.denom.tolist() == [1.0, 3.0, 5.0]
    with pytest.raises(ValueError):
        m.prune_by_contribution(st, 1e-12)          # 6 statistics, 3 Gaussians


def test_export_cameras_are_the_reference_lists():
    from dreamgaussian_b200.stage1 import Stage1Trainer
    assert len(Stage1Trainer.EXPORT_VERS) == len(Stage1Trainer.EXPORT_HORS) == 26
    assert Stage1Trainer.EXPORT_VERS[-2:] == [-89.9, 89.9] and Stage1Trainer.EXPORT_HORS[:8] == [0, 45, -45, 90, -90, 135, -135, 180]
