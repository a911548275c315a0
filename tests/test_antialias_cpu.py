"""The anti-aliased mode (DgrRasterOptions / DGR_RASTER_ANTIALIAS, include/dgr_b200.h) without a GPU: the *_ex symbols and their
refusals before device work, the oracles of the mode (tests/aa_oracle.py) against each other, against central differences and a
known answer, the property the mode exists for, and the SASS of its kernels."""
import ctypes
import os
import re
import shutil

import numpy as np
import pytest
import torch

import aa_oracle
import helpers
import trained_scenes as ts
from dreamgaussian_b200 import _lib, scene

EX = ("dgr_forward_preprocess_ex", "dgr_views_forward_preprocess_ex", "dgr_views_mixed_forward_preprocess_ex", "dgr_backward_ex",
      "dgr_views_backward_ex", "dgr_views_mixed_backward_ex", "dgr_backward_det_ex", "dgr_views_backward_det_ex",
      "dgr_views_mixed_backward_det_ex")


def test_ex_symbols_are_exported_and_the_abi_is_still_5():
    lib = _lib.load()
    for name in EX:
        assert hasattr(lib, name) and name in _lib.EXPORTS, name
    assert lib.dgr_abi_version() == 5 == _lib.ABI_VERSION
    assert ctypes.sizeof(_lib.DgrRasterOptions) == 4 and _lib.RASTER_ANTIALIAS == 1


# ---- refusals before device work (no pointer here is ever dereferenced) ----------------------------------------------------------
def _buf():
    buf = (ctypes.c_float * 64)()
    return buf, ctypes.cast(buf, ctypes.c_void_p)


def _refuse(call, want):
    lib = _lib.load()
    assert call() != 0, want
    assert want.encode() in lib.dgr_last_error(), (want, lib.dgr_last_error())


CAP = 1000
BAD = ctypes.byref(_lib.DgrRasterOptions(2))           # a bit no option has
AA = ctypes.byref(_lib.DgrRasterOptions(1))


def _single(p):
    s = _lib.DgrSettings(16, 16, 0.5, 0.5, 1.0, 0, 0, 0, p, p, p, p)
    g = _lib.DgrGaussians(1, 1, p, p, None, p, p, p, None, None, 0)
    return s, g, _lib.DgrImageGrads(p, None, None)


def test_single_view_ex_calls_refuse_unknown_flags_and_what_their_counterparts_refuse():
    lib = _lib.load()
    keep, p = _buf()
    s, g, gin = _single(p)
    gout = _lib.DgrGaussianGrads()
    det = (p, ctypes.c_uint64(lib.dgr_det_scratch_bytes(CAP, 1)), ctypes.c_uint64(CAP))
    bwd = (ctypes.byref(s), ctypes.byref(g), p, p, ctypes.c_uint64(CAP), 0, p, p, None, ctypes.byref(gin), ctypes.byref(gout))
    _refuse(lambda: lib.dgr_forward_preprocess_ex(ctypes.byref(s), ctypes.byref(g), p, p, p, BAD, None), "unknown flag bits")
    _refuse(lambda: lib.dgr_backward_ex(*bwd, BAD, None), "unknown flag bits")
    _refuse(lambda: lib.dgr_backward_det_ex(*bwd, *det, BAD, None), "unknown flag bits")
    # the counterparts' own refusals, with the anti-aliased flag set
    both = _lib.DgrGaussians(1, 1, p, p, p, p, p, p, None, None, 0)            # SHs and colours
    _refuse(lambda: lib.dgr_forward_preprocess_ex(ctypes.byref(s), ctypes.byref(both), p, p, p, AA, None), "excatly one of either SHs")
    _refuse(lambda: lib.dgr_forward_preprocess_ex(ctypes.byref(s), ctypes.byref(g), None, p, p, AA, None), "scratch is NULL")
    big = _lib.DgrSettings(70000, 16, 0.5, 0.5, 1.0, 0, 0, 0, p, p, p, p)
    _refuse(lambda: lib.dgr_forward_preprocess_ex(ctypes.byref(big), ctypes.byref(g), p, p, p, AA, None), "above 65535")
    bad_staging = (ctypes.byref(s), ctypes.byref(g), p, p, ctypes.c_uint64(CAP), 2, p, p, None, ctypes.byref(gin), ctypes.byref(gout))
    _refuse(lambda: lib.dgr_backward_ex(*bad_staging, AA, None), "staging")
    _refuse(lambda: lib.dgr_backward_det_ex(*bwd, None, det[1], det[2], AA, None), "det_scratch is NULL")
    push = _lib.DgrPeerPush(2, 0, 256, (ctypes.c_int64 * 16)())
    pushed = _lib.DgrGaussianGrads()
    pushed.push = ctypes.addressof(push)
    with_push = (ctypes.byref(s), ctypes.byref(g), p, p, ctypes.c_uint64(CAP), 0, p, p, None, ctypes.byref(gin), ctypes.byref(pushed))
    _refuse(lambda: lib.dgr_backward_det_ex(*with_push, *det, AA, None), "DgrPeerPush")
    bad_push = _lib.DgrPeerPush(2, 0, 100, (ctypes.c_int64 * 16)())             # the single-view backward takes a push: checked
    pushed.push = ctypes.addressof(bad_push)
    _refuse(lambda: lib.dgr_backward_ex(*with_push, AA, None), "gaussians_per_owner")


def test_batched_ex_calls_refuse_unknown_flags_and_what_their_counterparts_refuse():
    lib = _lib.load()
    keep, p = _buf()
    s = _lib.DgrViews(2, 16, 16, 1.0, 0, 0, p, p, p, p, p)
    g = _lib.DgrGaussians(1, 1, p, p, None, p, p, p, None, None, 0)
    gin, gout = _lib.DgrImageGrads(p, None, None), _lib.DgrGaussianGrads()
    hw = (ctypes.c_int32 * 4)(16, 16, 24, 8)
    det = (p, ctypes.c_uint64(lib.dgr_det_scratch_bytes(CAP, 2)), ctypes.c_uint64(CAP))
    common = (ctypes.byref(g), p, p, ctypes.c_uint64(CAP), 0, p, p, ctypes.byref(gin), ctypes.byref(gout))
    for opt, want in ((BAD, "unknown flag bits"),):
        _refuse(lambda: lib.dgr_views_forward_preprocess_ex(ctypes.byref(s), ctypes.byref(g), p, p, p, opt, None), want)
        _refuse(lambda: lib.dgr_views_mixed_forward_preprocess_ex(ctypes.byref(s), hw, ctypes.byref(g), p, p, p, opt, None), want)
        _refuse(lambda: lib.dgr_views_backward_ex(ctypes.byref(s), *common, opt, None), want)
        _refuse(lambda: lib.dgr_views_mixed_backward_ex(ctypes.byref(s), hw, *common, ctypes.c_uint64(0), opt, None), want)
        _refuse(lambda: lib.dgr_views_backward_det_ex(ctypes.byref(s), *common, *det, opt, None), want)
        _refuse(lambda: lib.dgr_views_mixed_backward_det_ex(ctypes.byref(s), hw, *common, ctypes.c_uint64(0), *det, opt, None), want)
    cov = _lib.DgrGaussians(1, 1, p, p, None, p, None, None, p, None, 0)
    _refuse(lambda: lib.dgr_views_forward_preprocess_ex(ctypes.byref(s), ctypes.byref(cov), p, p, p, AA, None), "not supported by the batched")
    _refuse(lambda: lib.dgr_views_mixed_forward_preprocess_ex(ctypes.byref(s), None, ctypes.byref(g), p, p, p, AA, None), "image_hw is NULL")
    _refuse(lambda: lib.dgr_views_mixed_backward_ex(ctypes.byref(s), hw, *common, ctypes.c_uint64(1 << 5), AA, None), "stats_views")
    _refuse(lambda: lib.dgr_views_backward_det_ex(ctypes.byref(s), *common, None, det[1], det[2], AA, None), "det_scratch is NULL")
    stats = _lib.DgrGaussianGrads()
    stats.denom = p
    with_stats = (ctypes.byref(g), p, p, ctypes.c_uint64(CAP), 0, p, p, ctypes.byref(gin), ctypes.byref(stats))
    _refuse(lambda: lib.dgr_views_backward_ex(ctypes.byref(s), *with_stats, AA, None), "densification statistics")


# ---- the oracles of the mode -------------------------------------------------------------------------------------------------------
def _small_case(seed=0, res=48, P=60, deg=1, needles=True):
    """A small float64 scene: ordinary Gaussians plus needles on both sides of the ratio floor (kept 10% away from the kink)."""
    s, i = helpers.make_case(P=P, res=res, deg=deg, seed=seed, sigma=0.02, opacity="trained")
    i = {k: np.asarray(v, np.float64) for k, v in i.items()}
    if needles:
        rng = np.random.default_rng(seed + 7)
        cam = scene.orbit_camera(0.0, 0.0, 2.0, res, res)
        n = 6
        view = ts.view_of_pixel(cam, rng.uniform(8, res - 8, n), rng.uniform(8, res - 8, n), rng.uniform(1.8, 2.2, n))
        fx, _ = ts.focal(cam)
        # cross-section sigma (px) of each needle: ratio det0 / det ~ s_short^2 / (s_short^2 + 0.3) for a long needle; half of them
        # far below the floor 2.5e-5, half far above it
        short = np.array([1e-4, 2e-4, 5e-4, 0.05, 0.2, 0.5])
        sig = np.stack([np.full(n, 12.0), short, short], 1)
        Rv = ts.axes_in_image_plane(rng.uniform(0, np.pi, n))
        g = ts.gaussians(cam, rng, view, sig, Rv, rng.uniform(0.3, 0.9, n), rng.uniform(0.1, 0.9, (n, 3)), deg)
        for k in i:
            i[k] = np.concatenate([i[k], g[k].reshape((n,) + i[k].shape[1:])], 0)
    return s, i


def _torch_inputs(i):
    return {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in i.items()}


def _torch_loss(s, t, grads):
    gC, gD, gA = (torch.tensor(np.asarray(x, np.float64)) for x in grads)
    kw = dict(s, bg=torch.tensor(np.asarray(s["bg"], np.float64)), viewmatrix=torch.tensor(np.asarray(s["viewmatrix"], np.float64)),
              projmatrix=torch.tensor(np.asarray(s["projmatrix"], np.float64)), campos=torch.tensor(np.asarray(s["campos"], np.float64)))
    means2D = torch.zeros_like(t["means3D"], requires_grad=True)
    color, radii, depth, alpha = aa_oracle.rasterize(**kw, means2D=means2D, **t)
    return (color * gC).sum() + (depth * gD).sum() + (alpha * gA).sum(), means2D, color, alpha


def test_needle_case_straddles_the_ratio_floor():
    s, i = _small_case()
    r = aa_oracle.ratio_of(*aa_oracle.cov2d(s, *(torch.tensor(i[k]) for k in ("means3D", "scales", "rotations")))).numpy()[-6:]
    floor = aa_oracle.AA_RATIO_FLOOR
    assert (r[:3] < 0.9 * floor).all() and (r[3:] > 1.1 * floor).all(), r


def test_c_oracle_backward_matches_torch_oracle_autograd():
    s, i = _small_case()
    grads = helpers.upstream_grads(s["image_height"], s["image_width"], seed=5)
    t = _torch_inputs(i)
    loss, means2D, color, alpha = _torch_loss(s, t, grads)
    loss.backward()
    ref = aa_oracle.run_oracle(s, i, grads)
    assert np.abs(ref["color"] - color.detach().numpy()).max() < 1e-12
    assert np.abs(ref["alpha"] - alpha.detach().numpy()).max() < 1e-12
    for k in i:
        a, b = ref["grads"][k].reshape(-1), t[k].grad.numpy().reshape(-1)
        assert np.abs(a - b).max() <= 1e-9 * max(np.abs(b).max(), 1e-30), k
    a, b = ref["grads"]["means2D"].reshape(-1), means2D.grad.numpy().reshape(-1)
    assert np.abs(a - b).max() <= 1e-9 * np.abs(b).max()


def test_torch_oracle_matches_central_differences():
    s, i = _small_case(res=32, P=12)
    grads = helpers.upstream_grads(s["image_height"], s["image_width"], seed=6)
    t = _torch_inputs(i)
    loss, _, _, _ = _torch_loss(s, t, grads)
    loss.backward()
    rng = np.random.default_rng(1)
    n = len(i["means3D"])
    checked = 0
    for k in ("means3D", "scales", "rotations", "opacities"):
        for g_ in list(rng.choice(n - 6, 3, replace=False)) + list(range(n - 6, n)):      # a few ordinary Gaussians and every needle
            for c in range(i[k].shape[1]):
                h = 1e-6 * max(1.0, abs(i[k][g_, c]))
                vals = []
                for sign in (1, -1):
                    j = {kk: vv.copy() for kk, vv in i.items()}
                    j[k][g_, c] += sign * h
                    with torch.no_grad():
                        vals.append(float(_torch_loss(s, {kk: torch.tensor(vv) for kk, vv in j.items()}, grads)[0]))
                fd = (vals[0] - vals[1]) / (2 * h)
                an = float(t[k].grad[g_, c])
                assert abs(fd - an) <= 1e-5 * max(1.0, abs(an)), (k, g_, c, fd, an)
                checked += 1
    assert checked == 9 * 11


def test_comp_matches_central_differences_on_both_sides_of_the_floor():
    s, i = _small_case()
    x = {k: torch.tensor(i[k], requires_grad=True) for k in ("means3D", "scales", "rotations")}
    w = torch.tensor(np.random.default_rng(3).normal(size=len(i["means3D"])))
    (aa_oracle.comp(s, **x) * w).sum().backward()
    for k in x:
        for g_ in range(len(i["means3D"]) - 6, len(i["means3D"])):
            for c in range(i[k].shape[1]):
                h = 1e-7 * max(1.0, abs(i[k][g_, c]))
                f = []
                for sign in (1, -1):
                    y = {kk: torch.tensor(i[kk]) for kk in x}
                    y[k][g_, c] += sign * h
                    f.append(float((aa_oracle.comp(s, **y) * w).sum()))
                fd = (f[0] - f[1]) / (2 * h)
                assert abs(fd - float(x[k].grad[g_, c])) <= 1e-5 * max(1.0, abs(fd)), (k, g_, c)
    # below the floor comp is the constant sqrt(floor) and has no gradient
    assert (x["scales"].grad[-6:-3] == 0).all()


# ---- known answer --------------------------------------------------------------------------------------------------------------
def known_answer_case(s_px=0.3, o=0.9):
    """One isotropic Gaussian at the origin seen by orbit_camera(0, 0, 2) at 800 x 800, pixel sigma s_px (sub-pixel).  Returns
    (settings, inputs, expected alpha at pixel (399, 399), comp)."""
    cam = scene.orbit_camera(0.0, 0.0, 2.0, 800, 800)
    fx = 800 / (2 * cam.tanfovx)
    sigma = s_px * 2.0 / fx
    s = ts.settings_of(cam, 0)
    i = dict(means3D=np.zeros((1, 3)), opacities=np.full((1, 1), o), shs=np.zeros((1, 1, 3)), scales=np.full((1, 3), sigma),
             rotations=np.array([[1.0, 0, 0, 0]]))
    comp = s_px ** 2 / (s_px ** 2 + 0.3)
    # the centre projects to pixel (399.5, 399.5): pixel (399, 399) is 0.5 px off in x and y
    return s, i, min(0.99, o * comp * np.exp(-0.25 / (s_px ** 2 + 0.3))), comp, fx


def test_known_answer_of_one_subpixel_gaussian():
    s, i, want, comp, fx = known_answer_case()
    assert abs(fx - 875.694) < 1e-3
    got = aa_oracle.run_oracle(s, i)
    assert abs(got["alpha"][0, 399, 399] - want) < 1e-6, (got["alpha"][0, 399, 399], want)
    plain = helpers.run_oracle(s, i)
    assert abs(plain["alpha"][0, 399, 399] - want / comp) < 1e-6          # the default mode: the same Gaussian without comp
    assert (got["radii"] == plain["radii"]).all()


# ---- the property the mode exists for ----------------------------------------------------------------------------------------
RES = (128, 256, 512)


def resolution_case(res, n_side=8, s128=0.2, o=0.95, seed=0):
    """Sparse isolated Gaussians on an 8 x 8 lattice (16 px apart at 128 x 128, a random sub-pixel phase each), pixel sigma s128 at
    128 x 128 (s128 res / 128 at res), all at depth 2, seen by one camera at res x res."""
    rng = np.random.default_rng(seed)
    c128 = ts.camera(128, 128)
    px = 8 + 16 * np.arange(n_side)
    gx, gy = np.meshgrid(px, px)
    view = ts.view_of_pixel(c128, gx.ravel() + rng.uniform(-0.5, 0.5, gx.size), gy.ravel() + rng.uniform(-0.5, 0.5, gx.size), 2.0)
    n = len(view)
    fx, _ = ts.focal(c128)
    i = dict(means3D=ts.view_to_world(c128, view), opacities=np.full((n, 1), o), shs=np.zeros((n, 1, 3)),
             scales=np.full((n, 3), s128 * 2.0 / fx), rotations=np.tile([1.0, 0, 0, 0], (n, 1)))
    return ts.settings_of(ts.camera(res, res), 0), i


def mean_alpha(run, aa):
    out = []
    for res in RES:
        s, i = resolution_case(res)
        out.append(float(run(s, i, aa)["alpha"].mean()))
    return np.array(out)


def _oracle_run(s, i, aa):
    return aa_oracle.run_oracle(s, i) if aa else helpers.run_oracle(s, i)


# Tolerances, from oracle runs (float64 C oracle through aa_oracle, this file's scene): sum(alpha) / (H W) at 128, 256, 512 is
#   anti-aliased  9.563e-4, 9.826e-4, 9.879e-4   spread max/min - 1 = 3.3 %
#   default       7.955e-3, 2.733e-3, 1.426e-3   spread max/min - 1 = 458 %
# The anti-aliased spread is what the 1/255 cutoff takes from the tails (1 / (255 o_eff) of each Gaussian's weight: 3.7 % at
# 128 x 128, 0.6 % at 512 x 512).  AA_SPREAD leaves 1.5x that; DEFAULT_SPREAD is far below what the default mode shows.
AA_SPREAD = 0.05
DEFAULT_SPREAD = 1.0


def test_antialiased_coverage_does_not_depend_on_resolution():
    aa, plain = mean_alpha(_oracle_run, True), mean_alpha(_oracle_run, False)
    print("mean alpha, anti-aliased:", aa, "default:", plain)
    assert aa.max() / aa.min() - 1 < AA_SPREAD, aa
    assert plain.max() / plain.min() - 1 > DEFAULT_SPREAD, plain


# ---- SASS --------------------------------------------------------------------------------------------------------------------------
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


def test_antialiased_kernels_keep_their_counterparts_budgets_and_staging():
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not found")
    import test_deterministic_cpu as dc
    import test_sass_contract as sc
    path, res = dc._resources()
    aa = [k for k in res if "_aa_kernel" in k]
    # single view: 14 input combinations + 8 staged; batched: 8 + 8 staged forward, 8 backward
    assert len([k for k in aa if "preprocess_fwd_aa" in k]) == 22 and len([k for k in aa if "preprocess_bwd_aa" in k]) == 22
    assert len([k for k in aa if "views_fwd_aa" in k]) == 16 and len([k for k in aa if "views_bwd_aa" in k]) == 8
    for k in aa:
        twin = res[re.sub(r"(\d+)(preprocess\w*?)_aa_kernel", lambda m: "%d%s_kernel" % (int(m.group(1)) - 3, m.group(2)), k)]
        assert res[k]["reg"] <= 80, (k, res[k])                               # __launch_bounds__(256, 3)
        # the twins already keep a few dozen bytes of local arrays on the stack; measured: the anti-aliased variant is within
        # -32 .. +56 bytes of its twin, and keeps no stack where the twin has none except in one kernel
        assert res[k]["stack"] <= twin["stack"] + 64, (k, res[k], twin)
        assert res[k]["shared"] == twin["shared"], (k, res[k], twin)
    count = lambda ops, prefix: sum(1 for o in ops if o.startswith(prefix))
    for name in ("preprocess_fwd_aa_kernelILi3ELb1ELb0ELb0ELb1E", "preprocess_bwd_aa_kernelILi3ELb1ELb0ELb0ELb1E",
                 "preprocess_views_fwd_aa_kernelILi3ELb0ELb1E"):
        assert count(sc._sass(path, sc._one(res, name)), "UBLKCP") >= 5, name
    for name in ("preprocess_fwd_aa_kernelILi3ELb1ELb0ELb0ELb0E", "preprocess_bwd_aa_kernelILi3ELb1ELb0ELb0ELb0E"):
        assert count(sc._sass(path, sc._one(res, name)), "UBLKCP") == 0, name
    # the mode costs a square root per Gaussian and view: one more MUFU.RSQ / MUFU.SQRT than the twin at least
    f_aa = sc._sass(path, sc._one(res, "preprocess_fwd_aa_kernelILi3ELb1ELb0ELb0ELb1E"))
    f = sc._sass(path, sc._one(res, "preprocess_fwd_kernelILi3ELb1ELb0ELb0ELb1E"))
    assert count(f_aa, "MUFU") > count(f, "MUFU")
