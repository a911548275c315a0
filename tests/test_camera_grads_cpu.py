"""Camera gradients (DGR_RASTER_CAMERA_GRADS, include/dgr_b200.h) without a GPU: the exports and refusals of the C ABI, the
float64 torch oracle's camera gradients against central differences, the torch MiniCam restatement against the goldens, and
the SASS of the two new kernels."""
import ctypes
import os
import shutil

import numpy as np
import pytest
import torch

import camgrad_helpers as C
import helpers
from dreamgaussian_b200 import _lib, scene

BWD_EX = ("dgr_backward_ex", "dgr_backward_det_ex", "dgr_views_backward_ex", "dgr_views_backward_det_ex", "dgr_views_mixed_backward_ex",
          "dgr_views_mixed_backward_det_ex")


def test_exports_and_layout():
    lib = _lib.load()
    assert hasattr(lib, "dgr_camera_grad_scratch_bytes") and "dgr_camera_grad_scratch_bytes" in _lib.EXPORTS
    assert lib.dgr_abi_version() == 5 == _lib.ABI_VERSION
    assert _lib.RASTER_CAMERA_GRADS == 4 and _lib.RASTER_CAMERA_GRADS & _lib.RASTER_ANTIALIAS == 0
    assert ctypes.sizeof(_lib.DgrCameraGrads) == 40 and ctypes.sizeof(_lib.DgrRasterOptionsCamera) == 16
    assert _lib.DgrRasterOptionsCamera.camera.offset == 8
    # one 27-float row per (256 Gaussians, view), at least the rows
    for V, P in ((1, 1), (1, 100000), (8, 500000), (64, 0)):
        assert lib.dgr_camera_grad_scratch_bytes(V, P) >= V * ((P + 255) // 256) * 27 * 4
    assert lib.dgr_camera_grad_scratch_bytes(8, 1000) > lib.dgr_camera_grad_scratch_bytes(1, 1000)


# ---- refusals before device work (no pointer here is ever dereferenced by a kernel) ----------------------------------------
def _buf():
    buf = (ctypes.c_float * 64)()
    return buf, ctypes.cast(buf, ctypes.c_void_p)


def _refuse(call, want):
    lib = _lib.load()
    assert call() != 0, want
    assert want.encode() in lib.dgr_last_error(), (want, lib.dgr_last_error())


def _opts(flags, camera):
    o = _lib.DgrRasterOptionsCamera(flags, ctypes.pointer(camera) if camera is not None else None)
    return o, ctypes.cast(ctypes.pointer(o), ctypes.POINTER(_lib.DgrRasterOptions))


CAP = 1000


def _calls(lib, p, P=3):
    """Every backward *_ex call as f(opt) on arguments that pass their own checks."""
    s = _lib.DgrSettings(16, 16, 0.5, 0.5, 1.0, 0, 0, 0, p, p, p, p)
    g = _lib.DgrGaussians(P, 1, p, p, None, p, p, p, None, None, 0)
    gin, gout = _lib.DgrImageGrads(p, None, None), _lib.DgrGaussianGrads()
    vs = _lib.DgrViews(2, 16, 16, 1.0, 0, 0, p, p, p, p, p)
    hw = (ctypes.c_int32 * 4)(16, 16, 24, 8)
    det1 = (p, ctypes.c_uint64(lib.dgr_det_scratch_bytes(CAP, P)), ctypes.c_uint64(CAP))
    det2 = (p, ctypes.c_uint64(lib.dgr_det_scratch_bytes(CAP, 2 * P)), ctypes.c_uint64(CAP))
    bwd = (ctypes.byref(s), ctypes.byref(g), p, p, ctypes.c_uint64(CAP), 0, p, p, None, ctypes.byref(gin), ctypes.byref(gout))
    common = (ctypes.byref(g), p, p, ctypes.c_uint64(CAP), 0, p, p, ctypes.byref(gin), ctypes.byref(gout))
    keep = (s, g, gin, gout, vs, hw)
    return keep, {
        "dgr_backward_ex": lambda o: lib.dgr_backward_ex(*bwd, o, None),
        "dgr_backward_det_ex": lambda o: lib.dgr_backward_det_ex(*bwd, *det1, o, None),
        "dgr_views_backward_ex": lambda o: lib.dgr_views_backward_ex(ctypes.byref(vs), *common, o, None),
        "dgr_views_backward_det_ex": lambda o: lib.dgr_views_backward_det_ex(ctypes.byref(vs), *common, *det2, o, None),
        "dgr_views_mixed_backward_ex": lambda o: lib.dgr_views_mixed_backward_ex(ctypes.byref(vs), hw, *common, ctypes.c_uint64(0), o, None),
        "dgr_views_mixed_backward_det_ex": lambda o: lib.dgr_views_mixed_backward_det_ex(ctypes.byref(vs), hw, *common, ctypes.c_uint64(0),
                                                                                         *det2, o, None),
    }, {"dgr_backward_ex": 1, "dgr_backward_det_ex": 1}


def test_backward_calls_refuse_a_missing_camera_and_short_or_missing_scratch():
    lib = _lib.load()
    keep, p = _buf()
    P = 3
    k2, calls, views = _calls(lib, p, P)
    for name in BWD_EX:
        V = views.get(name, 2)
        need = lib.dgr_camera_grad_scratch_bytes(V, P)
        for flags in (_lib.RASTER_CAMERA_GRADS, _lib.RASTER_CAMERA_GRADS | _lib.RASTER_ANTIALIAS):
            o, op = _opts(flags, None)
            _refuse(lambda: calls[name](op), "camera == NULL")
            cam = _lib.DgrCameraGrads(p, p, p, None, need)
            o, op = _opts(flags, cam)
            _refuse(lambda: calls[name](op), "scratch is NULL")
            cam = _lib.DgrCameraGrads(p, p, p, p, need - 1)
            o, op = _opts(flags, cam)
            _refuse(lambda: calls[name](op), "scratch is smaller")
        # unknown bits stay refused, with and without the camera bit
        for flags in (2, 8, 2 | _lib.RASTER_CAMERA_GRADS, 1 << 31):
            o, op = _opts(flags, _lib.DgrCameraGrads(p, p, p, p, 1 << 30))
            _refuse(lambda: calls[name](op), "unknown flag bits")


def test_forward_calls_refuse_the_camera_bit():
    lib = _lib.load()
    keep, p = _buf()
    s = _lib.DgrSettings(16, 16, 0.5, 0.5, 1.0, 0, 0, 0, p, p, p, p)
    g = _lib.DgrGaussians(3, 1, p, p, None, p, p, p, None, None, 0)
    vs = _lib.DgrViews(2, 16, 16, 1.0, 0, 0, p, p, p, p, p)
    hw = (ctypes.c_int32 * 4)(16, 16, 24, 8)
    cam = _lib.DgrCameraGrads(p, p, p, p, 1 << 30)
    for flags in (_lib.RASTER_CAMERA_GRADS, _lib.RASTER_CAMERA_GRADS | _lib.RASTER_ANTIALIAS):
        o, op = _opts(flags, cam)
        _refuse(lambda: lib.dgr_forward_preprocess_ex(ctypes.byref(s), ctypes.byref(g), p, p, p, op, None), "backward-only")
        _refuse(lambda: lib.dgr_views_forward_preprocess_ex(ctypes.byref(vs), ctypes.byref(g), p, p, p, op, None), "backward-only")
        _refuse(lambda: lib.dgr_views_mixed_forward_preprocess_ex(ctypes.byref(vs), hw, ctypes.byref(g), p, p, p, op, None), "backward-only")


def test_minicam_restatement_matches_the_goldens():
    z = np.load(os.path.join(helpers.ROOT, "tests", "golden", "reference_vectors.npz"))
    for k, (el, az, r, W, H) in enumerate(z["cam_params"]):
        V, PM, c, tx, ty = C.minicam(torch.tensor(scene.orbit_pose(el, az, r), dtype=torch.float64), int(W), int(H))
        np.testing.assert_allclose(V.numpy(), z["cam_view"][k], atol=2e-6)
        np.testing.assert_allclose(PM.numpy(), z["cam_fullproj"][k], atol=2e-6)
        np.testing.assert_allclose(c.numpy(), z["cam_center"][k], atol=1e-6)
        np.testing.assert_allclose((tx, ty), z["cam_tanfov"][k], rtol=1e-6)


# ---- the float64 torch oracle's camera gradients against central differences --------------------------------------------------
def _case(kind):
    """A tiny scene away from the 0.99, 1/255 and frustum clamps: Gaussians of opacity 0.2-0.5 well inside the view."""
    s, i = helpers.make_case(P=10, res=32, deg=0 if kind in ("colors", "cov") else 2, sigma=0.06, elev=15, azim=35, seed=4)
    rng = np.random.default_rng(11)
    i["opacities"] = rng.uniform(0.2, 0.5, (10, 1)).astype(np.float32)
    i["means3D"] = (i["means3D"] * 0.5).astype(np.float32)
    if kind == "colors":
        i.pop("shs")
        i["colors_precomp"] = rng.uniform(0.1, 0.9, (10, 3)).astype(np.float32)
    if kind == "cov":
        Rm = C.T._quat_to_R(torch.tensor(i.pop("rotations"), dtype=torch.float64))
        Mx = Rm * torch.tensor(i.pop("scales"), dtype=torch.float64)[:, None, :]
        S = (Mx @ Mx.transpose(1, 2)).numpy()
        i["cov3D_precomp"] = np.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1).astype(np.float32)
    return s, i


@pytest.mark.parametrize("kind,aa", [("plain", False), ("plain", True), ("colors", False), ("cov", True)])
def test_torch_oracle_camera_grads_match_central_differences(kind, aa):
    s, i = _case(kind)
    gC, gD, gA = (torch.tensor(x, dtype=torch.float64) for x in helpers.upstream_grads(32, 32, seed=9))
    loss = lambda c, d, a: (c * gC).sum() + (d * gD).sum() + (a * gA).sum()
    gV, gPM, gc = C.oracle_camera_grads(s, i, loss, antialiased=aa)
    tin = {k: torch.tensor(np.asarray(v, np.float64)) for k, v in i.items()}
    base = [torch.tensor(np.asarray(s[k], np.float64)) for k in ("viewmatrix", "projmatrix", "campos")]

    def f(which, idx, h):
        cam = [b.clone() for b in base]
        cam[which].view(-1)[idx] += h
        with torch.no_grad():
            c, _, d, a = C.oracle_render(s, tin, *cam, antialiased=aa)
        return float(loss(c, d, a))

    eps = 1e-6
    for which, g in enumerate((gV, gPM, gc)):
        g = torch.zeros_like(base[which]) if g is None else g
        fd = np.array([(f(which, k, eps) - f(which, k, -eps)) / (2 * eps) for k in range(base[which].numel())])
        ga = g.reshape(-1).numpy()
        scale = max(np.abs(fd).max(), 1e-6)
        assert np.abs(ga - fd).max() <= 2e-4 * scale + 1e-7, (which, np.abs(ga - fd).max(), scale)
    # the entries the forward never reads
    assert (gV[:, 3] == 0).all() and (gPM[:, 2] == 0).all()
    if kind in ("colors", "cov"):                          # colors_precomp or degree 0: no view-direction dependence
        assert gc is None or (gc == 0).all()


# ---- SASS of the new kernels ---------------------------------------------------------------------------------------------------
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


def test_camera_kernels_registers_stack_and_no_float_atomics():
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not found")
    import test_deterministic_cpu as dc
    import test_sass_contract as sc
    path, res = dc._resources()
    bwd = [k for k in res if "camera_bwd_kernel" in k]
    red = [k for k in res if "camera_reduce_kernel" in k]
    assert len(bwd) == 28 and len(red) == 1, (len(bwd), len(red))       # the 14 input combinations x {default, anti-aliased}
    for name in bwd + red:
        r = res[name]
        assert r["stack"] == 0 and r["reg"] <= 80, (name, r)
        ops = sc._sass(path, name)
        assert not any(op.startswith(("RED", "ATOM")) for op in ops), name
