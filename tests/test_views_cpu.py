"""The batched-camera call without a GPU: exports, the argument checks that run before any device work, the Python-side
settings checks, and the SASS of its kernels."""
import ctypes
import subprocess

import pytest

from dreamgaussian_b200 import _lib, build

import test_sass_contract as sass


def test_views_symbols_are_exported_and_the_abi_version_holds():
    lib = _lib.load()
    for name in ("dgr_views_geom_bytes", "dgr_views_image_bytes", "dgr_views_binning_bytes", "dgr_views_forward_preprocess",
                 "dgr_views_forward_render", "dgr_views_backward"):
        assert hasattr(lib, name), name
        assert name in _lib.EXPORTS
    assert lib.dgr_abi_version() == 5
    # scratch sizes grow with the views: V x P records, V x tiles
    assert lib.dgr_views_geom_bytes(4, 1000, 256, 256) > 3 * lib.dgr_geom_bytes(1000, 256, 256)
    assert lib.dgr_views_image_bytes(4, 256, 256) > 3 * lib.dgr_image_bytes(256, 256)
    assert lib.dgr_views_geom_bytes(1, 1000, 256, 256) == lib.dgr_geom_bytes(1000, 256, 256)


BAD = ctypes.c_void_p(0x10)          # never dereferenced: every call below must fail in its argument checks


def _views(V=2, H=64, W=64):
    return _lib.DgrViews(V, H, W, 1.0, 0, 0, BAD, BAD, BAD, BAD, BAD)


def _gaussians(P=100, cov=False, colors=False):
    return _lib.DgrGaussians(P, 1, BAD, None if colors else BAD, BAD if colors else None, BAD, None if cov else BAD,
                             None if cov else BAD, BAD if cov else None, None, 0)


def _err(code):
    assert code != 0
    return _lib.load().dgr_last_error().decode()


def _all_three(views, gaussians, gout=None, staging=0):
    lib = _lib.load()
    v, g = ctypes.byref(views), ctypes.byref(gaussians)
    out = _lib.DgrImages(BAD, BAD, BAD, BAD)
    gin = _lib.DgrImageGrads(None, None, None)
    gout = gout or _lib.DgrGaussianGrads()
    return [
        _err(lib.dgr_views_forward_preprocess(v, g, BAD, BAD, BAD, None)),
        _err(lib.dgr_views_forward_render(v, g, BAD, BAD, ctypes.c_uint64(1 << 20), BAD, ctypes.byref(out), 0, None, ctypes.c_uint64(0), None, None)),
        _err(lib.dgr_views_backward(v, g, BAD, BAD, ctypes.c_uint64(1 << 20), staging, BAD, BAD, ctypes.byref(gin), ctypes.byref(gout), None)),
    ]


@pytest.mark.parametrize("V", [0, 65])
def test_view_count_outside_1_to_64_is_refused(V):
    for e in _all_three(_views(V=V), _gaussians()):
        assert "V must be 1..64" in e, e


def test_more_than_51200_tiles_in_the_batch_is_refused():
    for e in _all_three(_views(V=51, H=512, W=512), _gaussians()):        # 51 x 1024 tiles
        assert "51200" in e, e


def test_more_records_than_the_bound_is_refused():
    P = _lib.VIEWS_MAX_RECORDS // 64 + 1
    for e in _all_three(_views(V=64, H=16, W=16), _gaussians(P=P)):
        assert "V x P" in e, e


@pytest.mark.parametrize("what", ["colors", "cov"])
def test_precomputed_colours_or_covariance_are_refused(what):
    for e in _all_three(_views(), _gaussians(colors=what == "colors", cov=what == "cov")):
        assert "precomputed colours / cov3D" in e, e


@pytest.mark.parametrize("field", ["xyz_gradient_accum", "denom", "max_radii2D", "push"])
def test_statistics_or_push_are_refused(field):
    gout = _lib.DgrGaussianGrads()
    setattr(gout, field, 0x10)
    e = _all_three(_views(), _gaussians(), gout=gout)[2]
    assert ("densification statistics" in e) if field != "push" else ("DgrPeerPush" in e), e


def test_bad_staging_is_refused():
    e = _all_three(_views(), _gaussians(), staging=7)[2]
    assert "staging must be" in e, e


def _settings(H=64, W=64, deg=0, sm=1.0, device="cpu"):
    import torch
    from dreamgaussian_b200.rasterizer import GaussianRasterizationSettings
    z = lambda n: torch.zeros(n, device=device)
    return GaussianRasterizationSettings(H, W, 0.5, 0.5, z(3), sm, torch.eye(4, device=device), torch.eye(4, device=device), deg, z(3),
                                         False, False)


@pytest.mark.parametrize("field", ["image_height", "image_width", "sh_degree", "scale_modifier"])
def test_mismatched_settings_raise(field):
    import torch
    from dreamgaussian_b200.rasterizer import rasterize_views
    other = dict(image_height=dict(H=32), image_width=dict(W=48), sh_degree=dict(deg=1), scale_modifier=dict(sm=0.5))[field]
    z = torch.zeros
    with pytest.raises(ValueError, match=field):
        rasterize_views([_settings(), _settings(**other)], z(10, 3), None, z(10, 1), z(10, 1, 3), z(10, 3), z(10, 4))


def test_cpu_tensors_raise_no_cpu_path():
    import torch
    from dreamgaussian_b200.rasterizer import rasterize_views
    z = torch.zeros
    with pytest.raises(RuntimeError, match="no CPU path"):
        rasterize_views([_settings(), _settings()], z(10, 3), None, z(10, 1), z(10, 1, 3), z(10, 3), z(10, 4))


# ---- SASS of the batched kernels -----------------------------------------------------------------------------------------
resources = sass.resources


def test_batched_kernels_sass(resources):
    path, res = resources
    count = lambda ops, prefix: sum(1 for o in ops if o.startswith(prefix))
    fwd_name, bwd_name = sass._one(res, "render_views_fwd_kernelILb0E"), sass._one(res, "render_views_bwd_kernelILb0E")
    for name in (fwd_name, bwd_name):
        assert res[name]["stack"] == 0, (name, res[name])
        ops = sass._sass(path, name)
        assert count(ops, "UBLKCP") >= 2 and count(ops, "SYNCS.ARRIVE.TRANS64") >= 2 and count(ops, "SYNCS.PHASECHK") >= 1, name
        assert count(ops, "HMMA") == 0 and count(ops, "UTCHMMA") == 0 and count(ops, "UTCMMA") == 0, name
    assert res[fwd_name]["reg"] <= 64                                                # 8 CTAs x 128 threads per SM
    # record staging by id: the forward has no stack either; the backward keeps a few bytes, no more than the single-view
    # by-id backward it shares its body with
    assert res[sass._one(res, "render_views_fwd_kernelILb1E")]["stack"] == 0
    lazy_bwd = res[sass._one(res, "render_views_bwd_kernelILb1E")]["stack"]
    assert lazy_bwd <= res[sass._one(res, "render_bwd_kernelILi1ELi2ELb1ELb1E")]["stack"] <= 16, lazy_bwd
    bwd = sass._sass(path, bwd_name)
    assert count(bwd, "REDG.E.ADD.F32") >= 10 and count(bwd, "ATOMG.E.ADD.F32") == 0
    per_gaussian = [k for k in res if "preprocess_views_fwd_kernel" in k or "preprocess_views_bwd_kernel" in k]
    assert len(per_gaussian) == 16 + 8, per_gaussian
    for k in per_gaussian:
        assert res[k]["reg"] <= 80, (k, res[k])                                       # three CTAs per SM
    # the staged forward issues the warp's bulk copies; the per-thread variant none
    assert count(sass._sass(path, sass._one(res, "preprocess_views_fwd_kernelILi3ELb0ELb1E")), "UBLKCP") >= 5
    assert count(sass._sass(path, sass._one(res, "preprocess_views_fwd_kernelILi3ELb0ELb0E")), "UBLKCP") == 0
