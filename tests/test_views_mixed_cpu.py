"""The batched call with a size per view (dgr_views_mixed_*, rasterize_views_mixed) without a GPU: exports, scratch sizes, the
argument checks that run before any device work, and the Python-side settings checks."""
import ctypes

import pytest

from dreamgaussian_b200 import _lib

MIXED = ("dgr_views_mixed_geom_bytes", "dgr_views_mixed_image_bytes", "dgr_views_mixed_forward_preprocess",
         "dgr_views_mixed_forward_render", "dgr_views_mixed_backward")


def test_mixed_symbols_are_exported_and_the_abi_version_holds():
    lib = _lib.load()
    for name in MIXED:
        assert hasattr(lib, name), name
        assert name in _lib.EXPORTS
    assert lib.dgr_abi_version() == 5


def _hw(sizes):
    flat = [x for hw in sizes for x in hw]
    return (ctypes.c_int32 * len(flat))(*flat)


@pytest.mark.parametrize("V,H,W,P", [(1, 64, 64, 1000), (2, 256, 256, 5000), (4, 72, 96, 2001), (3, 9, 17, 0), (64, 16, 16, 100)])
def test_scratch_sizes_equal_the_same_size_call_when_all_sizes_are_equal(V, H, W, P):
    lib = _lib.load()
    hw = _hw([(H, W)] * V)
    assert lib.dgr_views_mixed_geom_bytes(V, P, hw) == lib.dgr_views_geom_bytes(V, P, H, W)
    assert lib.dgr_views_mixed_image_bytes(V, hw) == lib.dgr_views_image_bytes(V, H, W)


def test_scratch_sizes_follow_the_totals():
    lib = _lib.load()
    a, b = lib.dgr_views_mixed_image_bytes(2, _hw([(256, 256), (512, 512)])), lib.dgr_views_mixed_image_bytes(2, _hw([(512, 512), (256, 256)]))
    assert a == b > lib.dgr_views_image_bytes(2, 256, 256)
    assert lib.dgr_views_mixed_geom_bytes(2, 100, None) == 0 and lib.dgr_views_mixed_image_bytes(2, _hw([(0, 5), (5, 5)])) == 0


BAD = ctypes.c_void_p(0x10)          # never dereferenced: every call below must fail in its argument checks


def _views(V=2):
    return _lib.DgrViews(V, 0, 0, 1.0, 0, 0, BAD, BAD, BAD, BAD, BAD)        # image_height / image_width are not read


def _gaussians(P=100, cov=False, colors=False):
    return _lib.DgrGaussians(P, 1, BAD, None if colors else BAD, BAD if colors else None, BAD, None if cov else BAD,
                             None if cov else BAD, BAD if cov else None, None, 0)


def _err(code):
    assert code != 0
    return _lib.load().dgr_last_error().decode()


def _all_three(views, hw, gaussians, gout=None, stats_views=0):
    lib = _lib.load()
    v, g = ctypes.byref(views), ctypes.byref(gaussians)
    out = _lib.DgrImages(BAD, BAD, BAD, BAD)
    gin = _lib.DgrImageGrads(None, None, None)
    gout = gout or _lib.DgrGaussianGrads()
    return [
        _err(lib.dgr_views_mixed_forward_preprocess(v, hw, g, BAD, BAD, BAD, None)),
        _err(lib.dgr_views_mixed_forward_render(v, hw, g, BAD, BAD, ctypes.c_uint64(1 << 20), BAD, ctypes.byref(out), 0, None,
                                                ctypes.c_uint64(0), None, None)),
        _err(lib.dgr_views_mixed_backward(v, hw, g, BAD, BAD, ctypes.c_uint64(1 << 20), 0, BAD, BAD, ctypes.byref(gin), ctypes.byref(gout),
                                          ctypes.c_uint64(stats_views), None)),
    ]


def _backward(views, hw, gaussians, gout=None, stats_views=0):
    return _all_three(views, hw, gaussians, gout, stats_views)[2]


def test_null_image_hw_is_refused():
    for e in _all_three(_views(), None, _gaussians()):
        assert "image_hw is NULL" in e, e


@pytest.mark.parametrize("bad", [(0, 64), (64, 0), (-3, 64)])
def test_non_positive_size_is_refused(bad):
    for e in _all_three(_views(), _hw([(64, 64), bad]), _gaussians()):
        assert "must be positive" in e, e


@pytest.mark.parametrize("bad", [(65536, 16), (16, 65536)])
def test_size_above_65535_is_refused(bad):
    for e in _all_three(_views(), _hw([(64, 64), bad]), _gaussians()):
        assert "above 65535" in e, e


def test_one_tile_over_51200_is_refused():
    # 49 x 1024 + 992 + 33 tiles: one tile more than 51,200, in views of three different sizes
    sizes = [(512, 512)] * 49 + [(512, 496), (16, 528)]
    tiles = sum(((h + 15) // 16) * ((w + 15) // 16) for h, w in sizes)
    assert tiles == 51201
    for e in _all_three(_views(V=len(sizes)), _hw(sizes), _gaussians()):
        assert "51200" in e, e


@pytest.mark.parametrize("V", [0, 65])
def test_view_count_outside_1_to_64_is_refused(V):
    for e in _all_three(_views(V=V), _hw([(16, 16)] * max(V, 1)), _gaussians()):
        assert "V must be 1..64" in e, e


def test_more_records_than_the_bound_is_refused():
    P = _lib.VIEWS_MAX_RECORDS // 64 + 1
    for e in _all_three(_views(V=64), _hw([(16, 16)] * 64), _gaussians(P=P)):
        assert "V x P" in e, e


def _stats(field="denom"):
    gout = _lib.DgrGaussianGrads()
    setattr(gout, field, 0x10)
    return gout


@pytest.mark.parametrize("bit", [2, 5, 63])
def test_a_stats_views_bit_at_or_above_V_is_refused(bit):
    e = _backward(_views(V=2), _hw([(16, 16), (32, 32)]), _gaussians(), gout=_stats(), stats_views=1 << bit)
    assert "at or above V" in e, e


def test_stats_views_without_a_statistic_buffer_is_refused():
    e = _backward(_views(), _hw([(16, 16), (32, 32)]), _gaussians(), stats_views=2)
    assert "no densification statistic buffer" in e, e


@pytest.mark.parametrize("field", ["xyz_gradient_accum", "denom", "max_radii2D"])
def test_a_statistic_buffer_without_stats_views_is_refused(field):
    e = _backward(_views(), _hw([(16, 16), (32, 32)]), _gaussians(), gout=_stats(field), stats_views=0)
    assert "stats_views is 0" in e, e


@pytest.mark.parametrize("what", ["colors", "cov"])
def test_precomputed_colours_or_covariance_are_refused(what):
    for e in _all_three(_views(), _hw([(16, 16), (32, 32)]), _gaussians(colors=what == "colors", cov=what == "cov")):
        assert "precomputed colours / cov3D" in e, e


def test_push_is_refused():
    gout = _lib.DgrGaussianGrads()
    gout.push = 0x10
    e = _backward(_views(), _hw([(16, 16), (32, 32)]), _gaussians(), gout=gout)
    assert "DgrPeerPush" in e, e


# ---- Python-side checks --------------------------------------------------------------------------------------------------
def _settings(H=64, W=64, deg=0, sm=1.0, device="cpu"):
    import torch
    from dreamgaussian_b200.rasterizer import GaussianRasterizationSettings
    z = lambda n: torch.zeros(n, device=device)
    return GaussianRasterizationSettings(H, W, 0.5, 0.5, z(3), sm, torch.eye(4, device=device), torch.eye(4, device=device), deg, z(3),
                                         False, False)


def _call(settings, raw=False, **kw):
    import torch
    z = torch.zeros
    if raw:
        from dreamgaussian_b200.fused import rasterize_views_mixed_raw
        return rasterize_views_mixed_raw(settings, z(10, 3), None, z(10, 1, 3), z(10, 0, 3), z(10, 1), z(10, 3), z(10, 4), **kw)
    from dreamgaussian_b200.rasterizer import rasterize_views_mixed
    return rasterize_views_mixed(settings, z(10, 3), None, z(10, 1), z(10, 1, 3), z(10, 3), z(10, 4))


@pytest.mark.parametrize("raw", [False, True])
def test_sizes_may_differ_and_cpu_tensors_raise_no_cpu_path(raw):
    with pytest.raises(RuntimeError, match="no CPU path"):
        _call([_settings(), _settings(H=32, W=48), _settings(H=9, W=17)], raw=raw)


@pytest.mark.parametrize("field", ["sh_degree", "scale_modifier"])
@pytest.mark.parametrize("raw", [False, True])
def test_mismatched_degree_or_scale_modifier_raise(field, raw):
    other = dict(sh_degree=dict(deg=1), scale_modifier=dict(sm=0.5))[field]
    with pytest.raises(ValueError, match=field):
        _call([_settings(), _settings(H=32, **other)], raw=raw)


@pytest.mark.parametrize("views", [(2,), (0, 5), (-1,)])
def test_a_stats_views_entry_outside_the_batch_raises(views):
    from dreamgaussian_b200.fused import DensifyStats
    with pytest.raises(ValueError, match="stats_views"):
        _call([_settings(), _settings(H=32)], raw=True, stats=DensifyStats(10, "cpu"), stats_views=views)


def test_batched_stage1_needs_the_fused_path():
    from dreamgaussian_b200.stage1 import Stage1Trainer
    with pytest.raises(ValueError, match="batched"):
        Stage1Trainer(device="cpu", fused=False, batched=True)
