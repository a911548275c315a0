"""GPU tests of every render-kernel variant, scheduling switch and image-size limit the library compiles and exposes.

Each variant is judged like the default path (tests/helpers.py: both CPU oracles, the suite's bounds) and its forward
images must be bit-identical to the default tuning's: DESIGN.md §4 holds the per-pixel arithmetic independent of the
sub-tile shape, of the hits evaluated together and of the record staging (sorted copy or by id: the same records in the
same order).  The tuning knobs are process-wide and may change between a forward and its backward: the backward must
run from what its forward left behind, whatever the knobs say by then.
"""
import numpy as np
import pytest
import torch

import helpers as h
from dreamgaussian_b200 import rasterizer as R
from dreamgaussian_b200 import scene

pytestmark = pytest.mark.gpu

SORTED, BY_ID = 1 << 22, 2 << 22          # dgr_set_tuning bits 22-23: record staging
PER_PIXEL = 1 << 26                      # backward render step 2 in its per-pixel form (sorted copy only)
SWITCHES = {"cost_order_off": 1 << 21, "two_ended": 1 << 20, "one_cta_per_sm": (1 << 12) | (1 << 16), "pdl_off": 1 << 3,
            "sort_2048_buckets": 1 << 28}
ALL_SWITCHES = sum(SWITCHES.values())

# (ppl_fwd, ppl_bwd, bits): forward / backward render kernels <PPL, U>
SHAPES = {
    "f11_b12": (1, 1, 1),                               # <1,1> / <1,2> row-sum (the default)
    "f11_b12_perpixel": (1, 1, 1 | PER_PIXEL),          # <1,1> / <1,2> per-pixel step 2
    "f14_b11": (1, 1, 1 | (4 << 4) | (1 << 8)),         # <1,4> / <1,1>
    "f22_b21": (2, 2, 1),                               # <2,2> / <2,1>, costed (same sub-tile shape)
    "f22_b22": (2, 2, 1 | (2 << 8)),                    # <2,2> / <2,2>
    "f11_b21": (1, 2, 1),                               # <1,1> / <2,1>: two forward items per backward item
    "f41_b12": (4, 1, 1),                               # <4,1> / <1,2>: 16x8 does not nest in 8x4, no costing
}
WORDS = {}
for _n, (_f, _b, _bits) in SHAPES.items():
    WORDS[_n + "_sorted"] = (_f, _b, _bits | SORTED)
    if not _bits & PER_PIXEL:
        WORDS[_n + "_byid"] = (_f, _b, _bits | BY_ID)
for _n, _bit in SWITCHES.items():
    WORDS[_n] = (1, 1, 1 | _bit)
WORDS["all_switches"] = (1, 1, 1 | ALL_SWITCHES)
WORDS["all_switches_byid"] = (1, 1, 1 | ALL_SWITCHES | BY_ID)


def _precomputed(i, seed=3):
    """The case's Gaussians as colors_precomp + cov3D_precomp (Sigma = R S S^T R^T from its scales / rotations)."""
    q, sc = i["rotations"].astype(np.float64), i["scales"].astype(np.float64)
    q = q / np.linalg.norm(q, axis=1, keepdims=True)
    Rm = np.stack([
        1 - 2 * (q[:, 2] ** 2 + q[:, 3] ** 2), 2 * (q[:, 1] * q[:, 2] - q[:, 0] * q[:, 3]), 2 * (q[:, 1] * q[:, 3] + q[:, 0] * q[:, 2]),
        2 * (q[:, 1] * q[:, 2] + q[:, 0] * q[:, 3]), 1 - 2 * (q[:, 1] ** 2 + q[:, 3] ** 2), 2 * (q[:, 2] * q[:, 3] - q[:, 0] * q[:, 1]),
        2 * (q[:, 1] * q[:, 3] - q[:, 0] * q[:, 2]), 2 * (q[:, 2] * q[:, 3] + q[:, 0] * q[:, 1]), 1 - 2 * (q[:, 1] ** 2 + q[:, 2] ** 2)],
        1).reshape(-1, 3, 3)
    Mx = Rm * sc[:, None, :]
    S = Mx @ Mx.transpose(0, 2, 1)
    cov6 = np.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1).astype(np.float32)
    rgb = np.random.default_rng(seed).random((q.shape[0], 3)).astype(np.float32)
    return dict(means3D=i["means3D"], opacities=i["opacities"], colors_precomp=rgb, cov3D_precomp=cov6)


CASES = {
    # sides that are multiples of neither 8 nor 16: every sub-tile shape is cut at the right and the bottom edge
    "edges_37x23_deg2": dict(P=400, res=0, width=37, height=23, deg=2, sigma=0.05, elev=5, azim=60, radius=1.2),
    "odd_size_deg1": dict(P=500, res=0, width=100, height=70, deg=1, sigma=0.04, elev=-20, azim=200),
    # the reference's initial opacity 0.1: no list ends early
    "cfg1_5k_256_init": dict(P=5000, res=256, deg=0, opacity="init", anisotropic=False),
    "big_tiles": dict(P=20000, res=32, deg=0, sigma=0.02),                # ~5k instances per tile: big-tile sorter
    "huge_tiles": dict(P=60000, res=32, deg=0, sigma=0.01),               # > 12288 per tile: in-place global sort
    "mid_20k_400_deg3_no_depth_grad": dict(P=20000, res=400, deg=3),
    "precomputed_colour_cov3D": dict(P=600, res=64, deg=0, sigma=0.05, elev=5, azim=140),
}

_CACHE = {}


def _case(name):
    """(settings, inputs, upstream grads, both oracle results, the default tuning's CUDA result) of a case, computed once."""
    if name not in _CACHE:
        s, i = h.make_case(**CASES[name])
        if name.startswith("precomputed"):
            i = _precomputed(i)
        g = h.upstream_grads(s["image_height"], s["image_width"], depth="no_depth" not in name)
        refs = h.oracles(s, i, g)
        base = h.run_tuned(h.DEFAULT_TUNING, lambda: h.run_cuda(s, i, g))
        _CACHE[name] = (s, i, g, refs, base)
    return _CACHE[name]


_HINTS = []                       # (compiled host layer?, key, capacity hint before the test changed it)


def _set_hint(key, cap, big):
    """Capacity hint of the CURRENT host layer for key = (device, P, H, W); the fixture puts the old one back."""
    _HINTS.append((R._FAST is not None, key, R.get_capacity_hint(*key)))
    R.set_capacity_hint(*key, cap, big)


@pytest.fixture(autouse=True)
def _restore_tuning_host_layer_and_hints():
    yield
    h.set_tuning(h.DEFAULT_TUNING)
    while _HINTS:
        fast, key, old = _HINTS.pop()
        R.set_fast_host(fast)
        if old is not None:
            R.set_capacity_hint(*key, *old)
        elif fast:
            R.set_capacity_hint(*key, max(65536, 16 * key[1]), True)       # what the layer assumes without a hint
        else:
            R._CAPACITY_HINT.pop(key, None)
    R.set_fast_host(True)


def _images_equal(a, b):
    return {k: float(np.abs(a[k].astype(np.float64) - b[k]).max()) for k in ("color", "depth", "alpha", "radii")
            if not np.array_equal(a[k], b[k])}


@pytest.mark.parametrize("word", list(WORDS))
@pytest.mark.parametrize("case", list(CASES))
def test_variant_matches_the_oracles_and_the_default_images(case, word):
    s, i, g, refs, base = _case(case)
    cu = h.run_tuned(WORDS[word], lambda: h.run_cuda(s, i, g))
    assert not _images_equal(cu, base), ("forward differs from the default tuning's", _images_equal(cu, base))
    h.both_oracles("%s/%s" % (case, word), s, i, g, refs=refs, cu=cu)


# ---------------------------------------------------------------------------------------------------------------------
# Tuning changed between a forward and its backward
# ---------------------------------------------------------------------------------------------------------------------
SWITCH_CASE = dict(P=6000, res=160, deg=2, seed=17, elev=8, azim=-35)
L2_BUSTING_HINT = 2_500_000          # instances: 2.5 M x 48-byte records = 120 MB, above twice the H100's 50 MB L2

SWITCH_PAIRS = {
    "byid_to_sorted": ((1, 1, 1 | BY_ID), (1, 1, 1 | SORTED), None),
    "auto_large_capacity_to_sorted": ((1, 1, 1), (1, 1, 1 | SORTED), L2_BUSTING_HINT),
    "sorted_to_byid": ((1, 1, 1 | SORTED), (1, 1, 1 | BY_ID), None),
    "ppl_bwd_1_to_2": ((1, 1, 1), (1, 2, 1), None),
    "ppl_bwd_2_to_1": ((1, 2, 1), (1, 1, 1), None),
    "cost_order_on_to_off": ((1, 1, 1), (1, 1, 1 | (1 << 21)), None),
    "cost_order_off_to_on": ((1, 1, 1 | (1 << 21)), (1, 1, 1), None),
}

_SWITCH_REFS = {}


def _switch_case():
    if not _SWITCH_REFS:
        s, i = h.make_case(**SWITCH_CASE)
        g = h.upstream_grads(s["image_height"], s["image_width"])
        _SWITCH_REFS["case"] = (s, i, g, h.oracles(s, i, g))
    return _SWITCH_REFS["case"]


@pytest.mark.parametrize("fast_host", [True, False], ids=["compiled_host", "ctypes_host"])
@pytest.mark.parametrize("pair", list(SWITCH_PAIRS))
def test_backward_follows_its_forward_when_the_tuning_changes_in_between(pair, fast_host):
    word_fwd, word_bwd, hint = SWITCH_PAIRS[pair]
    s, i, g, refs = _switch_case()

    def run():
        if hint is not None:
            _set_hint((torch.cuda.current_device(), i["means3D"].shape[0], s["image_height"], s["image_width"]), hint, True)
        return h.run_cuda(s, i, g, before_backward=lambda: h.set_tuning(word_bwd))

    h.both_oracles("switch/%s/%s" % (pair, "compiled" if fast_host else "ctypes"), s, i, g, refs=refs,
                   cu=h.run_tuned(word_fwd, run, fast_host))


@pytest.mark.parametrize("fast_host", [True, False], ids=["compiled_host", "ctypes_host"])
def test_two_retained_backwards_of_one_forward_under_different_tunings(fast_host):
    s, i, g, refs = _switch_case()
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda")

    def run():
        rs = R.GaussianRasterizationSettings(
            image_height=s["image_height"], image_width=s["image_width"], tanfovx=s["tanfovx"], tanfovy=s["tanfovy"], bg=t(s["bg"]),
            scale_modifier=s["scale_modifier"], viewmatrix=t(s["viewmatrix"]), projmatrix=t(s["projmatrix"]),
            sh_degree=s["sh_degree"], campos=t(s["campos"]), prefiltered=False, debug=False)
        leaves = {k: t(v).requires_grad_(True) for k, v in i.items()}
        m2d = torch.zeros_like(leaves["means3D"], requires_grad=True)
        color, radii, depth, alpha = R.GaussianRasterizer(rs)(means2D=m2d, **leaves)
        loss = (color * t(g[0])).sum() + (depth * t(g[1])).sum() + (alpha * t(g[2])).sum()
        names = list(leaves)
        img = dict(color=color.detach().cpu().numpy(), depth=depth.detach().cpu().numpy(), alpha=alpha.detach().cpu().numpy(),
                   radii=radii.cpu().numpy())
        outs = []
        for word, retain in (((1, 1, 1), True), ((1, 2, 1 | (1 << 21) | BY_ID), False)):
            h.set_tuning(word)
            gr = torch.autograd.grad(loss, [leaves[k] for k in names] + [m2d], retain_graph=retain)
            outs.append(dict(img, grads={k: v.detach().cpu().numpy() for k, v in zip(names + ["means2D"], gr)}))
        return outs

    for n, cu in enumerate(h.run_tuned(h.DEFAULT_TUNING, run, fast_host)):
        h.both_oracles("retained_backward_%d" % n, s, i, g, refs=refs, cu=cu)


# ---------------------------------------------------------------------------------------------------------------------
# Capacity repair (the instance buffer guess was too small: stage 2 re-runs) under each record staging
# ---------------------------------------------------------------------------------------------------------------------
REPAIR_CASE = dict(P=3000, res=128, deg=1, sigma=0.05)


@pytest.mark.parametrize("fast_host", [True, False], ids=["compiled_host", "ctypes_host"])
@pytest.mark.parametrize("word", [(1, 1, 1 | SORTED), (1, 1, 1 | BY_ID), (2, 2, 1)], ids=["sorted", "byid", "ppl2"])
def test_capacity_repair_under_each_staging(word, fast_host):
    s, i = h.make_case(**REPAIR_CASE)
    g = h.upstream_grads(128, 128)
    key = (torch.cuda.current_device(), REPAIR_CASE["P"], 128, 128)

    def run():
        plain = h.run_cuda(s, i, g)
        assert R.get_capacity_hint(*key)[0] > 64
        _set_hint(key, 64, False)                          # absurdly small instance buffer, no big-tile sorter
        repaired = h.run_cuda(s, i, g)
        assert R.get_capacity_hint(*key)[0] > 64
        return plain, repaired

    plain, repaired = h.run_tuned(word, run, fast_host)
    assert not _images_equal(plain, repaired), _images_equal(plain, repaired)
    h.both_oracles("repair/%r" % (word,), s, i, g, cu=repaired)


# ---------------------------------------------------------------------------------------------------------------------
# Image sizes at and beyond the library's limits
# ---------------------------------------------------------------------------------------------------------------------
def _exact_case(W, H, kxs, kys, deg=1, seed=5):
    """Gaussians whose projected centres float32 represents exactly, on a lattice over a W x H image.

    From pixel coordinate ~4096 on, the rounding of a projected centre alone (ulp(32768) = 0.004 px) moves the alpha >= 1/255
    edge of a footprint across pixels: decisions a float32 implementation may take either way but neither oracle flags.  So
    the camera looks down the world z axis from (0, 0, 2) with tan(half field of view) = 2 on both axes (ndc = x_view /
    (2 z_view)), the centres sit at ndc + 1 = k / 128 on both axes and at view depth 2 or 4: every step from the world
    position to the pixel position is then exact in float32 and float64 alike.  kxs / kys: the lattice's k values.  The
    lattice is a checkerboard of the view depths 2 and 4 and no footprint reaches a Gaussian of its own depth (no depth ties)."""
    rng = np.random.default_rng(seed)
    cam = scene.orbit_camera(0.0, 0.0, 2.0, W, H)
    V = cam.world_view_transform.astype(np.float64)                              # p_view = [p, 1] @ V
    Pm = np.zeros((4, 4)); Pm[0, 0] = Pm[1, 1] = 0.5; Pm[3, 2] = 1.0
    Pm[2, 2] = 100.0 / (100.0 - 0.01); Pm[2, 3] = -(100.0 * 0.01) / (100.0 - 0.01)
    full = (V @ Pm.T).astype(np.float32)
    ix, iy = np.meshgrid(np.arange(len(kxs)), np.arange(len(kys)), indexing="ij")
    ix, iy = ix.ravel(), iy.ravel()
    P = ix.size
    ndc_x, ndc_y = np.asarray(kxs, np.float64)[ix] / 128.0 - 1.0, np.asarray(kys, np.float64)[iy] / 128.0 - 1.0
    z = 2.0 ** (1 + (ix + iy) % 2)
    view = np.stack([2.0 * z * ndc_x, 2.0 * z * ndc_y, z, np.ones(P)], 1)
    world = (view @ np.linalg.inv(V))[:, :3]
    hom = np.concatenate([world.astype(np.float32).astype(np.float64), np.ones((P, 1))], 1) @ full.astype(np.float64)
    assert np.array_equal(hom[:, 0] / hom[:, 3], ndc_x) and np.array_equal(hom[:, 1] / hom[:, 3], ndc_y)

    def cap(ks, other, size):                     # pixel sigma whose footprint (<= 3.4 sigma) stays clear of its own depth
        if len(ks) == 1:
            return size / 3.5
        return size * (ks[1] - ks[0]) / 256.0 / (7.0 if len(other) > 1 else 4.5)      # diagonal neighbours share a depth
    sig = np.stack([rng.uniform(0.75, 1.0, P) * cap(kxs, kys, W) * 4.0 * z / W,        # focal = W / (2 tan) = W / 4 pixels per unit
                    rng.uniform(0.75, 1.0, P) * cap(kys, kxs, H) * 4.0 * z / H, rng.uniform(0.2, 1.0, P) * 4.0 * z / max(W, H)], 1)
    # near axis-aligned, so the caps hold per axis (with pixels W / H times wider than tall a tilt mixes the axes' scales that much)
    q = np.concatenate([np.ones((P, 1)), rng.normal(0.0, 0.05 * min(W, H) / max(W, H), (P, 3))], 1)
    M = (deg + 1) ** 2
    shs = np.zeros((P, M, 3))
    shs[:, 0] = (rng.random((P, 3)) - 0.5) / scene.SH_C0
    shs[:, 1:] = rng.normal(0.0, 0.1, (P, M - 1, 3))
    f32 = lambda a: np.ascontiguousarray(np.asarray(a, np.float64).astype(np.float32))
    inputs = dict(means3D=f32(world), opacities=f32(rng.uniform(0.5, 0.95, (P, 1))), shs=f32(shs), scales=f32(sig),
                  rotations=f32(q / np.linalg.norm(q, axis=1, keepdims=True)))
    settings = dict(image_height=H, image_width=W, tanfovx=2.0, tanfovy=2.0, bg=np.ones(3, np.float32), scale_modifier=1.0,
                    viewmatrix=cam.world_view_transform, projmatrix=full, sh_degree=deg, campos=cam.camera_center)
    return settings, inputs


ALL_K, K4 = list(range(0, 257)), list(range(0, 257, 4))
SIZE_CASES = {
    "2048sq_deg3": dict(P=3000, res=2048, deg=3, sigma=0.01),                  # 16,384 tiles: histogram above 48 KB, staged
    # exactly 51,200 tiles: a 200 KB histogram; at degree 3 with per-thread loads (histogram + staging > 227 KB), at degree 0 staged
    "4096x3200_deg3": dict(W=4096, H=3200, kxs=K4, kys=K4, deg=3),
    "4096x3200_deg0": dict(W=4096, H=3200, kxs=K4, kys=K4, deg=0),
    # pixel coordinates from 32640 on: the packed pixel AABB word bx0 | bx1 << 16 (by0 | by1 << 16) that travels as a float
    # is a NaN bit pattern, which the sort gather, the bulk copies and the shared-memory reads must pass on unchanged
    "65535x16": dict(W=65535, H=16, kxs=ALL_K, kys=[129]),
    "16x65535": dict(W=16, H=65535, kxs=[129], kys=ALL_K),
    "1x1": dict(P=30, res=0, width=1, height=1, deg=1, sigma=0.05),
    # (off the pixel centres: a centre on one puts power = 0 at that pixel, a decision the oracles flag as ambiguous)
    "1x200": dict(W=1, H=200, kxs=[129], kys=list(range(1, 257, 8)) + [256]),
    "200x1": dict(W=200, H=1, kxs=list(range(1, 257, 8)) + [256], kys=[129]),
}


@pytest.mark.parametrize("name", list(SIZE_CASES))
def test_image_size_limits(name):
    c = SIZE_CASES[name]
    s, i = _exact_case(**c) if "W" in c else h.make_case(**c)
    H, W = s["image_height"], s["image_width"]
    g = h.upstream_grads(H, W)
    refs = h.oracles(s, i, g)
    a = refs["f64"]["alpha"][0]
    if "W" in c:                                   # covered up to the far end of the long side
        assert a.max(axis=0)[-1] > 0 and a.max(axis=1)[-1] > 0
    if max(W, H) == 65535:                         # footprints that reach across 32640 from either side
        along = a.max(axis=0) if W > H else a.max(axis=1)
        assert along[32560:32720].min() > 0
    h.both_oracles("size/" + name, s, i, g, refs=refs)


@pytest.mark.parametrize("fast_host", [True, False], ids=["compiled_host", "ctypes_host"])
def test_images_beyond_the_limits_raise_the_library_error(fast_host):
    for (W, H), msg in (((4096, 3216), "more than 51200 tiles"), ((65536, 16), "above 65535"), ((16, 65536), "above 65535")):
        s, i = h.make_case(P=100, res=0, width=W, height=H, deg=0, sigma=0.05)
        with pytest.raises(RuntimeError, match=msg):
            h.run_tuned(h.DEFAULT_TUNING, lambda: h.run_cuda(s, i), fast_host)
    s, i = h.make_case(P=100, res=32, deg=0, sigma=0.05)          # nothing was left broken on the device
    h.both_oracles("after_size_errors", s, i, h.upstream_grads(32, 32))
