"""The rasterizer on trained-model parameters (tests/trained_scenes.py) against the CPU oracles: saturated opacities, dark and
over-bright colours, needles, faint and sub-pixel Gaussians, the near plane and the frustum edge, and all of them mixed;
plain and raw parameters, single view and batched cameras.  The float32 comparison keeps no decision-ambiguity exemption.

The support test needs no tolerance: on scenes where every pixel has at most one candidate Gaussian, CUDA alpha > 0 must
hold exactly where the float64 oracle's alpha >= 1/255, on every pixel the oracle does not flag, under every render-kernel
variant.  It is the test that catches an opacity-aware AABB or sub-tile ellipse cull that drops pixels."""
import numpy as np
import pytest

import helpers as h
import test_variants_gpu as variants
import test_views_gpu as views
import trained_scenes as ts
from oracle import c_oracle

pytestmark = pytest.mark.gpu

# Per-case max_ambig_frac: the measured fraction of pixels the float64 oracle flags, plus a margin.  Needles flag wide swaths:
# the quadratic form's terms are large there and cancel, so a float32 alpha >= 1/255 decision can go either way over much of
# a needle's footprint (bit 1).  The float32 comparison, which has no such exemption, judges those pixels too.
# The needle parity cases draw needles in random 3-D orientations with axis ratios 10-30 (trained_mix: 10-100).  At higher
# ratios two float32 evaluations (this kernel and the float32 oracle) disagree on a few colours and on the scale / rotation
# gradients of a few needles by more than the float32 comparison allows (ratios up to 100: 3 pixels at 1.5e-3 and 7
# Gaussians of 1500; up to 1000: 6 pixels and 13-24 Gaussians).  The needles of higher ratio and the screen-space needles
# of 20-400 px (condition numbers up to 5e5) are judged by the support test below, against the
# kernel's own float32 conic: their float32 det = cxx cyy - cxy^2 cancels to a relative error of ~eps times the condition
# number, so any float32 evaluation, the float32 oracle's included, differs from the float64 one across whole footprints
# (test_trained_regimes_cpu.py::test_float32_cancellation_of_screen_space_needles shows it without the GPU).
CASES = {
    "saturated": (ts.saturated, 0.13),          # measured 0.106: the sub-pixel pairs' T-stop knife edge (bit 2)
    "dark_deg0": (lambda: ts.dark(deg=0), h.MAX_AMBIG_FRAC),
    "dark_deg3": (lambda: ts.dark(deg=3), h.MAX_AMBIG_FRAC),
    "needles": (lambda: ts.needles(n=4000, constructed=0, max_ratio=30.0), 0.05),
    "needles_deg0": (lambda: ts.needles(deg=0, n=4000, constructed=0, max_ratio=30.0), 0.05),
    "faint": (ts.faint, h.MAX_AMBIG_FRAC),
    "subpixel": (ts.subpixel, 0.03),            # measured 0.016: centres on pixel centres (power = 0, bit 8)
    "frustum_edge": (ts.frustum_edge, h.MAX_AMBIG_FRAC),
    "trained_mix": (ts.trained_mix, 0.07),      # measured 0.051 (0.017 for the raw form)
}

_CACHE = {}


def _case(name):
    """(settings, inputs, upstream grads, both oracle results) of a case, computed once."""
    if name not in _CACHE:
        s, i = CASES[name][0]()
        g = h.upstream_grads(s["image_height"], s["image_width"])
        _CACHE[name] = (s, i, g, h.oracles(s, i, g))
    return _CACHE[name]


@pytest.mark.parametrize("name", list(CASES))
def test_plain_op_matches_both_oracles(name):
    s, i, g, refs = _case(name)
    h.both_oracles("trained/" + name, s, i, g, max_ambig_frac=CASES[name][1], refs=refs)


@pytest.mark.parametrize("name", ["saturated", "dark_deg3", "trained_mix"])
def test_raw_parameters_match_the_oracle(name):
    s, i, g, refs = _case(name)
    raw = ts.raw_of(i, seed=11, extremes=name == "trained_mix")
    ref = h.run_oracle_raw(s, raw, g)
    cu = h.run_cuda_raw(s, raw, g)
    ok, rep = h.compare(cu, ref, max_ambig_frac=CASES[name][1])
    h.report("trained raw/" + name, vs_f64=rep)
    assert ok, rep


@pytest.mark.parametrize("name", ["trained_mix", "needles_deg0"])
def test_batched_views_match_both_oracles(name):
    """View 0 is the case's own camera, view 1 the same pose with a black background and other upstream gradients.  (The
    scenes place their regimes for this pose: another pose would move the near-plane and frustum-edge Gaussians off their
    constructed values.)"""
    s0, i, g0, refs0 = _case(name)
    s1 = dict(s0, bg=np.zeros(3, np.float32))
    g1 = h.upstream_grads(s0["image_height"], s0["image_width"], seed=321)
    settings = [s0, s1]
    for v, (s, g, refs) in enumerate(((s0, g0, refs0), (s1, g1, None))):
        cu = views.run_views(settings, i, [g if u == v else None for u in range(2)])
        cv = views._view(cu, v)
        cv["grads"] = dict(cu["grads"], means2D=cu["grads"]["means2D"][v])
        h.both_oracles("trained views/%s v%d" % (name, v), s, i, g, max_ambig_frac=CASES[name][1], refs=refs, cu=cv)


# ---------------------------------------------------------------------------------------------------------------------------
# support: alpha > 0 exactly where the float64 oracle's alpha >= 1/255 (isolated Gaussians, every render-kernel variant)
# ---------------------------------------------------------------------------------------------------------------------------
ISOLATED = {
    "small": ts.isolated_small,
    "needles_45": lambda: ts.isolated_needles(theta=np.pi / 4),
    "needles_135": lambda: ts.isolated_needles(theta=3 * np.pi / 4),
}
_ISO = {}


def _isolated(name):
    """(settings, inputs, float64 alpha, pixels the float64 oracle judges): every pixel it does not flag with bit 1, except, for
    a Gaussian whose 3-sigma tile rect sits on a rounding boundary (bit 4), the ring of tiles either side of its rect's edge,
    the only tiles that decision can move."""
    if name not in _ISO:
        s, i = ISOLATED[name]()
        r = c_oracle.forward(**s, **i)
        apx, ag, _ = r.flags()
        judged = (apx & 1) == 0
        rects = r.state()["rect"]
        for g in np.nonzero((ag & 4) != 0)[0]:
            x0, y0, x1, y1 = (int(v) for v in rects[g])
            ring = np.zeros_like(judged)
            ring[max(0, y0 - 1) * 16:(y1 + 1) * 16, max(0, x0 - 1) * 16:(x1 + 1) * 16] = True
            ring[(y0 + 1) * 16:max(y0 + 1, y1 - 1) * 16, (x0 + 1) * 16:max(x0 + 1, x1 - 1) * 16] = False
            judged &= ~ring
        _ISO[name] = (s, i, r.alpha[0].copy(), judged)
        r.close()
    return _ISO[name]


def _f32(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


def _own_alpha(rec, radii, H, W):
    """The kernel's own per-pixel decision, from the records its forward preprocess wrote (Rec in dgr_common.cuh: q0 = mean x,
    mean y, -0.5 A log2e, -B log2e; q1 = -0.5 C log2e, opacity, ...): eval_power2's
    float32 fused multiply-adds emulated in float64 with one rounding each, alpha = o 2^power2, the 3-sigma tile rect from
    the same float32 steps.  Returns (contributes [H, W], near [H, W]): near = within 1e-5 relative of 1/255, where the
    approximate ex2 of the kernel may decide either way; every other pixel is decided."""
    want = np.zeros((H, W), bool)
    near = np.zeros((H, W), bool)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    for g in np.nonzero(radii > 0)[0]:
        mx, my, nA, nB = rec[g, 0:4]
        nC, o = rec[g, 4], rec[g, 5]
        rad = float(radii[g])
        x0 = min(gx, max(0, int(_f32(mx - rad) / 16))); x1 = min(gx, max(0, int(_f32(_f32(mx + rad) + 15) / 16)))
        y0 = min(gy, max(0, int(_f32(my - rad) / 16))); y1 = min(gy, max(0, int(_f32(_f32(my + rad) + 15) / 16)))
        ys, xs = np.mgrid[y0 * 16:min(y1 * 16, H), x0 * 16:min(x1 * 16, W)]
        dx, dy = _f32(mx - xs), _f32(my - ys)
        t = _f32(nA * dx + _f32(nB * dy))
        p2 = _f32(dx * t + _f32(_f32(nC * dy) * dy))
        a = np.minimum(0.99, o * np.exp2(p2))
        amin = float(np.float32(1.0 / 255.0))
        want[ys, xs] |= (p2 <= 0) & (a >= amin)
        near[ys, xs] |= np.abs(a / amin - 1.0) < 1e-5
    return want, near


def _forward_with_records(s, i):
    """One forward through the ctypes host layer: (alpha [H, W], radii, the [P, 12] float32 records)."""
    import torch
    from dreamgaussian_b200 import rasterizer as R
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda").contiguous()
    _, radii, _, alpha, state = R.forward_impl(views._rs(s), t(i["means3D"]), t(i["shs"]), None, t(i["opacities"]), t(i["scales"]),
                                               t(i["rotations"]), None)
    P = i["means3D"].shape[0]
    rec = state.geom[256:256 + 48 * P].view(torch.float32).reshape(P, 12)         # GeomLayout: records at byte 256
    return alpha[0].cpu().numpy(), radii.cpu().numpy(), rec.cpu().numpy().astype(np.float64)


@pytest.mark.parametrize("word", list(variants.WORDS))
@pytest.mark.parametrize("name", list(ISOLATED))
def test_support_matches_the_oracle_exactly(name, word):
    """CUDA alpha > 0 (a) exactly where the float64 oracle's alpha >= 1/255, on the pixels it judges, and (b) exactly where the
    kernel's own float32 record gives alpha >= 1/255 inside its 3-sigma tile rect, on every pixel not within 1e-5 of 1/255.
    (b) is what pins the opacity-aware AABB and the sub-tile ellipse test on needles, whose float64 footprints are flagged
    almost entirely; it must judge at least 500 pixels within a factor 2 of the 1/255 edge."""
    s, i, ref_alpha, judged = _isolated(name)
    alpha, radii, rec = h.run_tuned(variants.WORDS[word], lambda: _forward_with_records(s, i), fast_host=False)
    got = alpha > 0
    want = ref_alpha >= ts.ALPHA_MIN
    lost = int((want & ~got & judged).sum())
    extra = int((got & ~want & judged).sum())
    own, near = _own_alpha(rec, radii, s["image_height"], s["image_width"])
    own_lost = int((own & ~got & ~near).sum())
    own_extra = int((got & ~own & ~near).sum())
    edge = int(((alpha > 0) & (alpha < 2 * ts.ALPHA_MIN) & ~near).sum())
    h.report("support/%s/%s" % (name, word), support=dict(
        pixels=int(want.sum()), judged_footprint=int((want & judged).sum()), lost=lost, extra=extra,
        own_pixels=int(own.sum()), own_near=int((own & near).sum()), own_edge=edge, own_lost=own_lost, own_extra=own_extra))
    assert lost == 0 and extra == 0, (lost, extra)
    assert own_lost == 0 and own_extra == 0, (own_lost, own_extra)
    assert edge >= 500


# ---------------------------------------------------------------------------------------------------------------------------
# straight-through alpha clamp: gradients of a Gaussian whose only hit is clamped to 0.99
# ---------------------------------------------------------------------------------------------------------------------------
def test_straight_through_clamp_gradients():
    """The front Gaussian of every stack (trained_scenes.clamped_stacks) has o G in (0.99, 1]: alpha is clamped to 0.99, but
    the opacity and means2D gradients use the unclamped o G (dL/do = G dL/dalpha).  Against the float64 oracle, per
    Gaussian, to 1e-4 of its own value: a kernel that used the clamped alpha would be 0.1-1% off, one that masked the
    clamped hit would give zero."""
    checked = 0
    for n, (s, i) in enumerate(ts.clamped_stacks()):
        g = h.upstream_grads(1, 1, seed=500 + n)
        ref = h.run_oracle(s, i, g)
        cu = h.run_cuda(s, i, g)
        h.both_oracles("clamped_stack_%d" % n, s, i, g, cu=cu)
        if ref["ambig_px"][0, 0] or ref["ambig_g"][0]:
            continue
        checked += 1
        for k in ("opacities", "means2D"):
            r = np.asarray(ref["grads"][k][0], np.float64)
            c = np.asarray(cu["grads"][k][0], np.float64).reshape(r.shape)
            assert np.abs(r).max() > 0
            assert np.abs(c - r).max() <= 1e-4 * np.abs(r).max(), (n, k, c, r)
    assert checked >= 16
