"""SH storage wider than the active degree, on every render path: rows of M coefficients rendered at a degree that reads NB < M.

A 3DGS-style caller keeps (max_sh_degree + 1)^2 coefficients per Gaussian and renders at active_sh_degree (gs_renderer.py:806;
dreamgaussian_b200.stage1 does the same), so every per-Gaussian kernel takes M as a runtime row stride next to the compile-time
degree.  Each cell below renders a small compact scene (tests/trained_scenes.compact_mix: P not a multiple of 32, sides not
multiples of 16, near-plane, off-frustum, saturated, needle and clamped-colour Gaussians) whose padding holds +-10, so a read of it
shows in the image, and applies the rules the suite already has:

1. images, radii and gradients of the padded call: helpers.both_oracles (raw parameters: run_oracle_raw + helpers.compare;
   anti-aliased: tests/aa_oracle.py), through test_kernel_coverage_gpu's judges;
2. camera gradients by test_camera_grads_gpu's d <= max(1e-3, 3 d32); the AbsGS statistic and the contribution statistics by the
   check_rule of test_absgrad_gpu / test_contrib_gpu (tests/test_sh_padding_cpu.py shows these oracles ignore the padding);
3. the gradient of every padding coefficient is exactly 0.0, in dL/dshs and dL/d_features_rest; the gradient tensors are first
   dirtied with NaN in the caching allocator, so a skipped zero fill shows.  Accumulating into a buffer prefilled with a sentinel
   leaves the sentinel in the padding exactly;
4. the padded call and the unpadded one (M = NB) on the same input path: images, radii, depth and alpha bit-identical; the
   gradients (active coefficients and every other tensor), the camera gradients and the statistics bit-identical under
   torch.use_deterministic_algorithms(True).  A cell that runs without deterministic mode repeats both calls under it for this
   comparison: without it, float atomics move the needles' rotation gradients by more than 2e-5 of scale (test_parity_gpu's
   padded-test bound) from one run to the next, padded or not.

Input path: "staged" allows bulk-TMA staging of the per-Gaussian kernels' inputs, "thread" sets dgr_set_tuning bits 24 / 25
(test_kernel_coverage_gpu.PER_THREAD); each cell asserts from the profiler's kernel names which path its kernels took.

| cell                     | entry point                                   | (deg, M) | path   | options                         |
|--------------------------|-----------------------------------------------|----------|--------|---------------------------------|
| plain_d0m4_staged        | GaussianRasterizer                            | (0, 4)   | staged | camera                          |
| plain_d1m5_thread        | GaussianRasterizer                            | (1, 5)   | thread | camera, AA                      |
| plain_d2m16_staged       | GaussianRasterizer                            | (2, 16)  | staged | camera, AA, det, contributions  |
| plain_d0m16_thread       | GaussianRasterizer                            | (0, 16)  | thread | camera, det                     |
| fused_d1m16_staged       | FusedGaussianRasterizer + DensifyStats        | (1, 16)  | staged | camera, absgrad                 |
| fused_d0m16_thread       | FusedGaussianRasterizer + DensifyStats        | (0, 16)  | thread | camera, AA, contributions       |
| fused_d2m11_staged       | FusedGaussianRasterizer + DensifyStats        | (2, 11)  | staged | camera, AA, det, absgrad        |
| fused_d1m9_thread        | FusedGaussianRasterizer + DensifyStats        | (1, 9)   | thread | camera, det, contributions      |
| views_d1m9_staged        | rasterize_views                               | (1, 9)   | staged | camera, contributions           |
| views_d2m11_thread       | rasterize_views                               | (2, 11)  | thread | camera, AA, det                 |
| mixed_d0m4_staged        | rasterize_views_mixed                         | (0, 4)   | staged | camera, AA                      |
| mixed_d1m5_thread        | rasterize_views_mixed                         | (1, 5)   | thread | camera, det, contributions      |
| views_raw_d2m16_staged   | rasterize_views_raw                           | (2, 16)  | staged | camera, det                     |
| views_raw_d0m16_thread   | rasterize_views_raw                           | (0, 16)  | thread | camera, AA, contributions       |
| mixed_raw_d1m16_staged   | rasterize_views_mixed_raw, stats_views        | (1, 16)  | staged | camera, AA, det, absgrad        |
| mixed_raw_d2m11_thread   | rasterize_views_mixed_raw, stats_views        | (2, 11)  | thread | camera, absgrad, contributions  |
| sharded_d1m5_staged      | ViewShardedRasterizer.render_views, 2 views   | (1, 5)   | staged | accumulate                      |
| sharded_d2m16_thread     | ViewShardedRasterizer.render_views, 2 views   | (2, 16)  | thread | accumulate, AA, det             |
| fallback_d1m16           | GaussianRasterizer, 208 x 208 tiles           | (1, 16)  | staged allowed; the forward falls back to per-thread loads by itself | det, float64 rule only |

The batched cells back-propagate one view at a time (as test_kernel_coverage_gpu does), so each view's gradients meet the oracle
of that view.  The sharded cells judge their images by rule 1 and their summed gradients by rules 3 and 4.  test_stage1_* runs the
stage-1 loop with sh_degree 3 storage at active degree 1."""
import types

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import helpers as h
import kernel_names as KN
import test_kernel_coverage_gpu as KC
import trained_scenes as TS
from test_sh_padding_cpu import pad_raw, pad_shs
from dreamgaussian_b200 import rasterizer as R
from dreamgaussian_b200 import stage1
from dreamgaussian_b200.fused import DensifyStats, FusedGaussianRasterizer, rasterize_views_mixed_raw, rasterize_views_raw
from dreamgaussian_b200.multiview import ViewShardedRasterizer

pytestmark = pytest.mark.gpu
DEV = "cuda"
W, H = KC.W, KC.H
P_SINGLE, P_VIEWS = KC.P_SINGLE, KC.P_VIEWS
SENTINEL = 1234.5
RAW_APIS = ("fused", "views_raw", "mixed_raw")
STAT_KEYS = ("xyz_gradient_accum", "denom", "max_radii2D", "xyz_gradient_accum_abs")


# ---- inputs ---------------------------------------------------------------------------------------------------------------------
def _inputs(api, deg, M):
    """(unpadded, padded) inputs of a cell: test_kernel_coverage_gpu's scenes (same seeds), activated or raw."""
    if api in ("plain", "fused"):
        i = KC._scene(P_SINGLE, deg, (21 if api == "fused" else 11) + deg)
    else:
        i = KC._scene(P_VIEWS, deg, 41 + deg)
    if api in RAW_APIS:
        raw = TS.raw_of(i, seed=deg)
        return raw, pad_raw(raw, M)
    i = {k: i[k] for k in KC.ACT}
    return i, dict(i, shs=pad_shs(i["shs"], M))


def _views(api, deg):
    if api in ("plain", "fused"):
        return [KC._settings(W, H, deg)]
    sizes = KC.MIXED_SIZES if api.startswith("mixed") else [(W, H)] * (2 if api == "sharded" else 3)
    return [KC._settings(w, hh, deg, v) for v, (w, hh) in enumerate(sizes)]


def _dirty(P, M):
    """Leave NaN-filled blocks of the gradient rows' sizes in the caching allocator, so that torch::empty gradient outputs of the next
    call start as NaN rather than as whatever an earlier call left (often zeros)."""
    blocks = [torch.full((n,), float("nan"), device=DEV) for n in (P * M * 3, P * max(M - 1, 1) * 3) for _ in range(8)]
    del blocks


def _kernels(prof):
    return {n for n in (KN.normalize(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
            if KN.is_library_kernel(n)}


def _staged_flags(names):
    """{kernel family: set of STAGE template arguments seen} of the per-Gaussian forward / backward kernels that have a staged variant."""
    out = {}
    for n in names:
        fam = n.split("<")[0]
        if fam in ("dgr::preprocess_fwd_kernel", "dgr::preprocess_fwd_aa_kernel", "dgr::preprocess_bwd_kernel", "dgr::preprocess_bwd_aa_kernel",
                   "dgr::preprocess_views_fwd_kernel", "dgr::preprocess_views_fwd_aa_kernel"):
            out.setdefault(fam.replace("_aa", "").replace("views_", ""), set()).add(n.rstrip(">").split(",")[-1])
    return out


def _run(word, det, P, M, fn):
    """fn() under tuning `word` and deterministic mode `det`, with dirtied gradient memory; returns (result, launched kernel names)."""
    with KC._Det(det):
        torch.cuda.synchronize()
        _dirty(P, M)
        with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
            out = h.run_tuned(word, fn)
            torch.cuda.synchronize()
    return out, _kernels(prof)


# ---- one render call and its backward -------------------------------------------------------------------------------------------
def _render(spec, inputs, settings, grads, v):
    """The cell's entry point on `inputs`, loss of view v only; numpy results of that view."""
    api, aa, V = spec["api"], spec["aa"], len(settings)
    raw = api in RAW_APIS
    keys = h.RAW_KEYS if raw else KC.ACT
    P = len(inputs[keys[0]])
    rss, cams = zip(*(KC._rs(s, cam_grad=True) for s in settings))
    tin = {k: KC._t(inputs[k]).requires_grad_(True) for k in keys}
    cs = R.ContributionStats(P, DEV) if spec["contrib"] else None
    st = DensifyStats(P, DEV, absgrad=spec["absgrad"]) if api in ("fused", "mixed_raw") else None
    m2d = torch.zeros((P, 3) if V == 1 else (V, P, 3), device=DEV, requires_grad=True)
    if api == "plain":
        out = [[x] for x in R.GaussianRasterizer(rss[0], antialiasing=aa, contributions=cs)(means2D=m2d, **tin)]
    elif api == "fused":
        out = [[x] for x in FusedGaussianRasterizer(rss[0], aa, cs)(tin["xyz"], tin["features_dc"], tin["features_rest"], tin["opacity"],
                                                                     tin["scaling"], tin["rotation"], means2D=m2d, stats=st)]
    elif api in ("views", "mixed"):
        out = (R.rasterize_views if api == "views" else R.rasterize_views_mixed)(
            list(rss), tin["means3D"], m2d, tin["opacities"], tin["shs"], tin["scales"], tin["rotations"], antialiasing=aa, contributions=cs)
    else:
        args = (list(rss), tin["xyz"], m2d, tin["features_dc"], tin["features_rest"], tin["opacity"], tin["scaling"], tin["rotation"])
        if api == "views_raw":
            out = rasterize_views_raw(*args, antialiasing=aa, contributions=cs)
        else:
            out = rasterize_views_mixed_raw(*args, stats=st, stats_views=(v,), antialiasing=aa, contributions=cs)
    color, radii, depth, alpha = out
    KC._linear_loss(grads[v])(color[v], depth[v], alpha[v]).backward()
    res = dict(color=KC._np(color[v]), depth=KC._np(depth[v]), alpha=KC._np(alpha[v]), radii=radii[v].cpu().numpy(),
               grads=dict({k: KC._np(x.grad) if x.grad is not None else np.zeros(x.shape, np.float32) for k, x in tin.items()},
                          means2D=KC._np(m2d.grad if V == 1 else m2d.grad[v])),
               cam=[KC._np(c.grad) for c in cams[v]],
               stats={k: KC._np(getattr(st, k)) for k in STAT_KEYS if st is not None and getattr(st, k) is not None})
    if cs is not None:
        res["wsum"], res["wmax"] = KC._np(cs.weight_sum), KC._np(cs.weight_max)
        res["alpha_sum"] = sum(float(KC._np(alpha[u]).astype(np.float64).sum()) for u in range(V))
    return res


# ---- the rules --------------------------------------------------------------------------------------------------------------------
def _close(cid, what, got, want):
    """Rule 4 on a gradient-like quantity of two deterministic runs: bit-identical."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (cid, what, got.shape, want.shape)
    assert np.array_equal(got, want), (cid, what, "not bit-identical", float(np.abs(got.astype(np.float64) - want).max()) if got.size else 0.0)


def _active(k, a, NB):
    """The active coefficients of a padded gradient tensor."""
    if k == "shs":
        return a[:, :NB]
    if k == "features_rest":
        return a[:, :NB - 1]
    return a


def _padding(k, a, NB):
    return a[:, NB:] if k == "shs" else a[:, NB - 1:] if k == "features_rest" else None


def _same_result(cid, pad, ref, NB, det):
    """Rules 3 and 4: the padded result `pad` against the unpadded `ref` of the same input path (gradients and statistics only when
    both ran under deterministic mode)."""
    for k in ("color", "depth", "alpha", "radii"):
        assert np.array_equal(pad[k], ref[k]), (cid, k, "padded and unpadded renders differ")
    for k, g in ref["grads"].items():
        tail = _padding(k, pad["grads"][k], NB)
        if tail is not None:
            assert tail.size and not tail.any(), (cid, k, "padding gradient not zero", int(np.count_nonzero(tail)))
        if det:
            _close(cid, k, _active(k, pad["grads"][k], NB), g)
    if not det:
        return
    for n, a, b in zip(("viewmatrix", "projmatrix", "campos"), pad["cam"], ref["cam"]):
        _close(cid, "camera " + n, a, b)
    for k, b in ref["stats"].items():
        _close(cid, k, pad["stats"][k], b)
    for k in ("wsum", "wmax"):
        if k in ref:
            _close(cid, k, pad[k], ref[k])


def _assert_path(cid, names, staged):
    flags = _staged_flags(names)
    assert flags, (cid, "no per-Gaussian kernel with a staged variant launched", sorted(names))
    want = {"1"} if staged else {"0"}
    for fam, seen in flags.items():
        assert seen == want, (cid, fam, seen, "staged" if staged else "per-thread")


# ---- the cells ------------------------------------------------------------------------------------------------------------------
CELLS = {}


def _cell(cid, **spec):
    CELLS[cid] = dict(dict(aa=False, det=False, absgrad=False, contrib=False), **spec)


_cell("plain_d0m4_staged", api="plain", deg=0, M=4, thread=False)
_cell("plain_d1m5_thread", api="plain", deg=1, M=5, thread=True, aa=True)
_cell("plain_d2m16_staged", api="plain", deg=2, M=16, thread=False, aa=True, det=True, contrib=True)
_cell("plain_d0m16_thread", api="plain", deg=0, M=16, thread=True, det=True)
_cell("fused_d1m16_staged", api="fused", deg=1, M=16, thread=False, absgrad=True)
_cell("fused_d0m16_thread", api="fused", deg=0, M=16, thread=True, aa=True, contrib=True)
_cell("fused_d2m11_staged", api="fused", deg=2, M=11, thread=False, aa=True, det=True, absgrad=True)
_cell("fused_d1m9_thread", api="fused", deg=1, M=9, thread=True, det=True, contrib=True)
_cell("views_d1m9_staged", api="views", deg=1, M=9, thread=False, contrib=True)
_cell("views_d2m11_thread", api="views", deg=2, M=11, thread=True, aa=True, det=True)
_cell("mixed_d0m4_staged", api="mixed", deg=0, M=4, thread=False, aa=True)
_cell("mixed_d1m5_thread", api="mixed", deg=1, M=5, thread=True, det=True, contrib=True)
_cell("views_raw_d2m16_staged", api="views_raw", deg=2, M=16, thread=False, det=True)
_cell("views_raw_d0m16_thread", api="views_raw", deg=0, M=16, thread=True, aa=True, contrib=True)
_cell("mixed_raw_d1m16_staged", api="mixed_raw", deg=1, M=16, thread=False, aa=True, det=True, absgrad=True)
_cell("mixed_raw_d2m11_thread", api="mixed_raw", deg=2, M=11, thread=True, absgrad=True, contrib=True)


@pytest.mark.parametrize("cid", list(CELLS))
def test_padded_cell(cid):
    spec = CELLS[cid]
    api, deg, M, aa, det = spec["api"], spec["deg"], spec["M"], spec["aa"], spec["det"]
    NB = (deg + 1) ** 2
    raw = api in RAW_APIS
    small, padded = _inputs(api, deg, M)
    settings = _views(api, deg)
    V = len(settings)
    sizes = [(s["image_width"], s["image_height"]) for s in settings]
    grads = [h.upstream_grads(hh, w, seed=50 + v) for v, (w, hh) in enumerate(sizes)]
    word = (1, 1, 1 | (KC.PER_THREAD if spec["thread"] else 0))
    P = len(small["xyz" if raw else "means3D"])
    pads = []
    for v in range(V):
        pad, names = _run(word, det, P, M, lambda: _render(spec, padded, settings, grads, v))
        ref, ref_names = _run(word, det, P, NB, lambda: _render(spec, small, settings, grads, v))
        _assert_path(cid, names, not spec["thread"])
        _assert_path(cid, ref_names, not spec["thread"])
        _same_result("%s v%d" % (cid, v), pad, ref, NB, det)
        if not det:          # rule 4's gradients: the same two calls under deterministic mode
            pad_d, _ = _run(word, True, P, M, lambda: _render(spec, padded, settings, grads, v))
            ref_d, _ = _run(word, True, P, NB, lambda: _render(spec, small, settings, grads, v))
            _same_result("%s v%d det" % (cid, v), pad_d, ref_d, NB, True)
        pads.append(pad)
    # rules 1 and 2 on the padded inputs, view by view
    for v, s in enumerate(settings):
        name, key = "%s v%d" % (cid, v), ("shpad", cid, v)
        ambig = h.MAX_AMBIG_FRAC if V == 1 else KC._AMBIG.get((deg, v), 0.06)
        KC._judge_images(name, s, KC._image_refs(key, s, padded, grads[v], aa, raw), pads[v], raw, max_ambig_frac=ambig)
        act = KC._activated(padded) if raw else {k: np.asarray(x, np.float64) for k, x in padded.items()}
        cam = [types.SimpleNamespace(grad=torch.tensor(c)) for c in pads[v]["cam"]]
        KC._check_camera(name, key, s, act, grads[v], aa, cam)
        if spec["absgrad"]:
            KC._check_abs(name, key, s, KC._activated(padded, s, aa), grads[v], pads[v]["stats"]["xyz_gradient_accum_abs"])
    if spec["contrib"]:
        act = (lambda s: KC._activated(padded, s, aa)) if raw else (lambda s: KC._eff(padded, s, aa))
        KC._check_contrib(cid, [(("shpad", cid, v), s, act(s), grads[v]) for v, s in enumerate(settings)],
                          pads[0]["wsum"], pads[0]["wmax"], pads[0]["alpha_sum"])


# ---- ViewShardedRasterizer: two views accumulated into one flat buffer ---------------------------------------------------------
def _sharded(inputs, M, settings, grads, aa):
    P = len(inputs["means3D"])
    vs = ViewShardedRasterizer(P, M, DEV)
    params = {k: KC._t(inputs[k]) for k in KC.ACT}
    up = [tuple(KC._t(x) for x in g) for g in grads]
    rss = [KC._rs(s)[0] for s in settings]
    vs.grads.flat.fill_(SENTINEL)                   # the first view overwrites, the second adds
    images = vs.render_views(params, rss, up, keep_images=True, antialiasing=aa)
    torch.cuda.synchronize()
    g = vs.grads.views
    out = dict(images=[dict(color=KC._np(c), radii=r.cpu().numpy(), depth=KC._np(d), alpha=KC._np(a)) for c, r, d, a in images],
               grads={k: KC._np(g[k]) for k in ("means3D", "means2D", "shs", "opacities", "scales", "rotations")})
    # one more view ADDED to a buffer prefilled with the sentinel (accumulate=True from the first call on)
    vs.grads.flat.fill_(SENTINEL)
    _, _, _, _, state = R.forward_impl(rss[1], params["means3D"], params["shs"], None, params["opacities"], params["scales"],
                                       params["rotations"], None, antialiasing=aa)
    R.backward_impl(state, up[1][0], up[1][1], up[1][2], g["means3D"], g["means2D"], g["shs"], None, g["opacities"], g["scales"],
                    g["rotations"], None, accumulate=True)
    torch.cuda.synchronize()
    out["acc"] = {k: KC._np(g[k]) for k in out["grads"]}
    return out


@pytest.mark.parametrize("deg,M,thread,aa,det", [(1, 5, False, False, False), (2, 16, True, True, True)])
def test_padded_sharded_accumulation(deg, M, thread, aa, det):
    """Rules 1 (images) and 3 on a run in the cell's mode; rule 4 on the summed gradients under deterministic mode."""
    cid = "sharded_d%dm%d_%s" % (deg, M, "thread" if thread else "staged")
    NB = (deg + 1) ** 2
    small, padded = _inputs("sharded", deg, M)
    settings = _views("sharded", deg)
    grads = [h.upstream_grads(H, W, seed=50 + v) for v in range(len(settings))]
    word = (1, 1, 1 | (KC.PER_THREAD if thread else 0))
    runs = {}
    for mode in sorted({det, True}):
        pad, names = _run(word, mode, P_VIEWS, M, lambda: _sharded(padded, M, settings, grads, aa))
        ref, ref_names = _run(word, mode, P_VIEWS, NB, lambda: _sharded(small, NB, settings, grads, aa))
        _assert_path(cid, names, not thread)
        _assert_path(cid, ref_names, not thread)
        runs[mode] = pad, ref
    pad, ref = runs[True]
    for v, (a, b) in enumerate(zip(pad["images"], ref["images"])):
        for k in a:
            assert np.array_equal(a[k], b[k]), (cid, v, k)
    for part in ("grads", "acc"):
        for k, b in ref[part].items():
            a = pad[part][k]
            _close("%s %s" % (cid, part), k, a[:, :NB] if k == "shs" else a, b)
    pad = runs[det][0]
    for part in ("grads", "acc"):
        for k, a in pad[part].items():
            assert np.isfinite(a).all(), (cid, part, k)
        tail = pad[part]["shs"][:, NB:]
        if part == "grads":
            assert not tail.any(), (cid, "padding gradient not zero after write + accumulate")
        else:
            assert (tail == np.float32(SENTINEL)).all(), (cid, "accumulating changed the padding")
    for v, s in enumerate(settings):
        cu = dict(pad["images"][v], grads={})
        KC._judge_images("%s v%d" % (cid, v), s, KC._image_refs(("shpad", cid, v), s, padded, grads[v], aa, False), cu, False,
                         max_ambig_frac=KC._AMBIG.get((deg, v), 0.06))


# ---- the per-Gaussian forward falls back to per-thread loads on its own --------------------------------------------------------
def test_padded_rows_push_a_large_frame_to_per_thread_loads():
    """The staged forward needs the tile histogram plus 8 warps x 32 x (44 + 12 M) bytes of shared memory (dgr_api.cu pre_fwd_smem).
    At 208 x 208 tiles M = 4 fits in 227 KB and M = 16 does not: the padded call must take the per-thread forward (its backward
    stays staged), agree bit for bit with the unpadded call forced onto the same path, and pass the float64 oracle."""
    deg, M, NB, side = 1, 16, 4, 208 * 16
    s, i = TS.compact_mix(P_SINGLE, seed=71, W=side, H=side, deg=deg)
    small = {k: i[k] for k in KC.ACT}
    padded = dict(small, shs=pad_shs(small["shs"], M))
    g = h.upstream_grads(side, side, seed=72)
    spec = dict(api="plain", aa=False, absgrad=False, contrib=False)
    pad, names = _run(h.DEFAULT_TUNING, True, P_SINGLE, M, lambda: _render(spec, padded, [s], [g], 0))
    assert _staged_flags(names) == {"dgr::preprocess_fwd_kernel": {"0"}, "dgr::preprocess_bwd_kernel": {"1"}}, sorted(names)
    _, names4 = _run(h.DEFAULT_TUNING, True, P_SINGLE, NB, lambda: _render(spec, small, [s], [g], 0))
    assert _staged_flags(names4)["dgr::preprocess_fwd_kernel"] == {"1"}, sorted(names4)
    ref, names_ref = _run((1, 1, 1 | (1 << 24)), True, P_SINGLE, NB, lambda: _render(spec, small, [s], [g], 0))
    assert _staged_flags(names_ref) == _staged_flags(names), sorted(names_ref)
    _same_result("fallback_d1m16", pad, ref, NB, True)
    # the float64 rule (as the raw-parameter cells): on this frame the float32 rule's 99.9th percentile of dL/dscales is 6.9e-5
    # against its 3e-5, for the unpadded call too (the two are bit-identical above), so it says nothing about the padding
    ok, rep = h.compare(pad, h.run_oracle(s, padded, g))
    h.report("fallback_d1m16", vs_f64=rep)
    assert ok, rep


# ---- stage 1 with sh_degree 3 storage at active degree 1 ------------------------------------------------------------------------
def test_stage1_at_a_lowered_active_degree_tracks_the_reference_formulation():
    """Stage1Trainer at sh_degree=3 rendered at active_sh_degree 1: f_rest holds 15 columns of which 3 are read.  The padding columns
    hold +-10 and must get exactly zero gradient at every step; the fused path tracks fused=False by the bounds of
    test_stage1_gpu.test_stage1_loop_fused_tracks_the_reference_formulation_and_densifies, then densifies with finite losses."""
    cfg = stage1.Stage1Config(iters=40, num_pts=1500, ref_size=96, density_start_iter=6, densification_interval=6, seed=2, sh_degree=3)
    trainers = [stage1.Stage1Trainer(cfg, fused=True), stage1.Stage1Trainer(cfg, fused=False)]
    checked = []
    for t in trainers:
        g = t.gaussians
        g.active_sh_degree = 1
        t.fixed_cam = t.fixed_cam._replace(sh_degree=1)
        gen = torch.Generator(device=DEV).manual_seed(5)
        with torch.no_grad():
            g.p["f_rest"][:, 3:] = (torch.rand(g.p["f_rest"][:, 3:].shape, generator=gen, device=DEV) * 2 - 1) * 10.0

        def step(g=g, inner=g.optimizer_step):
            gr = g.p["f_rest"].grad
            assert gr is not None and gr.shape[1] == 15
            assert torch.isfinite(gr).all() and not gr[:, 3:].any(), "f_rest padding gradient not zero"
            assert gr[:, :3].abs().max() > 0
            checked.append(1)
            inner()
        g.optimizer_step = step
    a, b = trainers
    la, lb = [], []
    for _ in range(5):
        la.append(float(a.train_step().detach())); lb.append(float(b.train_step().detach()))
    np.testing.assert_allclose(la, lb, rtol=2e-3)
    for k in stage1.GROUPS:
        if k == "rotation":          # isotropic start: see test_stage1_gpu
            continue
        pa, pb = a.gaussians.p[k].detach(), b.gaussians.p[k].detach()
        assert float((pa - pb).abs().max()) <= 5e-3 * max(1.0, float(pb.abs().max())), k
    n0 = a.gaussians.num_points
    losses = a.train(20)
    assert np.isfinite(losses).all() and a.gaussians.num_points != n0
    assert len(checked) == 30
