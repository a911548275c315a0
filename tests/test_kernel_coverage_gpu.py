"""Kernel coverage: every __global__ instantiation of the library is launched by a small named call (a cell) whose outputs are
checked against an oracle, and the suite fails when one is not.

A cell runs under torch.profiler with CUDA activity tracing (process-wide, so kernels launched on autograd's backward thread are
seen too), checks every output with the rules the suite already has, and only then records the normalized names of the kernels it
launched.  tests/kernel_manifest.txt credits each instantiation to the cells that reach it; the last test asserts that the
checked cells reached every kernel the manifest does not excuse, and that each cell still launches what the manifest credits to
it (a dispatch change that routes a cell elsewhere fails here).

Rules (reused, not restated): images, radii and gradients by helpers.both_oracles / compare (raw-parameter cells: run_oracle_raw
and helpers.compare; anti-aliased cells: tests/aa_oracle.py), camera gradients by test_camera_grads_gpu's
d <= max(1e-3, 3 d32) against the float64 torch oracle, the AbsGS statistic and the contribution statistics by the check_rule of
test_absgrad_gpu / test_contrib_gpu against the C oracle; deterministic cells are also bit-identical across two runs.

The scene puts the kernels on their edges: P not a multiple of 32 (the staged kernels' partial last warp), image sides that are
not multiples of 16, Gaussians behind the near plane and outside the frustum (radius 0), saturated opacities, needles and clamped
colours (tests/trained_scenes.py).  Its needles have axis ratios 10-30 in random 3-D orientations, the needle regime
test_trained_regimes_gpu.py judges by the same rules (at higher ratios and for screen-space needles float32 cancellation in the
conic moves a few scale / rotation gradients past them in any float32 evaluation, the float32 oracle's included)."""
import itertools
import os

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import aa_oracle
import absgrad_oracle as AO
import camgrad_helpers as C
import contrib_oracle as CO
import helpers as h
import kernel_names as KN
import test_absgrad_gpu as TA
import test_contrib_gpu as TC
import test_variants_gpu as TV
import trained_scenes as TS
from dreamgaussian_b200 import fields, scene, stage1
from dreamgaussian_b200 import rasterizer as R
from dreamgaussian_b200.fused import DensifyStats, FusedGaussianRasterizer, rasterize_views_mixed_raw, rasterize_views_raw
from oracle import c_oracle, fields_oracle, knn_oracle

pytestmark = pytest.mark.gpu
MANIFEST = os.path.join(os.path.dirname(os.path.abspath(__file__)), "kernel_manifest.txt")
DEV = "cuda"

SORTED, BY_ID = TV.SORTED, TV.BY_ID
PER_THREAD = (1 << 24) | (1 << 25)                 # dgr_set_tuning bits 24 / 25: per-Gaussian kernels without bulk-TMA staging
# every render_fwd / render_bwd shape and record staging the tuning word selects (test_variants_gpu.WORDS minus the switches)
SHAPE_WORDS = [w for n, w in TV.WORDS.items() if n.endswith("_sorted") or n.endswith("_byid")]
STAGING = {"S": SORTED, "B": BY_ID}

P_SINGLE, P_VIEWS = 493, 1237                      # 15 and 38 full warps + a partial one; single-view cells stay small for the
W, H = 72, 56                                      # float64 torch oracle of the camera gradients
MIXED_SIZES = [(56, 72), (40, 40), (72, 48)]       # (W, H) per view
VIEW_POSES = [(0.0, 0.0, (1.0, 1.0, 1.0)), (10.0, 25.0, (0.0, 0.0, 0.0)), (-12.0, -30.0, (0.2, 0.5, 0.9))]
ACT = ("means3D", "opacities", "shs", "scales", "rotations")


# ---- scene, inputs, oracles (cached per scene, input form, mode and view) -------------------------------------------------------
_SCENES = {}


def _scene(P, deg, seed):
    """Activated inputs of P Gaussians (float32): trained_scenes.compact_mix in the view of the 72 x 56 camera."""
    key = (P, deg, seed)
    if key not in _SCENES:
        _SCENES[key] = TS.compact_mix(P, seed=seed, W=W, H=H, deg=deg)[1]
    return _SCENES[key]


def _settings(W_, H_, deg, v=0):
    elev, azim, bg = VIEW_POSES[v]
    cam = scene.orbit_camera(elev, azim, 2.0, W_, H_)
    return dict(image_height=H_, image_width=W_, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=np.asarray(bg, np.float32),
                scale_modifier=1.0, viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform, sh_degree=deg,
                campos=cam.camera_center)


def _form(i, form):
    """form: sh | sh_cov | colors | colors_cov (test_camera_grads_gpu._inputs in numpy)."""
    i = dict(i)
    if form.endswith("cov"):
        q = i.pop("rotations").astype(np.float64)
        q = q / np.linalg.norm(q, axis=1, keepdims=True)
        Mx = C.T._quat_to_R(torch.tensor(q)).numpy() * i.pop("scales").astype(np.float64)[:, None, :]
        S = Mx @ Mx.transpose(0, 2, 1)
        i["cov3D_precomp"] = np.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1).astype(np.float32)
    if form.startswith("colors"):
        i.pop("shs")
        i["colors_precomp"] = np.random.default_rng(5).uniform(0.05, 0.95, (len(i["means3D"]), 3)).astype(np.float32)
    return i


def _activated(raw, settings=None, aa=False):
    return TA.activated(raw, settings, aa)


_REFS = {}


def _refs(key, fn):
    if key not in _REFS:
        _REFS[key] = fn()
    return _REFS[key]


def _image_refs(key, s, inputs, g, aa, raw):
    """Oracle images / radii / gradients: both builds of the C oracle (raw: the float64 build through the activations)."""
    if raw:
        return _refs(("img",) + key, lambda: dict(f64=aa_oracle.run_oracle(s, inputs, g, raw=True) if aa else h.run_oracle_raw(s, inputs, g)))
    return _refs(("img",) + key, lambda: aa_oracle.oracles(s, inputs, g) if aa else h.oracles(s, inputs, g))


def _judge_images(name, s, refs, cu, raw, max_ambig_frac=h.MAX_AMBIG_FRAC):
    if raw:
        ok, rep = h.compare(cu, refs["f64"], max_ambig_frac=max_ambig_frac)
        h.report(name, vs_f64=rep)
        assert ok, (name, rep)
    else:
        h.both_oracles(name, s, None, None, refs=refs, cu=cu, max_ambig_frac=max_ambig_frac)


def _c_stats(key, s, act, g, dt):
    """(abs statistic, contribution sum, contribution max, flags) of the C oracle build dt on activated inputs act (o_eff included)."""
    def run():
        r = c_oracle.forward(**s, **act, dtype=dt)
        a, _ = AO.stat(AO.c_terms(r, *g), r.radii, r.H, r.W)
        ws, wm = CO.c_stats(r)
        _, flags, _ = r.flags()
        r.close()
        return a, ws, wm, flags
    return _refs(("stats", np.dtype(dt).name) + key, run)


def _eff(act, s, aa):
    """Activated inputs with the anti-aliased mode's o_eff (what the C oracle renders in that mode)."""
    act = {k: np.asarray(v, np.float64) for k, v in act.items()}
    if aa:
        t = {k: torch.tensor(act[k]) for k in ("means3D", "scales", "rotations") if k in act}
        act["opacities"] = act["opacities"] * aa_oracle.comp(s, t["means3D"], t.get("scales"), t.get("rotations"),
                                                             torch.tensor(act["cov3D_precomp"]) if "cov3D_precomp" in act else None
                                                             ).numpy().reshape(-1, 1)
    return act


def _check_contrib(name, views, wsum, wmax, alpha_sum):
    """test_contrib_gpu's rule on statistics accumulated over `views`, a list of (oracle key, settings, activated inputs with o_eff,
    upstream gradients): the sum of the sums, the max of the maxima, the union of the flags."""
    for dt in (np.float32, np.float64):
        ws = wm = flags = None
        for key, s, act, g in views:
            _, a, b, f = _c_stats(key, s, act, g, dt)
            ws = a if ws is None else ws + a
            wm = b if wm is None else np.maximum(wm, b)
            flags = f if flags is None else flags | f
        assert (wm > 0).sum() > 10
        TC.check_rule(wsum, ws, flags, "%s contrib %s sum" % (name, np.dtype(dt).name), f32=dt is np.float32)
        TC.check_rule(wmax, wm, flags, "%s contrib %s max" % (name, np.dtype(dt).name), f32=dt is np.float32)
    rel = abs(float(wsum.astype(np.float64).sum()) - alpha_sum) / alpha_sum
    assert rel <= 1e-5, (name, rel)


def _check_abs(name, key, s, act, g, a_cu):
    # the scene holds needles: like test_absgrad_gpu's needles regime, the statistic is held to the float64 build
    a, _, _, flags = _c_stats(key, s, act, g, np.float64)
    TA.check_rule(a_cu, a, flags, name + " abs float64")


class _Det:
    def __init__(self, on):
        self.on = on

    def __enter__(self):
        self.prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(self.on)

    def __exit__(self, *a):
        torch.use_deterministic_algorithms(self.prev)


def _t(a):
    return torch.tensor(np.asarray(a, np.float32), device=DEV)


def _rs(s, cam_grad=False):
    cam = [_t(s[k]).requires_grad_(cam_grad) for k in ("viewmatrix", "projmatrix", "campos")]
    return R.GaussianRasterizationSettings(
        image_height=s["image_height"], image_width=s["image_width"], tanfovx=s["tanfovx"], tanfovy=s["tanfovy"], bg=_t(s["bg"]),
        scale_modifier=s["scale_modifier"], viewmatrix=cam[0], projmatrix=cam[1], sh_degree=s["sh_degree"], campos=cam[2],
        prefiltered=False, debug=False), cam


def _linear_loss(g):
    def loss(color, depth, alpha):
        c = lambda a: torch.tensor(np.asarray(a, np.float64), dtype=color.dtype, device=color.device)
        return (color * c(g[0])).sum() + (depth * c(g[1])).sum() + (alpha * c(g[2])).sum()
    return loss


def _check_camera(name, key, s, act, g, aa, cam):
    loss = _linear_loss(g)
    g64, g32 = _refs(("cam",) + key, lambda: [[x.numpy() if x is not None else np.zeros(3) for x in
                                                C.oracle_camera_grads(s, act, loss, antialiased=aa, dtype=dt)]
                                               for dt in (torch.float64, torch.float32)])
    for n, c, b, f in zip(("viewmatrix", "projmatrix", "campos"), cam, g64, g32):
        a = c.grad.cpu().numpy().reshape(np.shape(b))
        scale = max(np.abs(b).max(), 1e-12)
        d, d32 = np.abs(a - b).max() / scale, np.abs(f - b).max() / scale
        h.report(name + " camera " + n, camera=dict(d=float(d), d32=float(d32)))
        assert d <= max(1e-3, 3 * d32), (name, n, d, d32)


def _np(x):
    return x.detach().cpu().numpy()


# ---- the cells ------------------------------------------------------------------------------------------------------------------
CELLS = {}


def _cell(cid, fn, **kw):
    assert cid not in CELLS, cid
    CELLS[cid] = lambda: fn(cid, **kw)


# single view, GaussianRasterizer, camera gradients on: 10 input forms x AA x (staged | per-thread where a staged kernel exists)
def single_plain(cid, form, deg, aa, per_thread, word):
    i = _form(_scene(P_SINGLE, deg, 11 + deg), form)
    s = _settings(W, H, deg)
    g = h.upstream_grads(H, W, seed=31)
    key = (form, deg, aa)

    def run():
        rs, cam = _rs(s, cam_grad=True)
        tin = {k: _t(v).requires_grad_(True) for k, v in i.items()}
        m2d = torch.zeros_like(tin["means3D"], requires_grad=True)
        color, radii, depth, alpha = R.GaussianRasterizer(rs, antialiasing=aa)(means2D=m2d, **tin)
        _linear_loss(g)(color, depth, alpha).backward()
        out = dict(color=_np(color), depth=_np(depth), alpha=_np(alpha), radii=radii.cpu().numpy(),
                   grads=dict({k: _np(v.grad) for k, v in tin.items()}, means2D=_np(m2d.grad)))
        return out, cam

    cu, cam = h.run_tuned((word[0], word[1], word[2] | (PER_THREAD if per_thread else 0)), run)
    _judge_images(cid, s, _image_refs(key, s, i, g, aa, False), cu, False)
    _check_camera(cid, key, s, {k: np.asarray(v, np.float64) for k, v in i.items()}, g, aa, cam)


_FORMS = [("sh", d) for d in range(4)] + [("sh_cov", d) for d in range(4)] + [("colors", 0), ("colors_cov", 0)]
_n = 0
for (_f, _d), _aa in itertools.product(_FORMS, (False, True)):
    for _pt in ((False, True) if _f == "sh" else (False,)):
        _cell("plain_%s%d_aa%d_%s" % (_f, _d, _aa, "thread" if _pt else "staged" if _f == "sh" else "thread"), single_plain,
              form=_f, deg=_d, aa=_aa, per_thread=_pt, word=SHAPE_WORDS[_n % len(SHAPE_WORDS)])
        _n += 1


# single view, FusedGaussianRasterizer + DensifyStats on raw parameters, camera gradients on
def single_raw(cid, deg, aa, per_thread, absgrad, det, staging, contrib):
    raw = TS.raw_of(_scene(P_SINGLE, deg, 21 + deg), seed=deg)
    s = _settings(W, H, deg)
    g = h.upstream_grads(H, W, seed=32)
    key = ("raw", deg, aa)
    word = (1, 1, 1 | STAGING[staging] | (PER_THREAD if per_thread else 0))

    def run():
        rs, cam = _rs(s, cam_grad=True)
        tin = {k: _t(raw[k]).requires_grad_(True) for k in h.RAW_KEYS}
        st = DensifyStats(P_SINGLE, DEV, absgrad=absgrad)
        cs = R.ContributionStats(P_SINGLE, DEV) if contrib else None
        m2d = torch.zeros_like(tin["xyz"], requires_grad=True)
        color, radii, depth, alpha = FusedGaussianRasterizer(rs, aa, cs)(tin["xyz"], tin["features_dc"], tin["features_rest"], tin["opacity"],
                                                                         tin["scaling"], tin["rotation"], means2D=m2d, stats=st)
        _linear_loss(g)(color, depth, alpha).backward()
        out = dict(color=_np(color), depth=_np(depth), alpha=_np(alpha), radii=radii.cpu().numpy(),
                   grads=dict({k: _np(v.grad) if v.grad is not None else np.zeros(v.shape, np.float32) for k, v in tin.items()},
                              means2D=_np(m2d.grad)),
                   abs=_np(st.xyz_gradient_accum_abs) if absgrad else None, cam=[_np(c.grad) for c in cam])
        if contrib:
            out["wsum"], out["wmax"] = _np(cs.weight_sum), _np(cs.weight_max)
        return out, cam

    with _Det(det):
        cu, cam = h.run_tuned(word, run)
        if det:
            again, _ = h.run_tuned(word, run)
            for k in cu["grads"]:
                assert np.array_equal(cu["grads"][k], again["grads"][k]), (cid, k)
            assert all(np.array_equal(a, b) for a, b in zip(cu["cam"], again["cam"])), cid
            if absgrad:
                assert np.array_equal(cu["abs"], again["abs"]), cid
    _judge_images(cid, s, _image_refs(key, s, raw, g, aa, True), cu, True)
    act = _activated(raw)
    _check_camera(cid, key, s, act, g, aa, cam)
    if absgrad or contrib:
        eff = _activated(raw, s, aa)
        if absgrad:
            _check_abs(cid, key, s, eff, g, cu["abs"])
        if contrib:
            _check_contrib(cid, [(key, s, eff, g)], cu["wsum"], cu["wmax"], float(cu["alpha"].astype(np.float64).sum()))


# (ABS, deterministic, record staging, contributions) spread so that every render_bwd_{abs,det,det_abs} and render_fwd_contrib
# instantiation is reached
_RAW_MODES = [(1, 0, "S", 0), (1, 0, "B", 0), (0, 1, "S", 0), (0, 1, "B", 0), (1, 1, "S", 0), (1, 1, "B", 0), (0, 0, "S", 1), (0, 0, "B", 1)]
for _n, (_d, _aa, _pt) in enumerate(itertools.product(range(4), (False, True), (False, True))):
    _ab, _det, _stg, _cb = _RAW_MODES[_n % len(_RAW_MODES)]
    _cell("raw_deg%d_aa%d_%s_%s%s%s%s" % (_d, _aa, "thread" if _pt else "staged", "abs_" * _ab, "det_" * _det, "contrib_" * _cb,
                                           "sorted" if _stg == "S" else "byid"),
          single_raw, deg=_d, aa=_aa, per_thread=_pt, absgrad=bool(_ab), det=bool(_det), staging=_stg, contrib=bool(_cb))


# batched: rasterize_views / _raw (same size) and rasterize_views_mixed / _mixed_raw; every view judged against the oracle
def batched(cid, api, deg, aa, per_thread, absgrad, det, staging, contrib):
    raw_api, mixed = api.endswith("raw"), api.startswith("mixed")
    inputs = _scene(P_VIEWS, deg, 41 + deg)
    if raw_api:
        inputs = TS.raw_of(inputs, seed=deg)
    sizes = MIXED_SIZES if mixed else [(W, H)] * 3
    settings = [_settings(w, hh, deg, v) for v, (w, hh) in enumerate(sizes)]
    V = len(settings)
    grads = [h.upstream_grads(hh, w, seed=50 + v) for v, (w, hh) in enumerate(sizes)]
    keys = h.RAW_KEYS if raw_api else ACT
    word = (1, 1, 1 | STAGING[staging] | ((1 << 24) if per_thread else 0))

    def run(v, want_contrib):
        rs = [_rs(s)[0] for s in settings]
        tin = {k: _t(inputs[k]).requires_grad_(True) for k in keys}
        m2d = torch.zeros((V, P_VIEWS, 3), device=DEV, requires_grad=True)
        cs = R.ContributionStats(P_VIEWS, DEV) if want_contrib else None
        st = DensifyStats(P_VIEWS, DEV, absgrad=True) if absgrad else None
        if api == "views":
            out = R.rasterize_views(rs, tin["means3D"], m2d, tin["opacities"], tin["shs"], tin["scales"], tin["rotations"], antialiasing=aa,
                                    contributions=cs)
        elif api == "mixed":
            out = R.rasterize_views_mixed(rs, tin["means3D"], m2d, tin["opacities"], tin["shs"], tin["scales"], tin["rotations"],
                                          antialiasing=aa, contributions=cs)
        else:
            args = (rs, tin["xyz"], m2d, tin["features_dc"], tin["features_rest"], tin["opacity"], tin["scaling"], tin["rotation"])
            if api == "views_raw":
                out = rasterize_views_raw(*args, antialiasing=aa, contributions=cs)
            else:
                out = rasterize_views_mixed_raw(*args, stats=st, stats_views=(v,) if absgrad else (), antialiasing=aa, contributions=cs)
        color, radii, depth, alpha = out
        _linear_loss(grads[v])(color[v], depth[v], alpha[v]).backward()
        res = dict(color=_np(color[v]), depth=_np(depth[v]), alpha=_np(alpha[v]), radii=radii[v].cpu().numpy(),
                   grads=dict({k: _np(x.grad) if x.grad is not None else np.zeros(x.shape, np.float32) for k, x in tin.items()},
                              means2D=_np(m2d.grad[v])),
                   abs=_np(st.xyz_gradient_accum_abs) if absgrad else None)
        if want_contrib:
            res["wsum"], res["wmax"] = _np(cs.weight_sum), _np(cs.weight_max)
            res["alpha_sum"] = sum(float(_np(alpha[u]).astype(np.float64).sum()) for u in range(V))
        return res

    with _Det(det):
        cus = [h.run_tuned(word, lambda: run(v, contrib and v == 0)) for v in range(V)]
        if det:
            again = h.run_tuned(word, lambda: run(0, False))
            for k in cus[0]["grads"]:
                assert np.array_equal(cus[0]["grads"][k], again["grads"][k]), (cid, k)
            if absgrad:
                assert np.array_equal(cus[0]["abs"], again["abs"]), cid
    sk = "mixed" if mixed else "same"
    for v in range(V):
        key = ("views", sk, raw_api, deg, aa, v)
        _judge_images("%s v%d" % (cid, v), settings[v], _image_refs(key, settings[v], inputs, grads[v], aa, raw_api), cus[v], raw_api,
                      max_ambig_frac=_AMBIG.get((deg, v), 0.06))
        if absgrad:
            _check_abs("%s v%d" % (cid, v), key, settings[v], _activated(inputs, settings[v], aa), grads[v], cus[v]["abs"])
    if contrib:
        act = (lambda s: _activated(inputs, s, aa)) if raw_api else (lambda s: _eff({k: inputs[k] for k in ACT}, s, aa))
        _check_contrib(cid, [(("views", sk, raw_api, deg, aa, v), s, act(s), grads[v]) for v, s in enumerate(settings)],
                       cus[0]["wsum"], cus[0]["wmax"], cus[0]["alpha_sum"])


# Flagged-pixel fraction allowed per view, the convention of test_views_gpu.py (0.06) except where measured otherwise: in the
# degree-2 scene the second view sees near-plane Gaussians of the first from close by, and the float64 oracle flags 7.4-10.0% of
# its pixels (same-size / mixed) as decisions a float32 implementation may take either way.
_AMBIG = {(2, 1): 0.12}

# (deterministic, record staging, contributions) for the plain and same-size calls; (ABS, deterministic, staging, contributions)
# for the mixed raw call, the only batched call that takes the absolute-gradient statistic
_VIEW_MODES = [(0, 0, "S", 0), (0, 1, "B", 0), (0, 0, "B", 1), (0, 1, "S", 1), (0, 0, "B", 0), (0, 1, "S", 0)]
_MIXED_RAW_MODES = [(1, 0, "S", 0), (1, 0, "B", 1), (1, 1, "S", 0), (1, 1, "B", 0)]
_counts = {}
for _d, _raw, _aa, _pt in itertools.product(range(4), (False, True), (False, True), (False, True)):
    _api = ("mixed" if (_d + _pt) % 2 else "views") + ("_raw" if _raw else "")
    _modes = _MIXED_RAW_MODES if _api == "mixed_raw" else _VIEW_MODES
    _j = _counts.get(_modes is _MIXED_RAW_MODES, 0)
    _counts[_modes is _MIXED_RAW_MODES] = _j + 1
    _ab, _det, _stg, _cb = _modes[_j % len(_modes)]
    _cell("%s_deg%d_aa%d_%s_%s%s%s%s" % (_api, _d, _aa, "thread" if _pt else "staged", "abs_" * _ab, "det_" * _det, "contrib_" * _cb,
                                          "sorted" if _stg == "S" else "byid"),
          batched, api=_api, deg=_d, aa=_aa, per_thread=_pt, absgrad=bool(_ab), det=bool(_det), staging=_stg, contrib=bool(_cb))


def big_tiles(cid):
    """More than 4096 instances per tile: the big-tile sorter (test_variants_gpu.CASES["big_tiles"])."""
    s, i = h.make_case(**TV.CASES["big_tiles"])
    g = h.upstream_grads(s["image_height"], s["image_width"])
    h.both_oracles(cid, s, i, g, refs=_refs(("big",), lambda: h.oracles(s, i, g)), cu=h.run_tuned(h.DEFAULT_TUNING, lambda: h.run_cuda(s, i, g)))


_cell("big_tiles", big_tiles)


def debug_geom(cid):
    """dgr_debug_geom's read-back of a forward's records against the C oracle's per-Gaussian state (state()), on the Gaussians
    both render (radius > 0) and the oracle does not flag.  Mean, depth, conic and colour by test_camera_grads_gpu's rule
    d <= max(1e-3, 3 d32) per quantity (d, d32: the largest deviation of CUDA / of the float32 build from the float64 build, over
    the quantity's largest value).  The opacity-aware pixel AABB: it holds every pixel where the float64 alpha reaches 1/255
    inside the oracle's tile rect and the image, and lies inside the kernel's padded extent (x 1.0005 + 0.02 px) of the float64
    one, 1e-3 px allowed for float32 rounding.  The tile count: the tiles of that AABB, exactly."""
    import ctypes
    from dreamgaussian_b200 import _lib
    i = _scene(P_SINGLE, 1, 61)
    s = _settings(W, H, 1)
    P = P_SINGLE

    def run():
        rs, _ = _rs(s)
        tin = {k: _t(v) for k, v in i.items()}
        _, radii, _, _, state = R.forward_impl(rs, tin["means3D"], tin["shs"], None, tin["opacities"], tin["scales"], tin["rotations"], None)
        out = dict(mean=torch.empty((P, 2), device=DEV), depth=torch.empty((P,), device=DEV), conic=torch.empty((P, 3), device=DEV),
                   rgb=torch.empty((P, 3), device=DEV), aabb=torch.empty((P, 4), dtype=torch.int32, device=DEV),
                   tiles=torch.empty((P,), dtype=torch.int32, device=DEV))
        p = lambda t: ctypes.c_void_p(t.data_ptr())
        _lib.check(_lib.load().dgr_debug_geom(P, H, W, p(state.geom), p(out["mean"]), p(out["depth"]), p(out["conic"]), p(out["rgb"]),
                                              p(out["aabb"]), p(out["tiles"]), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
        torch.cuda.synchronize()
        return {k: v.cpu().numpy() for k, v in out.items()}, radii.cpu().numpy()

    cu, radii = h.run_tuned(h.DEFAULT_TUNING, run, fast_host=False)          # the ctypes host layer keeps the geometry buffer
    st = {}
    for dt in (np.float64, np.float32):
        r = c_oracle.forward(**s, **i, dtype=dt)
        st[dt] = r.state()
        if dt is np.float64:
            _, ag, _ = r.flags()
            ref_radii = r.radii.copy()
        r.close()
    assert np.array_equal(radii[(ag & 4) == 0], ref_radii[(ag & 4) == 0]), cid
    m = (radii > 0) & (ag == 0)
    assert m.sum() > P // 4, (cid, int(m.sum()))
    f64, f32 = st[np.float64], st[np.float32]
    for name, c, a, b in (("mean", cu["mean"], np.stack([f64["px"], f64["py"]], 1), np.stack([f32["px"], f32["py"]], 1)),
                          ("depth", cu["depth"], f64["depth"], f32["depth"]), ("conic", cu["conic"], f64["conic"], f32["conic"]),
                          ("rgb", cu["rgb"], f64["rgb"], f32["rgb"])):
        a, b, c = (np.asarray(x, np.float64)[m] for x in (a, b, c))
        scale = max(float(np.abs(a).max()), 1e-12)
        d, d32 = float(np.abs(c - a).max()) / scale, float(np.abs(b - a).max()) / scale
        h.report(cid + " " + name, geom=dict(d=d, d32=d32))
        assert d <= max(1e-3, 3 * d32), (cid, name, d, d32)
    A, B, Cc = (f64["conic"][:, k].astype(np.float64) for k in range(3))
    inv = 1.0 / (A * Cc - B * B)
    o = i["opacities"][:, 0].astype(np.float64)
    tau = 2.0 * np.log(np.maximum(255.0 * o, 1.0))
    rect = f64["rect"]
    for g in np.nonzero(m)[0]:
        bx0, by0, bx1, by1 = (int(v) for v in cu["aabb"][g])
        empty = bx0 > bx1 or by0 > by1
        ntiles = 0 if empty else ((bx1 >> 4) - (bx0 >> 4) + 1) * ((by1 >> 4) - (by0 >> 4) + 1)
        assert int(cu["tiles"][g]) == ntiles, (cid, g, int(cu["tiles"][g]), ntiles)
        axes = []
        for lo, hi, mu, var, r0, r1, side in ((bx0, bx1, f64["px"][g], Cc[g] * inv[g], rect[g, 0], rect[g, 2], W),
                                              (by0, by1, f64["py"][g], A[g] * inv[g], rect[g, 1], rect[g, 3], H)):
            e = np.sqrt(tau[g] * var)
            axes.append((lo, hi, max(r0 * 16, int(np.ceil(mu - e))), min(min(r1 * 16, side) - 1, int(np.floor(mu + e))),
                         max(r0 * 16, int(np.ceil(mu - e * 1.0005 - 0.02 - 1e-3))),
                         min(min(r1 * 16, side) - 1, int(np.floor(mu + e * 1.0005 + 0.02 + 1e-3)))))
        if tau[g] > 0 and all(lo_in <= hi_in for _, _, lo_in, hi_in, _, _ in axes):
            assert not empty and all(lo <= lo_in and hi >= hi_in for lo, hi, lo_in, hi_in, _, _ in axes), (cid, g, axes)
        if not empty:
            assert all(lo >= lo_out and hi <= hi_out for lo, hi, _, _, lo_out, hi_out in axes), (cid, g, axes)


_cell("debug_geom", debug_geom)


# ---- rows next to the rasterizer ------------------------------------------------------------------------------------------------
FIELD_ATOL = 5e-5          # tests/test_fields_gpu.py


def fields_eval(cid, res, nb):
    raw = scene.to_raw_parameters(scene.make_cloud(3001, 0, seed=res + nb))
    args = [raw["xyz"], raw["opacity"], raw["scaling"], raw["rotation"]]
    want, wc, ws = fields_oracle.extract_fields(*args, res, nb, 1.5)
    occ, center, sc = fields.extract_fields(*[torch.tensor(a, device=DEV) for a in args], resolution=res, num_blocks=nb, relax_ratio=1.5)
    occ = occ.cpu().numpy()
    assert np.abs(occ - want).max() <= FIELD_ATOL * max(1.0, float(want.max())), cid
    assert np.array_equal(center.cpu().numpy(), wc) and float(sc) == np.float32(ws), cid


# voxels per block (res / nb)^3 = 8, 512, 1000, 1728, 4096 -> fields_eval_kernel<1, 2, 4, 8, 16>
for _res, _nb in ((32, 16), (64, 8), (80, 8), (96, 8), (64, 4)):
    _cell("fields_%d_%d" % (_res, _nb), fields_eval, res=_res, nb=_nb)


def knn(cid):
    from simple_knn._C import distCUDA2
    rng = np.random.default_rng(3)
    p = np.ascontiguousarray((rng.normal(size=(5003, 3)) * 0.3).astype(np.float32))
    got = distCUDA2(torch.tensor(p, device=DEV)).cpu().numpy()
    np.testing.assert_allclose(got, knn_oracle.dist2_f64(p), rtol=1e-6, atol=1e-30)       # tests/test_knn_gpu.py


_cell("knn", knn)


def adam(cid):
    """stage1's fused multi-tensor Adam against torch.optim.Adam (tests/test_stage1_gpu.py)."""
    rng = np.random.default_rng(3)
    shapes = dict(xyz=(1237, 3), f_dc=(1237, 1, 3), f_rest=(1237, 15, 3), opacity=(1237, 1), scaling=(1237, 3), rotation=(1237, 4))
    init = {k: rng.normal(0, 1, s).astype(np.float32) for k, s in shapes.items()}
    m = stage1.GaussianModelB200(3)
    m._set({k: torch.tensor(v, device=DEV) for k, v in init.items()})
    m.training_setup()
    assert m.fused_adam
    ref = {k: torch.nn.Parameter(torch.tensor(v)) for k, v in init.items()}
    opt = torch.optim.Adam([{"params": [ref[k]], "lr": m.lr[k]} for k in stage1.GROUPS], lr=0.0, eps=1e-15)
    for it in range(1, 4):
        opt.param_groups[0]["lr"] = m.update_learning_rate(it)
        for k in stage1.GROUPS:
            gr = (rng.normal(0, 1, shapes[k]) * 10.0 ** rng.integers(-5, 2)).astype(np.float32)
            m.p[k].grad = torch.tensor(gr, device=DEV)
            ref[k].grad = torch.tensor(gr)
        m.optimizer_step()
        opt.step()
    for k in stage1.GROUPS:
        want = ref[k].detach().numpy()
        np.testing.assert_allclose(m.p[k].detach().cpu().numpy(), want, rtol=5e-6, atol=1e-7 * np.abs(want).max(), err_msg=k)


_cell("adam", adam)


def densify(cid, absgrad):
    """The compaction kernels against the tensor-indexing path (tests/test_stage1_gpu.py), with and without AbsGS's split rule."""
    P, deg = 1237, 1
    rng = np.random.default_rng(P + absgrad)
    M = (deg + 1) ** 2
    init = dict(xyz=rng.normal(0, 0.3, (P, 3)), f_dc=rng.normal(0, 1, (P, 1, 3)), f_rest=rng.normal(0, 0.1, (P, M - 1, 3)),
                opacity=rng.normal(-1.0, 2.5, (P, 1)), scaling=rng.normal(-3.4, 0.6, (P, 3)), rotation=rng.normal(0, 1, (P, 4)))
    models = []
    for fused in (True, False):
        m = stage1.GaussianModelB200(deg)
        m.fused_adam, m.fused_densify = True, fused
        m._set({k: torch.tensor(v, dtype=torch.float32, device=DEV) for k, v in init.items()})
        m.training_setup()
        models.append(m)
    for k in stage1.GROUPS:
        m0 = torch.tensor(rng.normal(0, 1, init[k].shape), dtype=torch.float32, device=DEV)
        for m in models:
            m.exp_avg[k], m.exp_avg_sq[k] = m0.clone(), (m0 ** 2).clone()
    acc = torch.tensor(np.abs(rng.normal(0, 0.02, (P,))).astype(np.float32) * 3, device=DEV)
    acc_abs = acc * torch.tensor(rng.uniform(1.0, 3.0, (P,)).astype(np.float32), device=DEV)
    den = torch.tensor(rng.integers(0, 4, (P,)).astype(np.float32), device=DEV)
    draws = torch.randn((2 * P, 3), device=DEV)

    class Noise:
        def to(self, stds):
            return draws[: stds.shape[0]].to(stds)
    for m in models:
        m.stats = DensifyStats(P, DEV, absgrad=absgrad)
        m.stats.xyz_gradient_accum, m.stats.denom = acc.clone(), den.clone()
        if absgrad:
            m.stats.xyz_gradient_accum_abs = acc_abs.clone()
        m.densify_and_prune(0.01, min_opacity=0.01, extent=4, max_screen_size=1, noise=Noise(), max_abs_grad=0.02 if absgrad else None)
    a, b = models
    assert a.num_points == b.num_points and a.num_points != P
    for k in stage1.GROUPS:
        scale = max(1.0, float(b.p[k].abs().max()))
        assert float((a.p[k] - b.p[k]).abs().max()) <= 3e-6 * scale, k
        assert torch.equal(a.exp_avg[k], b.exp_avg[k]) and torch.equal(a.exp_avg_sq[k], b.exp_avg_sq[k]), k


_cell("densify", densify, absgrad=False)
_cell("densify_abs", densify, absgrad=True)


def mark_visible(cid):
    """markVisible against its rule: view depth > 0.2 (tests/test_parity_gpu.py)."""
    i = _scene(P_SINGLE, 0, 7)
    s = _settings(W, H, 0)
    pos = torch.tensor(i["means3D"], device=DEV)
    vis = R.GaussianRasterizer(_rs(s)[0]).markVisible(pos).cpu().numpy()
    tz = np.concatenate([i["means3D"].astype(np.float64), np.ones((P_SINGLE, 1))], 1) @ np.asarray(s["viewmatrix"], np.float64)[:, 2]
    assert (tz <= 0.2).any() and (tz > 0.2).any()
    assert (vis == (tz > 0.2)).all()


_cell("mark_visible", mark_visible)


# ---- running the cells, and the guard ---------------------------------------------------------------------------------------------
COVERED = {}                   # cell id -> normalized names of the library kernels it launched (recorded after its checks passed)


def _run_cell(cid):
    if cid in COVERED:
        return COVERED[cid]
    torch.cuda.synchronize()
    # acc_events: keep the activity of every profiler cycle; without it a cycle that closes inside a cell (the trace buffers
    # filling up) drops the kernels recorded before it
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        CELLS[cid]()
        torch.cuda.synchronize()
    names = sorted({n for n in (KN.normalize(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
                    if KN.is_library_kernel(n)})
    assert names, (cid, "no library kernel seen by the CUDA activity trace")
    h.report("coverage/" + cid, launched=dict(kernels=names))
    COVERED[cid] = set(names)
    return COVERED[cid]


@pytest.mark.parametrize("cid", list(CELLS))
def test_cell(cid):
    _run_cell(cid)


def test_every_manifest_kernel_is_reached_by_a_checked_call():
    for cid in CELLS:
        _run_cell(cid)
    manifest = KN.read_manifest(MANIFEST)
    need = {n for n, (_, reason) in manifest.items() if reason is None}
    covered = set().union(*COVERED.values())
    missing = sorted(need - covered)
    rerouted = sorted((n, c) for n, (ids, _) in manifest.items() for c in ids if n not in COVERED[c])
    print("covered = %d of %d (%d excused)" % (len(need & covered), len(manifest), len(manifest) - len(need)))
    for n, (_, reason) in sorted(manifest.items()):
        if reason is not None:
            print("excused: %s: %s" % (n, reason))
    assert not missing, ("manifest kernels no checked cell launched", missing)
    assert not rerouted, ("cells that no longer launch the kernels the manifest credits to them", rerouted)
