"""Shared test helpers: scene construction, running the oracle and the CUDA op, parity metrics.

Parity tolerances (fp32 CUDA vs float64 oracle), stated once:
  * images (color / depth / alpha): |cuda - oracle| <= IMG_ATOL = 1e-4 (depth scaled by max(1, max|depth|)) on every
    pixel the oracle does not flag as decision-ambiguous; flagged pixels (a float32 implementation may legitimately
    take the other side of alpha >= 1/255, the T-stop or a depth tie) must be few and within AMBIG_ATOL;
  * radii: exact on every Gaussian the oracle does not flag (ceil / tile-rect boundary within rounding);
  * gradients, per tensor, over the Gaussians the oracle does not flag, with e = |cuda - oracle| - GRAD_RTOL |oracle|
    and scale = max|oracle| of that tensor: the 99.9th percentile of e is <= GRAD_ATOL * scale and the maximum is
    <= GRAD_ATOL_MAX * scale.  (A per-Gaussian gradient is a SIGNED sum over ~10^3 pixel terms, so float32 evaluation
    — the reference's arithmetic type too — loses up to ~1e-3 of the net value on the few Gaussians whose terms cancel;
    the float32 build of the CPU oracle shows the same deviations from the float64 one, see DESIGN.md "Parity".)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from dreamgaussian_b200 import scene  # noqa: E402
from oracle import c_oracle  # noqa: E402

IMG_ATOL = 1e-4
AMBIG_ATOL = 2e-2
GRAD_RTOL = 2e-3
GRAD_ATOL = 1e-4
GRAD_ATOL_MAX = 1e-3
MAX_AMBIG_FRAC = 0.04
TIE_SLACK_FACTOR = 1.5
# float32 CUDA vs the float32 build of the oracle (compare_f32): NO decision-ambiguity exemption, only float32 depth-key
# ties (two consecutive contributors of a pixel whose view depths differ by < 1e-6 relative: either order is a valid
# float32 result) are set aside.  Bounds from tools/parity_report.py.
F32_IMG_ATOL = 2e-4            # every non-tie pixel ...
F32_IMG_OUTLIERS = 2e-5        # ... except this fraction of them (alpha >= 1/255 / T-stop decisions taken the other way) ...
F32_IMG_OUTLIER_ATOL = 1e-2    # ... which stay below this
F32_GRAD_ATOL_MAX = 3e-4       # of the tensor's scale, every non-tie Gaussian ...
F32_GRAD_OUTLIERS = 2e-4       # ... except this fraction of them (a Gaussian whose footprint edge crosses a pixel at alpha = 1/255
F32_GRAD_OUTLIER_ATOL = 2e-2   #     exactly where the two float32 evaluations of exp differ) which stay below this
F32_GRAD_ATOL = 3e-5           # 99.9th percentile


def make_case(P, res, deg, seed=0, elev=0.0, azim=0.0, opacity="trained", sigma=None, anisotropic=True, radius=2.0,
              bg=(1.0, 1.0, 1.0), scale_modifier=1.0, width=None, height=None):
    cloud = scene.make_cloud(P, deg, seed=seed, opacity=opacity, sigma=sigma, anisotropic=anisotropic)
    W = width or res
    Hh = height or res
    cam = scene.orbit_camera(elev, azim, radius, W, Hh)
    settings = dict(image_height=Hh, image_width=W, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy,
                    bg=np.asarray(bg, np.float32), scale_modifier=scale_modifier, viewmatrix=cam.world_view_transform,
                    projmatrix=cam.full_proj_transform, sh_degree=deg, campos=cam.camera_center)
    inputs = dict(means3D=cloud["means3D"], opacities=cloud["opacities"], shs=cloud["shs"], scales=cloud["scales"],
                  rotations=cloud["rotations"])
    return settings, inputs


def upstream_grads(H, W, seed=123, depth=True):
    rng = np.random.default_rng(seed)
    gC = rng.normal(size=(3, H, W)).astype(np.float32)
    gD = rng.normal(size=(1, H, W)).astype(np.float32) if depth else None
    gA = rng.normal(size=(1, H, W)).astype(np.float32)
    return gC, gD, gA


def run_oracle(settings, inputs, grads=None, dtype=np.float64, eps=2e-5):
    r = c_oracle.forward(**settings, **inputs, dtype=dtype, eps=eps)
    out = dict(color=r.color, depth=r.depth, alpha=r.alpha, radii=r.radii)
    apx, ag, n = r.flags()
    out.update(ambig_px=apx, ambig_g=ag, n_inst=n, tie_slack=r.tie_slack())
    if grads is not None:
        out["grads"] = r.backward(*grads)
    r.close()
    return out


def run_cuda(settings, inputs, grads=None, device="cuda", before_backward=None):
    """The product path: GaussianRasterizer on CUDA tensors. Returns numpy outputs (+ grads).  before_backward, if given, is
    called between the forward and the backward (e.g. to change the tuning knobs in between)."""
    import torch
    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device=device)
    rs = GaussianRasterizationSettings(
        image_height=settings["image_height"], image_width=settings["image_width"], tanfovx=settings["tanfovx"],
        tanfovy=settings["tanfovy"], bg=t(settings["bg"]), scale_modifier=settings["scale_modifier"],
        viewmatrix=t(settings["viewmatrix"]), projmatrix=t(settings["projmatrix"]), sh_degree=settings["sh_degree"],
        campos=t(settings["campos"]), prefiltered=False, debug=False)
    tin = {k: t(v).requires_grad_(grads is not None) for k, v in inputs.items()}
    means2D = torch.zeros_like(tin["means3D"], requires_grad=grads is not None)
    color, radii, depth, alpha = GaussianRasterizer(raster_settings=rs)(means2D=means2D, **tin)
    out = dict(color=color.detach().cpu().numpy(), depth=depth.detach().cpu().numpy(), alpha=alpha.detach().cpu().numpy(),
               radii=radii.cpu().numpy())
    if grads is not None:
        gC, gD, gA = grads
        loss = (color * t(gC)).sum() + (alpha * t(gA)).sum()
        if gD is not None:
            loss = loss + (depth * t(gD)).sum()
        if before_backward is not None:
            before_backward()
        loss.backward()
        g = {k: v.grad.detach().cpu().numpy() for k, v in tin.items()}
        g["means2D"] = means2D.grad.detach().cpu().numpy()
        out["grads"] = g
    return out


RAW_KEYS = ("xyz", "features_dc", "features_rest", "opacity", "scaling", "rotation")


def run_oracle_raw(settings, raw, grads):
    """Oracle for the fused-activation path (SURVEY §8 f1): the reference's activations (gs_renderer.py:127-138,196-216)
    in float64 torch, the rasterizer oracle on the activated values, and the activations' chain rule by autograd."""
    import torch
    t = {k: torch.tensor(np.asarray(raw[k], np.float64), requires_grad=True) for k in RAW_KEYS}
    act = dict(means3D=t["xyz"] * 1.0, shs=torch.cat((t["features_dc"], t["features_rest"]), dim=1),
               opacities=torch.sigmoid(t["opacity"]), scales=torch.exp(t["scaling"]),
               rotations=torch.nn.functional.normalize(t["rotation"]))
    ref = run_oracle(settings, {k: v.detach().numpy() for k, v in act.items()}, grads)
    keys = list(act)
    torch.autograd.backward([act[k] for k in keys], [torch.tensor(np.asarray(ref["grads"][k], np.float64)).reshape(act[k].shape) for k in keys])
    g = {k: t[k].grad.numpy() for k in RAW_KEYS}
    g["means2D"] = ref["grads"]["means2D"]
    ref["grads"] = g
    return ref


def run_cuda_raw(settings, raw, grads, stats=None, device="cuda"):
    """The fused product path: FusedGaussianRasterizer on the raw CUDA tensors."""
    import torch
    from dreamgaussian_b200.fused import FusedGaussianRasterizer
    from dreamgaussian_b200.rasterizer import GaussianRasterizationSettings
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device=device)
    rs = GaussianRasterizationSettings(
        image_height=settings["image_height"], image_width=settings["image_width"], tanfovx=settings["tanfovx"],
        tanfovy=settings["tanfovy"], bg=t(settings["bg"]), scale_modifier=settings["scale_modifier"],
        viewmatrix=t(settings["viewmatrix"]), projmatrix=t(settings["projmatrix"]), sh_degree=settings["sh_degree"],
        campos=t(settings["campos"]), prefiltered=False, debug=False)
    tin = {k: t(raw[k]).requires_grad_(True) for k in RAW_KEYS}
    means2D = torch.zeros_like(tin["xyz"], requires_grad=True)
    color, radii, depth, alpha = FusedGaussianRasterizer(rs)(tin["xyz"], tin["features_dc"], tin["features_rest"], tin["opacity"],
                                                             tin["scaling"], tin["rotation"], means2D=means2D, stats=stats)
    gC, gD, gA = grads
    loss = (color * t(gC)).sum() + (alpha * t(gA)).sum()
    if gD is not None:
        loss = loss + (depth * t(gD)).sum()
    loss.backward()
    g = {k: (v.grad.detach().cpu().numpy() if v.grad is not None else np.zeros(v.shape, np.float32)) for k, v in tin.items()}
    g["means2D"] = means2D.grad.detach().cpu().numpy()
    return dict(color=color.detach().cpu().numpy(), depth=depth.detach().cpu().numpy(), alpha=alpha.detach().cpu().numpy(),
                radii=radii.cpu().numpy(), grads=g)


def compare(cu, ref, check_grads=True, max_ambig_frac=MAX_AMBIG_FRAC, ambig_atol=AMBIG_ATOL):
    """Returns (ok, report dict). cu = CUDA outputs (float32), ref = oracle outputs with flags."""
    rep = {}
    ok = True
    apx = ref["ambig_px"].astype(bool)
    ag = ref["ambig_g"]
    rep["ambig_px_frac"] = float(apx.mean()) if apx.size else 0.0
    rep["ambig_g_frac"] = float((ag != 0).mean()) if ag.size else 0.0
    if rep["ambig_px_frac"] > max_ambig_frac:
        ok = False
    slack = TIE_SLACK_FACTOR * ref["tie_slack"].astype(np.float64) if "tie_slack" in ref else np.zeros(apx.shape)
    for name in ("color", "depth", "alpha"):
        d = np.abs(cu[name].astype(np.float64) - ref[name])
        scale = max(1.0, float(np.abs(ref[name]).max())) if name == "depth" else 1.0
        m = np.broadcast_to(apx[None], d.shape)
        clean = d[~m].max() if (~m).any() else 0.0
        # a pixel with a float32 depth-key tie may show the other (equally valid) order: the oracle reports how far that moves
        # the colour (sum over its ties of a1 a2 T |c1 - c2|); depth and alpha do not depend on the order of a tied pair
        bound = ambig_atol + (np.broadcast_to(slack[None], d.shape) if name == "color" else 0.0)
        excess = (d - bound)[m].max() if m.any() else -1.0
        amb = d[m].max() if m.any() else 0.0
        rep[name + "_err"] = float(clean / scale)
        rep[name + "_err_ambig"] = float(amb / scale)
        if clean / scale > IMG_ATOL or excess > 0.0:
            ok = False
    rad_bad = (cu["radii"] != ref["radii"]) & ((ag & 4) == 0)
    rep["radii_mismatch"] = int(rad_bad.sum())
    rep["radii_mismatch_flagged"] = int(((cu["radii"] != ref["radii"]) & ((ag & 4) != 0)).sum())
    if rad_bad.any():
        ok = False
    if check_grads and "grads" in ref:
        clean_g = ag == 0
        # a tensor whose true gradient vanishes by symmetry (e.g. rotations of isotropic Gaussians) is judged
        # against the scale of the other gradients, not against its own round-off
        floor = 1e-3 * max(float(np.abs(v).max()) if v.size else 0.0 for v in ref["grads"].values())
        for k, gr in ref["grads"].items():
            if k not in cu["grads"] or gr.size == 0:          # e.g. _features_rest of a degree-0 model: [P,0,3]
                continue
            gc = cu["grads"][k].astype(np.float64).reshape(gr.shape)
            scale = max(float(np.abs(gr).max()) if gr.size else 0.0, floor) or 1.0
            err = np.abs(gc - gr) - GRAD_RTOL * np.abs(gr)
            e2 = err.reshape(gr.shape[0], -1).max(axis=1) if gr.shape[0] else np.zeros(0)
            worst = float(e2[clean_g].max() / scale) if clean_g.any() else 0.0
            p999 = float(np.percentile(e2[clean_g], 99.9) / scale) if clean_g.any() else 0.0
            worst_amb = float(e2[~clean_g].max() / scale) if (~clean_g).any() else 0.0
            rep["grad_" + k] = worst
            rep["grad_" + k + "_p999"] = p999
            rep["grad_" + k + "_ambig"] = worst_amb
            rep["grad_" + k + "_scale"] = scale
            if p999 > GRAD_ATOL or worst > GRAD_ATOL_MAX or worst_amb > 0.05:
                ok = False
    return ok, rep


def compare_f32(cu, ref32):
    """CUDA (float32) against the float32 build of the oracle with NO decision-ambiguity exemption: only float32 depth-key
    ties (pixels with flag bit 4; Gaussians of a tied pair or compositing in front of a material one, bits 2 | 16) are set
    aside, and Gaussians whose radius sits on a rounding boundary (bit 4) are excused from the exact radii comparison.
    Returns (ok, report)."""
    rep = {}
    ok = True
    tie_px = (ref32["ambig_px"] & 4) != 0
    ag = ref32["ambig_g"]
    tie_g = (ag & (2 | 16)) != 0
    rep["tie_px_frac"] = float(tie_px.mean()) if tie_px.size else 0.0
    rep["tie_g_frac"] = float(tie_g.mean()) if tie_g.size else 0.0
    for name in ("color", "depth", "alpha"):
        d = np.abs(cu[name].astype(np.float64) - ref32[name].astype(np.float64))
        if name == "depth":
            d = d / max(1.0, float(np.abs(ref32[name]).max()))
        dd = d[~np.broadcast_to(tie_px[None], d.shape)]
        n_out = int((dd > F32_IMG_ATOL).sum())
        rep[name + "_max"] = float(dd.max()) if dd.size else 0.0
        rep[name + "_outliers"] = n_out
        if n_out > max(2, int(F32_IMG_OUTLIERS * dd.size)) or (dd.size and dd.max() > F32_IMG_OUTLIER_ATOL):
            ok = False
    bad = (cu["radii"] != ref32["radii"]) & ((ag & 4) == 0)
    rep["radii_mismatch"] = int(bad.sum())
    if bad.any():
        ok = False
    if "grads" in ref32 and "grads" in cu:
        floor = 1e-3 * max(float(np.abs(v).max()) if v.size else 0.0 for v in ref32["grads"].values())
        for k, gr in ref32["grads"].items():
            if k not in cu["grads"] or gr.size == 0:
                continue
            gr = gr.astype(np.float64)
            gc = cu["grads"][k].astype(np.float64).reshape(gr.shape)
            scale = max(float(np.abs(gr).max()), floor) or 1.0
            e = (np.abs(gc - gr) - GRAD_RTOL * np.abs(gr)).reshape(gr.shape[0], -1).max(axis=1) / scale
            e = e[~tie_g]
            rep["grad_" + k] = float(e.max()) if e.size else 0.0
            rep["grad_" + k + "_p999"] = float(np.percentile(e, 99.9)) if e.size else 0.0
            n_out = int((e > F32_GRAD_ATOL_MAX).sum())
            rep["grad_" + k + "_outliers"] = n_out
            if e.size and (n_out > max(2, int(F32_GRAD_OUTLIERS * e.size)) or e.max() > F32_GRAD_OUTLIER_ATOL
                           or np.percentile(e, 99.9) > F32_GRAD_ATOL):
                ok = False
    return ok, rep


def oracles(settings, inputs, grads, f64=True):
    """Both CPU oracle results of one case (float32 build, and float64 unless f64=False), to be reused for every CUDA run of it."""
    return dict(f32=run_oracle(settings, inputs, grads, dtype=np.float32), f64=run_oracle(settings, inputs, grads) if f64 else None)


def both_oracles(name, s, i, g, max_ambig_frac=MAX_AMBIG_FRAC, f64=True, refs=None, cu=None):
    """The rule of the suite: the CUDA result must agree (a) with the float64 oracle on everything that oracle does not flag
    as a decision a float32 implementation may take differently, and (b) with the float32 oracle with NO such exemption —
    only float32 depth-key ties are set aside there.  refs: oracles() of the case (computed here when None); cu: the CUDA
    result to judge (run here when None).  Returns the CUDA result."""
    if refs is None:
        refs = oracles(s, i, g, f64=f64)
    if cu is None:
        cu = run_cuda(s, i, g)
    ok32, rep32 = compare_f32(cu, refs["f32"])
    if refs["f64"] is not None:
        ok64, rep64 = compare(cu, refs["f64"], max_ambig_frac=max_ambig_frac)
    else:
        ok64, rep64 = True, {}
    report(name, vs_f64=rep64, vs_f32=rep32)
    assert ok64, ("float64 oracle", rep64)
    assert ok32, ("float32 oracle", rep32)
    return cu


DEFAULT_TUNING = (1, 1, 1)


def set_tuning(word):
    """dgr_set_tuning(ppl_fwd, ppl_bwd, bits) — process-wide until changed again."""
    from dreamgaussian_b200 import _lib
    _lib.check(_lib.load().dgr_set_tuning(*word))


def run_tuned(word, fn, fast_host=True):
    """fn() with the rasterizer tuned by `word` and the compiled (fast_host) or the ctypes host layer; the default tuning and
    the compiled host layer are restored afterwards, whatever fn does."""
    from dreamgaussian_b200 import rasterizer as R
    try:
        if R.set_fast_host(fast_host) != fast_host:
            raise RuntimeError("the compiled host layer is not available")
        set_tuning(word)
        return fn()
    finally:
        set_tuning(DEFAULT_TUNING)
        R.set_fast_host(True)


def report(name, **reps):
    """Flagged fractions and deviations of a parity case: printed (pytest -s / -rP shows it) and appended to
    gpurun_out/parity_suite.jsonl when that directory exists."""
    import json
    line = json.dumps({"case": name, **{k: {a: (round(b, 9) if isinstance(b, float) else b) for a, b in v.items()} for k, v in reps.items()}})
    print(line)
    d = os.path.join(ROOT, "gpurun_out")
    if os.path.isdir(d):
        with open(os.path.join(d, "parity_suite.jsonl"), "a") as f:
            f.write(line + "\n")
