"""Oracles of the anti-aliased mode (DGR_RASTER_ANTIALIAS, include/dgr_b200.h), built on the default-mode oracles.

The mode changes one thing: each Gaussian's activated opacity o becomes o_eff = o comp, with
comp = sqrt(max(AA_RATIO_FLOOR, det0 / det)) from its 2D covariance before (det0) and after (det) the 0.3 px^2 low-pass.  The
radii, the tile rectangle and the conic are those of the default mode.  So an anti-aliased render IS the default-mode render of
the cloud with opacities o_eff, and its gradients are the default-mode gradients plus the path through comp:
  * torch (float64, autograd): oracle.torch_oracle.rasterize with opacities = o * comp(inputs), comp differentiable;
  * C (float32 / float64, hand-derived): oracle.c_oracle on opacities o_eff, then dL/do = dL/do_eff comp and, for the geometry,
    the C oracle's gradient plus dL/do_eff o d comp / d(geometry) (comp's own chain rule by autograd).  Its decision-ambiguity
    flags are those of the o_eff render, the opacity the 1/255 and 0.99 decisions of the mode use.
comp is computed here with the projection of oracle/torch_oracle.py (same clamp rule inside J)."""
import numpy as np
import torch

import helpers
from oracle import torch_oracle as T

AA_RATIO_FLOOR = T._f(2.5e-5)            # include/dgr_constants.h DGR_AA_RATIO_FLOOR


def cov2d(settings, means3D, scales=None, rotations=None, cov3D_precomp=None):
    """(a, b, c): the 2D covariance in pixels WITH the low-pass, float64 torch, differentiable (torch_oracle's projection)."""
    dt = means3D.dtype
    V = torch.as_tensor(np.asarray(settings["viewmatrix"], np.float64)).to(dt)
    H, W = int(settings["image_height"]), int(settings["image_width"])
    tanfovx, tanfovy = float(settings["tanfovx"]), float(settings["tanfovy"])
    fx, fy = W / (2 * tanfovx), H / (2 * tanfovy)
    P = means3D.shape[0]
    t = torch.cat([means3D, torch.ones(P, 1, dtype=dt)], 1) @ V[:, :3]
    if cov3D_precomp is None:
        R = T._quat_to_R(rotations)
        Mx = R * (float(settings["scale_modifier"]) * scales)[:, None, :]
        Sigma = Mx @ Mx.transpose(1, 2)
    else:
        c = cov3D_precomp
        Sigma = torch.stack([c[:, 0], c[:, 1], c[:, 2], c[:, 1], c[:, 3], c[:, 4], c[:, 2], c[:, 4], c[:, 5]], 1).reshape(-1, 3, 3)
    tz = t[:, 2]
    tz_safe = torch.where(tz > T.NEAR_CULL_Z, tz, torch.ones_like(tz))
    limx, limy = T.FOV_CLAMP * tanfovx, T.FOV_CLAMP * tanfovy
    txtz, tytz = t[:, 0] / tz_safe, t[:, 1] / tz_safe
    clx, cly = (txtz < -limx) | (txtz > limx), (tytz < -limy) | (tytz > limy)
    tx = torch.where(clx, (txtz.clamp(-limx, limx) * tz_safe).detach(), t[:, 0])
    ty = torch.where(cly, (tytz.clamp(-limy, limy) * tz_safe).detach(), t[:, 1])
    zero = torch.zeros_like(tz)
    J = torch.stack([fx / tz_safe, zero, -fx * tx / (tz_safe * tz_safe), zero, fy / tz_safe, -fy * ty / (tz_safe * tz_safe)], 1).reshape(-1, 2, 3)
    Tm = J @ V[:3, :3].t()
    cov = Tm @ Sigma @ Tm.transpose(1, 2)
    return cov[:, 0, 0] + T.LOWPASS, cov[:, 0, 1], cov[:, 1, 1] + T.LOWPASS


def ratio_of(a, b, c):
    """det0 / det, as the kernels form it from the low-passed covariance."""
    det = a * c - b * b
    det_safe = torch.where(det != 0, det, torch.ones_like(det))
    return ((a - T.LOWPASS) * (c - T.LOWPASS) - b * b) / det_safe


def comp(settings, means3D, scales=None, rotations=None, cov3D_precomp=None):
    """The opacity factor of the anti-aliased mode, per Gaussian (differentiable; no gradient where the floor is active)."""
    return torch.sqrt(torch.clamp(ratio_of(*cov2d(settings, means3D, scales, rotations, cov3D_precomp)), min=AA_RATIO_FLOOR))


def rasterize(**kw):
    """oracle.torch_oracle.rasterize in the anti-aliased mode (same arguments and outputs)."""
    settings = dict(image_height=kw["image_height"], image_width=kw["image_width"], tanfovx=kw["tanfovx"], tanfovy=kw["tanfovy"],
                    viewmatrix=kw["viewmatrix"].detach().numpy() if torch.is_tensor(kw["viewmatrix"]) else kw["viewmatrix"],
                    scale_modifier=kw["scale_modifier"])
    k = comp(settings, kw["means3D"], kw.get("scales"), kw.get("rotations"), kw.get("cov3D_precomp"))
    kw = dict(kw, opacities=kw["opacities"] * k.reshape(kw["opacities"].shape))
    return T.rasterize(**kw)


ACT = {"xyz": "means3D", "scaling": "scales", "rotation": "rotations", "opacity": "opacities"}


def run_oracle(settings, inputs, grads=None, dtype=np.float64, eps=2e-5, raw=False):
    """helpers.run_oracle (raw=True: helpers.run_oracle_raw) in the anti-aliased mode; same outputs, flags of the o_eff render."""
    keys = helpers.RAW_KEYS if raw else [k for k, v in inputs.items() if v is not None]
    t = {k: torch.tensor(np.asarray(inputs[k], np.float64), requires_grad=True) for k in keys}
    if raw:
        act = dict(means3D=t["xyz"] * 1.0, shs=torch.cat((t["features_dc"], t["features_rest"]), dim=1), opacities=torch.sigmoid(t["opacity"]),
                   scales=torch.exp(t["scaling"]), rotations=torch.nn.functional.normalize(t["rotation"]))
    else:
        act = dict(t)
    o_eff = act["opacities"] * comp(settings, act["means3D"], act.get("scales"), act.get("rotations"),
                                    act.get("cov3D_precomp")).reshape(act["opacities"].shape)
    fed = {k: v.detach().numpy() for k, v in act.items()}
    fed["opacities"] = o_eff.detach().numpy()
    ref = helpers.run_oracle(settings, fed, grads, dtype=dtype, eps=eps)
    if grads is None:
        return ref
    g = ref["grads"]
    cot = lambda k: torch.tensor(np.asarray(g[k], np.float64)).reshape(act[k].shape)
    outs = [k for k in act if k != "opacities"]
    # the C oracle's gradients hold o_eff fixed: its opacity gradient is dL/do_eff, which flows back through o_eff = o comp
    torch.autograd.backward([act[k] for k in outs] + [o_eff], [cot(k) for k in outs] + [cot("opacities")])
    res = {k: t[k].grad.numpy().astype(np.float64) for k in keys}
    res["means2D"] = g["means2D"]
    if not raw:                  # gradients the forward did not use (colors_precomp / cov3D / shs absent) stay as the C oracle has them
        for k in g:
            res.setdefault(k, g[k])
    ref["grads"] = res
    return ref


def oracles(settings, inputs, grads, f64=True, raw=False):
    """helpers.oracles for the anti-aliased mode."""
    return dict(f32=run_oracle(settings, inputs, grads, dtype=np.float32, raw=raw),
                f64=run_oracle(settings, inputs, grads, raw=raw) if f64 else None)
