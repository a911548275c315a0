"""Helpers of the camera-gradient tests (DGR_RASTER_CAMERA_GRADS, include/dgr_b200.h).

* minicam: MiniCam's formulas (what dreamgaussian_b200.scene.make_camera restates in numpy) in differentiable torch ops, so a
  learnable camera-to-world pose drives viewmatrix / projmatrix / campos, the campos = -c2w[:3,3] sign quirk included.
* pose_of: a 6-DoF perturbation (axis-angle rotation applied on the left of c2w's rotation, translation added) of a c2w.
* oracle_loss: the float64 torch oracle (oracle/torch_oracle.py) with viewmatrix / projmatrix / campos as tensors, so autograd gives
  the reference camera gradients; antialiased=True multiplies the opacities by the mode's factor with the factor differentiable in
  the view matrix too (tests/aa_oracle.py holds V fixed)."""
import math

import numpy as np
import torch

from oracle import torch_oracle as T
import aa_oracle


def minicam(c2w, W, H, fovy_deg=49.1, znear=0.01, zfar=100.0):
    """c2w [4,4] (OpenGL convention, torch, any float dtype) -> (viewmatrix, projmatrix, campos, tanfovx, tanfovy)."""
    dt, dev = c2w.dtype, c2w.device
    fovy = math.radians(fovy_deg)
    fovx = 2 * math.atan(math.tan(fovy / 2) * W / H)
    w2c = torch.linalg.inv(c2w)
    flip = torch.tensor([1.0, -1.0, -1.0], dtype=dt, device=dev)
    R = w2c[:3, :3] * flip[:, None]                      # w2c[1:3, :3] *= -1
    t = -w2c[:3, 3]                                      # w2c[:3, 3] *= -1
    w2c = torch.cat([torch.cat([R, t[:, None]], 1), w2c[3:4]], 0)
    V = w2c.t()
    Pm = torch.zeros(4, 4, dtype=dt, device=dev)
    Pm[0, 0] = 1.0 / math.tan(fovx / 2)
    Pm[1, 1] = 1.0 / math.tan(fovy / 2)
    Pm[3, 2] = 1.0
    Pm[2, 2] = zfar / (zfar - znear)
    Pm[2, 3] = -(zfar * znear) / (zfar - znear)
    return V, V @ Pm.t(), -c2w[:3, 3], math.tan(fovx * 0.5), math.tan(fovy * 0.5)


def _skew(w):
    z = torch.zeros((), dtype=w.dtype, device=w.device)
    return torch.stack([torch.stack([z, -w[2], w[1]]), torch.stack([w[2], z, -w[0]]), torch.stack([-w[1], w[0], z])])


def pose_of(c2w0, delta):
    """delta [6] = (axis-angle, translation) -> c2w with rotation exp([w]x) R0 and position t0 + dt (differentiable)."""
    R = torch.linalg.matrix_exp(_skew(delta[:3])) @ c2w0[:3, :3]
    t = c2w0[:3, 3] + delta[3:]
    bottom = torch.tensor([[0.0, 0.0, 0.0, 1.0]], dtype=c2w0.dtype, device=c2w0.device)
    return torch.cat([torch.cat([R, t[:, None]], 1), bottom], 0)


def rotation_angle(Ra, Rb):
    """Angle (radians) of Ra^T Rb."""
    c = ((Ra.t() @ Rb).trace() - 1.0) * 0.5
    return float(torch.arccos(torch.clamp(c, -1.0, 1.0)))


def aa_comp(V, H, W, tanfovx, tanfovy, scale_modifier, means3D, scales=None, rotations=None, cov3D_precomp=None):
    """aa_oracle.comp with the view matrix V a (differentiable) tensor."""
    dt = means3D.dtype
    V = V.to(dt)
    fx, fy = W / (2 * tanfovx), H / (2 * tanfovy)
    P = means3D.shape[0]
    t = torch.cat([means3D, torch.ones(P, 1, dtype=dt)], 1) @ V[:, :3]
    if cov3D_precomp is None:
        R = T._quat_to_R(rotations)
        Mx = R * (scale_modifier * scales)[:, None, :]
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
    a, b, c = cov[:, 0, 0] + T.LOWPASS, cov[:, 0, 1], cov[:, 1, 1] + T.LOWPASS
    return torch.sqrt(torch.clamp(aa_oracle.ratio_of(a, b, c), min=aa_oracle.AA_RATIO_FLOOR))


def oracle_render(settings, inputs, V, PM, campos, antialiased=False, dtype=torch.float64):
    """The torch oracle's (color, radii, depth, alpha) with camera tensors V / PM / campos; inputs are tensors of `dtype`."""
    kw = dict(image_height=settings["image_height"], image_width=settings["image_width"], tanfovx=settings["tanfovx"],
              tanfovy=settings["tanfovy"], bg=torch.tensor(np.asarray(settings["bg"], np.float64), dtype=dtype),
              scale_modifier=settings["scale_modifier"], viewmatrix=V, projmatrix=PM, sh_degree=settings["sh_degree"], campos=campos,
              means2D=None, **inputs)
    if antialiased:
        k = aa_comp(V, settings["image_height"], settings["image_width"], settings["tanfovx"], settings["tanfovy"],
                    settings["scale_modifier"], inputs["means3D"], inputs.get("scales"), inputs.get("rotations"), inputs.get("cov3D_precomp"))
        kw["opacities"] = inputs["opacities"] * k.reshape(inputs["opacities"].shape)
    return T.rasterize(**kw)


def oracle_camera_grads(settings, inputs, loss_fn, antialiased=False, dtype=torch.float64):
    """(dL/dviewmatrix [4,4], dL/dprojmatrix [4,4], dL/dcampos [3]) of loss_fn(color, depth, alpha) by the torch oracle's autograd."""
    cam = [torch.tensor(np.asarray(settings[k], np.float64), dtype=dtype, requires_grad=True) for k in ("viewmatrix", "projmatrix", "campos")]
    tin = {k: torch.tensor(np.asarray(v, np.float64), dtype=dtype) for k, v in inputs.items() if v is not None}
    color, _, depth, alpha = oracle_render(settings, tin, *cam, antialiased=antialiased, dtype=dtype)
    return torch.autograd.grad(loss_fn(color, depth, alpha), cam, allow_unused=True)
