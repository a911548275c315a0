"""Oracles of the absolute-gradient densification statistic (DGR_RASTER_ABS_GRAD, include/dgr_b200.h; AbsGS, Ye et al., 2024).

Per render and Gaussian g with radius > 0:  stat = sqrt(a_x^2 + a_y^2),  a_x = sum_p |t_x(p)| W/2,  a_y = sum_p |t_y(p)| H/2,  where
t(p) is pixel p's term of dL/dmean_px (pixel units) and p runs over the pixels the backward render evaluates g at.  Two independent
restatements, both on the forward state of the C oracle (oracle/c_oracle.py):
  * c_terms: hand-derived, absgrad_oracle.c (the C oracle's backward loop with |.| sums; float32 and float64 builds);
  * autograd_terms: float64 torch, each (pixel, Gaussian) pair holding its OWN leaf copy of the 2D mean, so autograd returns every
    per-pixel term separately (their sum over the pixels is dL/dmean_px).
Both return dict(abs_x, abs_y, sum_x, sum_y) [P] in pixel units; stat() turns them into the statistic (NDC units)."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import torch

from oracle import torch_oracle as T

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SOURCES = [os.path.join(_HERE, "absgrad_oracle.c"), os.path.join(_HERE, "absgrad_oracle_impl.h"),
            os.path.join(_ROOT, "oracle", "dgr_oracle.c"), os.path.join(_ROOT, "oracle", "dgr_oracle_impl.h"),
            os.path.join(_ROOT, "include", "dgr_constants.h")]
_lib = None


def build():
    """gcc absgrad_oracle.c -> <tmp>/dgr_absgrad_oracle_<hash>.so (the repository tree is left as it is).  Returns the path."""
    h = hashlib.sha256()
    for s in _SOURCES:
        with open(s, "rb") as f:
            h.update(f.read())
    out = os.path.join(tempfile.gettempdir(), "dgr_absgrad_oracle_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
    if not os.path.exists(out):
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        tmp = out + ".%d.tmp" % os.getpid()
        subprocess.check_call([cc, "-O2", "-fopenmp", "-fPIC", "-std=c11", "-ffp-contract=off", "-w", "-shared", "-o", tmp,
                               _SOURCES[0], "-lm"], cwd=_HERE)
        os.replace(tmp, out)
    return out


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(build())
    return _lib


def c_terms(res, dL_dcolor=None, dL_ddepth=None, dL_dalpha=None):
    """res: an oracle.c_oracle.forward result (float32 or float64) -> the per-Gaussian sums of the hand-derived oracle."""
    dt = res._dt
    cv = lambda a: None if a is None else np.ascontiguousarray(np.asarray(a, dtype=dt))
    gC, gD, gA = cv(dL_dcolor), cv(dL_ddepth), cv(dL_dalpha)
    out = np.zeros((max(res.P, 1), 4), np.float64)
    p = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)
    getattr(lib(), "dgr_oracle_absgrad_" + res._suf)(ctypes.c_void_p(res._ctx), p(gC), p(gD), p(gA), p(out))
    out = out[: res.P]
    return dict(abs_x=out[:, 0], abs_y=out[:, 1], sum_x=out[:, 2], sum_y=out[:, 3])


def autograd_terms(res, opacities, bg, dL_dcolor=None, dL_ddepth=None, dL_dalpha=None, per_pixel=False):
    """The same sums from float64 autograd on the forward state of `res` (float64 C oracle result; opacities as fed to it).
    per_pixel=True also returns 'pixels': {g: (t_x [n], t_y [n])}, every per-pixel term of every Gaussian."""
    st = res.state()
    H, W, P = res.H, res.W, res.P
    f64 = lambda a: torch.as_tensor(np.asarray(a, np.float64))
    px, py, depth, conic, rgb, rect = f64(st["px"]), f64(st["py"]), f64(st["depth"]), f64(st["conic"]), f64(st["rgb"]), st["rect"]
    opac = f64(opacities).reshape(-1)
    bgt = f64(bg).reshape(3)
    gC = f64(dL_dcolor).reshape(3, H, W) if dL_dcolor is not None else torch.zeros(3, H, W, dtype=torch.float64)
    gD = f64(dL_ddepth).reshape(H, W) if dL_ddepth is not None else torch.zeros(H, W, dtype=torch.float64)
    gA = f64(dL_dalpha).reshape(H, W) if dL_dalpha is not None else torch.zeros(H, W, dtype=torch.float64)
    area = (rect[:, 2] - rect[:, 0]) * (rect[:, 3] - rect[:, 1])
    vis = (np.asarray(res.radii) > 0) & (area > 0)
    out = {k: np.zeros(P, np.float64) for k in ("abs_x", "abs_y", "sum_x", "sum_y")}
    pixels = {}
    gx, gy = (W + T.TILE - 1) // T.TILE, (H + T.TILE - 1) // T.TILE
    dep_np = np.asarray(st["depth"], np.float64)
    for ty_ in range(gy):
        for tx_ in range(gx):
            m = vis & (rect[:, 0] <= tx_) & (rect[:, 2] > tx_) & (rect[:, 1] <= ty_) & (rect[:, 3] > ty_)
            ids = np.nonzero(m)[0]
            if ids.size == 0:
                continue
            ids = ids[np.lexsort((ids, dep_np[ids]))]                   # the oracle's stable (depth, index) order
            it = torch.as_tensor(ids)
            x0, y0 = tx_ * T.TILE, ty_ * T.TILE
            x1, y1 = min(x0 + T.TILE, W), min(y0 + T.TILE, H)
            ys, xs = torch.meshgrid(torch.arange(y0, y1, dtype=torch.float64), torch.arange(x0, x1, dtype=torch.float64), indexing="ij")
            xs, ys = xs.reshape(-1, 1), ys.reshape(-1, 1)
            n = xs.shape[0]
            mxl = px[it][None, :].expand(n, -1).clone().requires_grad_(True)      # one leaf per (pixel, Gaussian)
            myl = py[it][None, :].expand(n, -1).clone().requires_grad_(True)
            dx, dy = mxl - xs, myl - ys
            cA, cB, cC = conic[it, 0][None], conic[it, 1][None], conic[it, 2][None]
            power = -0.5 * (cA * dx * dx + cC * dy * dy) - cB * dx * dy
            G = torch.exp(torch.clamp(power, max=0.0))
            a = T._StraightThroughMin.apply(opac[it][None] * G, T.ALPHA_MAX)
            with torch.no_grad():
                contrib = (power <= 0) & (a >= T.ALPHA_MIN)
            a = torch.where(contrib, a, torch.zeros_like(a))
            one_m = 1 - a
            Texcl = torch.cumprod(torch.cat([torch.ones_like(one_m[:, :1]), one_m[:, :-1]], 1), 1)
            with torch.no_grad():
                stopped = torch.cummax((contrib & (Texcl * one_m < T.T_STOP)).to(torch.int8), 1).values.bool()
            w = torch.where(stopped, torch.zeros_like(a), a * Texcl)
            Tfin = torch.prod(torch.where(stopped, torch.ones_like(one_m), one_m), 1)
            color = w @ rgb[it] + Tfin[:, None] * bgt[None, :]
            loss = ((color * gC[:, y0:y1, x0:x1].reshape(3, -1).t()).sum() + ((w @ depth[it]) * gD[y0:y1, x0:x1].reshape(-1)).sum()
                    + (w.sum(1) * gA[y0:y1, x0:x1].reshape(-1)).sum())
            tx, ty = torch.autograd.grad(loss, (mxl, myl))
            tx, ty = tx.numpy(), ty.numpy()
            np.add.at(out["abs_x"], ids, np.abs(tx).sum(0)); np.add.at(out["abs_y"], ids, np.abs(ty).sum(0))
            np.add.at(out["sum_x"], ids, tx.sum(0)); np.add.at(out["sum_y"], ids, ty.sum(0))
            if per_pixel:
                for j, g in enumerate(ids):
                    a_, b_ = pixels.get(int(g), (np.zeros(0), np.zeros(0)))
                    pixels[int(g)] = (np.concatenate([a_, tx[:, j]]), np.concatenate([b_, ty[:, j]]))
    if per_pixel:
        out["pixels"] = pixels
    return out


def stat(terms, radii, H, W):
    """-> (abs statistic, default statistic |dL/dmeans2D[:2]|) of one render, NDC units, 0 where radii == 0."""
    ax, ay = terms["abs_x"] * 0.5 * W, terms["abs_y"] * 0.5 * H
    sx, sy = terms["sum_x"] * 0.5 * W, terms["sum_y"] * 0.5 * H
    on = np.asarray(radii) > 0
    return np.where(on, np.sqrt(ax * ax + ay * ay), 0.0), np.where(on, np.sqrt(sx * sx + sy * sy), 0.0)
