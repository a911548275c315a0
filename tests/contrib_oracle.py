"""Oracles of the blending-weight statistics (DGR_RASTER_CONTRIB, include/dgr_b200.h).

Per render and Gaussian g:  weight_sum = sum_p w_p,  weight_max = max_p w_p,  w_p = alpha_p T_p over the pixels p where the forward
composites g.  Two independent restatements, both on the forward state of the C oracle (oracle/c_oracle.py):
  * c_stats: the C oracle's forward compositing with the weights summed per Gaussian (contrib_oracle.c; float32 and float64 builds);
  * torch_stats: float64 torch, the compositing of oracle/torch_oracle.py's forward restated per tile as a cumulative product.
Both return (weight_sum, weight_max) float64 [P]."""
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
_SOURCES = [os.path.join(_HERE, "contrib_oracle.c"), os.path.join(_HERE, "contrib_oracle_impl.h"),
            os.path.join(_ROOT, "oracle", "dgr_oracle.c"), os.path.join(_ROOT, "oracle", "dgr_oracle_impl.h"),
            os.path.join(_ROOT, "include", "dgr_constants.h")]
_lib = None


def build():
    """gcc contrib_oracle.c -> <tmp>/dgr_contrib_oracle_<hash>.so (the repository tree is left as it is).  Returns the path."""
    h = hashlib.sha256()
    for s in _SOURCES:
        with open(s, "rb") as f:
            h.update(f.read())
    out = os.path.join(tempfile.gettempdir(), "dgr_contrib_oracle_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
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


def c_stats(res):
    """res: an oracle.c_oracle.forward result (float32 or float64) -> (weight_sum, weight_max) float64 [P]."""
    out = np.zeros((max(res.P, 1), 2), np.float64)
    getattr(lib(), "dgr_oracle_contrib_" + res._suf)(ctypes.c_void_p(res._ctx), out.ctypes.data_as(ctypes.c_void_p))
    out = out[: res.P]
    return out[:, 0].copy(), out[:, 1].copy()


def torch_stats(res, opacities):
    """The same statistics in float64 torch on the forward state of `res` (opacities as fed to the oracle; o_eff in the
    anti-aliased mode): every tile's list in the oracle's (depth, index) order, the skip rules and the T stop as cumulative
    products over the list."""
    st = res.state()
    H, W, P = res.H, res.W, res.P
    f64 = lambda a: torch.as_tensor(np.asarray(a, np.float64))
    px, py, conic, rect = f64(st["px"]), f64(st["py"]), f64(st["conic"]), st["rect"]
    opac = f64(opacities).reshape(-1)
    area = (rect[:, 2] - rect[:, 0]) * (rect[:, 3] - rect[:, 1])
    vis = (np.asarray(res.radii) > 0) & (area > 0)
    wsum, wmax = np.zeros(P, np.float64), np.zeros(P, np.float64)
    gx, gy = (W + T.TILE - 1) // T.TILE, (H + T.TILE - 1) // T.TILE
    dep_np = np.asarray(st["depth"], np.float64)
    for ty_ in range(gy):
        for tx_ in range(gx):
            m = vis & (rect[:, 0] <= tx_) & (rect[:, 2] > tx_) & (rect[:, 1] <= ty_) & (rect[:, 3] > ty_)
            ids = np.nonzero(m)[0]
            if ids.size == 0:
                continue
            ids = ids[np.lexsort((ids, dep_np[ids]))]
            it = torch.as_tensor(ids)
            x0, y0 = tx_ * T.TILE, ty_ * T.TILE
            x1, y1 = min(x0 + T.TILE, W), min(y0 + T.TILE, H)
            ys, xs = torch.meshgrid(torch.arange(y0, y1, dtype=torch.float64), torch.arange(x0, x1, dtype=torch.float64), indexing="ij")
            dx, dy = px[it][None, :] - xs.reshape(-1, 1), py[it][None, :] - ys.reshape(-1, 1)
            cA, cB, cC = conic[it, 0][None], conic[it, 1][None], conic[it, 2][None]
            power = -0.5 * (cA * dx * dx + cC * dy * dy) - cB * dx * dy
            a = torch.clamp(opac[it][None] * torch.exp(torch.clamp(power, max=0.0)), max=T.ALPHA_MAX)
            contrib = (power <= 0) & (a >= T.ALPHA_MIN)
            a = torch.where(contrib, a, torch.zeros_like(a))
            one_m = 1 - a
            Texcl = torch.cumprod(torch.cat([torch.ones_like(one_m[:, :1]), one_m[:, :-1]], 1), 1)
            stopped = torch.cummax((contrib & (Texcl * one_m < T.T_STOP)).to(torch.int8), 1).values.bool()
            w = torch.where(stopped | ~contrib, torch.zeros_like(a), a * Texcl).numpy()
            np.add.at(wsum, ids, w.sum(0))
            np.maximum.at(wmax, ids, w.max(0))
    return wsum, wmax
