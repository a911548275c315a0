"""Float64 restatement of the MCMC densification rule (include/dgr_mcmc.h: dgr_mcmc_relocation, dgr_mcmc_refine,
dgr_mcmc_inject_noise; Kheradmand et al., NeurIPS 2024) in numpy: the relocation formula in both published forms and in 60-digit
decimal arithmetic, the sampling rule, one refinement, the position noise.  GaussianModelB200's torch restatement must reproduce
refine() exactly on the CPU; the kernels are held to it on the GPU."""
import math
from decimal import Decimal, localcontext

import numpy as np

GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")
N_MAX = 51
MIN_OPACITY = 0.005
OPACITY_MAX = 1.0 - 2.0 ** -23
GROW_PERCENT = 105
NOISE_K, NOISE_X0 = 100.0, 0.995


def add_count(P, cap_max):
    return max(0, min(int(cap_max), P * GROW_PERCENT // 100) - P)


def opacity(raw):
    """sigmoid in float64, rounded once to float32 (the sampling weights)."""
    return (1.0 / (1.0 + np.exp(-np.asarray(raw, np.float64)))).astype(np.float32)


def new_opacity(o, n):
    return -np.expm1(np.log1p(-np.asarray(o, np.float64)) / np.asarray(n, np.float64))


def hockey_stick(op, n):
    """D = sum_{m=1..n} C(n,m) (-1)^(m-1) op^m / sqrt(m), exact binomials, float64."""
    op, n = np.broadcast_arrays(np.asarray(op, np.float64), np.asarray(n, np.int64))
    D = np.zeros(op.shape)
    for m in range(1, N_MAX + 1):
        c = np.array([math.comb(int(k), m) for k in n.ravel()], np.float64).reshape(n.shape)
        D += (1 if m & 1 else -1) * c * op ** m / math.sqrt(m)
    return D


def double_sum(op, n):
    """The published form: D = sum_{i=1..n} sum_{k=0..i-1} C(i-1,k) (-1)^k op^(k+1) / sqrt(k+1), float64 terms, exactly rounded
    sum (scalar)."""
    return math.fsum(math.comb(i - 1, k) * (-1) ** k * op ** (k + 1) / math.sqrt(k + 1) for i in range(1, n + 1) for k in range(i))


def hockey_stick_fsum(op, n):
    """hockey_stick for one value with an exactly rounded sum (scalar): the form double_sum is compared with."""
    return math.fsum((1 if m & 1 else -1) * math.comb(n, m) * op ** m / math.sqrt(m) for m in range(1, n + 1))


def exact_D(op, n, digits=60):
    """D in `digits`-digit decimal arithmetic from the float64 value op."""
    with localcontext() as ctx:
        ctx.prec = digits
        x = Decimal(float(op))
        return float(sum(Decimal(math.comb(n, m)) * (-1) ** (m - 1) * x ** m / Decimal(m).sqrt() for m in range(1, n + 1)))


def relocate(o, n):
    """(o', o / D) in float64 for activated o and copy counts n (n clamped to [1, N_MAX]); factor 1 where D = 0."""
    o = np.asarray(o, np.float64)
    n = np.clip(np.asarray(n, np.int64), 1, N_MAX)
    op = new_opacity(o, n)
    D = hockey_stick(op, n)
    return op, np.where(D > 0, o / np.where(D > 0, D, 1.0), 1.0)


def sample(weights, u, fallback):
    """Smallest i with C_i > u C_last (C: float64 inclusive prefix of the float32 weights); `fallback` where none.  Also returns
    each draw's distance to the nearest prefix boundary over C_last (a draw within rounding of one may go either way)."""
    C = np.cumsum(np.asarray(weights, np.float32).astype(np.float64))
    t = np.asarray(u, np.float32).astype(np.float64) * C[-1]
    idx = np.searchsorted(C, t, side="right")
    idx = np.where(idx >= len(C), fallback, idx)
    lo = np.where(idx > 0, C[np.maximum(idx - 1, 0)], 0.0)
    margin = np.minimum(np.abs(t - lo), np.abs(C[np.minimum(idx, len(C) - 1)] - t)) / max(C[-1], 1e-300)
    return idx, margin


def update(op_raw, sc_raw, picks, min_opacity):
    """Raw opacity and scaling of rows picked `picks` times: logit(clamp(o')), scaling + log(o / D), float32."""
    o = opacity(op_raw).astype(np.float64)
    op, factor = relocate(o, np.asarray(picks) + 1)
    oc = np.clip(op, np.float64(np.float32(min_opacity)), OPACITY_MAX)
    return np.log(oc / (1 - oc)).astype(np.float32), (np.asarray(sc_raw, np.float64) + np.log(factor)[:, None]).astype(np.float32)


def refine(p, m, v, u_relocate, u_add, cap_max, min_opacity=MIN_OPACITY):
    """One refinement.  p / m / v: {group: float32 [P, ...]} (GROUPS).  Returns (p, m, v, n_relocated, info) with info = dict(
    dead, src (source per dead row), grow_src, margins (of every draw used))."""
    min_opacity = float(np.float32(min_opacity))
    P = p["xyz"].shape[0]
    n_add = add_count(P, cap_max)
    p, m, v = ({k: np.array(d[k], np.float32, copy=True) for k in GROUPS} for d in (p, m, v))
    o = opacity(p["opacity"][:, 0])
    dead = np.nonzero(o <= np.float32(min_opacity))[0]
    live = np.nonzero(o > np.float32(min_opacity))[0]
    info = dict(dead=dead, src=np.zeros(0, np.int64), grow_src=np.zeros(0, np.int64), margins=np.zeros(0))
    n_relocated = 0
    if len(dead) and len(live):
        src, mg = sample(np.where(o > np.float32(min_opacity), o, np.float32(0)), np.asarray(u_relocate)[:len(dead)], live[-1])
        picks = np.bincount(src, minlength=P)
        rows = np.nonzero(picks)[0]
        p["opacity"][rows, 0], p["scaling"][rows] = update(p["opacity"][rows, 0], p["scaling"][rows], picks[rows], min_opacity)
        for k in GROUPS:
            p[k][dead] = p[k][src]
            m[k][rows] = 0
            v[k][rows] = 0
        info.update(src=src, margins=mg)
        n_relocated = len(dead)
    if n_add:
        src, mg = sample(opacity(p["opacity"][:, 0]), u_add, P - 1)
        picks = np.bincount(src, minlength=P)
        rows = np.nonzero(picks)[0]
        p["opacity"][rows, 0], p["scaling"][rows] = update(p["opacity"][rows, 0], p["scaling"][rows], picks[rows], min_opacity)
        for k in GROUPS:
            m[k][rows] = 0
            v[k][rows] = 0
            p[k] = np.concatenate([p[k], p[k][src]])
            m[k] = np.concatenate([m[k], np.zeros_like(p[k][P:])])
            v[k] = np.concatenate([v[k], np.zeros_like(p[k][P:])])
        info.update(grow_src=src, margins=np.concatenate([info["margins"], mg]))
    return p, m, v, n_relocated, info


def rotation(q):
    q = np.asarray(q, np.float64)
    q = q / np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)


def noise_update(op_raw, sc_raw, rot_raw, z, scale):
    """scale g(o) R diag(s^2) R^T z in float64, g(o) = 1 / (1 + exp(-100 ((1 - o) - 0.995)))."""
    o = 1.0 / (1.0 + np.exp(-np.asarray(op_raw, np.float64).reshape(-1)))
    g = 1.0 / (1.0 + np.exp(-NOISE_K * ((1 - o) - NOISE_X0)))
    R = rotation(rot_raw)
    s2 = np.exp(np.asarray(sc_raw, np.float64)) ** 2
    a = np.einsum("pji,pj->pi", R, np.asarray(z, np.float64)) * s2
    return np.einsum("pij,pj->pi", R, a) * (float(scale) * g)[:, None]


def noise_bound(op_raw, sc_raw, z, scale):
    """scale g(o) max(s^2) |z| per row: the size of the terms of the noise update, which float32 rounding is relative to (the update
    itself can be far smaller where z points along a short axis)."""
    o = 1.0 / (1.0 + np.exp(-np.asarray(op_raw, np.float64).reshape(-1)))
    g = 1.0 / (1.0 + np.exp(-NOISE_K * ((1 - o) - NOISE_X0)))
    s2 = np.exp(np.asarray(sc_raw, np.float64)).max(axis=1) ** 2
    return (float(scale) * g * s2 * np.linalg.norm(np.asarray(z, np.float64), axis=1))[:, None]
