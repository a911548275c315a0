"""SH storage wider than the active degree, on the CPU: the oracles accept padded rows and ignore the padding.

Callers in the 3DGS style pass shs with (max_sh_degree + 1)^2 coefficients per Gaussian and render at active_sh_degree, so the
row holds M >= NB = (deg + 1)^2 coefficients of which only the first NB are read (gs_renderer.py:806 passes get_features next to
active_sh_degree; dreamgaussian_b200.stage1 does the same).  tests/test_sh_padding_gpu.py judges the kernels on such rows with the
oracles unchanged; this file shows that is sound: for every oracle a padded input gives exactly the images, statistics and active
gradients of the unpadded one, and zero gradient in the padding.  The padding holds large values (+-10), so an oracle that read
it would change its images.

The helpers pad_shs and pad_raw are shared with the GPU file."""
import numpy as np
import pytest
import torch

import aa_oracle
import absgrad_oracle as AO
import camgrad_helpers as C
import contrib_oracle as CO
import helpers as h
import trained_scenes as TS
from oracle import c_oracle
from oracle import torch_oracle as T

# (active degree, coefficients per row M): the layouts a 3DGS caller produces, plus rows the ABI accepts that it never does
# (M = 5 and 11: rows of 60 and 132 bytes, not multiples of 16)
PAIRS = [(0, 4), (0, 16), (1, 5), (1, 9), (1, 16), (2, 11), (2, 16)]
PAD_MAGNITUDE = 10.0


def pad_shs(shs, M, seed=0):
    """shs [P, NB, 3] -> [P, M, 3]: the rows extended with uniform values in +-PAD_MAGNITUDE."""
    P, NB, _ = shs.shape
    rng = np.random.default_rng(1000 + 17 * M + seed)
    pad = rng.uniform(-PAD_MAGNITUDE, PAD_MAGNITUDE, (P, M - NB, 3)).astype(shs.dtype)
    return np.ascontiguousarray(np.concatenate([shs, pad], axis=1))


def pad_raw(raw, M, seed=0):
    """Raw GaussianModel parameters with _features_rest widened from NB - 1 to M - 1 columns (the padding as in pad_shs)."""
    out = dict(raw)
    rest = raw["features_rest"]
    P = rest.shape[0]
    full = np.concatenate([np.zeros((P, 1, 3), rest.dtype), rest], axis=1)
    out["features_rest"] = np.ascontiguousarray(pad_shs(full, M, seed)[:, 1:])
    return out


@pytest.fixture(autouse=True)
def _one_oracle_thread():
    """The C oracles sum a Gaussian's gradient over pixels in thread order: bit-for-bit comparisons need one thread."""
    n = c_oracle.num_threads()
    c_oracle.set_threads(1)
    yield
    c_oracle.set_threads(n)


def _case(deg, P=97, W=40, H=24, seed=3):
    """A small compact_mix scene (P not a multiple of 32, sides not multiples of 16) with its settings and upstream gradients."""
    s, i = TS.compact_mix(P, seed=seed + deg, W=W, H=H, deg=deg)
    return s, i, h.upstream_grads(H, W, seed=40 + deg)


def _same(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and np.array_equal(a, b), (what, float(np.abs(a.astype(np.float64) - b).max()) if a.shape == b.shape else a.shape)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("deg,M", PAIRS)
def test_c_oracle_ignores_the_padding(deg, M, dtype):
    s, i, g = _case(deg)
    NB = (deg + 1) ** 2
    padded = dict(i, shs=pad_shs(i["shs"], M))
    outs = []
    for inputs in (i, padded):
        r = c_oracle.forward(**s, **inputs, dtype=dtype)
        o = dict(color=r.color.copy(), depth=r.depth.copy(), alpha=r.alpha.copy(), radii=r.radii.copy(), tie=r.tie_slack())
        o["px"], o["g"], o["n"] = r.flags()
        o["grads"] = r.backward(*g)
        o["abs"] = AO.c_terms(r, *g)
        o["wsum"], o["wmax"] = CO.c_stats(r)
        r.close()
        outs.append(o)
    a, b = outs
    assert (a["radii"] > 0).sum() > 20 and (a["alpha"] > 0.5).sum() > 50
    for k in ("color", "depth", "alpha", "radii", "tie", "px", "g", "n", "wsum", "wmax"):
        _same(b[k], a[k], k)
    for k in a["abs"]:
        _same(b["abs"][k], a["abs"][k], "abs " + k)
    for k, v in a["grads"].items():
        w = b["grads"][k]
        if k == "shs":
            assert w.shape == (len(v), M, 3)
            _same(w[:, :NB], v, k)
            assert not w[:, NB:].any(), "shs padding gradient"
        else:
            _same(w, v, k)


@pytest.mark.parametrize("deg,M", [(0, 16), (1, 5), (2, 11)])
def test_torch_oracle_and_camera_gradients_ignore_the_padding(deg, M):
    s, i, g = _case(deg)
    NB = (deg + 1) ** 2
    loss = lambda color, depth, alpha: sum((x * torch.tensor(np.asarray(u, np.float64))).sum() for x, u in zip((color, depth, alpha), g))
    outs = []
    for shs in (i["shs"], pad_shs(i["shs"], M)):
        tin = {k: torch.tensor(np.asarray(v, np.float64), requires_grad=True) for k, v in dict(i, shs=shs).items()}
        cam = [torch.tensor(np.asarray(s[k], np.float64), requires_grad=True) for k in ("viewmatrix", "projmatrix", "campos")]
        kw = {k: s[k] for k in ("image_height", "image_width", "tanfovx", "tanfovy", "scale_modifier", "sh_degree")}
        color, radii, depth, alpha = T.rasterize(**kw, bg=torch.tensor(np.asarray(s["bg"], np.float64)), viewmatrix=cam[0], projmatrix=cam[1],
                                                 campos=cam[2], means2D=None, **tin)
        loss(color, depth, alpha).backward()
        outs.append(dict(color=color.detach().numpy(), depth=depth.detach().numpy(), alpha=alpha.detach().numpy(), radii=radii.numpy(),
                         grads={k: v.grad.numpy() for k, v in tin.items()}, cam=[c.grad.numpy() if c.grad is not None else np.zeros(c.shape) for c in cam]))
    a, b = outs
    for k in ("color", "depth", "alpha", "radii"):
        _same(b[k], a[k], k)
    for k, v in a["grads"].items():
        _same(b["grads"][k][:, :NB] if k == "shs" else b["grads"][k], v, k)
    assert not b["grads"]["shs"][:, NB:].any()
    for x, y, n in zip(b["cam"], a["cam"], ("viewmatrix", "projmatrix", "campos")):
        _same(x, y, n)
    assert deg == 0 or np.abs(a["cam"][2]).max() > 0        # above degree 0 the SH colour depends on campos
    # and camgrad_helpers.oracle_camera_grads (the GPU rule's reference), float64 and float32, AA or not
    for aa, dt in ((False, torch.float64), (True, torch.float32)):
        ref = C.oracle_camera_grads(s, i, loss, antialiased=aa, dtype=dt)
        got = C.oracle_camera_grads(s, dict(i, shs=pad_shs(i["shs"], M)), loss, antialiased=aa, dtype=dt)
        for x, y in zip(got, ref):
            assert (x is None) == (y is None)
            if x is not None:
                _same(x.numpy(), y.numpy(), ("oracle_camera_grads", aa, dt))


@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("deg,M", [(0, 16), (1, 5), (2, 11)])
def test_raw_and_antialiased_oracles_ignore_the_padding(deg, M, aa):
    """helpers.run_oracle_raw and aa_oracle.run_oracle (activated and raw inputs): the padding of shs / _features_rest gets zero
    gradient, everything else is bit-identical."""
    s, i, g = _case(deg)
    raw = TS.raw_of(i, seed=deg)
    raw_p = pad_raw(raw, M)
    assert raw_p["features_rest"].shape == (len(i["means3D"]), M - 1, 3)
    if aa:
        runs = [(lambda x, d: aa_oracle.run_oracle(s, x, g, dtype=d, raw=True), raw, raw_p),
                (lambda x, d: aa_oracle.run_oracle(s, x, g, dtype=d), i, dict(i, shs=pad_shs(i["shs"], M)))]
    else:
        runs = [(lambda x, d: h.run_oracle_raw(s, x, g) if d is np.float64 else None, raw, raw_p)]
    for run, small, big in runs:
        for dt in (np.float64, np.float32):
            a, b = run(small, dt), run(big, dt)
            if a is None:
                continue
            for k in ("color", "depth", "alpha", "radii", "ambig_px", "ambig_g"):
                _same(b[k], a[k], k)
            for k, v in a["grads"].items():
                w = b["grads"][k]
                if k in ("shs", "features_rest") and v.ndim == 3 and w.shape != v.shape:
                    n = v.shape[1]
                    _same(w[:, :n], v, k)
                    assert not w[:, n:].any(), (k, "padding gradient")
                else:
                    _same(w, v, k)
