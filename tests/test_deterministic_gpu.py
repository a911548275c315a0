"""The deterministic backward on the GPU (torch.use_deterministic_algorithms(True)): its gradients pass both oracles, agree with
the default backward up to summation order, and are bit-identical from run to run whatever the scheduling knobs, the record
staging, a stage-2 re-run or the host layer; likewise the batched and mixed-size calls and two seeded stage-1 runs."""
import os
import subprocess
import sys

import numpy as np
import pytest

import helpers as h
import test_variants_gpu as tv
import test_views_gpu as tvw
from dreamgaussian_b200 import rasterizer as R

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


@pytest.fixture
def det():
    """torch.use_deterministic_algorithms(True) for the test; the flag, the tuning and the host layer are restored."""
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)
        h.set_tuning(h.DEFAULT_TUNING)
        R.set_fast_host(True)


def _same(a, b, what):
    for k in b["grads"]:
        assert np.array_equal(a["grads"][k], b["grads"][k]), (what, k, float(np.abs(a["grads"][k] - b["grads"][k]).max()))


def _agree(a, b, what, rtol=2e-5):
    """a, b: gradients of the same forward summed in different orders.  A tensor whose true gradient vanishes by symmetry (the
    rotations of isotropic Gaussians) is judged against the scale of the other gradients, as in helpers.compare."""
    floor = 1e-3 * max(float(np.abs(v).max()) if v.size else 0.0 for v in b["grads"].values())
    for k in b["grads"]:
        x, y = a["grads"][k].astype(np.float64), b["grads"][k].astype(np.float64)
        scale = max(float(np.abs(y).max()) if y.size else 0.0, floor)
        assert np.abs(x - y).max(initial=0.0) <= rtol * scale + 1e-7, (what, k, float(np.abs(x - y).max(initial=0.0)), scale)


PARITY = {
    "seeded_deg3": dict(P=3000, res=96, deg=3, seed=1),
    "opacity_0.1": dict(P=5000, res=128, deg=0, opacity="init", anisotropic=False, seed=2),
}


def _parity_case(name):
    if name in tv.CASES:
        s, i, g, refs, _ = tv._case(name)
        return s, i, g, refs
    s, i = h.make_case(**PARITY[name])
    g = h.upstream_grads(s["image_height"], s["image_width"])
    return s, i, g, h.oracles(s, i, g)


@pytest.mark.parametrize("name", list(PARITY) + ["big_tiles", "precomputed_colour_cov3D", "edges_37x23_deg2"])
def test_deterministic_gradients_pass_both_oracles_and_agree_with_the_default_backward(det, name):
    s, i, g, refs = _parity_case(name)
    cu = h.both_oracles("det " + name, s, i, g, refs=refs)
    torch.use_deterministic_algorithms(False)
    base = h.run_cuda(s, i, g)
    torch.use_deterministic_algorithms(True)
    _agree(cu, base, name)


def test_equal_depths_match_the_oracle(det):
    """All Gaussians at one view depth (the sort falls back to the Gaussian index): the rule of
    test_parity_gpu.py::test_equal_depths_resolve_by_index_like_the_reference, under the flag, and bit-identical twice."""
    s, i = h.make_case(P=3000, res=64, deg=1, sigma=0.03)
    i["means3D"] = i["means3D"].copy(); i["means3D"][:, 2] = 0.0
    g = h.upstream_grads(64, 64)
    ref = h.run_oracle(s, i, g)
    cu = h.run_cuda(s, i, g)
    for k in ("color", "depth", "alpha"):
        assert np.abs(cu[k] - ref[k]).max() < 1e-4, k
    assert (cu["radii"] == ref["radii"]).all()
    for k, v in ref["grads"].items():
        if k in cu["grads"]:
            assert np.abs(cu["grads"][k].reshape(v.shape) - v).max() <= 2e-3 * max(np.abs(v).max(), 1e-6), k
    _same(h.run_cuda(s, i, g), cu, "equal depths")


def _profiled_backward_kernels(fast, views):
    """Kernel names of one forward + backward driven on this thread (the library's events are per host thread)."""
    from dreamgaussian_b200 import _lib
    s, i = h.make_case(P=2000, res=64, deg=1, seed=13)
    rs = tvw._rs(s)
    t = {k: torch.tensor(v, device="cuda") for k, v in i.items()}
    P = 2000
    e = lambda *shape: torch.empty(shape, device="cuda")
    gC, gA = torch.randn((3, 64, 64), device="cuda"), torch.randn((1, 64, 64), device="cuda")
    R.set_fast_host(fast)
    lib = _lib.load()
    lib.dgr_profile_enable(1)
    try:
        if views:
            st = R.views_forward_impl([rs, rs], t["means3D"], t["shs"], t["opacities"], t["scales"], t["rotations"])[4]
            R.views_backward_impl(st, torch.stack([gC, gC]), None, torch.stack([gA, gA]), e(P, 3), e(2, P, 3), e(P, 4, 3), e(P, 1),
                                  e(P, 3), e(P, 4))
        else:
            st = R.forward_impl(rs, t["means3D"], t["shs"], None, t["opacities"], t["scales"], t["rotations"], None)[4]
            R.backward_impl(st, gC, None, gA, e(P, 3), e(P, 3), e(P, 4, 3), None, e(P, 1), e(P, 3), e(P, 4), None)
        torch.cuda.synchronize()
        return [n for n, _ in _lib.profile_collect()]
    finally:
        lib.dgr_profile_enable(0)
        R.set_fast_host(True)


@pytest.mark.parametrize("views", [False, True])
@pytest.mark.parametrize("fast", [True, False])
def test_the_flag_selects_the_deterministic_kernels_in_both_host_layers(fast, views):
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        for flag in (False, True):
            torch.use_deterministic_algorithms(flag)
            names = _profiled_backward_kernels(fast, views)
            bwd = "render_views_bwd" if views else "render_bwd"
            if flag:
                assert bwd + "_det" in names and "det_moments_gather" in names and bwd not in names, names
            else:
                assert bwd in names and not [n for n in names if "det" in n], names
    finally:
        torch.use_deterministic_algorithms(prev)


def test_an_instance_count_below_the_forwards_is_refused_in_debug_mode_and_never_silent(det):
    """`instances` is the caller's word: with debug set it is checked against the forward's own count; without, a count that
    is too small leaves NaN rows instead of quietly dropping moments."""
    s, i = h.make_case(P=2000, res=64, deg=1, seed=14)
    t = {k: torch.tensor(v, device="cuda") for k, v in i.items()}
    e = lambda *shape: torch.zeros(shape, device="cuda")
    gC, gA = torch.randn((3, 64, 64), device="cuda"), torch.randn((1, 64, 64), device="cuda")
    for debug in (False, True):
        rs = tvw._rs(s)._replace(debug=debug)
        for fast in (True, False):
            R.set_fast_host(fast)
            st = R.forward_impl(rs, t["means3D"], t["shs"], None, t["opacities"], t["scales"], t["rotations"], None)[4]
            n = st.num_rendered
            assert n > 100
            if fast:
                continue                              # the compiled layer always passes its own count
            st.num_rendered = n // 2
            d = [e(2000, 3), e(2000, 3), e(2000, 4, 3), None, e(2000, 1), e(2000, 3), e(2000, 4), None]
            if debug:
                with pytest.raises(RuntimeError, match="instances differs"):
                    R.backward_impl(st, gC, None, gA, *d)
            else:
                R.backward_impl(st, gC, None, gA, *d)
                assert torch.isnan(d[0]).any()
    R.set_fast_host(True)


@pytest.mark.parametrize("name", ["saturated", "dark_deg3", "needles", "faint", "trained_mix"])
def test_trained_regime_scenes_pass_both_oracles(det, name):
    import test_trained_regimes_gpu as tr
    s, i, g, refs = tr._case(name)
    h.both_oracles("det trained/" + name, s, i, g, max_ambig_frac=tr.CASES[name][1], refs=refs)


SCHEDULES = {
    "default": (1, 1, 1), "no_cost_order": (1, 1, 1 | 1 << 21), "two_ended": (1, 1, 1 | 1 << 20), "ctas_1": (1, 1, 1 | 1 << 16),
    "pdl_off": (1, 1, 1 | 1 << 3), "ppl_bwd_2": (1, 2, 1), "u_1": (1, 1, 1 | 1 << 8), "u_2": (1, 1, 1 | 2 << 8),
    "sorted_copy": (1, 1, 1 | 1 << 22), "by_id": (1, 1, 1 | 2 << 22),
}


def test_gradients_are_bit_identical_over_runs_knobs_staging_and_host_layers(det):
    s, i = h.make_case(P=20000, res=400, deg=3, seed=7)
    g = h.upstream_grads(s["image_height"], s["image_width"])
    first = h.run_tuned(h.DEFAULT_TUNING, lambda: h.run_cuda(s, i, g))
    for _ in range(2):
        _same(h.run_cuda(s, i, g), first, "repeat")
    for name, word in SCHEDULES.items():
        for fast in (True, False):
            _same(h.run_tuned(word, lambda: h.run_cuda(s, i, g), fast_host=fast), first, (name, fast))


def test_bit_identical_after_a_stage2_rerun(det):
    s, i = h.make_case(P=8000, res=128, deg=1, seed=9)
    g = h.upstream_grads(s["image_height"], s["image_width"])
    first = h.run_cuda(s, i, g)
    P, H, W = 8000, 128, 128
    for fast in (True, False):
        R.set_fast_host(fast)
        old = R.get_capacity_hint(0, P, H, W)
        R.set_capacity_hint(0, P, H, W, 64, False)               # far too small: stage 2 runs again with the real count
        try:
            _same(h.run_cuda(s, i, g), first, ("rerun", fast))
        finally:
            R.set_capacity_hint(0, P, H, W, *(old or (max(65536, 16 * P), True)))
    R.set_fast_host(True)


def test_fused_raw_path_with_densification_statistics_is_bit_identical(det):
    from dreamgaussian_b200.fused import DensifyStats
    s, i = h.make_case(P=3000, res=96, deg=3, seed=11)
    rng = np.random.default_rng(0)
    raw = dict(xyz=i["means3D"], features_dc=i["shs"][:, :1], features_rest=i["shs"][:, 1:],
               opacity=np.log(i["opacities"] / (1 - i["opacities"])).astype(np.float32), scaling=np.log(i["scales"]).astype(np.float32),
               rotation=i["rotations"] + 0.01 * rng.normal(size=i["rotations"].shape).astype(np.float32))
    g = h.upstream_grads(s["image_height"], s["image_width"])
    ref = h.run_oracle_raw(s, raw, g)
    outs = []
    for fast in (True, False, True):
        R.set_fast_host(fast)
        st = DensifyStats(3000, "cuda")
        cu = h.run_cuda_raw(s, raw, g, stats=st)
        cu["grads"].update(accum=st.xyz_gradient_accum.cpu().numpy(), denom=st.denom.cpu().numpy(), maxr=st.max_radii2D.cpu().numpy())
        outs.append(cu)
    R.set_fast_host(True)
    ok, rep = h.compare(outs[0], ref)
    h.report("det fused raw", vs_f64=rep)
    assert ok, rep
    for o in outs[1:]:
        _same(o, outs[0], "fused raw + stats")


def test_batched_calls_are_bit_identical(det):
    W, H = 96, 72
    cam = (10.0, 30.0, 49.1, (0.3, 0.3, 0.3))
    settings, inputs = tvw._cams(3000, W, H, 3, [cam] * 5, seed=3)
    g = h.upstream_grads(H, W, seed=5)
    a = tvw.run_views(settings, inputs, [g] * 5)
    m2d = a["grads"]["means2D"]
    for v in range(1, 5):                                # five identical cameras: five identical per-view means2D gradients
        assert np.array_equal(m2d[v], m2d[0]), v
    _same(tvw.run_views(settings, inputs, [g] * 5), a, "views repeat")
    R.set_fast_host(False)
    _same(tvw.run_views(settings, inputs, [g] * 5), a, "views ctypes")
    R.set_fast_host(True)


def test_mixed_size_calls_are_bit_identical(det):
    from dreamgaussian_b200.rasterizer import rasterize_views_mixed
    sizes = [(72, 96), (40, 130), (64, 64)]
    outs = []
    for fast in (True, True, False):
        R.set_fast_host(fast)
        settings = []
        for k, (Hh, Ww) in enumerate(sizes):
            s, _ = tvw._cams(10, Ww, Hh, 2, [(5.0 * k, 60.0 * k, 45.0, (0.1, 0.2, 0.3))])
            settings += s
        _, inputs = tvw._cams(4000, 96, 72, 2, [(0.0, 0.0, 45.0, (0, 0, 0))], seed=6)
        t = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda")
        tin = {k: t(v).requires_grad_(True) for k, v in inputs.items()}
        means2D = torch.zeros((3, 4000, 3), device="cuda", requires_grad=True)
        color, radii, depth, alpha = rasterize_views_mixed([tvw._rs(x) for x in settings], tin["means3D"], means2D, tin["opacities"],
                                                           tin["shs"], tin["scales"], tin["rotations"])
        gen = torch.Generator(device="cuda").manual_seed(1)
        loss = 0.0
        for c, d, a in zip(color, depth, alpha):          # per-view lists
            loss = loss + (c * torch.randn(c.shape, device="cuda", generator=gen)).sum() + a.sum() + d.sum()
        loss.backward()
        outs.append(dict(grads={k: v.grad.cpu().numpy() for k, v in tin.items()} | dict(means2D=means2D.grad.cpu().numpy())))
    R.set_fast_host(True)
    for o in outs[1:]:
        _same(o, outs[0], "mixed")


STAGE1 = r"""
import sys, numpy as np, torch
torch.use_deterministic_algorithms(True)
from dreamgaussian_b200 import stage1
cfg = stage1.Stage1Config(iters=200, num_pts=1500, ref_size=96, density_start_iter=100, densification_interval=100, seed=3)
t = stage1.Stage1Trainer(cfg, fused=sys.argv[2] == "fused")
t.train(200)
m = t.gaussians
out = {"n": np.array([m.num_points]), "losses": np.array([float(x) for x in t.losses])}
for k in stage1.GROUPS:
    out["p_" + k] = m.p[k].detach().cpu().numpy()
    out["m_" + k] = m.exp_avg[k].cpu().numpy()
    out["v_" + k] = m.exp_avg_sq[k].cpu().numpy()
np.savez(sys.argv[1], **out)
"""


@pytest.mark.parametrize("arm", ["fused", "reference"])
def test_two_seeded_stage1_runs_end_bit_identical(tmp_path, arm):
    """Two Stage1Trainer runs from one seed (200 iterations, densification at steps 100 and 200), each in its own process under
    torch.use_deterministic_algorithms(True): every parameter, Adam moment, loss and the point count are bit-identical."""
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8", PYTHONPATH=h.ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    res = []
    for k in range(2):
        path = str(tmp_path / ("run%d.npz" % k))
        p = subprocess.run([sys.executable, "-c", STAGE1, path, arm], env=env, cwd=h.ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                           text=True, timeout=1200)
        assert p.returncode == 0, p.stdout[-4000:]
        res.append(dict(np.load(path)))
    assert int(res[0]["n"][0]) != 1500                     # the densifications did change the cloud
    for k in res[0]:
        assert np.array_equal(res[0][k], res[1][k]), (arm, k)
