"""MCMC densification on the GPU (include/dgr_mcmc.h, libdgr_mcmc.so): the relocation kernel on the (o, n) grid against the float64
oracle, the refine kernels against GaussianModelB200's torch restatement from the same draws (which tests/test_mcmc_cpu.py holds to
tests/mcmc_oracle.py), the noise kernel against the float64 restatement, and stage-1 runs with densify_strategy="mcmc"."""
import numpy as np
import pytest
import torch

import helpers  # noqa: F401
import mcmc_oracle as O
import test_mcmc_cpu as TC
from dreamgaussian_b200 import stage1

pytestmark = pytest.mark.gpu
DEV = "cuda"
NEAR = 1e-10          # of C_last: above the float64 rounding of a prefix sum over up to 2M rows (2e6 x 2^-53 = 2e-10 at the most)


# ---- helpers shared with the kernel-coverage cells (tests/test_mcmc_kernel_coverage_gpu.py) -----------------------------------------
def check_relocation_grid():
    """dgr_mcmc_relocation on o in GRID_O x n in 1..51 (plus 60 and 400, clamped to 51): o' and s' within 1e-6 relative of float64."""
    oo, nn = np.meshgrid(np.array(TC.GRID_O, np.float32), np.array(list(range(1, O.N_MAX + 1)) + [60, 400], np.int32))
    oo, nn = oo.ravel(), nn.ravel()
    sc = np.exp(np.random.default_rng(5).normal(-3.0, 1.0, (oo.size, 3))).astype(np.float32)
    new_op, new_sc = stage1.mcmc_relocation(torch.tensor(oo, device=DEV), torch.tensor(sc, device=DEV), torch.tensor(nn, device=DEV))
    want_op, factor = O.relocate(oo.astype(np.float64), nn)
    want_sc = sc.astype(np.float64) * factor[:, None]
    got_op, got_sc = new_op.cpu().numpy().astype(np.float64), new_sc.cpu().numpy().astype(np.float64)
    e_op, e_sc = np.abs(got_op - want_op) / want_op, np.abs(got_sc - want_sc) / want_sc
    helpers.report("mcmc relocation grid", rel=dict(opacity=float(e_op.max()), scale=float(e_sc.max())))
    assert e_op.max() <= 1e-6 and e_sc.max() <= 1e-6, (e_op.max(), e_sc.max())


def refine_models(P, cap, seed, all_alive=False):
    """The kernels and the torch restatement (both on the GPU) from the same cloud and draws; returns (fused, torch, counts, oracle)."""
    p, m, v = TC._cloud(P, seed)
    if all_alive:
        p["opacity"] = np.maximum(p["opacity"], np.float32(-4.0))
    rng = np.random.default_rng(seed + 100)
    u, ua = rng.random(P, dtype=np.float32), rng.random(O.add_count(P, cap), dtype=np.float32)
    models, counts = [], []
    for fused in (True, False):
        g = TC._model(p, m, v, device=DEV, fused=fused)
        counts.append(int(g.relocate_and_grow_mcmc(cap, u_relocate=torch.tensor(u, device=DEV), u_add=torch.tensor(ua, device=DEV))))
        models.append(g)
    return models[0], models[1], counts, O.refine(p, m, v, u, ua, cap)


def check_refine(P, cap, seed, all_alive=False):
    """Picks identical, parameters within 2e-6 relative, moments bit-identical, the relocated count that of the oracle; a second run
    is bit-identical.  A draw within rounding of a prefix boundary may go either way (the kernels' fixed-order scan and the
    restatement's cumsum round differently, by about P 2^-53 of C_last): draws within NEAR of one are counted, expected none.
    (1e-6 of C_last is no such bound: at 100k rows the average row holds 1e-5 of it, and a fifth of the draws land that close.)"""
    a, b, (na, nb), want = refine_models(P, cap, seed, all_alive)
    close = int((want[4]["margins"] < NEAR).sum())
    helpers.report("mcmc refine P=%d cap=%d" % (P, cap), draws=dict(n=int(want[4]["margins"].size), near_boundary=close,
                                                                      within_1e6=int((want[4]["margins"] < 1e-6).sum())))
    assert close == 0
    assert na == nb == want[3] and (want[3] == 0) == (all_alive or len(want[4]["dead"]) == 0)
    assert a.num_points == b.num_points == want[0]["xyz"].shape[0] == max(P, min(cap, P * 105 // 100))
    for k in O.GROUPS:
        pa, pb = a.p[k].detach().cpu().numpy(), b.p[k].detach().cpu().numpy()
        np.testing.assert_allclose(pa, pb, rtol=2e-6, atol=1e-7, err_msg=k)
        np.testing.assert_allclose(pa, want[0][k], rtol=2e-6, atol=1e-7, err_msg=k)
        assert torch.equal(a.exp_avg[k], b.exp_avg[k]) and torch.equal(a.exp_avg_sq[k], b.exp_avg_sq[k]), k
        assert np.array_equal(a.exp_avg[k].cpu().numpy(), want[1][k]), k
    again = refine_models(P, cap, seed, all_alive)[0]
    assert all(torch.equal(again.p[k], a.p[k]) for k in O.GROUPS)
    return want


def check_noise(P, seed):
    p, m, v = TC._cloud(P, seed, op_mu=-3.0, op_sd=3.0)
    z = np.random.default_rng(seed + 1).normal(size=(P, 3)).astype(np.float32)
    g = TC._model(p, m, v, device=DEV, fused=True)
    g.inject_noise_mcmc(5000.0, normals=torch.tensor(z, device=DEV))
    upd = O.noise_update(p["opacity"], p["scaling"], p["rotation"], z, 5000.0)
    want = p["xyz"].astype(np.float64) + upd
    got = g.p["xyz"].detach().cpu().numpy().astype(np.float64)
    err = np.abs(got - want)
    tol = 1e-5 * O.noise_bound(p["opacity"], p["scaling"], z, 5000.0) + 2e-7 * np.abs(want) + 1e-30
    helpers.report("mcmc noise P=%d" % P, err=dict(max_over_tol=float((err / tol).max())))
    assert (err <= tol).all()
    opaque = O.opacity(p["opacity"][:, 0]) > 0.9
    assert opaque.sum() > 10 and (np.abs(upd[opaque]) <= 1e-30).all() and np.array_equal(got[opaque], p["xyz"][opaque])
    assert (np.abs(upd[~opaque]).max(axis=1) > 0).sum() > P // 4


# ---- kernels ---------------------------------------------------------------------------------------------------------------------
def test_relocation_kernel_on_the_grid():
    check_relocation_grid()


@pytest.mark.parametrize("P,cap,seed,all_alive", [(1237, 2000, 0, False), (1237, 1237, 1, False), (1237, 100, 2, False),
                                                  (1237, 5000, 3, True), (100_000, 200_000, 4, False), (100_000, 100_000, 5, False)])
def test_refine_kernels_equal_the_torch_restatement(P, cap, seed, all_alive):
    check_refine(P, cap, seed, all_alive)


@pytest.mark.parametrize("P", [1237, 100_003])
def test_noise_kernel_equals_the_float64_restatement(P):
    check_noise(P, 17)


def test_refine_without_host_synchronisation_and_empty_cloud():
    p, m, v = TC._cloud(3001, 6)
    g = TC._model(p, m, v, device=DEV, fused=True)
    torch.cuda.synchronize()
    n = g.relocate_and_grow_mcmc(4000)                        # draws from the default generator; the count stays on the device
    assert n.is_cuda and n.dtype == torch.int32 and g.num_points == 3151
    e = TC._model({k: x[:0] for k, x in p.items()}, {k: x[:0] for k, x in m.items()}, {k: x[:0] for k, x in v.items()}, device=DEV, fused=True)
    assert int(e.relocate_and_grow_mcmc(100)) == 0 and e.num_points == 0
    e.inject_noise_mcmc(1.0)


# ---- stage 1 -------------------------------------------------------------------------------------------------------------------
def _cfg(**kw):
    base = dict(iters=60, num_pts=1500, ref_size=96, density_start_iter=5, densification_interval=5, densify_strategy="mcmc",
                mcmc_cap_max=1700, seed=4)
    base.update(kw)
    return stage1.Stage1Config(**base)


def test_stage1_mcmc_holds_and_reaches_its_cap_and_leaves_no_dead_row():
    cfg = _cfg(num_pts=5000, mcmc_cap_max=5500, density_start_iter=10, densification_interval=10, iters=60)
    tr = stage1.Stage1Trainer(cfg)
    counts = []
    for step in range(1, 61):
        loss = tr.train_step()
        g = tr.gaussians
        assert g.num_points <= cfg.mcmc_cap_max
        if step % 10 == 0:
            o = torch.sigmoid(g._opacity.detach())
            # nothing below the floor right after a refinement (a relocated opacity clamped to it reads back at it, up to the
            # float32 round trip of the logit)
            assert float(o.min()) >= cfg.mcmc_min_opacity * (1 - 1e-5), (step, float(o.min()))
            counts.append(g.num_points)
        assert g.exp_avg["xyz"].shape[0] == g.num_points and g.stats.denom.shape[0] == g.num_points
        assert torch.isfinite(loss)
    assert counts[:3] == [5250, 5500, 5500] and g.num_points == 5500
    assert np.isfinite(torch.stack(tr.losses).cpu().numpy()).all()


def test_stage1_mcmc_fused_tracks_the_torch_restatement():
    cfg = _cfg(density_start_iter=3, densification_interval=3)
    a, b = stage1.Stage1Trainer(cfg), stage1.Stage1Trainer(cfg)
    b.gaussians.fused_densify = False
    la, lb = [], []
    for _ in range(8):                                      # refinements at steps 3 and 6, noise every step
        la.append(float(a.train_step())); lb.append(float(b.train_step()))
        assert a.gaussians.num_points == b.gaussians.num_points
    np.testing.assert_allclose(la, lb, rtol=2e-3)
    assert a.gaussians.num_points > cfg.num_pts


def test_stage1_mcmc_is_bit_reproducible():
    cfg = _cfg(density_start_iter=10, densification_interval=20, mcmc_cap_max=2200, iters=300)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        runs = []
        for _ in range(2):
            tr = stage1.Stage1Trainer(cfg)
            tr.train(300)
            runs.append((tr.gaussians.p, torch.stack(tr.losses)))
    finally:
        torch.use_deterministic_algorithms(prev)
    (pa, la), (pb, lb) = runs
    assert torch.equal(la, lb)
    assert pa["xyz"].shape[0] == 2200
    for k in stage1.GROUPS:
        assert torch.equal(pa[k], pb[k]), k


def test_stage1_mcmc_with_batched_antialiased_renders_and_the_reference_formulation():
    for kw in (dict(batched=True), dict(fused=False)):
        tr = stage1.Stage1Trainer(_cfg(antialiasing=True), **kw)
        losses = tr.train(12)
        assert np.isfinite(losses).all() and 1500 < tr.gaussians.num_points <= 1700


def test_default_strategy_never_calls_the_mcmc_library():
    """The default loop (a densification included) runs without touching libdgr_mcmc.so: any use of it would raise here."""
    from dreamgaussian_b200 import _lib

    class Untouchable:
        def __getattr__(self, name):
            raise AssertionError("the default strategy called libdgr_mcmc.so (%s)" % name)
    tr = stage1.Stage1Trainer(stage1.Stage1Config(iters=40, num_pts=1500, ref_size=96, density_start_iter=4, densification_interval=4))
    lib = _lib.load()
    saved, _lib._mcmc = _lib._mcmc, Untouchable()
    lib.dgr_profile_enable(1)
    try:
        tr.train(5)
        names = {n for n, _ in _lib.profile_collect()}
    finally:
        lib.dgr_profile_enable(0)
        _lib._mcmc = saved
    assert "densify_apply" in names, names                 # the default densification ran
