"""GPU tests of SURVEY.md §8 row f2: the fused multi-tensor Adam launch (dgr_adam_step) against the reference's optimiser
(golden from torch.optim.Adam as gs_renderer.py:370 builds it, and a CPU torch.optim.Adam run here), and the stage-1 loop
(main.py:182-287, guidance stubbed) in its fused form against the reference's formulation of the same loop."""
import numpy as np
import pytest
import torch

import helpers  # noqa: F401
import test_stage1_cpu as cpu
from dreamgaussian_b200 import stage1

pytestmark = pytest.mark.gpu


def test_fused_adam_reproduces_the_reference_optimiser_state():
    m = cpu._model_from_golden("cuda")
    assert m.fused_adam
    cpu._two_adam_steps(m)
    cpu.check_against(m, "after_adam_", rtol=2e-6, atol=1e-7)


def test_fused_adam_matches_torch_adam_on_odd_shapes_over_several_steps():
    rng = np.random.default_rng(3)
    shapes = dict(xyz=(1237, 3), f_dc=(1237, 1, 3), f_rest=(1237, 15, 3), opacity=(1237, 1), scaling=(1237, 3), rotation=(1237, 4))
    init = {k: rng.normal(0, 1, s).astype(np.float32) for k, s in shapes.items()}
    m = stage1.GaussianModelB200(3)
    m._set({k: torch.tensor(v, device="cuda") for k, v in init.items()})
    m.training_setup()
    ref = {k: torch.nn.Parameter(torch.tensor(v)) for k, v in init.items()}
    opt = torch.optim.Adam([{"params": [ref[k]], "lr": m.lr[k]} for k in stage1.GROUPS], lr=0.0, eps=1e-15)
    for it in range(1, 8):
        lr = m.update_learning_rate(it)
        opt.param_groups[0]["lr"] = lr
        for k in stage1.GROUPS:
            g = (rng.normal(0, 1, shapes[k]) * 10.0 ** rng.integers(-5, 2)).astype(np.float32)
            if it == 4 and k == "f_rest":
                m.p[k].grad = None; ref[k].grad = None          # a group without gradient is skipped by both
                continue
            m.p[k].grad = torch.tensor(g, device="cuda"); ref[k].grad = torch.tensor(g)
        m.optimizer_step(); opt.step()
    for k in stage1.GROUPS:
        want = ref[k].detach().numpy()
        np.testing.assert_allclose(m.p[k].detach().cpu().numpy(), want, rtol=5e-6, atol=1e-7 * np.abs(want).max(), err_msg=k)


def test_stage1_loop_fused_tracks_the_reference_formulation_and_densifies():
    cfg = stage1.Stage1Config(iters=40, num_pts=1500, ref_size=96, density_start_iter=6, densification_interval=6, seed=2)
    a = stage1.Stage1Trainer(cfg, fused=True)
    b = stage1.Stage1Trainer(cfg, fused=False)
    la, lb = [], []
    for i in range(5):                                  # before any densification the two formulations are the same computation
        la.append(float(a.train_step())); lb.append(float(b.train_step()))
    np.testing.assert_allclose(la, lb, rtol=2e-3)
    for k in stage1.GROUPS:
        pa, pb = a.gaussians.p[k].detach(), b.gaussians.p[k].detach()
        if pa.numel() == 0 or k == "rotation":
            # sh_degree 0: _features_rest is [P,0,3].  rotation: the initial Gaussians are isotropic, so the true rotation
            # gradient is zero and Adam (update = lr * m / sqrt(v)) turns the two paths' different round-off into +-lr steps
            continue
        assert float((pa - pb).abs().max()) <= 5e-3 * max(1.0, float(pb.abs().max())), k       # 5 Adam steps of lr <= 0.05
    n0 = a.gaussians.num_points
    losses = a.train(20)                                # runs through densify_and_prune at steps 6, 12, 18, 24
    assert np.isfinite(losses).all() and a.gaussians.num_points != n0
    assert a.gaussians.stats.denom.shape[0] == a.gaussians.num_points
    assert all(t.shape[0] == a.gaussians.num_points for t in a.gaussians.exp_avg.values())
    assert losses[-1] < losses[0]                       # the known-view MSE terms pull the loss down


def _golden_noise():
    noise = torch.tensor(cpu.GOLD["split_noise"])

    class Noise:                                   # sized lazily: the number of split points is known inside
        def to(self, stds):
            return noise[: stds.shape[0]].to(stds)
    return Noise()


def test_densify_compaction_kernels_reproduce_the_reference_methods():
    """dgr_densify_plan / dgr_densify_apply against the output of the reference's own densify_and_prune
    (tests/golden/make_golden_stage1.py: 400 -> 684 points, parameters and both Adam moments), then reset_opacity + one more
    optimiser step against the reference's."""
    m = cpu._model_from_golden("cuda")
    assert m.fused_densify
    cpu._two_adam_steps(m)
    m.stats.xyz_gradient_accum = torch.tensor(cpu.GOLD["stats_xyz_gradient_accum"], device="cuda").reshape(-1)
    m.stats.denom = torch.tensor(cpu.GOLD["stats_denom"], device="cuda").reshape(-1)
    m.stats.max_radii2D = torch.tensor(cpu.GOLD["stats_max_radii2D"], device="cuda").reshape(-1)
    m.densify_and_prune(0.01, min_opacity=0.01, extent=4, max_screen_size=1, noise=_golden_noise())
    assert m.num_points == cpu.GOLD["after_densify_xyz"].shape[0] == 684
    cpu.check_against(m, "after_densify_", rtol=3e-6, atol=1e-7)
    assert not m.stats.xyz_gradient_accum.any() and m.stats.denom.shape[0] == 684
    m.reset_opacity()
    cpu.check_against(m, "after_reset_", rtol=3e-6, atol=1e-7)
    m.update_learning_rate(3)
    for k in stage1.GROUPS:
        m.p[k].grad = torch.tensor(cpu.GOLD["grad3_" + k], device="cuda")
    m.optimizer_step()
    cpu.check_against(m, "after_reset_adam_", rtol=5e-6, atol=1e-7)


@pytest.mark.parametrize("P,deg,screen", [(5000, 0, 1), (30011, 3, 0), (257, 1, 1), (1, 0, 1), (262401, 1, 1)])
def test_densify_compaction_equals_the_tensor_indexing_path(P, deg, screen):
    """Same decisions, same order, same values as the device-agnostic restatement (stage1.py, pinned on the CPU by the
    reference's outputs) on random models, including the no-world-size-prune variant and tiny point counts.  P = 262401 is
    1026 blocks of 256: the one-CTA scan of the per-block counts (1024 threads) carries over into a second pass."""
    rng = np.random.default_rng(P)
    M = (deg + 1) ** 2
    init = dict(xyz=rng.normal(0, 0.3, (P, 3)), f_dc=rng.normal(0, 1, (P, 1, 3)), f_rest=rng.normal(0, 0.1, (P, M - 1, 3)),
                opacity=rng.normal(-1.0, 2.5, (P, 1)), scaling=rng.normal(-3.4, 0.6, (P, 3)), rotation=rng.normal(0, 1, (P, 4)))
    models = []
    for fused in (True, False):
        m = stage1.GaussianModelB200(deg)
        m.fused_adam, m.fused_densify = True, fused
        m._set({k: torch.tensor(v, dtype=torch.float32, device="cuda") for k, v in init.items()})
        m.training_setup()
        for k in stage1.GROUPS:
            m.exp_avg[k] = torch.tensor(rng.normal(0, 1, init[k].shape), dtype=torch.float32, device="cuda")
            m.exp_avg_sq[k] = m.exp_avg[k] ** 2
        models.append(m)
    for k in stage1.GROUPS:
        models[1].exp_avg[k] = models[0].exp_avg[k].clone(); models[1].exp_avg_sq[k] = models[0].exp_avg_sq[k].clone()
    acc = torch.tensor(np.abs(rng.normal(0, 0.02, (P,))).astype(np.float32) * 3, device="cuda")
    den = torch.tensor(rng.integers(0, 4, (P,)).astype(np.float32), device="cuda")
    draws = torch.randn((2 * P, 3), device="cuda")

    class Noise:                                   # both paths read row child * n_selected + rank of the same draws
        def to(self, stds):
            return draws[: stds.shape[0]].to(stds)
    noise = Noise()
    for m in models:
        m.stats.xyz_gradient_accum, m.stats.denom = acc.clone(), den.clone()
        m.densify_and_prune(0.01, min_opacity=0.01, extent=4, max_screen_size=screen, noise=noise)
    a, b = models
    assert a.num_points == b.num_points
    for k in stage1.GROUPS:
        if a.p[k].numel() == 0:
            assert a.p[k].shape == b.p[k].shape
            continue
        scale = max(1.0, float(b.p[k].abs().max()))
        assert float((a.p[k] - b.p[k]).abs().max()) <= 3e-6 * scale, k
        assert torch.equal(a.exp_avg[k], b.exp_avg[k]) and torch.equal(a.exp_avg_sq[k], b.exp_avg_sq[k]), k
