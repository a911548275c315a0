"""SURVEY.md §8 row f2: the stage-1 optimisation loop around the rasterizer (BASELINE.json configs[3]) — GaussianModel's
optimiser plumbing restated B200-first.

Reference: /root/reference/gs_renderer.py:25-47 (LR schedule), :331-382 (create_from_pcd, training_setup,
update_learning_rate), :464-622 (optimizer-state surgery, densify_and_clone / _split / _prune, prune),
main.py:182-287 (train_step).  What changes:
  * the six parameter tensors are stepped by ONE fused Adam launch (dgr_adam_step) instead of torch.optim.Adam's
    six groups x ~6 element-wise kernels; Adam state lives in plain tensors, so the reference's optimizer-state surgery
    (replace / prune / cat on `optimizer.state`) becomes ordinary tensor indexing;
  * rendering goes through FusedGaussianRasterizer (row f1): activations, SH dc/rest split and the three densification
    statistics happen inside the per-Gaussian kernels;
  * initial scales come from this library's distCUDA2 (row f3).
The densification exists twice: as device-agnostic tensor logic (tests/test_stage1_cpu.py runs it on the CPU against outputs
of the reference's own methods) and as stream-compaction kernels (dgr_densify_plan / dgr_densify_apply, csrc/dgr_densify.cuh)
that the CUDA loop uses and tests/test_stage1_gpu.py pins against the same reference outputs."""
import ctypes
import math
from typing import NamedTuple, Optional

import numpy as np
import torch

from . import _lib
from .fused import DensifyStats, FusedGaussianRasterizer
from .rasterizer import GaussianRasterizationSettings

SH_C0 = 0.28209479177387814


def get_expon_lr_func(lr_init, lr_final, lr_delay_steps=0, lr_delay_mult=1.0, max_steps=1000000):
    """gs_renderer.py:25-47: log-linear decay from lr_init to lr_final with an optional sine warm-up."""
    def helper(step):
        if lr_init == lr_final:
            return lr_init
        if step < 0 or (lr_init == 0.0 and lr_final == 0.0):
            return 0.0
        if lr_delay_steps > 0:
            delay_rate = lr_delay_mult + (1 - lr_delay_mult) * math.sin(0.5 * math.pi * min(max(step / lr_delay_steps, 0.0), 1.0))
        else:
            delay_rate = 1.0
        t = min(max(step / max_steps, 0.0), 1.0)
        return delay_rate * math.exp(math.log(lr_init) * (1 - t) + math.log(lr_final) * t)
    return helper


class OptimConfig(NamedTuple):
    """configs/image.yaml:60-80"""
    position_lr_init: float = 0.001
    position_lr_final: float = 0.00002
    position_lr_delay_mult: float = 0.02
    position_lr_max_steps: int = 500
    feature_lr: float = 0.01
    opacity_lr: float = 0.05
    scaling_lr: float = 0.005
    rotation_lr: float = 0.005
    percent_dense: float = 0.01


GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")

# MCMC densification: include/dgr_constants.h DGR_MCMC_* (tests/test_mcmc_cpu.py holds the two equal)
MCMC_N_MAX = 51
MCMC_MIN_OPACITY = 0.005
MCMC_OPACITY_MAX = 1.0 - 2.0 ** -23
MCMC_GROW_PERCENT = 105
MCMC_NOISE_K, MCMC_NOISE_X0 = 100.0, 0.995
MCMC_NOISE_LR = 5e5
MCMC_OPACITY_REG = MCMC_SCALE_REG = 0.01


def mcmc_add_count(P, cap_max):
    """Rows one MCMC refinement appends: max(0, min(cap_max, floor(1.05 P)) - P)."""
    return max(0, min(int(cap_max), P * MCMC_GROW_PERCENT // 100) - P)


def mcmc_relocation(opacity, scale, ratio):
    """The relocation formula alone on activated values (gsplat's `relocation` op), one launch of dgr_mcmc_relocation (float64
    inside): n = ratio clamped to [1, 51], o' = 1 - (1 - o)^(1/n), s' = s o / D with D = sum_{m=1..n} C(n,m) (-1)^(m-1) o'^m / sqrt(m)
    (1 where D = 0); no clamp.  opacity [K] (or [K,1]), scale [K,3] float32 and ratio [K] integer CUDA tensors -> (o' shaped like
    opacity, s' [K,3])."""
    if not (opacity.is_cuda and scale.is_cuda and ratio.is_cuda):
        raise ValueError("mcmc_relocation: CUDA tensors expected (the formula runs in dgr_mcmc_relocation)")
    K = opacity.numel()
    if tuple(scale.shape) != (K, 3) or ratio.numel() != K:
        raise ValueError("mcmc_relocation: opacity [K], scale [K,3], ratio [K]")
    op = opacity.detach().float().contiguous()
    sc = scale.detach().float().contiguous()
    r = ratio.to(torch.int32).contiguous()
    new_op, new_sc = torch.empty_like(op), torch.empty_like(sc)
    lib = _lib.load_mcmc()
    with torch.cuda.device(op.device):
        st = ctypes.c_void_p(torch.cuda.current_stream(op.device).cuda_stream)
        _lib.check_mcmc(lib.dgr_mcmc_relocation(K, op.data_ptr(), sc.data_ptr(), r.data_ptr(), new_op.data_ptr(), new_sc.data_ptr(), st))
    return new_op, new_sc


def _mcmc_relocate(o, n):
    """(o', o / D) in float64, the operation order of csrc/dgr_mcmc.cuh::mcmc_relocate (terms past m = n are +-0)."""
    o_new = -torch.expm1(torch.log1p(-o) / n)
    c, p, D = torch.ones_like(o), torch.ones_like(o), torch.zeros_like(o)
    nd = n.double()
    for m in range(1, MCMC_N_MAX + 1):
        c = c * (nd - m + 1) / m
        p = p * o_new
        t = c * p / math.sqrt(m)
        D = D + t if m & 1 else D - t
    return o_new, torch.where(D > 0, o / D, torch.ones_like(o))


def _mcmc_opacity(raw):
    """sigmoid in float64 rounded once to float32: the weights the kernels compute."""
    return torch.sigmoid(raw.double()).float()


def _mcmc_update(op_raw, sc_raw, picks, min_opacity):
    """Raw opacity / scaling of rows picked `picks` times: logit(clamp(o', min_opacity, 1 - 2^-23)), scaling + log(o / D)."""
    o = _mcmc_opacity(op_raw).double()
    o_new, factor = _mcmc_relocate(o, (picks.to(torch.int64) + 1).clamp(max=MCMC_N_MAX))
    oc = o_new.clamp(min_opacity, MCMC_OPACITY_MAX)
    return torch.log(oc / (1 - oc)).float(), (sc_raw.double() + torch.log(factor)[:, None]).float()


def build_rotation(r):
    """gs_renderer.py:85-107 (normalises the quaternion)."""
    q = r / torch.sqrt((r * r).sum(dim=1, keepdim=True))
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                        2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                        2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], dim=1).reshape(-1, 3, 3)


class GaussianModelB200:
    """The reference GaussianModel's training state: raw parameters (same attribute names), Adam moments, statistics."""

    def __init__(self, sh_degree: int):
        self.max_sh_degree = sh_degree
        self.active_sh_degree = sh_degree          # main.py:147: no progressive SH
        self.p = {}                                # name -> leaf tensor (requires_grad)
        self.exp_avg, self.exp_avg_sq = {}, {}
        self.lr = {}
        self.steps = {k: 0 for k in GROUPS}          # torch.optim.Adam keeps state['step'] per tensor
        self.stats: Optional[DensifyStats] = None
        self.absgrad = False                       # keep AbsGS's statistic too (DensifyStats.xyz_gradient_accum_abs)
        self.percent_dense = 0.01
        self.spatial_lr_scale = 1.0
        self.betas, self.eps = (0.9, 0.999), 1e-15
        self.fused_adam = True

    # reference attribute names (gs_renderer.py:140-160) so that fused.render_gaussian_model / fields work on this object
    _xyz = property(lambda s: s.p["xyz"]); _features_dc = property(lambda s: s.p["f_dc"]); _features_rest = property(lambda s: s.p["f_rest"])
    _opacity = property(lambda s: s.p["opacity"]); _scaling = property(lambda s: s.p["scaling"]); _rotation = property(lambda s: s.p["rotation"])

    @property
    def num_points(self):
        return self.p["xyz"].shape[0]

    def create_from_points(self, points, colors, spatial_lr_scale=1.0, device="cuda"):
        """gs_renderer.py:331-354 (colors in [0,1], SH dc = RGB2SH; scales from the 3-NN mean squared distance)."""
        from .knn import distCUDA2
        self.spatial_lr_scale = spatial_lr_scale
        xyz = torch.tensor(np.asarray(points), dtype=torch.float32, device=device)
        rgb = torch.tensor(np.asarray(colors), dtype=torch.float32, device=device)
        M = (self.max_sh_degree + 1) ** 2
        dist2 = torch.clamp_min(distCUDA2(xyz), 0.0000001)
        self._set(dict(xyz=xyz, f_dc=((rgb - 0.5) / SH_C0).reshape(-1, 1, 3).contiguous(),
                       f_rest=torch.zeros((xyz.shape[0], M - 1, 3), device=device),
                       opacity=torch.full((xyz.shape[0], 1), math.log(0.1 / 0.9), device=device),
                       scaling=torch.log(torch.sqrt(dist2))[..., None].repeat(1, 3),
                       rotation=torch.tensor([[1.0, 0, 0, 0]], device=device).repeat(xyz.shape[0], 1)))

    def _set(self, tensors):
        self.p = {k: tensors[k].detach().float().contiguous().requires_grad_(True) for k in GROUPS}

    def training_setup(self, cfg: OptimConfig = OptimConfig()):
        """gs_renderer.py:356-374"""
        self.percent_dense = cfg.percent_dense
        self._reset_stats()
        s = self.spatial_lr_scale
        self.lr = dict(xyz=cfg.position_lr_init * s, f_dc=cfg.feature_lr, f_rest=cfg.feature_lr / 20.0, opacity=cfg.opacity_lr,
                       scaling=cfg.scaling_lr, rotation=cfg.rotation_lr)
        self.exp_avg = {k: torch.zeros_like(v) for k, v in self.p.items()}
        self.exp_avg_sq = {k: torch.zeros_like(v) for k, v in self.p.items()}
        self.steps = {k: 0 for k in GROUPS}
        self.xyz_scheduler = get_expon_lr_func(cfg.position_lr_init * s, cfg.position_lr_final * s, lr_delay_mult=cfg.position_lr_delay_mult,
                                               max_steps=cfg.position_lr_max_steps)

    def _reset_stats(self):
        self.stats = DensifyStats(self.num_points, self.p["xyz"].device, absgrad=self.absgrad)

    def update_learning_rate(self, iteration):
        self.lr["xyz"] = self.xyz_scheduler(iteration)
        return self.lr["xyz"]

    def zero_grad(self):
        for v in self.p.values():
            v.grad = None

    def optimizer_step(self):
        """torch.optim.Adam.step() of the reference (main.py:275) as one launch; a group whose .grad is None is skipped,
        as torch does."""
        names = [k for k in GROUPS if self.p[k].grad is not None]
        for k in names:
            self.steps[k] += 1
        names = [k for k in names if self.p[k].numel() > 0]
        if not names:
            return
        if not self.fused_adam or not self.p["xyz"].is_cuda:
            return self._adam_torch(names)
        lib = _lib.load()
        arr = (_lib.DgrAdamGroup * len(names))()
        keep = []
        for i, k in enumerate(names):
            g = self.p[k].grad.contiguous(); keep.append(g)
            arr[i] = _lib.DgrAdamGroup(self.p[k].data_ptr(), g.data_ptr(), self.exp_avg[k].data_ptr(), self.exp_avg_sq[k].data_ptr(),
                                       self.p[k].numel(), self.lr[k], self.steps[k])
        dev = self.p["xyz"].device
        with torch.cuda.device(dev):
            st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            _lib.check(lib.dgr_adam_step(arr, len(names), self.betas[0], self.betas[1], self.eps, st))

    def _adam_torch(self, names):
        """The same update with torch ops (device-agnostic; used by the CPU tests of the host logic)."""
        b1, b2 = self.betas
        with torch.no_grad():
            for k in names:
                bc1, bc2 = 1 - b1 ** self.steps[k], 1 - b2 ** self.steps[k]
                g = self.p[k].grad
                self.exp_avg[k].lerp_(g, 1 - b1)
                self.exp_avg_sq[k].mul_(b2).addcmul_(g, g, value=1 - b2)
                denom = (self.exp_avg_sq[k].sqrt() / math.sqrt(bc2)).add_(self.eps)
                self.p[k].addcdiv_(self.exp_avg[k], denom, value=-self.lr[k] / bc1)

    # ---- densification (gs_renderer.py:464-622): optimizer-state surgery == tensor indexing here
    def _select(self, mask):
        with torch.no_grad():
            self.p = {k: v[mask].detach().contiguous().requires_grad_(True) for k, v in self.p.items()}
            self.exp_avg = {k: v[mask].contiguous() for k, v in self.exp_avg.items()}
            self.exp_avg_sq = {k: v[mask].contiguous() for k, v in self.exp_avg_sq.items()}
            st = self.stats
            st.xyz_gradient_accum, st.denom, st.max_radii2D = st.xyz_gradient_accum[mask], st.denom[mask], st.max_radii2D[mask]
            if st.xyz_gradient_accum_abs is not None:
                st.xyz_gradient_accum_abs = st.xyz_gradient_accum_abs[mask]

    def _append(self, new):
        """densification_postfix + cat_tensors_to_optimizer (:515-552): new points get zero Adam moments, stats reset."""
        with torch.no_grad():
            self.p = {k: torch.cat((self.p[k].detach(), new[k]), dim=0).contiguous().requires_grad_(True) for k in GROUPS}
            self.exp_avg = {k: torch.cat((v, torch.zeros_like(new[k])), dim=0) for k, v in self.exp_avg.items()}
            self.exp_avg_sq = {k: torch.cat((v, torch.zeros_like(new[k])), dim=0) for k, v in self.exp_avg_sq.items()}
        self._reset_stats()

    def prune_points(self, mask):
        self._select(~mask)

    def densify_and_clone(self, grads, grad_threshold, scene_extent):
        with torch.no_grad():
            sel = (grads >= grad_threshold) & (torch.exp(self.p["scaling"]).max(dim=1).values <= self.percent_dense * scene_extent)
            self._append({k: self.p[k].detach()[sel] for k in GROUPS})

    def densify_and_split(self, grads, grad_threshold, scene_extent, N=2, noise=None):
        """:555-580.  noise: optional standard-normal [N * n_selected, 3] (tests pass the reference's draws)."""
        with torch.no_grad():
            n_init = self.num_points
            padded = torch.zeros((n_init,), device=grads.device)
            padded[:grads.shape[0]] = grads
            scaling = torch.exp(self.p["scaling"].detach())
            sel = (padded >= grad_threshold) & (scaling.max(dim=1).values > self.percent_dense * scene_extent)
            stds = scaling[sel].repeat(N, 1)
            if noise is None:
                noise = torch.randn(stds.shape, device=stds.device, generator=getattr(self, "noise_gen", None))
            samples = noise.to(stds) * stds
            rots = build_rotation(self.p["rotation"].detach()[sel]).repeat(N, 1, 1)
            new = dict(xyz=torch.bmm(rots, samples.unsqueeze(-1)).squeeze(-1) + self.p["xyz"].detach()[sel].repeat(N, 1),
                       scaling=torch.log(scaling[sel].repeat(N, 1) / (0.8 * N)),
                       rotation=self.p["rotation"].detach()[sel].repeat(N, 1),
                       f_dc=self.p["f_dc"].detach()[sel].repeat(N, 1, 1), f_rest=self.p["f_rest"].detach()[sel].repeat(N, 1, 1),
                       opacity=self.p["opacity"].detach()[sel].repeat(N, 1))
            n_new = new["xyz"].shape[0]
            self._append(new)
            self.prune_points(torch.cat((sel, torch.zeros((n_new,), dtype=torch.bool, device=sel.device))))

    def _prune_mask(self, min_opacity, extent, max_screen_size):
        m = (torch.sigmoid(self.p["opacity"].detach()) < min_opacity).squeeze(1)
        if max_screen_size:
            m = m | (self.stats.max_radii2D > max_screen_size) | (torch.exp(self.p["scaling"].detach()).max(dim=1).values > 0.1 * extent)
        return m

    def _densify_fused(self, max_grad, min_opacity, extent, max_screen_size, noise=None, max_abs_grad=None):
        """densify_and_prune as two launches of compaction kernels (csrc/dgr_densify.cuh: classify + block scan, then ONE pass
        that writes the six parameter tensors and both Adam moments in the reference's final order) with one host read-back
        of the new point count between them — instead of ~30 boolean-mask indexing / torch.cat calls.  max_abs_grad: split by
        the absolute-gradient statistic (dgr_densify_plan_ex)."""
        lib = _lib.load()
        P, dev = self.num_points, self.p["xyz"].device
        with torch.no_grad(), torch.cuda.device(dev):
            st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            scratch = torch.empty((lib.dgr_densify_scratch_bytes(P),), dtype=torch.uint8, device=dev)
            if getattr(self, "_counts_host", None) is None:
                self._counts_host = torch.zeros((4,), dtype=torch.int32).pin_memory()
            acc, den = self.stats.xyz_gradient_accum.contiguous(), self.stats.denom.contiguous()
            if max_abs_grad is None:
                _lib.check(lib.dgr_densify_plan(P, acc.data_ptr(), den.data_ptr(), self.p["opacity"].data_ptr(), self.p["scaling"].data_ptr(),
                                                float(max_grad), float(self.percent_dense * extent), float(min_opacity), float(0.1 * extent),
                                                1 if max_screen_size else 0, scratch.data_ptr(), self._counts_host.data_ptr(), st))
            else:
                acc_abs = self.stats.xyz_gradient_accum_abs.contiguous()
                _lib.check(lib.dgr_densify_plan_ex(P, acc.data_ptr(), acc_abs.data_ptr(), den.data_ptr(), self.p["opacity"].data_ptr(),
                                                   self.p["scaling"].data_ptr(), float(max_grad), float(max_abs_grad),
                                                   float(self.percent_dense * extent), float(min_opacity), float(0.1 * extent),
                                                   1 if max_screen_size else 0, scratch.data_ptr(), self._counts_host.data_ptr(), st))
            torch.cuda.current_stream(dev).synchronize()
            n_keep, n_clone, n_sel, n_child = (int(x) for x in self._counts_host)
            n_out = n_keep + n_clone + 2 * n_child
            if noise is None:
                noise = torch.randn((max(2 * n_sel, 1), 3), device=dev, generator=getattr(self, "noise_gen", None))
            else:                                   # tests hand over the reference's draws: row = child * n_selected + rank
                noise = noise.to(torch.empty((2 * n_sel, 3), device=dev)) if hasattr(noise, "to") else noise
            noise = noise.contiguous().float()
            t = _lib.DgrDensifyTensors()
            new_p, new_m, new_v, keep = {}, {}, {}, [noise, scratch]
            for i, k in enumerate(GROUPS):
                src = self.p[k].detach()
                w = int(src[0].numel()) if src.shape[0] else int(np.prod(src.shape[1:]))
                new_p[k] = torch.empty((n_out,) + tuple(src.shape[1:]), dtype=torch.float32, device=dev)
                new_m[k], new_v[k] = torch.empty_like(new_p[k]), torch.empty_like(new_p[k])
                t.inp[i], t.exp_avg_in[i], t.exp_avg_sq_in[i] = src.data_ptr(), self.exp_avg[k].data_ptr(), self.exp_avg_sq[k].data_ptr()
                t.out[i], t.exp_avg_out[i], t.exp_avg_sq_out[i] = new_p[k].data_ptr(), new_m[k].data_ptr(), new_v[k].data_ptr()
                t.width[i] = w
            _lib.check(lib.dgr_densify_apply(P, ctypes.byref(t), noise.data_ptr(), scratch.data_ptr(), st))
            self.p = {k: v.requires_grad_(True) for k, v in new_p.items()}
            self.exp_avg, self.exp_avg_sq = new_m, new_v
        self._reset_stats()

    def densify_and_prune(self, max_grad, min_opacity, extent, max_screen_size, noise=None, max_abs_grad=None):
        """max_abs_grad (needs stats with xyz_gradient_accum_abs): AbsGS's rule (Ye et al., 2024) — clone by the default statistic,
        split by the absolute one (xyz_gradient_accum_abs / denom >= max_abs_grad)."""
        if max_abs_grad is not None and self.stats.xyz_gradient_accum_abs is None:
            raise ValueError("densify_and_prune: max_abs_grad needs the absolute-gradient statistic (GaussianModelB200.absgrad = True)")
        if getattr(self, "fused_densify", False) and self.p["xyz"].is_cuda and self.num_points > 0:
            return self._densify_fused(max_grad, min_opacity, extent, max_screen_size, noise=noise, max_abs_grad=max_abs_grad)
        with torch.no_grad():
            grads = self.stats.xyz_gradient_accum / self.stats.denom
            grads[grads.isnan()] = 0.0
            if max_abs_grad is not None:
                grads_abs = self.stats.xyz_gradient_accum_abs / self.stats.denom
                grads_abs[grads_abs.isnan()] = 0.0
        self.densify_and_clone(grads, max_grad, extent)
        if max_abs_grad is None:
            self.densify_and_split(grads, max_grad, extent, noise=noise)
        else:
            self.densify_and_split(grads_abs, max_abs_grad, extent, noise=noise)
        self.prune_points(self._prune_mask(min_opacity, extent, max_screen_size))

    def prune(self, min_opacity, extent, max_screen_size):
        self.prune_points(self._prune_mask(min_opacity, extent, max_screen_size))

    # ---- MCMC densification (Kheradmand et al., NeurIPS 2024): relocate dead rows, grow to a cap, position noise
    def relocate_and_grow_mcmc(self, cap_max, min_opacity=MCMC_MIN_OPACITY, u_relocate=None, u_add=None):
        """One MCMC refinement of the P rows: relocation of the rows with sigmoid(opacity) <= min_opacity onto live rows drawn in
        proportion to their opacity, then growth by n_add = max(0, min(cap_max, floor(1.05 P)) - P) rows drawn from all rows in
        proportion to their opacity (include/dgr_mcmc.h dgr_mcmc_refine has the rule).  Sources get the relocation formula and zero
        Adam moments; relocated dead rows keep their own moments (as the published code); appended rows get zero moments.  Nothing is
        pruned.  u_relocate [P] / u_add [n_add]: uniform draws in [0, 1), by default from `noise_gen`.  With `fused_densify` on CUDA
        it runs the kernels (no host synchronisation), otherwise the torch restatement.  Returns the number of relocated rows as a
        device int32 scalar."""
        P, dev = self.num_points, self.p["xyz"].device
        n_add = mcmc_add_count(P, cap_max)
        min_opacity = float(np.float32(min_opacity))
        gen = getattr(self, "noise_gen", None)
        if u_relocate is None:
            u_relocate = torch.rand((P,), device=dev, generator=gen)
        if u_add is None:
            u_add = torch.rand((n_add,), device=dev, generator=gen)
        u_relocate, u_add = u_relocate.to(dev, torch.float32).contiguous(), u_add.to(dev, torch.float32).contiguous()
        if u_relocate.shape != (P,) or u_add.shape != (n_add,):
            raise ValueError("relocate_and_grow_mcmc: u_relocate must be [%d] and u_add [%d]" % (P, n_add))
        with torch.no_grad():
            if getattr(self, "fused_densify", False) and self.p["xyz"].is_cuda and P > 0:
                n = self._mcmc_refine_fused(n_add, u_relocate, u_add, min_opacity)
            else:
                n = self._mcmc_refine_torch(n_add, u_relocate, u_add, min_opacity)
        self._reset_stats()
        return n

    def _mcmc_refine_fused(self, n_add, u_relocate, u_add, min_opacity):
        lib = _lib.load_mcmc()
        P, dev = self.num_points, self.p["xyz"].device
        with torch.cuda.device(dev):
            st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            nbytes = lib.dgr_mcmc_scratch_bytes(P, n_add)
            scratch = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
            n_relocated = torch.zeros((), dtype=torch.int32, device=dev)
            t = _lib.DgrDensifyTensors()
            new_p, new_m, new_v = {}, {}, {}
            for i, k in enumerate(GROUPS):
                src = self.p[k].detach()
                new_p[k] = torch.empty((P + n_add,) + tuple(src.shape[1:]), dtype=torch.float32, device=dev)
                new_m[k], new_v[k] = torch.empty_like(new_p[k]), torch.empty_like(new_p[k])
                t.inp[i], t.exp_avg_in[i], t.exp_avg_sq_in[i] = src.data_ptr(), self.exp_avg[k].data_ptr(), self.exp_avg_sq[k].data_ptr()
                t.out[i], t.exp_avg_out[i], t.exp_avg_sq_out[i] = new_p[k].data_ptr(), new_m[k].data_ptr(), new_v[k].data_ptr()
                t.width[i] = int(np.prod(src.shape[1:]))
            _lib.check_mcmc(lib.dgr_mcmc_refine(P, n_add, ctypes.byref(t), u_relocate.data_ptr(), u_add.data_ptr() if n_add else None,
                                           min_opacity, scratch.data_ptr(), nbytes, n_relocated.data_ptr(), st))
            self.p = {k: v.requires_grad_(True) for k, v in new_p.items()}
            self.exp_avg, self.exp_avg_sq = new_m, new_v
        return n_relocated

    def _mcmc_refine_torch(self, n_add, u_relocate, u_add, min_opacity):
        """The rule of dgr_mcmc_refine with torch ops: searchsorted on a float64 cumsum, then tensor indexing (what the GPU tests hold the kernels to)."""
        P, dev = self.num_points, self.p["xyz"].device
        out = {k: v.detach().clone() for k, v in self.p.items()}
        m = {k: v.clone() for k, v in self.exp_avg.items()}
        v = {k: x.clone() for k, x in self.exp_avg_sq.items()}
        n_relocated = torch.zeros((), dtype=torch.int32, device=dev)
        if P > 0:
            o = _mcmc_opacity(out["opacity"][:, 0])
            dead = o <= min_opacity
            C = torch.cumsum(torch.where(dead, torch.zeros_like(o), o).double(), 0)
            dead_idx = dead.nonzero()[:, 0]
            if float(C[-1]) > 0 and dead_idx.numel() > 0:
                src = torch.searchsorted(C, u_relocate[:dead_idx.numel()].double() * C[-1], right=True)
                src = torch.where(src >= P, (~dead).nonzero()[-1, 0], src)
                picks = torch.bincount(src, minlength=P)
                rows = (picks > 0).nonzero()[:, 0]
                out["opacity"][rows, 0], out["scaling"][rows] = _mcmc_update(out["opacity"][rows, 0], out["scaling"][rows], picks[rows],
                                                                             min_opacity)
                for k in GROUPS:
                    out[k][dead_idx] = out[k][src]
                    m[k][rows] = 0
                    v[k][rows] = 0
                n_relocated.fill_(dead_idx.numel())
            if n_add > 0:
                C = torch.cumsum(_mcmc_opacity(out["opacity"][:, 0]).double(), 0)
                src = torch.searchsorted(C, u_add.double() * C[-1], right=True).clamp(max=P - 1)
                picks = torch.bincount(src, minlength=P)
                rows = (picks > 0).nonzero()[:, 0]
                out["opacity"][rows, 0], out["scaling"][rows] = _mcmc_update(out["opacity"][rows, 0], out["scaling"][rows], picks[rows],
                                                                             min_opacity)
                for k in GROUPS:
                    m[k][rows] = 0
                    v[k][rows] = 0
                    out[k] = torch.cat((out[k], out[k][src]), 0)
                    m[k] = torch.cat((m[k], torch.zeros_like(out[k][P:])), 0)
                    v[k] = torch.cat((v[k], torch.zeros_like(out[k][P:])), 0)
        self.p = {k: x.contiguous().requires_grad_(True) for k, x in out.items()}
        self.exp_avg = {k: x.contiguous() for k, x in m.items()}
        self.exp_avg_sq = {k: x.contiguous() for k, x in v.items()}
        return n_relocated

    def inject_noise_mcmc(self, scale, normals=None):
        """xyz += scale g(o) R diag(s^2) R^T z in place, g(o) = 1 / (1 + exp(-100 ((1 - o) - 0.995))) (near-transparent Gaussians
        move, opaque ones do not); scale = lr_xyz(step) * noise_lr in the published rule.  normals [P,3]: standard normals, by default
        from `noise_gen`.  With `fused_densify` on CUDA one launch (dgr_mcmc_inject_noise), otherwise torch ops."""
        P, dev = self.num_points, self.p["xyz"].device
        if normals is None:
            normals = torch.randn((P, 3), device=dev, generator=getattr(self, "noise_gen", None))
        normals = normals.to(dev, torch.float32).contiguous()
        if normals.shape != (P, 3):
            raise ValueError("inject_noise_mcmc: normals must be [%d, 3]" % P)
        with torch.no_grad():
            if getattr(self, "fused_densify", False) and self.p["xyz"].is_cuda and P > 0:
                lib = _lib.load_mcmc()
                with torch.cuda.device(dev):
                    st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
                    _lib.check_mcmc(lib.dgr_mcmc_inject_noise(P, self.p["xyz"].data_ptr(), self.p["opacity"].data_ptr(), self.p["scaling"].data_ptr(),
                                                         self.p["rotation"].data_ptr(), normals.data_ptr(), float(scale), st))
                return
            o = torch.sigmoid(self.p["opacity"].detach())
            gate = 1.0 / (1.0 + torch.exp(-MCMC_NOISE_K * ((1 - o) - MCMC_NOISE_X0)))
            R = build_rotation(self.p["rotation"].detach())
            s2 = torch.exp(self.p["scaling"].detach()) ** 2
            a = torch.bmm(R.transpose(1, 2), normals[:, :, None])[:, :, 0] * s2 * (scale * gate)
            self.p["xyz"].add_(torch.bmm(R, a[:, :, None])[:, :, 0])

    def prune_by_contribution(self, stats, min_weight_max):
        """Removes the Gaussians whose largest blending weight over the renders in `stats` (rasterizer.ContributionStats) is below
        min_weight_max: with a tiny threshold, those no render composited at all (outside every view or hidden behind others),
        which the opacity prune keeps.  Through prune_points, so the Adam moments and densification statistics follow.
        Returns how many were removed."""
        wmax = stats.weight_max
        if wmax.shape[0] != self.num_points:
            raise ValueError("prune_by_contribution: the statistics have %d Gaussians, the model %d" % (wmax.shape[0], self.num_points))
        mask = (wmax < min_weight_max).to(self.p["xyz"].device)
        n = int(mask.sum())
        self.prune_points(mask)
        return n

    def reset_opacity(self):
        """gs_renderer.py:417-420 + replace_tensor_to_optimizer :464-477: opacity = inverse_sigmoid(min(sigmoid(o), 0.01)) and
        that group's Adam moments zeroed (torch keeps the group's step count: `stored_state["step"]` is left alone)."""
        with torch.no_grad():
            o = torch.sigmoid(self.p["opacity"].detach())
            o = torch.min(o, torch.full_like(o, 0.01))
            self.p["opacity"] = torch.log(o / (1 - o)).contiguous().requires_grad_(True)
            self.exp_avg["opacity"] = torch.zeros_like(self.p["opacity"])
            self.exp_avg_sq["opacity"] = torch.zeros_like(self.p["opacity"])


# ---------------------------------------------------------------------------------------------------------------------
class Stage1Config(NamedTuple):
    """configs/image.yaml + main.py defaults used by train_step (SURVEY.md Appendix B)."""
    iters: int = 500
    ref_size: int = 256
    num_pts: int = 5000
    sh_degree: int = 0
    radius: float = 2.0
    fovy: float = 49.1
    elevation: float = 0.0
    min_ver: int = -30
    max_ver: int = 30
    invert_bg_prob: float = 0.5
    lambda_zero123: float = 1.0
    density_start_iter: int = 100
    density_end_iter: int = 3000
    densification_interval: int = 100
    opacity_reset_interval: int = 700
    densify_grad_threshold: float = 0.01
    seed: int = 0
    antialiasing: bool = False          # every render with the 2D Mip filter and opacity compensation (GaussianRasterizer's switch)
    # AbsGS densification: split by the absolute-gradient statistic at this threshold (clone as before); None = the default loop.
    # Needs fused=True: the statistic exists only inside the backward render.
    densify_abs_grad_threshold: Optional[float] = None
    # "mcmc": 3DGS-MCMC's rule instead of clone / split / prune — relocate dead Gaussians and grow by 5 % per refinement up to
    # mcmc_cap_max (in the density window at the densification interval), position noise every step, the two regularisers in the loss,
    # no opacity reset.  The cap's default is about the count the default loop reaches in 500 iterations; nobody has measured it
    # for quality.
    densify_strategy: str = "default"
    mcmc_cap_max: int = 43000
    mcmc_noise_lr: float = MCMC_NOISE_LR
    mcmc_opacity_reg: float = MCMC_OPACITY_REG
    mcmc_scale_reg: float = MCMC_SCALE_REG
    mcmc_min_opacity: float = MCMC_MIN_OPACITY


class GuidanceStub:
    """Deterministic stand-in for guidance.zero123_utils.Zero123.train_step (SURVEY.md Appendix B): a differentiable
    scalar 0.5 * sum((downsample(pred, 32x32) - fixed_target)^2), as the real one returns 0.5 * ||latents - target||^2."""

    def __init__(self, device, seed=0):
        g = torch.Generator(device="cpu").manual_seed(seed + 99)
        self.target = torch.rand((1, 3, 32, 32), generator=g).to(device)

    def train_step(self, images, vers, hors, radii, step_ratio=None, default_elevation=0):
        pred = torch.nn.functional.interpolate(images, (32, 32), mode="bilinear", align_corners=False)
        return 0.5 * ((pred - self.target) ** 2).sum()


def synthetic_rgba(size):
    """Synthetic RGBA input (BASELINE.json configs[3]): a shaded disc on a transparent background, [1,3,S,S] and [1,1,S,S]."""
    y, x = np.mgrid[0:size, 0:size].astype(np.float32)
    c = (size - 1) / 2.0
    r = np.sqrt((x - c) ** 2 + (y - c) ** 2) / (0.35 * size)
    mask = (r < 1.0).astype(np.float32)
    shade = np.clip(1.0 - 0.6 * r, 0, 1)
    rgb = np.stack([0.9 * shade, 0.4 + 0.3 * shade, 0.2 + 0.5 * (x / size)], 0) * mask + (1 - mask)      # white background (main.py:100-104)
    return rgb[None].astype(np.float32), mask[None, None].astype(np.float32)


class Stage1Trainer:
    """main.py:182-287 train_step, guidance stubbed.  `fused=True`: FusedGaussianRasterizer + fused Adam (rows f1 + f2);
    `fused=False`: the reference's formulation through this library's plain op — torch activations + torch.cat, the three
    torch statistic updates, torch.optim.Adam-style per-tensor updates — the baseline tools/stage1_bench.py times.
    `batched=True` (needs fused=True): the known and the novel view of a step are ONE mixed-size batched render
    (fused.rasterize_views_mixed_raw) with one forward and one backward, the statistics taken from the novel view only; same
    cameras, rng draws and loss terms as the default path, whose gradient summation order it does not share."""

    def __init__(self, cfg: Stage1Config = Stage1Config(), optim: OptimConfig = OptimConfig(), device="cuda", fused=True, batched=False):
        from . import scene
        if batched and not fused:
            raise ValueError("Stage1Trainer: batched=True needs fused=True (the batched call takes the raw parameters)")
        if cfg.densify_abs_grad_threshold is not None and not fused:
            raise ValueError("Stage1Trainer: densify_abs_grad_threshold needs fused=True (the reference formulation takes its statistics "
                             "from means2D.grad, which has no per-pixel absolute values)")
        if cfg.densify_strategy not in ("default", "mcmc"):
            raise ValueError("Stage1Trainer: densify_strategy must be 'default' or 'mcmc', not %r" % (cfg.densify_strategy,))
        if cfg.densify_strategy == "mcmc" and cfg.densify_abs_grad_threshold is not None:
            raise ValueError("Stage1Trainer: densify_strategy='mcmc' does not split by a gradient statistic; "
                             "densify_abs_grad_threshold must be None")
        self.cfg, self.device, self.fused, self.batched = cfg, torch.device(device), fused, batched
        self.mcmc = cfg.densify_strategy == "mcmc"
        self.rng = np.random.default_rng(cfg.seed)
        self.scene = scene
        cloud = scene.make_cloud(cfg.num_pts, cfg.sh_degree, seed=cfg.seed, anisotropic=False, sigma=1.0)      # positions only
        colors = self.rng.random((cfg.num_pts, 3)) / 255.0 * SH_C0 + 0.5                                         # SH2RGB(rand/255), gs_renderer.py:703-706
        self.gaussians = GaussianModelB200(cfg.sh_degree)
        self.gaussians.fused_adam = fused
        self.gaussians.fused_densify = fused
        self.gaussians.absgrad = cfg.densify_abs_grad_threshold is not None
        # the split children's noise comes from the trainer's own generator: torch's default one is seeded differently in every
        # process, so two runs from one seed would split differently at the first densification
        self.gaussians.noise_gen = torch.Generator(device=self.device).manual_seed(cfg.seed)
        self.gaussians.create_from_points(cloud["means3D"], colors, spatial_lr_scale=10.0, device=device)      # gs_renderer.py:709
        self.gaussians.training_setup(optim)
        rgb, mask = synthetic_rgba(cfg.ref_size)
        self.input_img, self.input_mask = torch.tensor(rgb, device=device), torch.tensor(mask, device=device)
        self.guidance = GuidanceStub(self.device, cfg.seed)
        self.step = 0
        self.fixed_cam = self._settings(cfg.elevation, 0.0, cfg.radius, cfg.ref_size, (1.0, 1.0, 1.0))
        self.losses = []

    def _settings(self, elev, azim, radius, res, bg):
        cam = self.scene.orbit_camera(elev, azim, radius, res, res, fovy_deg=self.cfg.fovy)
        # one host-to-device copy for the four small camera tensors (the loop is host-bound: every copy is a driver call)
        buf = np.concatenate([np.append(np.asarray(bg, np.float32).ravel(), 0.0).astype(np.float32), cam.world_view_transform.ravel(), cam.full_proj_transform.ravel(),
                              cam.camera_center.ravel(), np.zeros(1, np.float32)]).astype(np.float32)
        t = torch.from_numpy(buf).to(self.device)
        return GaussianRasterizationSettings(image_height=res, image_width=res, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=t[0:3],
                                             scale_modifier=1.0, viewmatrix=t[4:20].view(4, 4), projmatrix=t[20:36].view(4, 4),
                                             sh_degree=self.gaussians.active_sh_degree, campos=t[36:39], prefiltered=False, debug=False)

    def render(self, rs, track_stats):
        g = self.gaussians
        means2D = torch.zeros_like(g._xyz, requires_grad=True)
        if self.fused:
            color, radii, depth, alpha = FusedGaussianRasterizer(rs, self.cfg.antialiasing)(g._xyz, g._features_dc, g._features_rest, g._opacity, g._scaling,
                                                                     g._rotation, means2D=means2D, stats=g.stats if track_stats else None)
        else:
            from .rasterizer import GaussianRasterizer
            color, radii, depth, alpha = GaussianRasterizer(rs, self.cfg.antialiasing)(
                means3D=g._xyz, means2D=means2D, shs=torch.cat((g._features_dc, g._features_rest), dim=1),
                opacities=torch.sigmoid(g._opacity), scales=torch.exp(g._scaling), rotations=torch.nn.functional.normalize(g._rotation))
        return {"image": color.clamp(0, 1), "alpha": alpha, "viewspace_points": means2D, "visibility_filter": radii > 0, "radii": radii}

    def train_step(self):
        cfg, g = self.cfg, self.gaussians
        self.step += 1
        step_ratio = min(1, self.step / cfg.iters)
        g.update_learning_rate(self.step)
        g.zero_grad()
        densify_window = cfg.density_start_iter <= self.step <= cfg.density_end_iter
        track = densify_window and not self.mcmc          # the MCMC rule needs no densification statistics
        if self.batched:
            loss = self._batched_loss(step_ratio, track)
        else:
            loss = self._loss(step_ratio, track)
        if self.mcmc:
            loss = loss + cfg.mcmc_opacity_reg * torch.sigmoid(g._opacity).mean() + cfg.mcmc_scale_reg * torch.exp(g._scaling).mean()
        loss.backward()
        g.optimizer_step()
        if self.mcmc:
            if densify_window and self.step % cfg.densification_interval == 0:
                g.relocate_and_grow_mcmc(cfg.mcmc_cap_max, cfg.mcmc_min_opacity)
            g.inject_noise_mcmc(g.lr["xyz"] * cfg.mcmc_noise_lr)
        elif densify_window:
            if not self.fused:          # the reference's three torch updates (main.py:279-281, gs_renderer.py:625-627)
                with torch.no_grad():
                    vis, radii, st = self._last["visibility_filter"], self._last["radii"], g.stats
                    st.max_radii2D[vis] = torch.max(st.max_radii2D[vis], radii[vis].float())
                    st.xyz_gradient_accum[vis] += torch.norm(self._last["viewspace_points"].grad[vis, :2], dim=-1)
                    st.denom[vis] += 1
            if self.step % cfg.densification_interval == 0:
                g.densify_and_prune(cfg.densify_grad_threshold, min_opacity=0.01, extent=4, max_screen_size=1,
                                    max_abs_grad=cfg.densify_abs_grad_threshold)
            if self.step % cfg.opacity_reset_interval == 0:          # main.py:285-286 (700 > 500 iterations in image.yaml)
                g.reset_opacity()
        self._last = None
        self.losses.append(loss.detach())
        return loss

    def _novel_camera(self, step_ratio):
        """The novel view's camera (main.py:210-226): its resolution by step_ratio, then ver, hor, bg drawn from the rng."""
        cfg = self.cfg
        res = 128 if step_ratio < 0.3 else (256 if step_ratio < 0.6 else 512)
        min_ver = max(min(cfg.min_ver, cfg.min_ver - cfg.elevation), -80 - cfg.elevation)
        max_ver = min(max(cfg.max_ver, cfg.max_ver - cfg.elevation), 80 - cfg.elevation)
        ver, hor = int(self.rng.integers(min_ver, max_ver)), int(self.rng.integers(-180, 180))
        bg = (1.0, 1.0, 1.0) if self.rng.random() > cfg.invert_bg_prob else (0.0, 0.0, 0.0)
        return self._settings(cfg.elevation + ver, hor, cfg.radius, res, bg), ver, hor

    def _batched_loss(self, step_ratio, densify_window):
        """The loss of the step from ONE batched render of [known view, novel view] (sizes ref_size and res)."""
        from .fused import rasterize_views_mixed_raw
        cfg, g = self.cfg, self.gaussians
        novel, ver, hor = self._novel_camera(step_ratio)
        colors, radii, depths, alphas = rasterize_views_mixed_raw(
            [self.fixed_cam, novel], g._xyz, None, g._features_dc, g._features_rest, g._opacity, g._scaling, g._rotation,
            stats=g.stats if densify_window else None, stats_views=(1,) if densify_window else (), antialiasing=cfg.antialiasing)
        loss = 10000 * step_ratio * torch.nn.functional.mse_loss(colors[0].clamp(0, 1).unsqueeze(0), self.input_img)
        loss = loss + 1000 * step_ratio * torch.nn.functional.mse_loss(alphas[0].unsqueeze(0), self.input_mask)
        return loss + cfg.lambda_zero123 * self.guidance.train_step(colors[1].clamp(0, 1).unsqueeze(0), [ver], [hor], [0], step_ratio=step_ratio,
                                                                     default_elevation=cfg.elevation)

    def _loss(self, step_ratio, densify_window):
        cfg = self.cfg
        # known view (main.py:196-208)
        out = self.render(self.fixed_cam, track_stats=False)
        loss = 10000 * step_ratio * torch.nn.functional.mse_loss(out["image"].unsqueeze(0), self.input_img)
        loss = loss + 1000 * step_ratio * torch.nn.functional.mse_loss(out["alpha"].unsqueeze(0), self.input_mask)
        # novel view (main.py:210-240); the statistics come from this LAST render of the step (main.py:278-281)
        novel, ver, hor = self._novel_camera(step_ratio)
        out = self.render(novel, track_stats=densify_window)
        self._last = out
        return loss + cfg.lambda_zero123 * self.guidance.train_step(out["image"].unsqueeze(0), [ver], [hor], [0], step_ratio=step_ratio,
                                                                    default_elevation=cfg.elevation)

    def train(self, iters=None):
        for _ in range(iters or self.cfg.iters):
            self.train_step()
        return torch.stack(self.losses).cpu().numpy()

    # the 26 cameras the reference's save_model bakes the texture from (main.py:428-429): elevation, azimuth in degrees
    EXPORT_VERS = [0] * 8 + [-45] * 8 + [45] * 8 + [-89.9, 89.9]
    EXPORT_HORS = [0, 45, -45, 90, -90, 135, -135, 180] * 3 + [0, 0]

    def export_settings(self, resolution=512):
        """The export cameras at cfg.radius / cfg.fovy, resolution x resolution, white background."""
        return [self._settings(v, h, self.cfg.radius, resolution, (1.0, 1.0, 1.0)) for v, h in zip(self.EXPORT_VERS, self.EXPORT_HORS)]

    def prune_unseen(self, min_weight_max, resolution=512):
        """Before extracting the mesh or saving the PLY: renders the 26 export cameras in one batched forward (no gradients) with
        the blending-weight statistics and removes the Gaussians whose largest weight in any of them is below min_weight_max
        (GaussianModelB200.prune_by_contribution).  Returns how many were removed.  train() does not call it."""
        from .fused import rasterize_views_raw
        from .rasterizer import ContributionStats
        g = self.gaussians
        stats = ContributionStats(g.num_points, self.device)
        with torch.no_grad():
            rasterize_views_raw(self.export_settings(resolution), g._xyz, None, g._features_dc, g._features_rest, g._opacity, g._scaling,
                                g._rotation, antialiasing=self.cfg.antialiasing, contributions=stats)
        return g.prune_by_contribution(stats, min_weight_max)

    def save_mesh(self, path, density_thresh=1.0, resolution=128):
        """save_model(mode='geo') (main.py:405-410) without the texture half: extract_fields, marching cubes, the world transform and
        the small-component removal on the device (meshing.extract_mesh_of_model), written as a binary PLY.  Returns (v, f).
        train() does not call it; prune_unseen stays a separate call."""
        from . import meshing
        from .ply import save_mesh_ply
        v, f = meshing.extract_mesh_of_model(self.gaussians, density_thresh, resolution)
        save_mesh_ply(path, v, f)
        return v, f
