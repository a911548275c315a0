"""SURVEY.md §8 row f1: the rasterizer taking GaussianModel's RAW parameters, activations fused into the kernels.

The reference renders with (gs_renderer.py:196-216, :762-806)

    means3D = _xyz;  opacity = sigmoid(_opacity);  scales = exp(_scaling);  rotations = F.normalize(_rotation)
    shs = torch.cat((_features_dc, _features_rest), dim=1)

i.e. four element-wise passes over the parameters, a 12·M-byte-per-Gaussian concatenation copy, and the mirror-image
passes in the backward — then, after the optimiser step (main.py:279-281, gs_renderer.py:625-627),

    max_radii2D[vis] = max(max_radii2D[vis], radii[vis]);  xyz_gradient_accum[vis] += |means2D.grad[vis, :2]|;  denom[vis] += 1

Here the per-Gaussian kernels read the raw tensors directly (`DgrGaussians.activations`), apply the activations in
registers, return gradients with respect to the raw tensors, and update the three densification statistics in the same
backward kernel.  Same C ABI entry points as the plain path (include/dgr_b200.h)."""
from typing import Optional

import torch
import torch.nn as nn

from . import rasterizer as _r


class DensifyStats:
    """The three per-Gaussian statistics of the reference's densification (float32 [P]; the reference keeps [P,1] / [P]).
    absgrad=True adds xyz_gradient_accum_abs (float32 [P], else None): AbsGS's statistic, the per-render norm of the summed ABSOLUTE
    per-pixel terms of dL/dmeans2D (DGR_RASTER_ABS_GRAD, include/dgr_b200.h), which the renders below then update as well."""

    def __init__(self, P: int, device, absgrad: bool = False):
        self.xyz_gradient_accum = torch.zeros((P,), dtype=torch.float32, device=device)
        self.denom = torch.zeros((P,), dtype=torch.float32, device=device)
        self.max_radii2D = torch.zeros((P,), dtype=torch.float32, device=device)
        self.xyz_gradient_accum_abs = torch.zeros((P,), dtype=torch.float32, device=device) if absgrad else None

    def as_tuple(self):
        return (self.xyz_gradient_accum, self.denom, self.max_radii2D)


class _RasterizeRaw(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xyz, means2D, features_dc, features_rest, opacity_raw, scaling_raw, rotation_raw, raster_settings, stats,
                antialiasing=False, contributions=None, *cams):
        ctx.cams = cams                  # (viewmatrix, projmatrix, campos) when their gradient is asked for
        if _r._FAST is not None:
            color, radii, depth, alpha, state = _r.forward_impl(raster_settings, xyz, features_dc, None, opacity_raw, scaling_raw, rotation_raw,
                                                                None, sh_rest=features_rest, activations=True, antialiasing=antialiasing,
                                                                contrib=contributions is not None)
            _r._add_contributions(contributions, state)
            ctx.state, ctx.stats = state, stats
            ctx.mark_non_differentiable(radii)
            return color, radii, depth, alpha
        xyz = _r._dev_f32(xyz, "xyz")
        dc = _r._dev_f32(features_dc, "features_dc")
        rest = _r._opt(features_rest, "features_rest")
        if rest is not None and rest.numel() == 0:
            rest = None
        op, sc, rot = _r._dev_f32(opacity_raw, "opacity"), _r._dev_f32(scaling_raw, "scaling"), _r._dev_f32(rotation_raw, "rotation")
        color, radii, depth, alpha, state = _r.forward_impl(raster_settings, xyz, dc, None, op, sc, rot, None, sh_rest=rest,
                                                            activations=True, antialiasing=antialiasing, contrib=contributions is not None)
        _r._add_contributions(contributions, state)
        ctx.state, ctx.stats = state, stats
        ctx.mark_non_differentiable(radii)
        return color, radii, depth, alpha

    @staticmethod
    def backward(ctx, grad_color, grad_radii, grad_depth, grad_alpha):
        state = ctx.state
        # the statistics describe the RENDER, not the backward call: a retain_graph / second backward of the same forward
        # must not count the view twice (gs_renderer.py:625-627 runs once per render)
        if getattr(state, "stats_applied", False):
            ctx.stats = None
        state.stats_applied = True
        needs = ctx.needs_input_grad[11:]
        cam_needed = any(needs)
        if state.fast is not None:
            stats = ctx.stats.as_tuple() if ctx.stats is not None else (None, None, None)
            absgrad = ctx.stats.xyz_gradient_accum_abs if ctx.stats is not None else None
            g = _r._FAST.backward(state.fast, grad_color, grad_depth, grad_alpha, False, [], *stats, camera=cam_needed, absgrad=absgrad)
            cg = _r._camera_input_grads(ctx.cams, needs, g[9:12]) if cam_needed else [None] * len(ctx.cams)
            return (g[0], g[1], g[2], g[8], g[4], g[5], g[6], None, None, None, None, *cg)
        xyz, dc, _, op, sc, rot, _, rest = state.tensors
        P = state.frame.P
        f32 = dict(dtype=torch.float32, device=xyz.device)
        gC = _r._dev_f32(grad_color, "grad_color") if grad_color is not None else None
        gD = _r._dev_f32(grad_depth, "grad_depth") if grad_depth is not None else None
        gA = _r._dev_f32(grad_alpha, "grad_alpha") if grad_alpha is not None else None
        d_xyz, d_m2d = torch.empty((P, 3), **f32), torch.empty((P, 3), **f32)
        d_dc = torch.empty((P, 1, 3), **f32)
        d_rest = torch.empty(rest.shape, **f32) if rest is not None else None
        d_op, d_sc, d_rot = torch.empty((P, 1), **f32), torch.empty((P, 3), **f32), torch.empty((P, 4), **f32)
        stats = ctx.stats.as_tuple() if ctx.stats is not None else None
        absgrad = ctx.stats.xyz_gradient_accum_abs if ctx.stats is not None else None
        camera = _r._camera_outputs(0, xyz.device) if cam_needed else None
        _r.backward_impl(state, gC, gD, gA, d_xyz, d_m2d, d_dc, None, d_op, d_sc, d_rot, None, d_sh_rest=d_rest, densify=stats, camera=camera,
                         absgrad=absgrad)
        cg = _r._camera_input_grads(ctx.cams, needs, camera) if cam_needed else [None] * len(ctx.cams)
        return (d_xyz, d_m2d if ctx.needs_input_grad[1] else None, d_dc, d_rest, d_op, d_sc, d_rot, None, None, None, None, *cg)


class FusedGaussianRasterizer(nn.Module):
    """`GaussianRasterizer` for raw parameters.  forward(xyz, features_dc, features_rest, opacity, scaling, rotation,
    means2D=None, stats=None) -> (color [3,H,W], radii int32 [P], depth [1,H,W], alpha [1,H,W]); `stats` (DensifyStats) is
    updated during the backward, its xyz_gradient_accum_abs too when it has one.  antialiasing: as GaussianRasterizer (the 2D Mip filter with opacity compensation).  Camera
    tensors of the settings that require grad receive their gradient, as with GaussianRasterizer.  contributions
    (rasterizer.ContributionStats): every forward adds its blending-weight statistics to it, as with GaussianRasterizer."""

    def __init__(self, raster_settings: _r.GaussianRasterizationSettings, antialiasing: bool = False, contributions=None):
        super().__init__()
        self.raster_settings = raster_settings
        self.antialiasing = bool(antialiasing)
        self.contributions = contributions

    def forward(self, xyz, features_dc, features_rest, opacity, scaling, rotation, means2D: Optional[torch.Tensor] = None,
                stats: Optional[DensifyStats] = None):
        if means2D is None:
            means2D = torch.zeros_like(xyz, requires_grad=xyz.requires_grad)
        return _RasterizeRaw.apply(xyz, means2D, features_dc, features_rest, opacity, scaling, rotation, self.raster_settings, stats,
                                   self.antialiasing, self.contributions, *_r._camera_tensors([self.raster_settings]))


def render_gaussian_model(gaussians, raster_settings, stats: Optional[DensifyStats] = None, antialiasing: bool = False,
                          contributions=None):
    """Renders an object with the reference GaussianModel's attribute names (_xyz, _features_dc, _features_rest, _opacity,
    _scaling, _rotation: gs_renderer.py:140-160).  Returns the reference Renderer.render's dict (gs_renderer.py:812-822).
    contributions: as FusedGaussianRasterizer."""
    xyz = gaussians._xyz
    means2D = torch.zeros_like(xyz, requires_grad=True)
    color, radii, depth, alpha = FusedGaussianRasterizer(raster_settings, antialiasing, contributions)(
        xyz, gaussians._features_dc, gaussians._features_rest, gaussians._opacity, gaussians._scaling, gaussians._rotation,
        means2D=means2D, stats=stats)
    return {"image": color.clamp(0, 1), "depth": depth, "alpha": alpha, "viewspace_points": means2D,
            "visibility_filter": radii > 0, "radii": radii}


class _RasterizeViewsRaw(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xyz, means2D, features_dc, features_rest, opacity_raw, scaling_raw, rotation_raw, settings_list, antialiasing=False,
                contributions=None, *cams):
        ctx.cams = cams
        xyz = _r._dev_f32(xyz, "xyz")
        dc = _r._dev_f32(features_dc, "features_dc")
        rest = _r._opt(features_rest, "features_rest")
        if rest is not None and rest.numel() == 0:
            rest = None
        op, sc, rot = _r._dev_f32(opacity_raw, "opacity"), _r._dev_f32(scaling_raw, "scaling"), _r._dev_f32(rotation_raw, "rotation")
        color, radii, depth, alpha, state = _r.views_forward_impl(settings_list, xyz, dc, op, sc, rot, sh_rest=rest, activations=True,
                                                                  antialiasing=antialiasing, contrib=contributions is not None)
        _r._add_contributions(contributions, state)
        ctx.state = state
        ctx.mark_non_differentiable(radii)
        return color, radii, depth, alpha

    @staticmethod
    def backward(ctx, grad_color, grad_radii, grad_depth, grad_alpha):
        (d_xyz, d_m2d, d_dc, d_rest, d_op, d_sc, d_rot), cg = _r._views_backward_with_cameras(ctx, grad_color, grad_depth, grad_alpha,
                                                                                                True, 10)
        return (d_xyz, d_m2d if ctx.needs_input_grad[1] else None, d_dc, d_rest, d_op, d_sc, d_rot, None, None, None, *cg)


def rasterize_views_raw(settings_list, xyz, means2D, features_dc, features_rest, opacity, scaling, rotation, antialiasing=False,
                        contributions=None):
    """rasterize_views (rasterizer.py) for GaussianModel's RAW parameters: one cloud, a batch of same-size cameras, the
    activations applied in the kernels and the gradients summed over the views with respect to the raw tensors.  means2D
    [V,P,3] receives the per-view screen-space gradient.  The densification statistics are not updated by the batched call.
    antialiasing: as GaussianRasterizer; contributions: as rasterizer.rasterize_views."""
    settings_list = _r._check_views_settings(settings_list)
    if means2D is not None and tuple(means2D.shape) != (len(settings_list), xyz.shape[0], 3):
        raise ValueError("means2D must have dimensions (num_views, num_points, 3)")
    return _RasterizeViewsRaw.apply(xyz, means2D, features_dc, features_rest, opacity, scaling, rotation, settings_list, bool(antialiasing),
                                    contributions, *_r._camera_tensors(settings_list))


class _RasterizeViewsMixedRaw(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xyz, means2D, features_dc, features_rest, opacity_raw, scaling_raw, rotation_raw, settings_list, stats, stats_mask,
                antialiasing=False, contributions=None, *cams):
        ctx.cams = cams
        xyz = _r._dev_f32(xyz, "xyz")
        dc = _r._dev_f32(features_dc, "features_dc")
        rest = _r._opt(features_rest, "features_rest")
        if rest is not None and rest.numel() == 0:
            rest = None
        op, sc, rot = _r._dev_f32(opacity_raw, "opacity"), _r._dev_f32(scaling_raw, "scaling"), _r._dev_f32(rotation_raw, "rotation")
        color, radii, depth, alpha, state = _r.views_forward_impl(settings_list, xyz, dc, op, sc, rot, sh_rest=rest, activations=True,
                                                                  mixed=True, antialiasing=antialiasing, contrib=contributions is not None)
        _r._add_contributions(contributions, state)
        ctx.state, ctx.stats, ctx.stats_mask = state, (stats if stats_mask else None), stats_mask
        ctx.mark_non_differentiable(radii)
        return color, radii, depth, alpha

    @staticmethod
    def backward(ctx, grad_color, grad_radii, grad_depth, grad_alpha):
        state = ctx.state
        # as _RasterizeRaw: the statistics describe the forward, a retain_graph / second backward must not count its views twice
        if getattr(state, "stats_applied", False):
            ctx.stats = None
        state.stats_applied = True
        (d_xyz, d_m2d, d_dc, d_rest, d_op, d_sc, d_rot), cg = _r._views_backward_with_cameras(
            ctx, grad_color, grad_depth, grad_alpha, True, 12, stats=ctx.stats, stats_views=ctx.stats_mask)
        return (d_xyz, d_m2d if ctx.needs_input_grad[1] else None, d_dc, d_rest, d_op, d_sc, d_rot, None, None, None, None, None, *cg)


def rasterize_views_mixed_raw(settings_list, xyz, means2D, features_dc, features_rest, opacity, scaling, rotation, stats=None,
                              stats_views=(), antialiasing=False, contributions=None):
    """rasterize_views_mixed (rasterizer.py) for GaussianModel's RAW parameters: one cloud, cameras of any image sizes, the
    activations applied in the kernels and the gradients summed over the views with respect to the raw tensors.  Returns
    (colors, radii, depths, alphas) as rasterize_views_mixed.  `stats` (DensifyStats) is updated during the backward for the views
    listed in `stats_views` (indices into settings_list), in view order, as one fused single-view render of each would update it;
    once per forward.  antialiasing: as GaussianRasterizer; contributions: as rasterizer.rasterize_views."""
    settings_list = _r._check_views_mixed_settings(settings_list)
    if means2D is not None and tuple(means2D.shape) != (len(settings_list), xyz.shape[0], 3):
        raise ValueError("means2D must have dimensions (num_views, num_points, 3)")
    mask = _r._stats_mask(stats_views, len(settings_list))
    color, radii, depth, alpha = _RasterizeViewsMixedRaw.apply(xyz, means2D, features_dc, features_rest, opacity, scaling, rotation,
                                                               settings_list, stats if mask else None, mask, bool(antialiasing),
                                                               contributions, *_r._camera_tensors(settings_list))
    colors, depths, alphas = _r.split_views(settings_list, color, depth, alpha)
    return colors, radii, depths, alphas
