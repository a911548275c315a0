"""Host-side mirror of the reference's rasterizer operator: ``GaussianRasterizationSettings`` / ``GaussianRasterizer``.

Drop-in for the import at /root/reference/gs_renderer.py:10-13 and the call at gs_renderer.py:745-809:

    rasterizer = GaussianRasterizer(raster_settings=GaussianRasterizationSettings(...12 fields...))
    color, radii, depth, alpha = rasterizer(means3D=, means2D=, shs=, colors_precomp=, opacities=,
                                            scales=, rotations=, cov3D_precomp=)

Same names, argument meaning, return shapes/dtypes (color [3,H,W], radii int32 [P], depth [1,H,W], alpha [1,H,W]) and
error behaviour (the two "Please provide ..." exceptions) as the un-vendored package the reference imports [EXT].
All arithmetic runs in libdgr_b200.so (hand-written sm_90a CUDA) through the C ABI of include/dgr_b200.h; torch is
used for device memory, the current stream and autograd plumbing only.  There is no CPU path: non-CUDA tensors raise.
"""
import ctypes
from typing import NamedTuple, Optional

import torch
import torch.nn as nn

from . import _lib


def _load_fast():
    """The compiled host layer (csrc/dgr_torch.cpp -> lib/dgr_torch_host.so): same C-ABI calls, ~10x less host time per
    call than ctypes.  Optional: without it (or with DGR_NO_FASTHOST=1) the ctypes path below does the same work."""
    import importlib.util
    import os
    if os.environ.get("DGR_NO_FASTHOST") == "1":
        return None
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "dgr_torch_host.so")
    if not os.path.exists(path):
        return None
    try:
        from . import build as _build
        if not os.path.exists(_build.HOST_HASH) or open(_build.HOST_HASH).read().strip() != _build._host_hash():
            import warnings
            warnings.warn("dgr_torch_host.so is stale (csrc/dgr_torch.cpp or include/dgr_b200.h changed since it was built): "
                          "using the ctypes host layer; run dreamgaussian_b200/build.py", RuntimeWarning)
            return None
        _lib.load()
        spec = importlib.util.spec_from_file_location("dgr_torch_host", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return mod if mod.abi_version() == _lib.ABI_VERSION else None
    except Exception as e:  # noqa: BLE001  (a torch / compiler mismatch: fall back to ctypes, never to a CPU path)
        import warnings
        warnings.warn("dgr_torch_host.so could not be loaded (%r): using the ctypes host layer" % (e,), RuntimeWarning)
        return None


_FAST = _load_fast()


def set_fast_host(enabled: bool):
    """Switch between the compiled host layer and the ctypes one (tests exercise both)."""
    global _FAST
    _FAST = _load_fast() if enabled else None
    return _FAST is not None


def get_capacity_hint(device_index, P, H, W):
    if _FAST is not None:
        return _FAST.get_hint(device_index, P, H, W)
    return _CAPACITY_HINT.get((device_index, P, H, W))


def set_capacity_hint(device_index, P, H, W, cap, big):
    if _FAST is not None:
        _FAST.set_hint(device_index, P, H, W, cap, big)
    else:
        _CAPACITY_HINT[(device_index, P, H, W)] = (cap, big)


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _dev_f32(t: torch.Tensor, name: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor):
        raise TypeError("%s must be a torch.Tensor" % name)
    if not t.is_cuda:
        raise RuntimeError(
            "%s is on %s: this rasterizer has no CPU path (it runs as sm_90a CUDA kernels in libdgr_b200.so)" % (name, t.device))
    if t.dtype != torch.float32:
        t = t.float()
    return _aligned16(t.contiguous())


def _aligned16(t: torch.Tensor) -> torch.Tensor:
    """The kernels read rotations / SH rows with 128-bit loads and stage their inputs with bulk TMA: a contiguous view that starts
    off a 16-byte boundary (e.g. ``flat[1:].view(P, 4)``) gets its own allocation, which is aligned."""
    if t.numel() > 0 and t.data_ptr() % 16 != 0:
        t = t.clone(memory_format=torch.contiguous_format)
    return t


def _opt(t, name):
    if t is None or (isinstance(t, torch.Tensor) and t.numel() == 0 and t.dim() <= 1):
        return None
    return _dev_f32(t, name)


class _Frame:
    """ctypes views of one forward call's settings + inputs (keeps the tensors alive)."""

    def __init__(self, rs: GaussianRasterizationSettings, means3D, sh, colors_precomp, opacities, scales, rotations, cov3D,
                 sh_rest=None, activations=False):
        self.keep = []
        k = self.keep.append
        self.bg = _dev_f32(rs.bg, "bg"); k(self.bg)
        self.view = _dev_f32(rs.viewmatrix, "viewmatrix"); k(self.view)
        self.proj = _dev_f32(rs.projmatrix, "projmatrix"); k(self.proj)
        self.campos = _dev_f32(rs.campos, "campos"); k(self.campos)
        if self.bg.numel() != 3 or self.view.numel() != 16 or self.proj.numel() != 16 or self.campos.numel() != 3:
            raise ValueError("bg/campos must have 3 elements, viewmatrix/projmatrix 16")
        self.settings = _lib.DgrSettings(
            int(rs.image_height), int(rs.image_width), float(rs.tanfovx), float(rs.tanfovy), float(rs.scale_modifier),
            int(rs.sh_degree), int(bool(rs.prefiltered)), int(bool(rs.debug)),
            _ptr(self.bg), _ptr(self.view), _ptr(self.proj), _ptr(self.campos))
        if means3D.dim() != 2 or means3D.shape[1] != 3:
            raise ValueError("means3D must have dimensions (num_points, 3)")
        P = means3D.shape[0]
        M = 0
        if sh is not None:
            if sh.dim() != 3 or sh.shape[0] != P or sh.shape[2] != 3:
                raise ValueError("shs must have dimensions (num_points, num_coeffs, 3)")
            M = sh.shape[1]
        if activations:
            # raw GaussianModel parameters: sh = _features_dc [P,1,3], sh_rest = _features_rest [P,M-1,3]
            if sh is None or sh.shape[1] != 1:
                raise ValueError("features_dc must have dimensions (num_points, 1, 3)")
            if sh_rest is not None and sh_rest.numel() > 0:
                if sh_rest.dim() != 3 or sh_rest.shape[0] != P or sh_rest.shape[2] != 3:
                    raise ValueError("features_rest must have dimensions (num_points, num_coeffs - 1, 3)")
                M = 1 + sh_rest.shape[1]
            else:
                sh_rest = None
        for t, n, w in ((colors_precomp, "colors_precomp", 3), (scales, "scales", 3), (rotations, "rotations", 4), (cov3D, "cov3D_precomp", 6)):
            if t is not None and (t.numel() != P * w):
                raise ValueError("%s must have dimensions (num_points, %d)" % (n, w))
        if opacities.numel() != P:
            raise ValueError("opacities must have dimensions (num_points, 1)")
        self.P, self.M = P, M
        self.gaussians = _lib.DgrGaussians(P, M, _ptr(means3D), _ptr(sh), _ptr(colors_precomp), _ptr(opacities),
                                           _ptr(scales), _ptr(rotations), _ptr(cov3D), _ptr(sh_rest if activations else None),
                                           1 if activations else 0)


def _stream_ptr(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _contrib_opts(contrib, records, dev):
    """The DgrRasterOptions argument of a stage-2 render *_ex call: None without contrib; with it, DGR_RASTER_CONTRIB and its
    outputs -> (options pointer, (weight_sum, weight_max) float32 [records], the structs and scratch to keep alive)."""
    if not contrib:
        return None, None, None
    lib = _lib.load()
    ws = torch.empty((records,), dtype=torch.float32, device=dev)
    wm = torch.empty((records,), dtype=torch.float32, device=dev)
    scratch = torch.empty((max(1, lib.dgr_contrib_scratch_bytes(int(records))),), dtype=torch.uint8, device=dev)
    c = _lib.DgrContrib(_ptr(ws) if records else None, _ptr(wm) if records else None, _ptr(scratch), scratch.numel())
    opt = _lib.DgrRasterOptionsContrib(_lib.RASTER_CONTRIB, None, None, ctypes.pointer(c))
    return ctypes.cast(ctypes.pointer(opt), ctypes.POINTER(_lib.DgrRasterOptions)), (ws, wm), (c, opt, scratch)


class ContributionStats:
    """Per-Gaussian blending-weight statistics accumulated over renders (DGR_RASTER_CONTRIB, include/dgr_b200.h): for every
    rendered view, weight_sum adds the sum over the pixels where the Gaussian is composited of its weight w = alpha T, and
    weight_max keeps the largest such w seen.  A Gaussian that no render composites (outside every view, or hidden behind
    others) keeps weight_max == 0, whatever its radius; prune with GaussianModelB200.prune_by_contribution.
    Pass it as contributions= to a render call: the forward updates it once per call (after its last stage-2 run, in view
    order), under torch.no_grad too; the backward never touches it.  renders counts the views added."""

    def __init__(self, P: int, device):
        self.weight_sum = torch.zeros((P,), dtype=torch.float32, device=device)
        self.weight_max = torch.zeros((P,), dtype=torch.float32, device=device)
        self.renders = 0

    def add(self, weight_sum, weight_max):
        """Adds one render's ([P]) or one batch's ([V,P], view order) statistics."""
        if weight_sum.dim() == 1:
            weight_sum, weight_max = weight_sum.unsqueeze(0), weight_max.unsqueeze(0)
        if weight_sum.shape[-1] != self.weight_sum.shape[0]:
            raise ValueError("ContributionStats: %d Gaussians, the render has %d" % (self.weight_sum.shape[0], weight_sum.shape[-1]))
        with torch.no_grad():
            for v in range(weight_sum.shape[0]):
                self.weight_sum.add_(weight_sum[v])
                torch.maximum(self.weight_max, weight_max[v], out=self.weight_max)
        self.renders += int(weight_sum.shape[0])


def _add_contributions(contributions, state):
    """After a forward that ran with contrib: its statistics into `contributions`, and out of the state."""
    if contributions is not None:
        contributions.add(*state.contrib)
    state.contrib = None


def _raster_opts(antialiasing):
    """The DgrRasterOptions argument of the *_ex calls."""
    return ctypes.byref(_lib.DgrRasterOptions(_lib.RASTER_ANTIALIAS if antialiasing else 0))


def _backward_opts(antialiasing, camera, V, P, dev, absgrad=None):
    """The DgrRasterOptions argument of a backward *_ex call.  camera = (dL/dviewmatrix, dL/dprojmatrix, dL/dcampos) float32 outputs
    ([16], [16], [3] or [V,16], [V,16], [V,3]) or None; with them, DGR_RASTER_CAMERA_GRADS and its scratch (the returned pointer
    keeps the option structs alive, the scratch stays alive until the call returns).  absgrad = xyz_gradient_accum_abs float32 [P]
    or None; with it, DGR_RASTER_ABS_GRAD."""
    if camera is None and absgrad is None:
        return _raster_opts(antialiasing), None
    flags = _lib.RASTER_ANTIALIAS if antialiasing else 0
    cg, scratch = None, None
    if camera is not None:
        lib = _lib.load()
        scratch = torch.empty((lib.dgr_camera_grad_scratch_bytes(int(V), int(P)),), dtype=torch.uint8, device=dev)
        cg = ctypes.pointer(_lib.DgrCameraGrads(*(_ptr(t) for t in camera), _ptr(scratch), scratch.numel()))
        flags |= _lib.RASTER_CAMERA_GRADS
    if absgrad is not None:
        flags |= _lib.RASTER_ABS_GRAD
    opt = _lib.DgrRasterOptionsFull(flags, cg, _ptr(absgrad))
    return ctypes.cast(ctypes.pointer(opt), ctypes.POINTER(_lib.DgrRasterOptions)), scratch


# ---- camera gradients (DGR_RASTER_CAMERA_GRADS) -----------------------------------------------------------------------------
# The settings are a non-tensor argument of the autograd functions; when grad mode is on and a camera tensor of the settings
# requires grad, the calls below hand every view's (viewmatrix, projmatrix, campos) to the function as extra tensor inputs, and
# its backward returns their gradients (the C ABI's per-view [16] / [16] / [3]) in each tensor's own shape and dtype.
def _camera_tensors(settings_list):
    """() unless grad mode is on and some viewmatrix / projmatrix / campos of the settings requires grad; else every view's
    (viewmatrix, projmatrix, campos), flattened in view order."""
    if not torch.is_grad_enabled():
        return ()
    flat = tuple(t for s in settings_list for t in (s.viewmatrix, s.projmatrix, s.campos))
    if not any(isinstance(t, torch.Tensor) and t.requires_grad for t in flat):
        return ()
    return flat


def _camera_outputs(V, dev):
    """Output tensors of the camera gradients: [V,16], [V,16], [V,3] (V = 0: single view, [16], [16], [3])."""
    f32 = dict(dtype=torch.float32, device=dev)
    lead = (V,) if V else ()
    return torch.empty(lead + (16,), **f32), torch.empty(lead + (16,), **f32), torch.empty(lead + (3,), **f32)


def _camera_input_grads(cams, needs, grads):
    """grads = (dL/dviewmatrix, dL/dprojmatrix, dL/dcampos), per view or single -> the gradients of the flattened camera inputs
    `cams` (None where needs is False), each in its input's shape and dtype."""
    out = []
    for i, t in enumerate(cams):
        if not needs[i] or not isinstance(t, torch.Tensor):
            out.append(None)
            continue
        g = grads[i % 3]
        g = g.reshape(-1, g.shape[-1])[i // 3]
        out.append(g.reshape(t.shape).to(dtype=t.dtype, device=t.device))
    return out


class ForwardState:
    """Everything one forward leaves behind for its backward (upstream: ctx + geom/binning/img buffers)."""
    __slots__ = ("rs", "frame", "num_rendered", "capacity", "staging", "geom", "binning", "image", "radii", "alpha", "tensors",
                 "fast", "stats_applied", "antialiasing", "contrib")


def forward_impl(rs, means3D, sh, colors_precomp, opacities, scales, rotations, cov3D, sh_rest=None, activations=False,
                 antialiasing=False, contrib=False):
    """Runs both forward stages through the C ABI. Inputs are validated CUDA float32 tensors (or None).
    Returns (color, radii, depth, alpha, ForwardState).  antialiasing: the 2D Mip filter with opacity compensation
    (DGR_RASTER_ANTIALIAS, include/dgr_b200.h); the state remembers it for the backward.  contrib: the render also leaves the
    blending-weight statistics (DGR_RASTER_CONTRIB) of its last stage-2 run in state.contrib = (weight_sum, weight_max) [P]
    (None without it).

    No host round trip sits between the kernels: the instance buffer is sized from a per-shape capacity hint, every
    kernel of the forward is enqueued, and only then does the host wait for the (early) instance-count event.  If the
    guess was too small, stage 2 is re-run with a large enough buffer (the kernels clip safely to the capacity)."""
    if _FAST is not None:
        color, radii, depth, alpha, cst = _FAST.forward(
            int(rs.image_height), int(rs.image_width), float(rs.tanfovx), float(rs.tanfovy), float(rs.scale_modifier), int(rs.sh_degree),
            bool(rs.prefiltered), bool(rs.debug), rs.bg, rs.viewmatrix, rs.projmatrix, rs.campos, means3D, sh, colors_precomp, opacities,
            scales, rotations, cov3D, sh_rest, bool(activations), bool(antialiasing), bool(contrib))
        state = ForwardState()
        state.fast, state.rs, state.num_rendered, state.capacity = cst, rs, cst.num_rendered, cst.capacity
        state.contrib = (cst.weight_sum, cst.weight_max) if contrib else None
        state.antialiasing = bool(antialiasing)
        state.radii, state.alpha = radii, None
        state.tensors = (means3D, sh, colors_precomp, opacities, scales, rotations, cov3D, sh_rest)
        return color, radii, depth, alpha, state
    lib = _lib.load()
    dev = means3D.device
    with torch.cuda.device(dev):
        fr = _Frame(rs, means3D, sh, colors_precomp, opacities, scales, rotations, cov3D, sh_rest, activations)
        H, W, P = int(rs.image_height), int(rs.image_width), fr.P
        u8 = dict(dtype=torch.uint8, device=dev)
        color = torch.empty((3, H, W), dtype=torch.float32, device=dev)
        depth = torch.empty((1, H, W), dtype=torch.float32, device=dev)
        alpha = torch.empty((1, H, W), dtype=torch.float32, device=dev)
        radii = torch.empty((P,), dtype=torch.int32, device=dev)
        geom = torch.empty((lib.dgr_geom_bytes(P, H, W),), **u8)
        image = torch.empty((lib.dgr_image_bytes(H, W),), **u8)
        n_host, event = _host_sync_objects(dev)
        st = _stream_ptr(dev)
        _lib.check(lib.dgr_forward_preprocess_ex(ctypes.byref(fr.settings), ctypes.byref(fr.gaussians), _ptr(geom), _ptr(image),
                                                 _ptr(radii), _raster_opts(antialiasing), st))
        out = _lib.DgrImages(_ptr(color), _ptr(depth), _ptr(alpha), _ptr(radii))
        key = (dev.index, P, H, W)
        cap, big = _CAPACITY_HINT.get(key, (max(65536, 16 * P), True))
        rerun = 0
        copt, cout, _ckeep = _contrib_opts(contrib, P, dev)      # every stage-2 run rewrites it: the last run's values are kept
        while True:
            binning = torch.empty((lib.dgr_binning_bytes(cap, H, W),), **u8)
            args = (ctypes.byref(fr.settings), ctypes.byref(fr.gaussians), _ptr(geom), _ptr(binning), ctypes.c_uint64(cap), _ptr(image),
                    ctypes.byref(out), (1 if big else 0) | rerun, ctypes.c_void_p(n_host.data_ptr()), ctypes.c_uint64(0), event)
            if contrib:
                _lib.check(lib.dgr_forward_render_ex(*args, copt, st))
            else:
                _lib.check(lib.dgr_forward_render(*args, st))
            _lib.check(lib.dgr_event_synchronize(event))
            n_inst, n_big = int(n_host[0]), int(n_host[1])
            if n_inst <= cap and (big or n_big == 0):
                break
            cap = max(cap, int(n_inst * 1.25) + 4096)  # a guess was wrong: redo stage 2 (rare)
            big = big or n_big > 0
            rerun = 2                                   # DGR_FLAG_RERUN
        _CAPACITY_HINT[key] = (max(int(n_inst * 1.25) + 4096, 65536), n_big > 0)
    state = ForwardState()
    state.fast, state.antialiasing, state.contrib = None, bool(antialiasing), cout
    state.rs, state.frame, state.num_rendered, state.capacity = rs, fr, n_inst, cap
    state.staging = int(n_host[3])                  # record staging of the last stage-2 run: its backward must use the same
    # alpha is a differentiable OUTPUT: storing it here would close the cycle state -> alpha -> grad_fn -> ctx -> state and leave
    # ~100 MB of scratch per call to the cyclic garbage collector (the C ABI's out_alpha argument is unused)
    state.geom, state.binning, state.image, state.radii, state.alpha = geom, binning, image, radii, None
    state.tensors = (means3D, sh, colors_precomp, opacities, scales, rotations, cov3D, sh_rest)
    return color, radii, depth, alpha, state


_SYNC = {}
_CAPACITY_HINT = {}


def _host_sync_objects(dev):
    """(pinned uint64 for the instance count, cudaEvent handle) per (host thread, device)."""
    import threading
    key = (threading.get_ident(), dev.index)
    t = _SYNC.get(key)
    if t is None:
        ev = _lib.load().dgr_event_create()
        if not ev:
            raise RuntimeError("libdgr_b200: could not create a CUDA event")
        t = (torch.zeros((4,), dtype=torch.int64).pin_memory(), ctypes.c_void_p(ev))
        _SYNC[key] = t
    return t


def backward_impl(state, grad_color, grad_depth, grad_alpha, d_means3D, d_means2D, d_sh, d_col, d_opac, d_scales, d_rot,
                  d_cov, accumulate=False, d_sh_rest=None, densify=None, push=None, camera=None, absgrad=None):
    """Runs the backward through the C ABI, writing (or accumulating) into the given gradient tensors.
    densify = (xyz_gradient_accum, denom, max_radii2D) float32 [P] tensors (any may be None) updated in the same kernel.
    push = a _lib.DgrPeerPush (multi-GPU: rows of Gaussians another rank owns go straight to that rank, include/dgr_b200.h).
    camera = (dL/dviewmatrix [16], dL/dprojmatrix [16], dL/dcampos [3]) float32 tensors, written (never accumulated), or None.
    absgrad = xyz_gradient_accum_abs float32 [P], updated with the absolute-gradient statistic (DGR_RASTER_ABS_GRAD), or None."""
    push_addr = ctypes.addressof(push) if push is not None else 0
    if state.fast is not None:
        g = _FAST.backward(state.fast, grad_color, grad_depth, grad_alpha, bool(accumulate),
                           [d_means3D, d_means2D, d_sh, d_col, d_opac, d_scales, d_rot, d_cov, d_sh_rest], *(densify or (None, None, None)),
                           push_addr, camera=camera is not None, absgrad=absgrad)
        if camera is not None:
            for dst, src in zip(camera, g[9:12]):
                dst.copy_(src)
        return
    lib = _lib.load()
    fr = state.frame
    dev = state.radii.device
    with torch.cuda.device(dev):
        gin = _lib.DgrImageGrads(_ptr(grad_color), _ptr(grad_depth), _ptr(grad_alpha))
        gout = _lib.DgrGaussianGrads(_ptr(d_means3D), _ptr(d_means2D), _ptr(d_sh), _ptr(d_col), _ptr(d_opac), _ptr(d_scales),
                                     _ptr(d_rot), _ptr(d_cov), 1 if accumulate else 0, _ptr(d_sh_rest),
                                     *((_ptr(t) for t in densify) if densify is not None else (None, None, None)), push_addr or None)
        args = (ctypes.byref(fr.settings), ctypes.byref(fr.gaussians), _ptr(state.geom), _ptr(state.binning),
                ctypes.c_uint64(state.capacity), state.staging, _ptr(state.image), _ptr(state.radii), _ptr(state.alpha),
                ctypes.byref(gin), ctypes.byref(gout))
        opts, _scratch = _backward_opts(state.antialiasing, camera, 1, fr.P, dev, absgrad)
        if torch.are_deterministic_algorithms_enabled():
            det = _det_scratch(lib, state.num_rendered, fr.P, dev)
            _lib.check(lib.dgr_backward_det_ex(*args, *_det_args(det, state.num_rendered), opts, _stream_ptr(dev)))
        else:
            _lib.check(lib.dgr_backward_ex(*args, opts, _stream_ptr(dev)))


def _det_scratch(lib, instances, records, dev):
    """Scratch of the deterministic backward (dgr_*_backward_det), used when torch.use_deterministic_algorithms(True) is in effect
    (warn_only included) at the time the backward runs."""
    return torch.empty((lib.dgr_det_scratch_bytes(int(instances), int(records)),), dtype=torch.uint8, device=dev)


def _det_args(det, instances):
    return _ptr(det), ctypes.c_uint64(det.numel()), ctypes.c_uint64(int(instances))


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings,
                antialiasing=False, contributions=None, *cams):
        ctx.cams = cams                  # (viewmatrix, projmatrix, campos) when their gradient is asked for (_camera_tensors)
        means3D = _dev_f32(means3D, "means3D")
        opacities = _dev_f32(opacities, "opacities")
        sh, colors_precomp = _opt(sh, "shs"), _opt(colors_precomp, "colors_precomp")
        scales, rotations, cov3D = _opt(scales, "scales"), _opt(rotations, "rotations"), _opt(cov3Ds_precomp, "cov3D_precomp")
        color, radii, depth, alpha, state = forward_impl(raster_settings, means3D, sh, colors_precomp, opacities, scales,
                                                         rotations, cov3D, antialiasing=antialiasing, contrib=contributions is not None)
        _add_contributions(contributions, state)
        ctx.state = state
        ctx.mark_non_differentiable(radii)
        return color, radii, depth, alpha

    @staticmethod
    def backward(ctx, grad_color, grad_radii, grad_depth, grad_alpha):
        state = ctx.state
        cams = ctx.cams
        cam_needed = any(ctx.needs_input_grad[11:])
        if state.fast is not None:
            g = _FAST.backward(state.fast, grad_color, grad_depth, grad_alpha, False, [], None, None, None,
                               camera=cam_needed)      # undefined -> None
            cg = _camera_input_grads(cams, ctx.needs_input_grad[11:], g[9:12]) if cam_needed else [None] * len(cams)
            return (g[0], g[1], g[2], g[3], g[4], g[5], g[6], g[7], None, None, None, *cg)
        means3D, sh, colors_precomp, opacities, scales, rotations, cov3D, _ = state.tensors
        dev = means3D.device
        P, M = state.frame.P, state.frame.M
        f32 = dict(dtype=torch.float32, device=dev)
        gC = _dev_f32(grad_color, "grad_color") if grad_color is not None else None
        gD = _dev_f32(grad_depth, "grad_depth") if grad_depth is not None else None
        gA = _dev_f32(grad_alpha, "grad_alpha") if grad_alpha is not None else None
        d_means3D = torch.empty((P, 3), **f32)
        d_means2D = torch.empty((P, 3), **f32)
        d_opac = torch.empty((P, 1), **f32)
        d_sh = torch.empty((P, M, 3), **f32) if sh is not None else None
        d_col = torch.empty((P, 3), **f32) if colors_precomp is not None else None
        d_scales = torch.empty((P, 3), **f32) if scales is not None else None
        d_rot = torch.empty((P, 4), **f32) if rotations is not None else None
        d_cov = torch.empty((P, 6), **f32) if cov3D is not None else None
        camera = _camera_outputs(0, dev) if cam_needed else None
        backward_impl(state, gC, gD, gA, d_means3D, d_means2D, d_sh, d_col, d_opac, d_scales, d_rot, d_cov, camera=camera)
        cg = _camera_input_grads(cams, ctx.needs_input_grad[11:], camera) if cam_needed else [None] * len(cams)
        # ctx.state stays: a retain_graph backward runs again from the same buffers (they go away with the graph node)
        return (d_means3D, d_means2D, d_sh, d_col, d_opac, d_scales, d_rot, d_cov, None, None, None, *cg)


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings,
                        antialiasing=False, contributions=None):
    """antialiasing=True: the 2D Mip filter with opacity compensation (Mip-Splatting), DGR_RASTER_ANTIALIAS of include/dgr_b200.h.
    A viewmatrix / projmatrix / campos of raster_settings that requires grad receives its gradient (DGR_RASTER_CAMERA_GRADS).
    contributions (ContributionStats): the forward adds this render's blending-weight statistics to it (DGR_RASTER_CONTRIB)."""
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                                     raster_settings, bool(antialiasing), contributions, *_camera_tensors([raster_settings]))


class GaussianRasterizer(nn.Module):
    """Constructed per render call by the reference (gs_renderer.py:760): construction is trivial.  antialiasing=True renders
    with the 2D Mip filter and opacity compensation (include/dgr_b200.h, DGR_RASTER_ANTIALIAS); the settings keep their 12 fields.
    contributions (ContributionStats): every forward adds its blending-weight statistics to it (DGR_RASTER_CONTRIB)."""

    def __init__(self, raster_settings: GaussianRasterizationSettings, antialiasing: bool = False, contributions=None):
        super().__init__()
        self.raster_settings = raster_settings
        self.antialiasing = bool(antialiasing)
        self.contributions = contributions

    def markVisible(self, positions):
        with torch.no_grad():
            rs = self.raster_settings
            lib = _lib.load()
            pos = _dev_f32(positions, "positions")
            view, proj = _dev_f32(rs.viewmatrix, "viewmatrix"), _dev_f32(rs.projmatrix, "projmatrix")
            present = torch.empty((pos.shape[0],), dtype=torch.uint8, device=pos.device)
            with torch.cuda.device(pos.device):
                _lib.check(lib.dgr_mark_visible(pos.shape[0], _ptr(pos), _ptr(view), _ptr(proj), _ptr(present), _stream_ptr(pos.device)))
            return present.bool()

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None):
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception("Please provide excatly one of either SHs or precomputed colors!")
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp,
                                   self.raster_settings, self.antialiasing, self.contributions)


# ---------------------------------------------------------------------------------------------------------------------------
# Batched cameras: one cloud, V views of the same image size in one forward / backward (include/dgr_b200.h, DgrViews).
# ---------------------------------------------------------------------------------------------------------------------------
def get_views_capacity_hint(device_index, P, H, W, V):
    """Instance-capacity hint of the batched call, kept apart from the single-view hints."""
    if _FAST is not None:
        return _FAST.get_views_hint(device_index, P, H, W, V)
    return _CAPACITY_HINT.get(("views", device_index, P, H, W, V))


def set_views_capacity_hint(device_index, P, H, W, V, cap, big):
    if _FAST is not None:
        _FAST.set_views_hint(device_index, P, H, W, V, cap, big)
    else:
        _CAPACITY_HINT[("views", device_index, P, H, W, V)] = (cap, big)


_MAX_CAPACITY = 2 ** 32 - 2          # tile-instance positions are 32-bit in the kernels


def _views_capacity_ceiling(lib, dev, V, H, W):
    """Largest instance capacity a batched call sizes its binning buffer for: the kernels' 32-bit positions, and half the free
    device memory (the first-call guess of 16 instances per record would ask for tens of GB at 64 views x 1M Gaussians)."""
    free, _ = torch.cuda.mem_get_info(dev)
    per = max(1, lib.dgr_views_binning_bytes(1 << 20, V, H, W) >> 20)
    return min(_MAX_CAPACITY, max(65536, (free // 2) // per))


def get_views_mixed_capacity_hint(device_index, P, sizes):
    """Instance-capacity hint of the mixed-size batched call, keyed by the tuple of (height, width) sizes."""
    sizes = tuple((int(h), int(w)) for h, w in sizes)
    if _FAST is not None:
        return _FAST.get_views_mixed_hint(device_index, P, [x for hw in sizes for x in hw])
    return _CAPACITY_HINT.get(("views_mixed", device_index, P, sizes))


def set_views_mixed_capacity_hint(device_index, P, sizes, cap, big):
    sizes = tuple((int(h), int(w)) for h, w in sizes)
    if _FAST is not None:
        _FAST.set_views_mixed_hint(device_index, P, [x for hw in sizes for x in hw], cap, big)
    else:
        _CAPACITY_HINT[("views_mixed", device_index, P, sizes)] = (cap, big)


def _check_views_settings(settings_list, fields=("image_height", "image_width", "sh_degree", "scale_modifier"), what="rasterize_views"):
    settings_list = list(settings_list)
    if not settings_list:
        raise ValueError("%s needs at least one camera" % what)
    if len(settings_list) > _lib.VIEWS_MAX:
        raise ValueError("%s takes at most %d cameras per call, got %d" % (what, _lib.VIEWS_MAX, len(settings_list)))
    s0 = settings_list[0]
    for i, s in enumerate(settings_list[1:], 1):
        for f in fields:
            if getattr(s, f) != getattr(s0, f):
                raise ValueError("%s: every camera of a batch must share %s (camera 0 has %r, camera %d has %r)"
                                 % (what, f, getattr(s0, f), i, getattr(s, f)))
    return settings_list


def _check_views_mixed_settings(settings_list):
    """The cameras of a mixed-size batch: any image sizes, one sh_degree and scale_modifier."""
    return _check_views_settings(settings_list, ("sh_degree", "scale_modifier"), "rasterize_views_mixed")


def _stats_mask(stats_views, V):
    """View indices -> the stats_views bit mask of dgr_views_mixed_backward."""
    mask = 0
    for v in stats_views:
        v = int(v)
        if v < 0 or v >= V:
            raise ValueError("stats_views: view %d is not in the batch of %d views" % (v, V))
        mask |= 1 << v
    return mask


def _views_cameras(settings_list, dev):
    """The per-view device arrays of a batch: tanfov [V,2], bg [V,3], viewmatrix [V,16], projmatrix [V,16], campos [V,3]."""
    stack = lambda name: torch.stack([_dev_f32(getattr(s, name), name).reshape(-1) for s in settings_list]).to(dev)
    bg, view, proj, campos = stack("bg"), stack("viewmatrix"), stack("projmatrix"), stack("campos")
    if bg.shape[1] != 3 or view.shape[1] != 16 or proj.shape[1] != 16 or campos.shape[1] != 3:
        raise ValueError("bg/campos must have 3 elements, viewmatrix/projmatrix 16")
    tanfov = torch.tensor([[float(s.tanfovx), float(s.tanfovy)] for s in settings_list], dtype=torch.float32, device=dev)
    return tanfov, bg, view, proj, campos


class _Views:
    """ctypes views of one batched call's cameras + inputs (keeps the tensors alive)."""

    def __init__(self, settings_list, means3D, sh, opacities, scales, rotations, sh_rest=None, activations=False, mixed=False):
        dev = means3D.device
        s0 = settings_list[0]
        V = len(settings_list)
        self.tanfov, self.bg, self.view, self.proj, self.campos = _views_cameras(settings_list, dev)
        self.keep = [self.bg, self.view, self.proj, self.campos, self.tanfov]
        self.V, self.H, self.W = V, int(s0.image_height), int(s0.image_width)
        # mixed sizes: the host [V,2] (height, width) array the dgr_views_mixed_* calls take
        self.sizes = tuple((int(s.image_height), int(s.image_width)) for s in settings_list)
        self.hw = (ctypes.c_int32 * (2 * V))(*[x for hw in self.sizes for x in hw]) if mixed else None
        self.settings = _lib.DgrViews(V, self.H, self.W, float(s0.scale_modifier), int(s0.sh_degree), int(bool(s0.debug)),
                                      _ptr(self.tanfov), _ptr(self.bg), _ptr(self.view), _ptr(self.proj), _ptr(self.campos))
        # the per-Gaussian checks of the single-view call (shapes, raw-parameter layout)
        fr = _Frame(s0, means3D, sh, None, opacities, scales, rotations, None, sh_rest, activations)
        self.P, self.M, self.gaussians = fr.P, fr.M, fr.gaussians
        self.keep.append(fr)


class ViewsState:
    """Everything one batched forward leaves behind for its backward."""
    __slots__ = ("views", "capacity", "staging", "num_rendered", "geom", "binning", "image", "radii", "tensors", "fast", "mixed",
                 "stats_applied", "antialiasing", "contrib")


def views_forward_impl(settings_list, means3D, sh, opacities, scales, rotations, sh_rest=None, activations=False, mixed=False,
                       antialiasing=False, contrib=False):
    """Both forward stages of the batched call through the C ABI; inputs are validated CUDA float32 tensors.
    Returns (color [V,3,H,W], radii [V,P], depth [V,1,H,W], alpha [V,1,H,W], ViewsState).  Same speculative-capacity
    protocol as forward_impl, with hints keyed by (device, P, H, W, V); the compiled host layer when it is loaded.
    mixed=True: every camera has its own image size (dgr_views_mixed_*); color [sum 3 H_v W_v], depth / alpha [sum H_v W_v]
    are flat, view v's blocks one after the other, and the hints are keyed by (device, P, the sizes).  antialiasing: as forward_impl.
    contrib: as forward_impl, state.contrib = (weight_sum, weight_max) [V,P]."""
    lib = _lib.load()
    dev = means3D.device
    if _FAST is not None:
        s0 = settings_list[0]
        with torch.cuda.device(dev):
            cams = _views_cameras(settings_list, dev)
        if mixed:
            hw = [int(x) for s in settings_list for x in (s.image_height, s.image_width)]
            color, radii, depth, alpha, cst = _FAST.views_mixed_forward(
                hw, float(s0.scale_modifier), int(s0.sh_degree), bool(s0.debug), *cams, means3D, sh, opacities, scales, rotations, sh_rest,
                bool(activations), bool(antialiasing), bool(contrib))
        else:
            color, radii, depth, alpha, cst = _FAST.views_forward(
                int(s0.image_height), int(s0.image_width), float(s0.scale_modifier), int(s0.sh_degree), bool(s0.debug), *cams,
                means3D, sh, opacities, scales, rotations, sh_rest, bool(activations), bool(antialiasing), bool(contrib))
        state = ViewsState()
        state.contrib = (cst.weight_sum, cst.weight_max) if contrib else None
        state.fast, state.capacity, state.num_rendered, state.radii = cst, cst.capacity, cst.num_rendered, radii
        state.tensors = (means3D, sh, opacities, scales, rotations, sh_rest)
        state.mixed, state.antialiasing = mixed, bool(antialiasing)
        return color, radii, depth, alpha, state
    with torch.cuda.device(dev):
        vw = _Views(settings_list, means3D, sh, opacities, scales, rotations, sh_rest, activations, mixed=mixed)
        V, H, W, P = vw.V, vw.H, vw.W, vw.P
        u8 = dict(dtype=torch.uint8, device=dev)
        f32 = dict(dtype=torch.float32, device=dev)
        if mixed:
            pix = sum(h * w for h, w in vw.sizes)
            color, depth, alpha = torch.empty((3 * pix,), **f32), torch.empty((pix,), **f32), torch.empty((pix,), **f32)
        else:
            color, depth, alpha = torch.empty((V, 3, H, W), **f32), torch.empty((V, 1, H, W), **f32), torch.empty((V, 1, H, W), **f32)
        radii = torch.empty((V, P), dtype=torch.int32, device=dev)
        n_host, event = _host_sync_objects(dev)
        st = _stream_ptr(dev)
        if mixed:
            geom = torch.empty((max(1, lib.dgr_views_mixed_geom_bytes(V, P, vw.hw)),), **u8)
            image = torch.empty((max(1, lib.dgr_views_mixed_image_bytes(V, vw.hw)),), **u8)
            _lib.check(lib.dgr_views_mixed_forward_preprocess_ex(ctypes.byref(vw.settings), vw.hw, ctypes.byref(vw.gaussians), _ptr(geom),
                                                                 _ptr(image), _ptr(radii), _raster_opts(antialiasing), st))
            key = ("views_mixed", dev.index, P, vw.sizes)
        else:
            geom = torch.empty((lib.dgr_views_geom_bytes(V, P, H, W),), **u8)
            image = torch.empty((lib.dgr_views_image_bytes(V, H, W),), **u8)
            _lib.check(lib.dgr_views_forward_preprocess_ex(ctypes.byref(vw.settings), ctypes.byref(vw.gaussians), _ptr(geom), _ptr(image),
                                                           _ptr(radii), _raster_opts(antialiasing), st))
            key = ("views", dev.index, P, H, W, V)
        out = _lib.DgrImages(_ptr(color), _ptr(depth), _ptr(alpha), _ptr(radii))
        ceiling = _views_capacity_ceiling(lib, dev, V, H, W)
        cap, big = _CAPACITY_HINT.get(key, (min(max(65536, 16 * P * V), ceiling), True))
        rerun = 0
        copt, cout, _ckeep = _contrib_opts(contrib, V * P, dev)
        while True:
            binning = torch.empty((lib.dgr_views_binning_bytes(cap, V, H, W),), **u8)
            args = (ctypes.byref(vw.gaussians), _ptr(geom), _ptr(binning), ctypes.c_uint64(cap), _ptr(image), ctypes.byref(out),
                    (1 if big else 0) | rerun, ctypes.c_void_p(n_host.data_ptr()), ctypes.c_uint64(0), event)
            if mixed and contrib:
                _lib.check(lib.dgr_views_mixed_forward_render_ex(ctypes.byref(vw.settings), vw.hw, *args, copt, st))
            elif mixed:
                _lib.check(lib.dgr_views_mixed_forward_render(ctypes.byref(vw.settings), vw.hw, *args, st))
            elif contrib:
                _lib.check(lib.dgr_views_forward_render_ex(ctypes.byref(vw.settings), *args, copt, st))
            else:
                _lib.check(lib.dgr_views_forward_render(ctypes.byref(vw.settings), *args, st))
            _lib.check(lib.dgr_event_synchronize(event))
            n_inst, n_big = int(n_host[0]), int(n_host[1])
            if n_inst <= cap and (big or n_big == 0):
                break
            if n_inst > _MAX_CAPACITY:
                raise RuntimeError("libdgr_b200: the batch has %d tile instances, above the 2^32-1 the kernels address" % n_inst)
            cap = min(max(cap, int(n_inst * 1.25) + 4096), _MAX_CAPACITY)
            big = big or n_big > 0
            rerun = 2                                   # DGR_FLAG_RERUN
        _CAPACITY_HINT[key] = (min(max(int(n_inst * 1.25) + 4096, 65536), _MAX_CAPACITY), n_big > 0)
    state = ViewsState()
    state.fast, state.mixed, state.antialiasing = None, mixed, bool(antialiasing)
    state.contrib = (cout[0].view(V, P), cout[1].view(V, P)) if contrib else None
    state.views, state.capacity, state.staging, state.num_rendered = vw, cap, int(n_host[3]), n_inst
    state.geom, state.binning, state.image, state.radii = geom, binning, image, radii
    state.tensors = (means3D, sh, opacities, scales, rotations, sh_rest)
    return color, radii, depth, alpha, state


def views_backward_impl(state, grad_color, grad_depth, grad_alpha, d_means3D, d_means2D, d_sh, d_opac, d_scales, d_rot,
                        accumulate=False, d_sh_rest=None, densify=None, stats_views=0, camera=None, absgrad=None):
    """Backward of a batched forward: the per-Gaussian gradients are the sums over the views (written, or added with
    accumulate); d_means2D is per view, [V,P,3].  Mixed-size forwards only: densify = (xyz_gradient_accum, denom, max_radii2D)
    float32 [P] tensors (any may be None), updated for the views whose bit is set in the stats_views mask, and absgrad =
    xyz_gradient_accum_abs float32 [P] (DGR_RASTER_ABS_GRAD) or None, updated for the same views.
    camera = (dL/dviewmatrix [V,16], dL/dprojmatrix [V,16], dL/dcampos [V,3]) float32 tensors, each view's own, or None."""
    if state.fast is not None:
        outs = [d_means3D, d_means2D, d_sh, d_opac, d_scales, d_rot, d_sh_rest]
        if state.mixed:
            g = _FAST.views_mixed_backward(state.fast, grad_color, grad_depth, grad_alpha, bool(accumulate), outs,
                                           *(densify or (None, None, None)), int(stats_views), camera=camera is not None, absgrad=absgrad)
        else:
            g = _FAST.views_backward(state.fast, grad_color, grad_depth, grad_alpha, bool(accumulate), outs, camera=camera is not None)
        if camera is not None:
            for dst, src in zip(camera, g[7:10]):
                dst.copy_(src)
        return
    lib = _lib.load()
    vw = state.views
    dev = state.radii.device
    with torch.cuda.device(dev):
        gin = _lib.DgrImageGrads(_ptr(grad_color), _ptr(grad_depth), _ptr(grad_alpha))
        gout = _lib.DgrGaussianGrads(_ptr(d_means3D), _ptr(d_means2D), _ptr(d_sh), None, _ptr(d_opac), _ptr(d_scales), _ptr(d_rot),
                                     None, 1 if accumulate else 0, _ptr(d_sh_rest),
                                     *((_ptr(t) for t in densify) if densify is not None else (None, None, None)), None)
        common = (ctypes.byref(vw.gaussians), _ptr(state.geom), _ptr(state.binning), ctypes.c_uint64(state.capacity), state.staging,
                  _ptr(state.image), _ptr(state.radii), ctypes.byref(gin), ctypes.byref(gout))
        opts, _scratch = _backward_opts(state.antialiasing, camera, vw.V, vw.P, dev, absgrad)
        if torch.are_deterministic_algorithms_enabled():
            det = _det_scratch(lib, state.num_rendered, vw.P * vw.V, dev)
            if state.mixed:
                _lib.check(lib.dgr_views_mixed_backward_det_ex(ctypes.byref(vw.settings), vw.hw, *common, ctypes.c_uint64(stats_views),
                                                               *_det_args(det, state.num_rendered), opts, _stream_ptr(dev)))
            else:
                _lib.check(lib.dgr_views_backward_det_ex(ctypes.byref(vw.settings), *common, *_det_args(det, state.num_rendered), opts,
                                                         _stream_ptr(dev)))
            return
        if state.mixed:
            _lib.check(lib.dgr_views_mixed_backward_ex(ctypes.byref(vw.settings), vw.hw, *common, ctypes.c_uint64(stats_views), opts,
                                                       _stream_ptr(dev)))
        else:
            _lib.check(lib.dgr_views_backward_ex(ctypes.byref(vw.settings), *common, opts, _stream_ptr(dev)))


def _views_grads(state, grad_color, grad_depth, grad_alpha, raw, stats=None, stats_views=0, camera=False):
    """-> (means3D, means2D [V,P,3], shs | features_dc, features_rest, opacities, scales, rotations) gradients, and with camera=True
    also (dL/dviewmatrix [V,16], dL/dprojmatrix [V,16], dL/dcampos [V,3]) as an 8th element.
    stats (DensifyStats) / stats_views (bit mask): the densification statistics of a mixed-size forward (with the absolute-gradient
    one when stats carries it)."""
    densify = stats.as_tuple() if stats is not None else None
    absgrad = stats.xyz_gradient_accum_abs if stats is not None else None
    if state.fast is not None:
        if state.mixed:
            g = _FAST.views_mixed_backward(state.fast, grad_color, grad_depth, grad_alpha, False, [], *(densify or (None, None, None)),
                                           int(stats_views) if densify is not None else 0, camera=bool(camera), absgrad=absgrad)
        else:
            g = _FAST.views_backward(state.fast, grad_color, grad_depth, grad_alpha, False, [], camera=bool(camera))   # undefined -> None
        out = (g[0], g[1], g[2], g[6], g[3], g[4], g[5])
        return out + (tuple(g[7:10]),) if camera else out
    means3D, sh, opacities, scales, rotations, sh_rest = state.tensors
    vw = state.views
    P, M, V = vw.P, vw.M, vw.V
    f32 = dict(dtype=torch.float32, device=means3D.device)
    gC = _dev_f32(grad_color, "grad_color") if grad_color is not None else None
    gD = _dev_f32(grad_depth, "grad_depth") if grad_depth is not None else None
    gA = _dev_f32(grad_alpha, "grad_alpha") if grad_alpha is not None else None
    d_means3D, d_means2D, d_opac = torch.empty((P, 3), **f32), torch.empty((V, P, 3), **f32), torch.empty((P, 1), **f32)
    d_sh = torch.empty((P, 1 if raw else M, 3), **f32)
    d_rest = torch.empty(sh_rest.shape, **f32) if (raw and sh_rest is not None) else None
    d_scales, d_rot = torch.empty((P, 3), **f32), torch.empty((P, 4), **f32)
    cam = _camera_outputs(V, means3D.device) if camera else None
    views_backward_impl(state, gC, gD, gA, d_means3D, d_means2D, d_sh, d_opac, d_scales, d_rot, d_sh_rest=d_rest, densify=densify,
                        stats_views=stats_views if densify is not None else 0, camera=cam, absgrad=absgrad)
    out = (d_means3D, d_means2D, d_sh, d_rest, d_opac, d_scales, d_rot)
    return out + (cam,) if camera else out


def _views_backward_with_cameras(ctx, grad_color, grad_depth, grad_alpha, raw, first_cam, **kw):
    """_views_grads for a batched autograd function whose camera inputs (if any) start at input index first_cam -> (the 7
    per-Gaussian gradients, the list of camera-input gradients)."""
    needs = ctx.needs_input_grad[first_cam:]
    cam_needed = any(needs)
    r = _views_grads(ctx.state, grad_color, grad_depth, grad_alpha, raw=raw, camera=cam_needed, **kw)
    cg = _camera_input_grads(ctx.cams, needs, r[7]) if cam_needed else [None] * len(ctx.cams)
    return r[:7], cg


class _RasterizeViews(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, opacities, scales, rotations, settings_list, antialiasing=False, contributions=None, *cams):
        ctx.cams = cams
        means3D, opacities = _dev_f32(means3D, "means3D"), _dev_f32(opacities, "opacities")
        sh, scales, rotations = _dev_f32(sh, "shs"), _dev_f32(scales, "scales"), _dev_f32(rotations, "rotations")
        color, radii, depth, alpha, state = views_forward_impl(settings_list, means3D, sh, opacities, scales, rotations,
                                                               antialiasing=antialiasing, contrib=contributions is not None)
        _add_contributions(contributions, state)
        ctx.state = state
        ctx.mark_non_differentiable(radii)
        return color, radii, depth, alpha

    @staticmethod
    def backward(ctx, grad_color, grad_radii, grad_depth, grad_alpha):
        (d_means3D, d_means2D, d_sh, _, d_opac, d_scales, d_rot), cg = _views_backward_with_cameras(ctx, grad_color, grad_depth, grad_alpha,
                                                                                                      False, 9)
        # ctx.state stays: a retain_graph backward runs again from the same buffers.  means2D may be None (no per-view gradient wanted)
        return (d_means3D, d_means2D if ctx.needs_input_grad[1] else None, d_sh, d_opac, d_scales, d_rot, None, None, None, *cg)


def rasterize_views(settings_list, means3D, means2D, opacities, shs, scales, rotations, antialiasing=False, contributions=None):
    """Renders ONE cloud from every camera of `settings_list` (GaussianRasterizationSettings, at most 64, all with the same
    image_height / image_width / sh_degree / scale_modifier) in one batched forward, and one batched backward.
    Returns (color [V,3,H,W], radii int32 [V,P], depth [V,1,H,W], alpha [V,1,H,W]); view v equals what GaussianRasterizer
    returns for camera v.  The gradients of means3D / shs / opacities / scales / rotations are summed over the views;
    means2D is [V,P,3] (e.g. zeros with requires_grad) or None: its gradient is per view, for densification.  SH colours and
    scale / rotation inputs only; no CPU path.  antialiasing: as GaussianRasterizer.  A camera tensor of a settings entry that
    requires grad receives that view's own gradient (DGR_RASTER_CAMERA_GRADS).  contributions (ContributionStats): the forward adds
    every view's blending-weight statistics to it, in view order (DGR_RASTER_CONTRIB)."""
    settings_list = _check_views_settings(settings_list)
    if means2D is not None and tuple(means2D.shape) != (len(settings_list), means3D.shape[0], 3):
        raise ValueError("means2D must have dimensions (num_views, num_points, 3)")
    return _RasterizeViews.apply(means3D, means2D, shs, opacities, scales, rotations, settings_list, bool(antialiasing), contributions,
                                 *_camera_tensors(settings_list))


class GaussianViewsRasterizer(nn.Module):
    """`GaussianRasterizer` for a batch of same-size cameras: forward(means3D, means2D, opacities, shs, scales, rotations)
    -> (color [V,3,H,W], radii [V,P], depth [V,1,H,W], alpha [V,1,H,W]), see rasterize_views."""

    def __init__(self, settings_list, antialiasing=False, contributions=None):
        super().__init__()
        self.settings_list = _check_views_settings(settings_list)
        self.antialiasing = bool(antialiasing)
        self.contributions = contributions

    def forward(self, means3D, means2D, opacities, shs, scales, rotations):
        return rasterize_views(self.settings_list, means3D, means2D, opacities, shs, scales, rotations, self.antialiasing,
                               self.contributions)


# ---------------------------------------------------------------------------------------------------------------------------
# Batched cameras of different image sizes: one cloud, V views, each with its own size (include/dgr_b200.h, dgr_views_mixed_*).
# ---------------------------------------------------------------------------------------------------------------------------
def split_views(settings_list, color, depth, alpha):
    """The flat outputs of a mixed-size call -> per-view lists: colour [3,H_v,W_v], depth / alpha [1,H_v,W_v] (views of the flat
    tensors, so gradients flow back into them)."""
    colors, depths, alphas, off = [], [], [], 0
    for s in settings_list:
        h, w = int(s.image_height), int(s.image_width)
        colors.append(color.narrow(0, 3 * off, 3 * h * w).view(3, h, w))
        depths.append(depth.narrow(0, off, h * w).view(1, h, w))
        alphas.append(alpha.narrow(0, off, h * w).view(1, h, w))
        off += h * w
    return colors, depths, alphas


class _RasterizeViewsMixed(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, opacities, scales, rotations, settings_list, antialiasing=False, contributions=None, *cams):
        ctx.cams = cams
        means3D, opacities = _dev_f32(means3D, "means3D"), _dev_f32(opacities, "opacities")
        sh, scales, rotations = _dev_f32(sh, "shs"), _dev_f32(scales, "scales"), _dev_f32(rotations, "rotations")
        color, radii, depth, alpha, state = views_forward_impl(settings_list, means3D, sh, opacities, scales, rotations, mixed=True,
                                                               antialiasing=antialiasing, contrib=contributions is not None)
        _add_contributions(contributions, state)
        ctx.state = state
        ctx.mark_non_differentiable(radii)
        return color, radii, depth, alpha

    @staticmethod
    def backward(ctx, grad_color, grad_radii, grad_depth, grad_alpha):
        (d_means3D, d_means2D, d_sh, _, d_opac, d_scales, d_rot), cg = _views_backward_with_cameras(ctx, grad_color, grad_depth, grad_alpha,
                                                                                                      False, 9)
        return (d_means3D, d_means2D if ctx.needs_input_grad[1] else None, d_sh, d_opac, d_scales, d_rot, None, None, None, *cg)


def rasterize_views_mixed(settings_list, means3D, means2D, opacities, shs, scales, rotations, antialiasing=False, contributions=None):
    """rasterize_views for cameras of DIFFERENT image sizes (at most 64, one sh_degree / scale_modifier): one batched forward
    and one batched backward.  Returns (colors, radii, depths, alphas): colors a list of [3,H_v,W_v], depths / alphas lists of
    [1,H_v,W_v] (views of one flat tensor each), radii int32 [V,P]; view v equals what GaussianRasterizer returns for camera v.
    The gradients of means3D / shs / opacities / scales / rotations are summed over the views; means2D is [V,P,3] or None.
    antialiasing, contributions: as rasterize_views."""
    settings_list = _check_views_mixed_settings(settings_list)
    if means2D is not None and tuple(means2D.shape) != (len(settings_list), means3D.shape[0], 3):
        raise ValueError("means2D must have dimensions (num_views, num_points, 3)")
    color, radii, depth, alpha = _RasterizeViewsMixed.apply(means3D, means2D, shs, opacities, scales, rotations, settings_list,
                                                            bool(antialiasing), contributions, *_camera_tensors(settings_list))
    colors, depths, alphas = split_views(settings_list, color, depth, alpha)
    return colors, radii, depths, alphas
