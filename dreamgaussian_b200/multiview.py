"""View-sharded data parallelism for the rasterizer path (SURVEY.md §8e).

The reference loops over views sequentially and sums their losses (/root/reference/main.py:219-255); each view's
rasterisation is independent given the Gaussian parameters.  Here the Gaussians are replicated on every GPU, the views
of one iteration are split across ranks (one process per GPU), every rank accumulates the per-Gaussian gradients of its
local views into ONE flat float32 buffer — the backward kernels add straight into it (DgrGaussianGrads.accumulate), so
there is no pack step — and a single NCCL all-reduce(sum) over NVLink makes the buffer identical on all ranks.

Flat layout (floats): [means3D 3P | shs 3MP | opacities P | scales 3P | rotations 4P | means2D 3P].
"""
import ctypes
import os
from typing import List, Optional, Sequence

import torch

from . import rasterizer as _r


class FlatGrads:
    """One contiguous gradient buffer with typed views for every op input.

    symmetric=True allocates it in symmetric (peer-mapped) memory so the ranks can reduce it with the library's own
    NVLink kernel; the buffer is padded to a multiple of 64 floats so it splits into float4 slices for any world size."""

    def __init__(self, P: int, M: int, device, with_means2D: bool = True, symmetric: bool = False, flag_floats: int = 0,
                 stage_slots: int = 0):
        self.P, self.M = P, M
        sizes = [("means3D", 3 * P, (P, 3)), ("shs", 3 * M * P, (P, M, 3)), ("opacities", P, (P, 1)),
                 ("scales", 3 * P, (P, 3)), ("rotations", 4 * P, (P, 4))]
        if with_means2D:
            sizes.append(("means2D", 3 * P, (P, 3)))
        total = sum(n for _, n, _ in sizes)
        self.numel = total
        padded = (total + 63) // 64 * 64
        self.padded = padded
        if symmetric:
            import torch.distributed._symmetric_memory as symm_mem
            # [gradient data | cross-rank barrier flags of the collective kernels | staging area: one flat-buffer-sized slot per
            # source rank, where the other ranks' backward kernels push the rows this rank owns]: one symmetric allocation
            self.storage = symm_mem.empty(padded + flag_floats + stage_slots * padded, dtype=torch.float32, device=device)
            self.storage.zero_()
            self.stage_offset = padded + flag_floats
        else:
            self.storage = torch.zeros((padded,), dtype=torch.float32, device=device)
        self.data = self.storage[:padded]                 # what the all-reduce covers
        self.flat = self.storage[:total]
        self.views = {}
        self.segments = []                                # (offset in floats, floats per Gaussian) of every [P, stride] segment
        o = 0
        for name, n, shape in sizes:
            self.views[name] = self.flat[o:o + n].view(shape)
            self.segments.append((o, n // P if P else 0))
            o += n
        if not with_means2D:
            self.views["means2D"] = None

    def nbytes(self):
        return self.flat.numel() * 4


class ViewShardedRasterizer:
    """Forward + backward of this rank's views with gradient accumulation, then one all-reduce.

    params: dict(means3D, shs, opacities, scales, rotations) of CUDA float32 tensors (replicated on every rank).
    The cameras are constants here: unlike the autograd render calls, this path computes no camera gradients.
    """

    def __init__(self, P: int, M: int, device, process_group=None, peer_allreduce: bool = True):
        import torch.distributed as dist
        self.device = torch.device(device)
        self.pg = process_group
        self.collective = "none"
        self._hdl = None
        self._use_push = False
        self._pushed = False
        multi = dist.is_available() and dist.is_initialized() and dist.get_world_size(process_group) > 1
        if os.environ.get("DGR_NO_PEER") == "1":          # A/B switch: plain NCCL all_reduce instead of the library's kernels
            peer_allreduce = False
        if multi and peer_allreduce and self.device.type == "cuda":
            # the gradient buffer in symmetric memory + this library's NVLink all-reduce kernel; NCCL is the fallback
            try:
                import torch.distributed._symmetric_memory as symm_mem
                from . import _lib
                flag_floats = int(_lib.load().dgr_peer_flag_bytes()) // 4
                world = dist.get_world_size(process_group)
                # DGR_PUSH=1 (opt-in): the reduce-scatter half fused into the last local backward (rows of other owners stored
                # straight into the owner's staging area) + dgr_peer_reduce_staged, instead of the two-shot all-reduce kernel.
                # Measured slower at 2 GPUs (the backward kernel is a single wave: the pushes do not overlap its arithmetic).
                self._use_push = os.environ.get("DGR_PUSH") == "1" and P > 0
                self.grads = FlatGrads(P, M, self.device, symmetric=True, flag_floats=flag_floats,
                                       stage_slots=world if self._use_push else 0)
                group = process_group if process_group is not None else dist.group.WORLD
                self._hdl = symm_mem.rendezvous(self.grads.storage, group)
                mc = int(getattr(self._hdl, "multicast_ptr", 0) or 0)
                self._mc = mc if (mc and os.environ.get("DGR_NO_MULTIMEM") != "1") else 0
                self._ptrs = (ctypes.c_uint64 * len(self._hdl.buffer_ptrs))(*[int(p) for p in self._hdl.buffer_ptrs])
                # the flag area follows the gradient data in every rank's copy.  DGR_INKERNEL_BARRIERS=1: the all-reduce kernel
                # carries its own two cross-rank barriers (no extra launches); default: symmetric-memory barriers around it
                self._flags = (ctypes.c_uint64 * len(self._hdl.buffer_ptrs))(*[int(p) + 4 * self.grads.padded for p in self._hdl.buffer_ptrs])
                self._inkernel = os.environ.get("DGR_INKERNEL_BARRIERS", "1") == "1"
                self._epoch = 0
                self._pushed = False
                if self._use_push:
                    self._setup_push(P, world)
                self._hdl.barrier(channel=0)              # every rank has zeroed its flags before anyone signals
                self.collective = "own kernel: multimem (NVLS)" if self._mc else "own kernel: p2p two-shot"
                if self._use_push:
                    self.collective = "push fused into the backward + own reduce/publish kernel: " + ("multimem.st (NVLS)" if self._mc else "peer stores")
                if self._mc and os.environ.get("DGR_FORCE_MULTIMEM") != "1":
                    self._autotune(group)
            except Exception as e:          # no symmetric memory on this system / backend
                self._hdl = None
                self._why_nccl = repr(e)
        if self._hdl is None:
            self.grads = FlatGrads(P, M, self.device)
            if multi:
                self.collective = "nccl all_reduce" if self.device.type == "cuda" else "gloo all_reduce"

    def _setup_push(self, P, world):
        """Ownership of the Gaussians (rank g // per, per a multiple of the backward kernel's 256-thread block) and, for every
        owner, where this rank's rows land in that owner's staging area (include/dgr_b200.h: DgrPeerPush)."""
        from . import _lib
        rank = self._hdl.rank
        per = (-(-P // world) + 255) // 256 * 256
        push = _lib.DgrPeerPush()
        push.world, push.rank, push.gaussians_per_owner = world, rank, per
        local = int(self._hdl.buffer_ptrs[rank])
        for o in range(world):
            slot = int(self._hdl.buffer_ptrs[o]) + 4 * (self.grads.stage_offset + rank * self.grads.padded)
            assert (slot - local) % 4 == 0
            push.delta_floats[o] = 0 if o == rank else (slot - local) // 4
        self._push = push
        n = len(self.grads.segments)
        self._seg_off = (ctypes.c_int64 * n)(*[o for o, _ in self.grads.segments])
        self._seg_stride = (ctypes.c_int32 * n)(*[s for _, s in self.grads.segments])
        self._stage_ptr = local + 4 * self.grads.stage_offset

    def _autotune(self, group):
        """Both NVLink variants are available: time each on the real buffer and keep the faster one (in-switch reduction wins on
        8 GPUs, plain peer loads on 2).  Timed the way the step uses it — back to back, launch latency hidden: 3 batches of 4 calls,
        best batch, max over ranks (every rank takes the same decision)."""
        import torch.distributed as dist
        mc, best = self._mc, None
        names = ("own kernel: multimem (NVLS)", "own kernel: p2p two-shot")
        if self._use_push:
            names = tuple("push fused into the backward + own reduce/publish kernel: " + x for x in ("multimem.st (NVLS)", "peer stores"))
        for cand, name in ((mc, names[0]), (0, names[1])):
            self._mc = cand
            self.all_reduce()                                   # warm-up
            ts = []
            for _ in range(3):
                torch.cuda.synchronize(self.device)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(4):
                    self.all_reduce()
                e1.record(); torch.cuda.synchronize(self.device)
                ts.append(e0.elapsed_time(e1) / 4)
            t = torch.tensor([min(ts)], device=self.device)
            dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
            if best is None or float(t) < best[0]:
                best = (float(t), cand, name)
        self._mc, self.collective = best[1], best[2] + " (auto-tuned, %.0f us%s)" % (best[0] * 1e3, ", barriers inside the kernel" if self._inkernel else "")
        self.grads.data.zero_()

    def render_views(self, params: dict, settings: Sequence[_r.GaussianRasterizationSettings],
                     upstream: Sequence[tuple], keep_images: bool = False, antialiasing: bool = False):
        """upstream[i] = (dL_dcolor [3,H,W] or None, dL_ddepth or None, dL_dalpha or None) for local view i.  antialiasing: as
        GaussianRasterizer."""
        g = self.grads.views
        images = []
        if len(settings) == 0:
            # a rank without a view this iteration (fewer views than ranks) contributes ZERO to the all-reduce; without this
            # its buffer would still hold the previous iteration's reduced sum
            self.grads.data.zero_()
        fused = self._hdl is not None and self._use_push
        self._pushed = False
        for i, (rs, up) in enumerate(zip(settings, upstream)):
            color, radii, depth, alpha, state = _r.forward_impl(
                rs, params["means3D"], params["shs"], None, params["opacities"], params["scales"], params["rotations"], None,
                antialiasing=antialiasing)
            # the backward of the LAST local view also delivers the rows other ranks own (local sum of all this rank's views)
            # to their owners' staging areas: the reduce-scatter half of the all-reduce rides on that kernel
            # (not under torch.use_deterministic_algorithms: the deterministic backward takes no push, so the rows travel by
            #  dgr_peer_push_flat after the last view instead, as for a rank without a view)
            last = fused and i == len(settings) - 1 and not torch.are_deterministic_algorithms_enabled()
            _r.backward_impl(state, up[0], up[1], up[2], g["means3D"], g["means2D"], g["shs"], None, g["opacities"],
                             g["scales"], g["rotations"], None, accumulate=(i > 0), push=self._push if last else None)
            self._pushed = self._pushed or last
            if keep_images:
                images.append((color, radii, depth, alpha))
        return images

    def use_nccl(self, why: str):
        """Drop the library's own all-reduce kernels for this object (e.g. after a failed self-check): plain NCCL from now on."""
        self._hdl = None
        self.collective = "nccl all_reduce (%s)" % why

    def all_reduce(self):
        """Sum the flat gradient over ranks: this library's NVLink kernel on the symmetric buffer (its two cross-rank
        barriers are inside the kernel), else NCCL (gloo in the CPU tests of the host logic)."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized() and dist.get_world_size(self.pg) > 1):
            return self.grads.flat
        if self._hdl is not None:
            from . import _lib
            lib = _lib.load()
            self._epoch += 1
            with torch.cuda.device(self.device):
                st = ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
                flags = ctypes.cast(self._flags, ctypes.c_void_p) if self._inkernel else None
                if self._use_push:
                    n = len(self.grads.segments)
                    if not self._pushed:      # no backward carried the push (no local view, or the buffer was filled by hand)
                        _lib.check(lib.dgr_peer_push_flat(ctypes.c_void_p(int(self._hdl.buffer_ptrs[self._hdl.rank])), ctypes.byref(self._push),
                                                          self.grads.P, n, self._seg_off, self._seg_stride, st))
                    self._pushed = False
                    if not self._inkernel:
                        self._hdl.barrier(channel=0)
                    _lib.check(lib.dgr_peer_reduce_staged(ctypes.cast(self._ptrs, ctypes.c_void_p), ctypes.byref(self._push), self.grads.P, n,
                                                          self._seg_off, self._seg_stride, ctypes.c_uint64(self._stage_ptr),
                                                          ctypes.c_uint64(self.grads.padded), ctypes.c_uint64(self._mc), flags,
                                                          ctypes.c_uint32(self._epoch), st))
                    if not self._inkernel:
                        self._hdl.barrier(channel=1)
                    return self.grads.flat
            if not self._inkernel:
                self._hdl.barrier(channel=0)
            with torch.cuda.device(self.device):
                _lib.check(lib.dgr_peer_allreduce(ctypes.cast(self._ptrs, ctypes.c_void_p), self._hdl.world_size, self._hdl.rank,
                                                  ctypes.c_uint64(self.grads.padded), ctypes.c_uint64(self._mc), flags,
                                                  ctypes.c_uint32(self._epoch), st))
            if not self._inkernel:
                self._hdl.barrier(channel=1)
        else:
            dist.all_reduce(self.grads.data if self.grads.data.is_cuda else self.grads.flat, op=dist.ReduceOp.SUM, group=self.pg)
        return self.grads.flat


def shard_views(num_views: int, rank: int, world: int) -> List[int]:
    """Contiguous block partition of view indices (rank r gets views [r*V/G, (r+1)*V/G))."""
    per = num_views // world
    rem = num_views % world
    start = rank * per + min(rank, rem)
    return list(range(start, start + per + (1 if rank < rem else 0)))
