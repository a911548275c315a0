"""Mesh export on the device: the geometry half of the reference's `GaussianModel.extract_mesh` (gs_renderer.py:296-322) over
libdgr_mesh.so (include/dgr_mesh.h).

    extract_fields -> marching_cubes(occ, density_thresh) -> v / (res - 1) * 2 - 1, then / scale + center
    -> remove_small_components (the floater removal of clean_mesh: by face count and by bounding-box diagonal)

The rest of clean_mesh (vertex merging, duplicate / null face removal, non-manifold repair, isotropic remeshing), decimation and the
texture half are not done here.  Every call runs on CUDA tensors; there is no CPU path."""
import ctypes

import torch

from . import _lib

MIN_FACES = 64            # include/dgr_mesh.h DGR_MESH_MIN_FACES (UNVERIFIED-EXT)
MIN_DIAG_PCT = 20.0       # include/dgr_mesh.h DGR_MESH_MIN_DIAG_PCT (UNVERIFIED-EXT)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def marching_cubes(occ, thr):
    """mcubes.marching_cubes's call shape: occ [NX,NY,NZ] float32 CUDA, inside iff occ > thr -> (v float32 [Nv,3] in index space,
    f int32 [Nf,3]) CUDA tensors, faces facing from inside to outside.  One host synchronisation (the output sizes)."""
    if not isinstance(occ, torch.Tensor) or not occ.is_cuda:
        raise RuntimeError("occ must be a CUDA tensor: marching_cubes has no CPU path")
    if occ.dim() != 3 or occ.dtype != torch.float32:
        raise ValueError("occ must be a float32 [NX,NY,NZ] tensor")
    occ = occ.contiguous()
    NX, NY, NZ = occ.shape
    dev = occ.device
    lib = _lib.load_mesh()
    scratch = torch.empty((max(1, lib.dgr_mesh_scratch_bytes(NX, NY, NZ)),), dtype=torch.uint8, device=dev)
    counts = (ctypes.c_int64 * 2)()
    with torch.cuda.device(dev):
        st = _stream(dev)
        args = (_ptr(occ), NX, NY, NZ, ctypes.c_float(thr), _ptr(scratch), scratch.numel())
        _lib.check_mesh(lib.dgr_mesh_marching_cubes_count(*args, counts, st))
        v = torch.empty((counts[0], 3), dtype=torch.float32, device=dev)
        f = torch.empty((counts[1], 3), dtype=torch.int32, device=dev)
        _lib.check_mesh(lib.dgr_mesh_marching_cubes_emit(*args, counts[0], counts[1], _ptr(v), _ptr(f), st))
    return v, f


def remove_small_components(v, f, min_faces=MIN_FACES, min_diag_pct=MIN_DIAG_PCT):
    """Drop the components (faces connected through shared vertices) with fewer than min_faces faces or a bounding-box diagonal
    below min_diag_pct % of the mesh's (0 disables a rule), and the vertices no kept face references.  Order is kept, faces are
    re-indexed.  -> (v float32 [Nv',3], f int32 [Nf',3]).  One host synchronisation (the kept sizes)."""
    for name, t in (("v", v), ("f", f)):
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise RuntimeError("%s must be a CUDA tensor: remove_small_components has no CPU path" % name)
    if v.dim() != 2 or v.shape[1] != 3 or f.dim() != 2 or f.shape[1] != 3:
        raise ValueError("v and f must be [N,3]")
    v = v.detach().float().contiguous()
    f = f.detach().to(torch.int32).contiguous()
    dev = v.device
    lib = _lib.load_mesh()
    Nv, Nf = v.shape[0], f.shape[0]
    scratch = torch.empty((lib.dgr_mesh_components_scratch_bytes(Nv, Nf),), dtype=torch.uint8, device=dev)
    counts = (ctypes.c_int64 * 2)()
    with torch.cuda.device(dev):
        st = _stream(dev)
        _lib.check_mesh(lib.dgr_mesh_remove_components_count(_ptr(v), Nv, _ptr(f), Nf, int(min_faces), float(min_diag_pct), _ptr(scratch),
                                                             scratch.numel(), counts, st))
        vo = torch.empty((counts[0], 3), dtype=torch.float32, device=dev)
        fo = torch.empty((counts[1], 3), dtype=torch.int32, device=dev)
        _lib.check_mesh(lib.dgr_mesh_remove_components_emit(_ptr(v), Nv, _ptr(f), Nf, _ptr(scratch), scratch.numel(), counts[0], counts[1],
                                                            _ptr(vo), _ptr(fo), st))
    return vo, fo


def to_world(v, resolution, center, scale):
    """Index space -> world space the way extract_mesh writes it: v / (res - 1) * 2 - 1, then / scale + center."""
    v = v / (resolution - 1.0) * 2 - 1
    return v / scale + center


def extract_mesh_of_model(gaussians, density_thresh=1.0, resolution=128, min_faces=MIN_FACES, min_diag_pct=MIN_DIAG_PCT):
    """extract_mesh's geometry on the device: -> world-space (v float32 [Nv,3], f int32 [Nf,3]) CUDA tensors.  Sets
    gaussians.center / gaussians.scale as extract_fields does."""
    from .fields import extract_fields_of_model
    occ = extract_fields_of_model(gaussians, resolution)
    v, f = marching_cubes(occ, density_thresh)
    v = to_world(v, resolution, gaussians.center, gaussians.scale)
    return remove_small_components(v, f, min_faces, min_diag_pct)
