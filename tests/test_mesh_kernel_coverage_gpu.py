"""Kernel coverage of libdgr_mesh.so, the rule tests/test_mcmc_kernel_coverage_gpu.py applies to libdgr_mcmc.so: every __global__
instantiation is launched by a small named call (a cell) whose outputs are checked against tests/mesh_oracle.py (through the checks of
tests/test_mesh_gpu.py), and the suite fails when one is not.  A cell runs under torch.profiler with CUDA activity tracing, passes its
checks, and only then records the normalized names of the library kernels it launched; tests/mesh_kernel_manifest.txt credits each
kernel to the cells that reach it, and the last test asserts both directions."""
import os

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import helpers as h
import kernel_names as KN
import test_mesh_gpu as TM

pytestmark = pytest.mark.gpu
MANIFEST = os.path.join(os.path.dirname(os.path.abspath(__file__)), "mesh_kernel_manifest.txt")

# marching cubes on a closed surface and on noise; one component removal with both rules on
CELLS = {
    "mesh_mc_sphere": lambda: TM.check_field("sphere"),
    "mesh_mc_noise": lambda: TM.check_field("noise"),
    "mesh_components": lambda: TM.check_components(2, 64, 20.0),
}
COVERED = {}


def _run_cell(cid):
    if cid in COVERED:
        return COVERED[cid]
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        # a throwaway kernel first: late in a long session the trace has been seen to miss the first library kernel of a cell
        torch.ones(1, device="cuda").add_(1)
        torch.cuda.synchronize()
        CELLS[cid]()
        torch.cuda.synchronize()
    names = sorted({n for n in (KN.normalize(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
                    if n.startswith("dgr::mesh_")})
    assert names, (cid, "no mesh kernel seen by the CUDA activity trace")
    h.report("mesh coverage/" + cid, launched=dict(kernels=names))
    COVERED[cid] = set(names)
    return COVERED[cid]


@pytest.mark.parametrize("cid", list(CELLS))
def test_cell(cid):
    _run_cell(cid)


def test_every_mesh_kernel_is_reached_by_a_checked_call():
    for cid in CELLS:
        _run_cell(cid)
    manifest = KN.read_manifest(MANIFEST)
    covered = set().union(*COVERED.values())
    missing = sorted(set(manifest) - covered)
    rerouted = sorted((n, c) for n, (ids, _) in manifest.items() for c in ids if n not in COVERED[c])
    assert not missing, ("manifest kernels no checked cell launched", missing)
    assert not rerouted, ("cells that no longer launch the kernels the manifest credits to them", rerouted)
