"""Kernel coverage of libdgr_mcmc.so, the rule tests/test_kernel_coverage_gpu.py applies to libdgr_b200.so: every __global__
instantiation is launched by a small named call (a cell) whose outputs are checked against tests/mcmc_oracle.py (through the checks
of tests/test_mcmc_gpu.py), and the suite fails when one is not.  A cell runs under torch.profiler with CUDA activity tracing,
passes its checks, and only then records the normalized names of the library kernels it launched; tests/mcmc_kernel_manifest.txt
credits each kernel to the cells that reach it, and the last test asserts both directions."""
import os

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import helpers as h
import kernel_names as KN
import test_mcmc_gpu as TM

pytestmark = pytest.mark.gpu
MANIFEST = os.path.join(os.path.dirname(os.path.abspath(__file__)), "mcmc_kernel_manifest.txt")

# the relocation formula on the (o, n) grid; one refinement with dead rows and growth; one at the cap (relocation only); the noise
CELLS = {
    "mcmc_relocation": TM.check_relocation_grid,
    "mcmc_refine": lambda: TM.check_refine(1237, 2000, 0),
    "mcmc_refine_at_cap": lambda: TM.check_refine(1237, 1237, 1),
    "mcmc_noise": lambda: TM.check_noise(1237, 17),
}
COVERED = {}


def _run_cell(cid):
    if cid in COVERED:
        return COVERED[cid]
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        CELLS[cid]()
        torch.cuda.synchronize()
    names = sorted({n for n in (KN.normalize(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
                    if n.startswith("dgr::mcmc_")})
    assert names, (cid, "no MCMC kernel seen by the CUDA activity trace")
    h.report("mcmc coverage/" + cid, launched=dict(kernels=names))
    COVERED[cid] = set(names)
    return COVERED[cid]


@pytest.mark.parametrize("cid", list(CELLS))
def test_cell(cid):
    _run_cell(cid)


def test_every_mcmc_kernel_is_reached_by_a_checked_call():
    for cid in CELLS:
        _run_cell(cid)
    manifest = KN.read_manifest(MANIFEST)
    covered = set().union(*COVERED.values())
    missing = sorted(set(manifest) - covered)
    rerouted = sorted((n, c) for n, (ids, _) in manifest.items() for c in ids if n not in COVERED[c])
    assert not missing, ("manifest kernels no checked cell launched", missing)
    assert not rerouted, ("cells that no longer launch the kernels the manifest credits to them", rerouted)
