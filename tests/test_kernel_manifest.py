"""The kernel manifest (tests/kernel_manifest.txt) lists every __global__ instantiation the compiled sm_90a library holds, each with
the cells of tests/test_kernel_coverage_gpu.py that launch it and check its output against an oracle, or with the reason it is
excused.  This test (no GPU: cuobjdump reads the library) holds the manifest equal to the library, so adding or removing a kernel
or a template instantiation forces a manifest edit, and that edit has to name the cell that checks the new kernel."""
import os
import re
import shutil
import subprocess

import pytest

import kernel_names as KN
from dreamgaussian_b200 import build

HERE = os.path.dirname(os.path.abspath(__file__))
MANIFEST = os.path.join(HERE, "kernel_manifest.txt")
CUDA_BIN = "/usr/local/cuda/bin"
CUOBJDUMP = shutil.which("cuobjdump") or os.path.join(CUDA_BIN, "cuobjdump")
CUFILT = shutil.which("cu++filt") or os.path.join(CUDA_BIN, "cu++filt")


def library_kernels():
    """Normalized names of every __global__ function in the built library."""
    if not (os.path.exists(CUOBJDUMP) and os.path.exists(CUFILT)):
        pytest.skip("cuobjdump / cu++filt not found")
    path = build.build()
    out = subprocess.run([CUOBJDUMP, "--dump-resource-usage", path], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-500:]
    mangled = sorted({m.group(1) for m in (re.match(r"\s*Function\s+(\S+?):?\s*$", l) for l in out.stdout.splitlines()) if m})
    assert len(mangled) > 40, "no kernels found in %s" % path
    dem = subprocess.run([CUFILT], input="\n".join(mangled) + "\n", stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=60)
    assert dem.returncode == 0, dem.stderr[-500:]
    names = [KN.normalize(l) for l in dem.stdout.splitlines() if l.strip()]
    assert len(names) == len(mangled), (len(names), len(mangled))
    assert len(set(names)) == len(names), "two instantiations normalize to one name"
    return set(names)


def test_manifest_lists_exactly_the_compiled_kernels():
    have = library_kernels()
    listed = KN.read_manifest(MANIFEST)
    missing, stale = sorted(have - set(listed)), sorted(set(listed) - have)
    assert not missing and not stale, ("kernels compiled but not in tests/kernel_manifest.txt: %s; listed but not compiled: %s"
                                       % (missing, stale))


def test_every_manifest_line_names_a_cell_or_an_excuse():
    import test_kernel_coverage_gpu as cov
    cells = set(cov.CELLS)
    for name, (ids, reason) in KN.read_manifest(MANIFEST).items():
        assert ids or reason, name
        unknown = [c for c in ids if c not in cells]
        assert not unknown, (name, unknown)


@pytest.mark.parametrize("raw,want", [
    ("void dgr::preprocess_fwd_kernel<(int)3, (bool)1, (bool)0, (bool)0, (bool)1>", "dgr::preprocess_fwd_kernel<3,1,0,0,1>"),
    ("void dgr::preprocess_fwd_kernel<3, true, false, false, true>(int, int, int, int, float, float, float, float const*)",
     "dgr::preprocess_fwd_kernel<3,1,0,0,1>"),
    ("dgr::adam_multi_kernel(dgr::AdamGroups, float, float, float, float)", "dgr::adam_multi_kernel"),
    ("<unnamed>::debug_geom_kernel(int, const dgr::Rec *, const unsigned int *)", "(anonymous)::debug_geom_kernel"),
    ("(anonymous namespace)::debug_geom_kernel(int, dgr::Rec const*, unsigned int const*)", "(anonymous)::debug_geom_kernel"),
])
def test_both_demangler_forms_normalize_alike(raw, want):
    assert KN.normalize(raw) == want
