"""What the compiled sm_90a library must look like (no GPU needed: cuobjdump reads dreamgaussian_b200/lib/libdgr_b200.so).

Guards the properties DESIGN.md §4 states about the step kernels against silent regressions: register budgets that decide how many
CTAs fit per SM, no spills in the render / sort kernels, bulk-TMA (UBLKCP) + mbarrier (SYNCS) staging where it is claimed and nowhere
else, reductions as RED (no returning atomics) in the backward render, and no tensor-core instructions on a path without a contraction."""
import re
import shutil
import subprocess

import pytest

from dreamgaussian_b200 import build

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.fixture(scope="module")
def resources():
    import os
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not found")
    path = build.build()
    out = subprocess.run([CUOBJDUMP, "--dump-resource-usage", path], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-500:]
    res, name = {}, None
    for line in out.stdout.splitlines():
        m = re.match(r"\s*Function\s+(\S+?):?\s*$", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+)\s+STACK:(\d+)\s+SHARED:(\d+)", line)
        if m and name:
            res[name] = dict(reg=int(m.group(1)), stack=int(m.group(2)), shared=int(m.group(3)))
            name = None
    assert len(res) > 40, "no kernels found in %s" % path
    return path, res


def _one(res, *parts):
    hits = [k for k in res if all(p in k for p in parts)]
    assert len(hits) == 1, (parts, hits)
    return hits[0]


def _sass(path, fn):
    out = subprocess.run([CUOBJDUMP, "-sass", "-fun", fn, path], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-500:]
    ops = []
    for line in out.stdout.splitlines():
        m = re.match(r"\s*/\*[0-9a-f]{4,6}\*/\s+(?:@!?U?P\d\s+)?([A-Z0-9_.]+)", line)
        if m:
            ops.append(m.group(1))
    assert len(ops) > 100, fn
    return ops


def test_register_budgets_and_no_spills_in_the_render_and_sort_kernels(resources):
    _, res = resources
    fwd = res[_one(res, "render_fwd_kernelILi1ELi1ELb0E")]            # default forward: 8 CTAs x 128 threads per SM need <= 64
    bwd = res[_one(res, "render_bwd_kernelILi1ELi2ELb0ELb1E")]        # default backward (per-row step 2): 6 CTAs per SM need <= 80
    srt = res[_one(res, "tile_sort_gather_kernelILi1024E")]           # 4 CTAs x 512 threads per SM need <= 32
    assert fwd["reg"] <= 64 and fwd["stack"] == 0, fwd
    assert bwd["reg"] <= 80 and bwd["stack"] == 0, bwd
    assert srt["reg"] <= 32 and srt["stack"] == 0, srt
    for k, v in res.items():
        if "preprocess_fwd_kernel" in k or "preprocess_bwd_kernel" in k:
            assert v["reg"] <= 80, (k, v)                             # __launch_bounds__(256, 3): three CTAs per SM


def test_bulk_tma_staging_is_where_the_design_says_it_is(resources):
    path, res = resources
    count = lambda ops, prefix: sum(1 for o in ops if o.startswith(prefix))
    # render kernels: private ring of bulk copies per warp, completion on mbarriers with transaction bytes
    for parts in (("render_fwd_kernelILi1ELi1ELb0E",), ("render_bwd_kernelILi1ELi2ELb0ELb1E",)):
        ops = _sass(path, _one(res, *parts))
        assert count(ops, "UBLKCP") >= 2 and count(ops, "SYNCS.ARRIVE.TRANS64") >= 2 and count(ops, "SYNCS.PHASECHK") >= 1, parts
        assert count(ops, "HMMA") == 0 and count(ops, "UTCHMMA") == 0 and count(ops, "UTCMMA") == 0      # no contraction on this path
    fwd = _sass(path, _one(res, "render_fwd_kernelILi1ELi1ELb0E"))
    assert count(fwd, "MUFU.EX2") >= 1 and count(fwd, "LDS.128") >= 3
    bwd = _sass(path, _one(res, "render_bwd_kernelILi1ELi2ELb0ELb1E"))
    assert count(bwd, "REDG.E.ADD.F32") >= 10 and count(bwd, "ATOMG.E.ADD.F32") == 0                      # moments leave as reductions
    # per-Gaussian kernels, degree 3, scale / rotation inputs: staged variant = five bulk copies per warp (issued once for the first
    # block iteration and once for the look-ahead in the forward), per-thread variant = none
    staged_f = _sass(path, _one(res, "preprocess_fwd_kernelILi3ELb1ELb0ELb0ELb1E"))
    plain_f = _sass(path, _one(res, "preprocess_fwd_kernelILi3ELb1ELb0ELb0ELb0E"))
    staged_b = _sass(path, _one(res, "preprocess_bwd_kernelILi3ELb1ELb0ELb0ELb1E"))
    plain_b = _sass(path, _one(res, "preprocess_bwd_kernelILi3ELb1ELb0ELb0ELb0E"))
    assert count(staged_f, "UBLKCP") >= 5 and count(staged_b, "UBLKCP") >= 5
    assert count(plain_f, "UBLKCP") == 0 and count(plain_b, "UBLKCP") == 0
    # (the staged variants keep the per-thread loads for a partial warp at the end of the cloud; what they add are the reads of the
    #  staged values out of shared memory)
    assert count(staged_f, "LDS") > count(plain_f, "LDS") + 10 and count(staged_b, "LDS") > count(plain_b, "LDS") + 10
