"""The deterministic backward (dgr_backward_det, dgr_views_backward_det, dgr_views_mixed_backward_det) without a GPU: its symbols,
its scratch size query, every refusal it makes before device work (the pointers here are never dereferenced), and what its kernels
look like in SASS (no float atomics, bulk-TMA staging, registers, no stack)."""
import ctypes
import os
import shutil

import pytest

import helpers  # noqa: F401  (sets sys.path)
from dreamgaussian_b200 import _lib

NEW = ("dgr_det_scratch_bytes", "dgr_backward_det", "dgr_views_backward_det", "dgr_views_mixed_backward_det")


def test_new_symbols_are_exported_and_the_scratch_size_needs_no_gpu():
    lib = _lib.load()
    for name in NEW:
        assert hasattr(lib, name) and name in _lib.EXPORTS, name
    b = lib.dgr_det_scratch_bytes
    assert b(0, 0) > 0
    assert b(1000, 100) < b(2000, 100) and b(1000, 100) < b(1000, 100000)
    assert b(1 << 20, 1000) >= (1 << 20) * 48 and b(0, 1 << 20) >= (1 << 20) * 4


def _buf():
    buf = (ctypes.c_float * 64)()
    return buf, ctypes.cast(buf, ctypes.c_void_p)


def _refuse(call, want):
    lib = _lib.load()
    rc = call()
    assert rc != 0, want
    assert want.encode() in lib.dgr_last_error(), (want, lib.dgr_last_error())


CAP = 1000


def _cases(p):
    """(name, scratch, scratch bytes, instances, push, staging) -> expected error text: exactly one thing wrong in each."""
    lib = _lib.load()
    ok_bytes = lib.dgr_det_scratch_bytes(CAP, 64 * 64)
    push = _lib.DgrPeerPush(2, 0, 256, (ctypes.c_int64 * 16)())
    return [
        (dict(scratch=None, nbytes=ok_bytes, inst=CAP, push=None, staging=0), "det_scratch is NULL"),
        (dict(scratch=p, nbytes=ok_bytes // 2, inst=CAP, push=None, staging=0), "smaller than dgr_det_scratch_bytes"),
        (dict(scratch=p, nbytes=ok_bytes, inst=CAP + 1, push=None, staging=0), "instances above capacity_instances"),
        (dict(scratch=p, nbytes=ok_bytes, inst=CAP, push=push, staging=0), "DgrPeerPush"),
        (dict(scratch=p, nbytes=ok_bytes, inst=CAP, push=None, staging=2), "staging"),          # the counterpart's own refusal
    ]


def test_single_view_call_refuses_before_device_work():
    lib = _lib.load()
    keep, p = _buf()
    s = _lib.DgrSettings(16, 16, 0.5, 0.5, 1.0, 0, 0, 0, p, p, p, p)
    g = _lib.DgrGaussians(1, 1, p, p, None, p, p, p, None, None, 0)
    gin = _lib.DgrImageGrads(p, None, None)
    for c, want in _cases(p):
        gout = _lib.DgrGaussianGrads()
        gout.push = ctypes.addressof(c["push"]) if c["push"] is not None else None
        _refuse(lambda: lib.dgr_backward_det(ctypes.byref(s), ctypes.byref(g), p, p, ctypes.c_uint64(CAP), c["staging"], p, p, None,
                                             ctypes.byref(gin), ctypes.byref(gout), c["scratch"], ctypes.c_uint64(c["nbytes"]),
                                             ctypes.c_uint64(c["inst"]), None), want)


def _views_args(p, V=2):
    s = _lib.DgrViews(V, 16, 16, 1.0, 0, 0, p, p, p, p, p)
    g = _lib.DgrGaussians(1, 1, p, p, None, p, p, p, None, None, 0)
    return s, g, _lib.DgrImageGrads(p, None, None)


def test_batched_calls_refuse_before_device_work():
    lib = _lib.load()
    keep, p = _buf()
    s, g, gin = _views_args(p)
    hw = (ctypes.c_int32 * 4)(16, 16, 24, 8)
    for c, want in _cases(p):
        gout = _lib.DgrGaussianGrads()
        gout.push = ctypes.addressof(c["push"]) if c["push"] is not None else None
        common = (ctypes.byref(g), p, p, ctypes.c_uint64(CAP), c["staging"], p, p, ctypes.byref(gin), ctypes.byref(gout))
        det = (c["scratch"], ctypes.c_uint64(c["nbytes"]), ctypes.c_uint64(c["inst"]), None)
        _refuse(lambda: lib.dgr_views_backward_det(ctypes.byref(s), *common, *det), want)
        _refuse(lambda: lib.dgr_views_mixed_backward_det(ctypes.byref(s), hw, *common, ctypes.c_uint64(0), *det), want)
    # the mixed call's own refusals come first as well
    gout = _lib.DgrGaussianGrads()
    ok = (p, ctypes.c_uint64(lib.dgr_det_scratch_bytes(CAP, 2)), ctypes.c_uint64(CAP), None)
    common = (ctypes.byref(g), p, p, ctypes.c_uint64(CAP), 0, p, p, ctypes.byref(gin), ctypes.byref(gout))
    _refuse(lambda: lib.dgr_views_mixed_backward_det(ctypes.byref(s), hw, *common, ctypes.c_uint64(1 << 5), *ok), "stats_views")
    _refuse(lambda: lib.dgr_views_mixed_backward_det(ctypes.byref(s), None, *common, ctypes.c_uint64(0), *ok), "image_hw is NULL")


# ---- SASS of the new kernels ---------------------------------------------------------------------------------------------------
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"

# registers ptxas gives the deterministic render kernels (256 threads, ~51 KB of shared memory per CTA): the sorted-copy variants fit
# three CTAs per SM at <= 80, the by-id variants (lane-wise bulk copies) two at <= 128
REG_LIMITS = {"render_bwd_det_kernelILb0E": 80, "render_views_bwd_det_kernelILb0E": 80,
              "render_bwd_det_kernelILb1E": 128, "render_views_bwd_det_kernelILb1E": 128,
              "det_moments_gather_kernel": 40, "det_counts_kernel": 32}


@pytest.fixture(scope="module")
def resources():
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not found")
    return _resources()


def _resources():
    import re
    import subprocess
    from dreamgaussian_b200 import build
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
    return path, res


def _sass(path, fn):
    import re
    import subprocess
    out = subprocess.run([CUOBJDUMP, "-sass", "-fun", fn, path], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-500:]
    ops = [m.group(1) for m in (re.match(r"\s*/\*[0-9a-f]{4,6}\*/\s+(?:@!?U?P\d\s+)?([A-Z0-9_.]+)", l) for l in out.stdout.splitlines()) if m]
    assert len(ops) > 10, fn
    return ops


def test_new_kernels_use_no_float_atomics_stage_by_bulk_tma_and_keep_their_register_budget(resources):
    import test_sass_contract as sc
    path, res = resources
    for part, limit in REG_LIMITS.items():
        name = sc._one(res, part)
        r = res[name]
        assert r["reg"] <= limit and r["stack"] == 0, (part, r)
        ops = _sass(path, name)
        assert not [o for o in ops if (o.startswith("REDG") or o.startswith("ATOMG") or o.startswith("RED.") or o.startswith("ATOM."))
                    and "F32" in o], part
        if "render" in part:
            count = lambda prefix: sum(1 for o in ops if o.startswith(prefix))
            assert count("UBLKCP") >= 1 and count("SYNCS.ARRIVE.TRANS64") >= 1 and count("SYNCS.PHASECHK") >= 1, part
            assert count("BAR.SYNC") >= 2, part                       # the CTA barrier before the warp-ordered sum
