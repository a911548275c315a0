"""MCMC densification (include/dgr_mcmc.h, libdgr_mcmc.so; Kheradmand et al., NeurIPS 2024) without a GPU: the exports and refusals of the
C ABI, the constants, the float64 oracle against itself and 60-digit arithmetic, the torch restatement of GaussianModelB200 against
the oracle on hand-built snapshots and seeded clouds, the stage-1 switches, and the SASS of the new kernels."""
import ctypes
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import mcmc_oracle as O
from dreamgaussian_b200 import _lib, stage1

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("dgr_mcmc_relocation", "dgr_mcmc_scratch_bytes", "dgr_mcmc_refine", "dgr_mcmc_inject_noise")


def _declared(header):
    with open(os.path.join(ROOT, "include", header)) as f:
        src = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    return set(re.findall(r"\b(dgr_[a-z_0-9]+)\s*\(", src))


def test_exports_and_constants():
    lib = _lib.load_mcmc()
    declared = _declared("dgr_mcmc.h")
    assert declared == set(_lib.MCMC_EXPORTS) == set(NEW_SYMBOLS) | {"dgr_mcmc_last_error"}
    for name in declared:
        assert hasattr(lib, name), name
    # the rasterizer library and its header are untouched by the feature
    assert not any(n.startswith("dgr_mcmc") for n in _declared("dgr_b200.h") | set(_lib.EXPORTS))
    assert not hasattr(_lib.load(), "dgr_mcmc_refine") and _lib.load().dgr_abi_version() == 5
    with open(os.path.join(ROOT, "include", "dgr_constants.h")) as f:
        hdr = f.read()
    val = lambda name: re.search(r"#define %s\s+(\S+(?: - 1\.0 / 8388608\.0\))?)" % name, hdr).group(1)
    assert int(val("DGR_MCMC_N_MAX")) == stage1.MCMC_N_MAX == O.N_MAX
    assert float(val("DGR_MCMC_MIN_OPACITY").rstrip("f")) == stage1.MCMC_MIN_OPACITY == O.MIN_OPACITY
    assert val("DGR_MCMC_OPACITY_MAX") == "(1.0 - 1.0 / 8388608.0)" and stage1.MCMC_OPACITY_MAX == O.OPACITY_MAX == 1 - 2.0 ** -23
    assert int(val("DGR_MCMC_GROW_PERCENT")) == stage1.MCMC_GROW_PERCENT == O.GROW_PERCENT
    assert float(val("DGR_MCMC_NOISE_K").rstrip("f")) == stage1.MCMC_NOISE_K == O.NOISE_K
    assert float(val("DGR_MCMC_NOISE_X0").rstrip("f")) == stage1.MCMC_NOISE_X0 == O.NOISE_X0
    assert float(val("DGR_MCMC_NOISE_LR").rstrip("f")) == stage1.MCMC_NOISE_LR
    assert float(val("DGR_MCMC_OPACITY_REG").rstrip("f")) == stage1.MCMC_OPACITY_REG
    assert float(val("DGR_MCMC_SCALE_REG").rstrip("f")) == stage1.MCMC_SCALE_REG
    # scratch grows with P and n_add
    assert 0 < lib.dgr_mcmc_scratch_bytes(0, 0) < lib.dgr_mcmc_scratch_bytes(1000, 0) < lib.dgr_mcmc_scratch_bytes(1000, 500)


# ---- refusals before any device work (no pointer here is ever dereferenced) ---------------------------------------------------
def _refuse(call, want):
    lib = _lib.load_mcmc()
    assert call() != 0, want
    assert want.encode() in lib.dgr_mcmc_last_error(), (want, lib.dgr_mcmc_last_error())


def _tensors(p, widths=(3, 3, 0, 1, 3, 4), null=None):
    t = _lib.DgrDensifyTensors()
    for i in range(6):
        t.inp[i] = t.exp_avg_in[i] = t.exp_avg_sq_in[i] = t.out[i] = t.exp_avg_out[i] = t.exp_avg_sq_out[i] = p
        t.width[i] = widths[i]
    if null is not None:
        t.exp_avg_out[null] = None
    return t


def test_refusals():
    lib = _lib.load_mcmc()
    buf = ctypes.create_string_buffer(64)
    p = ctypes.addressof(buf)
    P, A = 40, 2
    need = lib.dgr_mcmc_scratch_bytes(P, A)
    t = _tensors(p)
    refine = lambda P_, A_, t_, u, ua, mo, scr, nb: lib.dgr_mcmc_refine(P_, A_, ctypes.byref(t_) if t_ is not None else None, u, ua, mo,
                                                                       scr, nb, None, None)
    _refuse(lambda: lib.dgr_mcmc_relocation(-1, p, p, p, p, p, None), "dgr_mcmc_relocation: n < 0")
    _refuse(lambda: lib.dgr_mcmc_relocation(3, p, None, p, p, p, None), "dgr_mcmc_relocation: NULL argument")
    _refuse(lambda: refine(-1, 0, t, p, p, 0.005, p, need), "dgr_mcmc_refine: negative P or n_add")
    _refuse(lambda: refine(P, -1, t, p, p, 0.005, p, need), "dgr_mcmc_refine: negative P or n_add")
    _refuse(lambda: refine(P, A, None, p, p, 0.005, p, need), "dgr_mcmc_refine: NULL tensors")
    for mo in (-0.1, 1.0, float("nan")):
        _refuse(lambda: refine(P, A, t, p, p, mo, p, need), "dgr_mcmc_refine: min_opacity outside [0, 1)")
    _refuse(lambda: refine(P, A, _tensors(p, (3, 3, -3, 1, 3, 4)), p, p, 0.005, p, need), "dgr_mcmc_refine: negative row width")
    _refuse(lambda: refine(P, A, _tensors(p, null=4), p, p, 0.005, p, need), "dgr_mcmc_refine: NULL tensor")
    _refuse(lambda: refine(P, A, _tensors(p, (3, 3, 0, 1, 3, 3)), p, p, 0.005, p, need), "dgr_mcmc_refine: row widths must be")
    _refuse(lambda: refine(0, 1, t, p, p, 0.005, p, need), "dgr_mcmc_refine: n_add > 0 needs P > 0")
    _refuse(lambda: refine(P, A, t, None, p, 0.005, p, need), "dgr_mcmc_refine: NULL draws")
    _refuse(lambda: refine(P, A, t, p, None, 0.005, p, need), "dgr_mcmc_refine: NULL draws")
    _refuse(lambda: refine(P, A, t, p, p, 0.005, None, need), "dgr_mcmc_refine: scratch NULL or smaller")
    _refuse(lambda: refine(P, A, t, p, p, 0.005, p, need - 1), "dgr_mcmc_refine: scratch NULL or smaller")
    _refuse(lambda: lib.dgr_mcmc_inject_noise(-1, p, p, p, p, p, 1.0, None), "dgr_mcmc_inject_noise: P < 0")
    _refuse(lambda: lib.dgr_mcmc_inject_noise(3, p, p, p, p, None, 1.0, None), "dgr_mcmc_inject_noise: NULL argument")
    for sc in (-1.0, float("inf"), float("nan")):
        _refuse(lambda: lib.dgr_mcmc_inject_noise(3, p, p, p, p, p, sc, None), "dgr_mcmc_inject_noise: scale must be finite")
    # empty calls succeed without touching the device
    assert lib.dgr_mcmc_relocation(0, None, None, None, None, None, None) == 0
    assert lib.dgr_mcmc_inject_noise(0, None, None, None, None, None, 1.0, None) == 0


# ---- the oracle ----------------------------------------------------------------------------------------------------------------
GRID_O = [0.005, 0.01, 0.1, 0.5, 0.9, 0.99, 0.999, float(np.float32(1 - 2.0 ** -23))]


def test_formula_identities_and_forms():
    for o in GRID_O:
        op, f = O.relocate([o], [1])
        assert op[0] == pytest.approx(o, rel=1e-15) and f[0] == pytest.approx(1.0, rel=1e-15)       # n = 1 is the identity
        for n in range(1, O.N_MAX + 1):
            op = float(O.new_opacity(o, n))
            assert abs(1 - (1 - op) ** n - o) <= 1e-12 * o, (o, n)                               # 1 - (1 - o')^n = o
            exact = O.exact_D(op, n)
            assert abs(O.double_sum(op, n) - O.hockey_stick_fsum(op, n)) <= 1e-12 * exact, (o, n)
            assert abs(float(O.hockey_stick(op, n)) - exact) <= 1e-11 * exact, (o, n)          # the vectorized oracle
    # n = 2 by hand: o' = 1 - sqrt(1 - o), D = 2 o' - o'^2 / sqrt(2)
    o = 0.3
    op, f = O.relocate([o], [2])
    want_op = 1 - math.sqrt(1 - o)
    assert op[0] == pytest.approx(want_op, rel=1e-14)
    assert f[0] == pytest.approx(o / (2 * want_op - want_op ** 2 / math.sqrt(2)), rel=1e-13)
    # ratio past the table is clamped
    assert np.array_equal(np.array(O.relocate([0.5], [400])), np.array(O.relocate([0.5], [O.N_MAX])))


def test_sampling_rule():
    w = np.array([0.5, 0.0, 0.25, 0.25], np.float32)
    idx, margin = O.sample(w, np.array([0.0, 0.49, 0.5, 0.74, 0.75, 0.9999], np.float32), fallback=3)
    assert idx.tolist() == [0, 0, 2, 2, 3, 3]                 # smallest i with C_i > u C_last; the zero-weight row is never picked
    assert margin[2] == 0.0 and margin[0] == 0.0              # draws on a boundary have zero margin
    idx, _ = O.sample(np.zeros(3, np.float32), np.array([0.5], np.float32), fallback=2)
    assert idx.tolist() == [2]                                # no C_i above the draw: the fallback


# ---- snapshots of the torch restatement against the oracle ---------------------------------------------------------------------
def _cloud(P, seed, deg=1, op_mu=-1.0, op_sd=2.5):
    rng = np.random.default_rng(seed)
    M = (deg + 1) ** 2
    p = dict(xyz=rng.normal(0, 0.3, (P, 3)), f_dc=rng.normal(0, 1, (P, 1, 3)), f_rest=rng.normal(0, 0.1, (P, M - 1, 3)),
             opacity=rng.normal(op_mu, op_sd, (P, 1)), scaling=rng.normal(-3.4, 0.6, (P, 3)), rotation=rng.normal(0, 1, (P, 4)))
    p = {k: v.astype(np.float32) for k, v in p.items()}
    m = {k: rng.normal(0, 1, v.shape).astype(np.float32) for k, v in p.items()}
    v = {k: (x ** 2).astype(np.float32) for k, x in m.items()}
    return p, m, v


def _model(p, m, v, device="cpu", fused=False):
    g = stage1.GaussianModelB200(1)
    g._set({k: torch.tensor(x, device=device) for k, x in p.items()})
    g.training_setup()
    g.exp_avg = {k: torch.tensor(x, device=device) for k, x in m.items()}
    g.exp_avg_sq = {k: torch.tensor(x, device=device) for k, x in v.items()}
    g.fused_adam = g.fused_densify = fused
    return g


def _np(g):
    return ({k: x.detach().cpu().numpy() for k, x in g.p.items()}, {k: x.cpu().numpy() for k, x in g.exp_avg.items()},
            {k: x.cpu().numpy() for k, x in g.exp_avg_sq.items()})


def _run_torch(p, m, v, cap, u, ua, min_opacity=O.MIN_OPACITY):
    g = _model(p, m, v)
    n = g.relocate_and_grow_mcmc(cap, min_opacity, u_relocate=torch.tensor(u), u_add=torch.tensor(ua))
    assert g.stats.denom.shape[0] == g.num_points
    return _np(g) + (int(n),)


def _assert_equal(a, b, what):
    for k in O.GROUPS:
        np.testing.assert_allclose(a[k], b[k], rtol=2e-7, atol=0, err_msg="%s %s" % (what, k))


@pytest.mark.parametrize("P,cap,seed", [(1237, 2000, 0), (1237, 1237, 1), (1237, 500, 2), (4000, 4100, 3)])
def test_torch_restatement_equals_the_oracle(P, cap, seed):
    p, m, v = _cloud(P, seed)
    rng = np.random.default_rng(seed + 100)
    n_add = O.add_count(P, cap)
    u, ua = rng.random(P, dtype=np.float32), rng.random(n_add, dtype=np.float32)
    want = O.refine(p, m, v, u, ua, cap)
    tp, tm, tv, n = _run_torch(p, m, v, cap, u, ua)
    assert n == want[3] and len(want[4]["dead"]) > 20 and n == len(want[4]["dead"])
    assert tp["xyz"].shape[0] == P + n_add == max(P, min(cap, P * 105 // 100))
    for a, b, what in ((tp, want[0], "param"), (tm, want[1], "exp_avg"), (tv, want[2], "exp_avg_sq")):
        _assert_equal(a, b, what)
    for k in O.GROUPS:                                           # moments are copies or zeros: bit-identical
        assert np.array_equal(tm[k], want[1][k]) and np.array_equal(tv[k], want[2][k]), k


def test_relocation_snapshot_by_hand():
    P = 5
    p, m, v = _cloud(P, 7)
    o = np.array([0.9, 0.001, 0.5, 0.002, 0.3])
    p["opacity"] = np.log(o / (1 - o)).astype(np.float32)[:, None]
    u = np.array([0.1, 0.7, 0.0, 0.0, 0.0], np.float32)     # live weights 0.9, 0.5, 0.3: C = 0.9, 0.9, 1.4, 1.4, 1.7
    tp, tm, tv, n = _run_torch(p, m, v, P, u, np.zeros(0, np.float32))
    assert n == 2 and tp["xyz"].shape[0] == P                # floor(1.05 * 5) = 5: no growth
    for k in O.GROUPS:
        assert np.array_equal(tp[k][1], tp[k][0]) and np.array_equal(tp[k][3], tp[k][2]), k      # dead rows became copies
        assert np.array_equal(tp[k][4], p[k][4]), k                                                # untouched row
        for r in (0, 2):                                                                           # sources: zero moments
            assert not tm[k][r].any() and not tv[k][r].any(), k
        for r in (1, 3, 4):                                                                        # the rest keep theirs
            assert np.array_equal(tm[k][r], m[k][r]) and np.array_equal(tv[k][r], v[k][r]), k
        if k not in ("opacity", "scaling"):
            assert np.array_equal(tp[k][0], p[k][0]) and np.array_equal(tp[k][2], p[k][2]), k
    o32 = O.opacity(p["opacity"][:, 0]).astype(np.float64)
    for r in (0, 2):                                         # n = 2: o' = 1 - sqrt(1 - o), s' = s o / (2 o' - o'^2 / sqrt 2)
        op = 1 - math.sqrt(1 - o32[r])
        assert 1 / (1 + math.exp(-float(tp["opacity"][r, 0]))) == pytest.approx(op, rel=1e-6)
        want_s = np.exp(p["scaling"][r].astype(np.float64)) * o32[r] / (2 * op - op * op / math.sqrt(2))
        np.testing.assert_allclose(np.exp(tp["scaling"][r].astype(np.float64)), want_s, rtol=1e-6)


def test_growth_snapshot_cases():
    P = 40
    p, m, v = _cloud(P, 8, op_mu=1.0, op_sd=0.5)            # every row alive
    ua = np.array([0.3, 0.3], np.float32)                    # n_add = floor(42) - 40 = 2, both draws pick the same row
    tp, tm, tv, n = _run_torch(p, m, v, 10 ** 6, np.random.default_rng(0).random(P, dtype=np.float32), ua)
    assert n == 0 and tp["xyz"].shape[0] == 42
    C = np.cumsum(O.opacity(p["opacity"][:, 0]).astype(np.float64))
    r = int(np.searchsorted(C, np.float64(np.float32(0.3)) * C[-1], side="right"))
    for k in O.GROUPS:
        assert np.array_equal(tp[k][40], tp[k][r]) and np.array_equal(tp[k][41], tp[k][r]), k         # appended in pick order
        assert not tm[k][40:].any() and not tv[k][40:].any() and not tm[k][r].any() and not tv[k][r].any(), k
        others = [i for i in range(P) if i != r]
        assert np.array_equal(tm[k][others], m[k][others]) and np.array_equal(tp[k][others], p[k][others]), k
    o32 = float(O.opacity(p["opacity"][r:r + 1, 0])[0])
    assert 1 / (1 + math.exp(-float(tp["opacity"][r, 0]))) == pytest.approx(1 - (1 - o32) ** (1 / 3), rel=1e-6)    # n = 1 + 2
    # the cap: at the cap and below the current count nothing is added, P + n_add = min(cap, floor(1.05 P)) otherwise
    for cap, want in ((41, 41), (42, 42), (10 ** 6, 42), (40, 40), (3, 40)):
        assert _run_torch(p, m, v, cap, np.zeros(P, np.float32), np.zeros(O.add_count(P, cap), np.float32))[0]["xyz"].shape[0] == want


def test_no_live_and_no_dead_rows():
    P = 30
    p, m, v = _cloud(P, 9)
    p["opacity"][:] = -8.0                                   # every row dead, none alive: relocation does nothing
    tp, tm, tv, n = _run_torch(p, m, v, P, np.full(P, 0.5, np.float32), np.zeros(0, np.float32))
    assert n == 0
    for k in O.GROUPS:
        assert np.array_equal(tp[k], p[k]) and np.array_equal(tm[k], m[k]) and np.array_equal(tv[k], v[k]), k
    p["opacity"][:] = 2.0                                    # none dead: nothing moves either
    tp, tm, tv, n = _run_torch(p, m, v, P, np.full(P, 0.5, np.float32), np.zeros(0, np.float32))
    assert n == 0 and all(np.array_equal(tp[k], p[k]) and np.array_equal(tm[k], m[k]) for k in O.GROUPS)


def test_noise_torch_restatement_equals_the_oracle():
    P = 500
    p, m, v = _cloud(P, 10, op_mu=-3.0, op_sd=3.0)
    z = np.random.default_rng(4).normal(size=(P, 3)).astype(np.float32)
    g = _model(p, m, v)
    g.inject_noise_mcmc(5000.0, normals=torch.tensor(z))
    want = p["xyz"].astype(np.float64) + O.noise_update(p["opacity"], p["scaling"], p["rotation"], z, 5000.0)
    got = g.p["xyz"].detach().numpy().astype(np.float64)
    assert (np.abs(got - want) <= 1e-5 * O.noise_bound(p["opacity"], p["scaling"], z, 5000.0) + 2e-7 * np.abs(want) + 1e-30).all()
    o = O.opacity(p["opacity"][:, 0])
    op = o > 0.9                                             # opaque rows: the gate is below 1e-38, they do not move
    assert op.sum() > 10 and np.array_equal(got[op], p["xyz"][op])
    assert (np.abs(O.noise_update(p["opacity"], p["scaling"], p["rotation"], z, 5000.0)[op]) <= 1e-30).all()


def test_stage1_switches():
    cfg = stage1.Stage1Config()
    assert cfg.densify_strategy == "default" and cfg.mcmc_min_opacity == O.MIN_OPACITY and cfg.mcmc_noise_lr == 5e5
    with pytest.raises(ValueError, match="densify_abs_grad_threshold must be None"):
        stage1.Stage1Trainer(stage1.Stage1Config(densify_strategy="mcmc", densify_abs_grad_threshold=0.02), device="cpu")
    with pytest.raises(ValueError, match="densify_strategy must be"):
        stage1.Stage1Trainer(stage1.Stage1Config(densify_strategy="abs"), device="cpu")
    with pytest.raises(ValueError, match="CUDA tensors"):
        stage1.mcmc_relocation(torch.ones(2), torch.ones(2, 3), torch.ones(2, dtype=torch.int32))
    g = _model(*_cloud(10, 1))
    with pytest.raises(ValueError, match="u_relocate"):
        g.relocate_and_grow_mcmc(10, u_relocate=torch.zeros(9), u_add=torch.zeros(0))


# ---- the compiled MCMC library: its kernel manifest and SASS ------------------------------------------------------------------
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
CUFILT = shutil.which("cu++filt") or "/usr/local/cuda/bin/cu++filt"
MANIFEST = os.path.join(ROOT, "tests", "mcmc_kernel_manifest.txt")


def mcmc_resources():
    """{mangled name: dict(reg, stack)} of every __global__ function in libdgr_mcmc.so."""
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not found")
    from dreamgaussian_b200 import build
    path = build.build_mcmc()
    out = subprocess.run([CUOBJDUMP, "--dump-resource-usage", path], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-500:]
    res, name = {}, None
    for line in out.stdout.splitlines():
        m = re.match(r"\s*Function\s+(\S+?):?\s*$", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+)\s+STACK:(\d+)", line)
        if m and name:
            res[name] = dict(reg=int(m.group(1)), stack=int(m.group(2)))
            name = None
    return path, res


def test_mcmc_manifest_lists_exactly_the_compiled_kernels_and_names_cells():
    """tests/mcmc_kernel_manifest.txt is to libdgr_mcmc.so what tests/kernel_manifest.txt is to libdgr_b200.so: every __global__
    instantiation, each with the cells of tests/test_mcmc_kernel_coverage_gpu.py that launch it and check its output."""
    import kernel_names as KN
    import test_mcmc_kernel_coverage_gpu as cov
    if not os.path.exists(CUFILT):
        pytest.skip("cu++filt not found")
    _, res = mcmc_resources()
    dem = subprocess.run([CUFILT], input="\n".join(sorted(res)) + "\n", stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=60)
    have = {KN.normalize(l) for l in dem.stdout.splitlines() if l.strip()}
    assert len(have) == len(res) == 11, sorted(have)
    listed = KN.read_manifest(MANIFEST)
    assert set(listed) == have, (sorted(have - set(listed)), sorted(set(listed) - have))
    for name, (ids, reason) in listed.items():
        assert ids and reason is None, name                    # nothing here is excused
        assert all(c in cov.CELLS for c in ids), (name, ids)


def test_new_kernels_no_spills_no_local_memory_float64_where_claimed():
    path, res = mcmc_resources()
    for part in NEW_KERNELS:
        hits = [k for k in res if "%d%s" % (len(part), part) in k]
        assert len(hits) == 1, (part, hits)
        name = hits[0]
        assert res[name]["stack"] == 0, (part, res[name])
        out = subprocess.run([CUOBJDUMP, "-sass", "-fun", name, path], stdout=-1, stderr=-1, text=True, timeout=300)
        ops = re.findall(r"/\*[0-9a-f]{4,6}\*/\s+(?:@!?U?P\d\s+)?([A-Z0-9_.]+)", out.stdout)
        assert ops and not any(op.startswith(("STL", "LDL")) for op in ops), part
        if part in ("mcmc_relocation_kernel", "mcmc_relocate_update_kernel", "mcmc_grow_update_kernel"):
            assert sum(op.startswith(("DFMA", "DADD", "DMUL")) for op in ops) >= 20, part          # the formula runs in float64
        if part in ("mcmc_relocate_pick_kernel", "mcmc_grow_pick_kernel"):
            assert not any(op.startswith(("RED.E.ADD.F", "REDG.E.ADD.F", "ATOMG.E.ADD.F")) for op in ops), part   # integer atomics only
        if part == "mcmc_noise_kernel":
            assert not any(op.startswith(("DFMA", "DADD", "DMUL")) for op in ops), part            # the per-step kernel stays float32


NEW_KERNELS = ("mcmc_relocation_kernel", "mcmc_scan_local_kernel", "mcmc_scan_blocks_kernel", "mcmc_scan_add_kernel",
               "mcmc_relocate_pick_kernel", "mcmc_relocate_write_kernel", "mcmc_relocate_update_kernel", "mcmc_grow_pick_kernel",
               "mcmc_grow_update_kernel", "mcmc_append_kernel", "mcmc_noise_kernel")
