"""Mesh export (include/dgr_mesh.h, libdgr_mesh.so) without a GPU: the triangle table over all 256 cases, the numpy oracle against
its per-cell restatement and against scipy, the exports and refusals of the C ABI, the kernel manifest and SASS of the library, and
the mesh PLY layout."""
import ctypes
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

import mesh_oracle as O
from dreamgaussian_b200 import _lib, meshing, ply

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_mc_table as T  # noqa: E402


def grid(shape, fn):
    ii = np.meshgrid(*[np.arange(s, dtype=np.float64) for s in shape], indexing="ij")
    return fn(*ii).astype(np.float32)


def sphere(shape, R, c):
    return grid(shape, lambda x, y, z: R - np.sqrt((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2))


# ---- the table ------------------------------------------------------------------------------------------------------------------
def test_committed_header_is_what_the_script_writes():
    with open(T.HEADER) as f:
        assert f.read() == T.render(T.build_table())
    assert [list(map(tuple, t)) for t in T.build_table()] == O.TRIS


def _face_rule(case, f):
    """The segments a face's four corners give, restated: cut edges in cyclic order; two of them form one segment, four (the
    inside corners on a diagonal) form one segment around each inside corner.  Directed so that the inside corner(s) lie to the
    right of the segment seen from outside the cube."""
    a, s, cyc = T.FACES[f]
    ins = [(case >> c) & 1 for c in cyc]
    out = set()
    n = np.zeros(3)
    n[a] = 1 if s else -1
    pos = lambda c: np.array(T.corner_pos(c), float)
    mid = lambda e: (pos(T.EDGE_CORNER[e]) + pos(T.EDGE_OTHER[e])) / 2
    cuts = [i for i in range(4) if ins[i] != ins[(i + 1) % 4]]
    edges = [T.edge_of(cyc[i], cyc[(i + 1) % 4]) for i in cuts]
    pairs = [tuple(edges)] if len(edges) == 2 else [] if not edges else \
        [(T.edge_of(cyc[i - 1], cyc[i]), T.edge_of(cyc[i], cyc[(i + 1) % 4])) for i in range(4) if ins[i]]
    for e0, e1 in pairs:
        d = mid(e1) - mid(e0)
        inside_pts = [pos(c) for c, x in zip(cyc, ins) if x]
        m = (mid(e0) + mid(e1)) / 2
        # the inside corner nearest the segment decides the side
        c = min(inside_pts, key=lambda p: np.linalg.norm(p - m))
        out.add((e0, e1) if np.dot(np.cross(n, d), c - m) < 0 else (e1, e0))
    return out


def test_table_boundary_is_the_face_rule_interior_edges_pair_and_no_inadmissible_diagonal():
    for case in range(256):
        tris = O.TRIS[case]
        directed = [(t[i], t[(i + 1) % 3]) for t in tris for i in range(3)]
        assert len(set(directed)) == len(directed), case
        boundary = {e for e in directed if (e[1], e[0]) not in set(directed)}
        want = set().union(*(_face_rule(case, f) for f in range(6)))
        assert boundary == want, (case, sorted(boundary), sorted(want))
        interior = [e for e in directed if e not in boundary]
        for e0, e1 in interior:                                  # used by exactly two triangles, in opposite directions
            assert directed.count((e0, e1)) == 1 and directed.count((e1, e0)) == 1, case
            assert not T.share_face(e0, e1), (case, e0, e1)      # an in-face diagonal that is not a segment
        assert (case in (0, 255)) == (not tris)


# ---- the oracle -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,seed", [((5, 6, 7), 0), ((2, 2, 2), 1), ((4, 3, 5), 2), ((6, 2, 3), 3)])
def test_vectorised_oracle_equals_the_per_cell_loop(shape, seed):
    rng = np.random.default_rng(seed)
    for occ in (rng.random(shape).astype(np.float32), np.round(rng.random(shape) * 4).astype(np.float32) / 4):
        a, b = O.marching_cubes(occ, 0.5), O.marching_cubes_loop(occ, 0.5)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_vertex_set_is_the_sign_changing_edges():
    rng = np.random.default_rng(5)
    occ = rng.normal(size=(7, 8, 9)).astype(np.float32)
    v, _ = O.marching_cubes(occ, 0.1)
    want = []
    for i in range(7):
        for j in range(8):
            for k in range(9):
                for a, (di, dj, dk) in enumerate(((1, 0, 0), (0, 1, 0), (0, 0, 1))):
                    q = (i + di, j + dj, k + dk)
                    if q[a] >= occ.shape[a] or (occ[i, j, k] > np.float32(0.1)) == (occ[q] > np.float32(0.1)):
                        continue
                    t = (np.float64(np.float32(0.1)) - occ[i, j, k]) / (np.float64(occ[q]) - occ[i, j, k])
                    want.append(np.array([i, j, k], float) + t * np.array([di, dj, dk]))
    np.testing.assert_array_equal(v, np.array(want))


def test_oracle_sphere_volume_euler_and_closed_edges():
    for R, c in ((20.0, (22.3, 24.1, 26.7)), (24.5, (26.0, 27.5, 28.2))):
        shape = tuple(int(x + R + 3) for x in c)
        v, f = O.marching_cubes(sphere(shape, R, c), 0.0)
        vol = O.signed_volume(v, f)
        assert vol > 0 and abs(vol / (4 / 3 * np.pi * R ** 3) - 1) < 0.01
        assert O.euler_characteristic(v, f) == 2 and O.closed_edge_violations(f) == 0


def test_component_labels_match_scipy_and_the_rule():
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components
    rng = np.random.default_rng(2)
    v, f = O.marching_cubes(rng.random((14, 15, 16)).astype(np.float32), 0.6)
    lab = O.component_labels(len(v), f)
    A = sp.coo_matrix((np.ones(3 * len(f)), (np.repeat(f[:, 0], 3), f.reshape(-1))), shape=(len(v), len(v)))
    n, sl = connected_components(A, directed=False)
    assert n == len(np.unique(lab)) > 20
    for c in range(n):                                           # same partition, labelled by its least vertex
        members = np.nonzero(sl == c)[0]
        assert (lab[members] == members.min()).all()
    vk, fk = O.remove_small_components(v, f, 8, 0)
    sizes = np.bincount(lab[f[:, 0]], minlength=len(v))
    assert len(fk) == int(sizes[sizes >= 8].sum()) and (fk < len(vk)).all()
    assert len(O.remove_small_components(v, f, 0, 0)[1]) == len(f)


# ---- the C ABI --------------------------------------------------------------------------------------------------------------------
def _declared(header):
    with open(os.path.join(ROOT, "include", header)) as f:
        src = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    return set(re.findall(r"\b(dgr_[a-z_0-9]+)\s*\(", src))


def test_exports_and_constants():
    lib = _lib.load_mesh()
    assert _declared("dgr_mesh.h") == set(_lib.MESH_EXPORTS)
    for name in _lib.MESH_EXPORTS:
        assert hasattr(lib, name), name
    assert not any(n.startswith("dgr_mesh") for n in _declared("dgr_b200.h") | set(_lib.EXPORTS))
    with open(os.path.join(ROOT, "include", "dgr_mesh.h")) as f:
        hdr = f.read()
    assert int(re.search(r"#define DGR_MESH_MIN_FACES (\d+)", hdr).group(1)) == meshing.MIN_FACES == 64
    assert float(re.search(r"#define DGR_MESH_MIN_DIAG_PCT (\S+)", hdr).group(1)) == meshing.MIN_DIAG_PCT == 20.0
    assert "UNVERIFIED-EXT" in hdr
    assert 0 < lib.dgr_mesh_scratch_bytes(2, 2, 2) < lib.dgr_mesh_scratch_bytes(37, 45, 53)
    assert lib.dgr_mesh_scratch_bytes(1, 5, 5) == 0 and lib.dgr_mesh_scratch_bytes(2048, 1024, 1024) == 0
    assert 0 < lib.dgr_mesh_components_scratch_bytes(0, 0) < lib.dgr_mesh_components_scratch_bytes(100, 200)


def _refuse(call, want):
    lib = _lib.load_mesh()
    assert call() != 0, want
    assert want.encode() in lib.dgr_mesh_last_error(), (want, lib.dgr_mesh_last_error())


def test_refusals_before_any_device_work():
    """No pointer here is ever dereferenced: every call is refused by its checks."""
    lib = _lib.load_mesh()
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 16
    cnt = (ctypes.c_int64 * 2)()
    need = lib.dgr_mesh_scratch_bytes(4, 5, 6)
    mc = lambda occ, X, Y, Z, thr, scr, nb, counts=cnt: lib.dgr_mesh_marching_cubes_count(occ, X, Y, Z, thr, scr, nb, counts, None)
    em = lambda occ, X, Y, Z, nv, nf, vv, ff, nb=need: lib.dgr_mesh_marching_cubes_emit(occ, X, Y, Z, 0.5, p, nb, nv, nf, vv, ff, None)
    _refuse(lambda: mc(p, 1, 5, 6, 0.5, p, need), "every grid side must be >= 2")
    _refuse(lambda: mc(p, 4, 5, 0, 0.5, p, need), "every grid side must be >= 2")
    _refuse(lambda: mc(p, 2048, 1024, 1024, 0.5, p, need), "2^31 points or more")
    _refuse(lambda: mc(None, 4, 5, 6, 0.5, p, need), "NULL occ")
    _refuse(lambda: mc(p + 2, 4, 5, 6, 0.5, p, need), "occ is not 4-byte aligned")
    _refuse(lambda: mc(p, 4, 5, 6, float("nan"), p, need), "thr is NaN")
    _refuse(lambda: mc(p, 4, 5, 6, 0.5, None, need), "scratch NULL or smaller")
    _refuse(lambda: mc(p, 4, 5, 6, 0.5, p, need - 1), "scratch NULL or smaller")
    _refuse(lambda: mc(p, 4, 5, 6, 0.5, p + 4, need), "scratch is not 16-byte aligned")
    _refuse(lambda: mc(p, 4, 5, 6, 0.5, p, need, None), "NULL counts")
    _refuse(lambda: em(p, 4, 5, 6, -1, 0, p, p), "counts outside")
    _refuse(lambda: em(p, 4, 5, 6, 2 ** 31, 0, p, p), "counts outside")
    _refuse(lambda: em(p, 4, 5, 6, 3, 1, None, p), "NULL output")
    _refuse(lambda: em(p, 4, 5, 6, 3, 1, p, None), "NULL output")
    _refuse(lambda: em(p, 4, 5, 6, 3, 1, p + 2, p), "not 4-byte aligned")
    _refuse(lambda: em(p, 4, 5, 6, 0, 1, p, p), "faces without vertices")
    assert em(p, 4, 5, 6, 0, 0, None, None) == 0                  # an empty surface: nothing to write
    cneed = lib.dgr_mesh_components_scratch_bytes(10, 20)
    cc = lambda v, nv, f, nf, mf=64, pct=20.0, scr=p, nb=cneed, counts=cnt: lib.dgr_mesh_remove_components_count(
        v, nv, f, nf, mf, pct, scr, nb, counts, None)
    _refuse(lambda: cc(p, -1, p, 20), "negative Nv or Nf")
    _refuse(lambda: cc(None, 10, p, 20), "NULL vertices or faces")
    _refuse(lambda: cc(p, 10, None, 20), "NULL vertices or faces")
    _refuse(lambda: cc(p, 10, p + 1, 20), "not 4-byte aligned")
    _refuse(lambda: cc(p, 10, p, 20, nb=cneed - 1), "scratch NULL or smaller")
    _refuse(lambda: cc(p, 10, p, 20, scr=p + 8), "scratch is not 16-byte aligned")
    _refuse(lambda: cc(p, 10, p, 20, counts=None), "NULL counts")
    _refuse(lambda: cc(p, 10, p, 20, mf=-1), "min_faces < 0 or min_diag_pct")
    for pct in (-1.0, 100.5, float("nan")):
        _refuse(lambda: cc(p, 10, p, 20, pct=pct), "min_faces < 0 or min_diag_pct")
    ce = lambda kv, kf, vo, fo: lib.dgr_mesh_remove_components_emit(p, 10, p, 20, p, cneed, kv, kf, vo, fo, None)
    _refuse(lambda: ce(11, 1, p, p), "kept counts outside")
    _refuse(lambda: ce(3, 1, None, p), "NULL output")
    assert cc(p, 10, p, 0) == 0 and list(cnt) == [0, 0]          # no face: nothing is kept, no device work
    with pytest.raises(RuntimeError, match="no CPU path"):
        meshing.marching_cubes(torch.zeros(3, 3, 3), 0.5)
    with pytest.raises(RuntimeError, match="no CPU path"):
        meshing.remove_small_components(torch.zeros(3, 3), torch.zeros(1, 3, dtype=torch.int32))


# ---- the compiled library: its kernel manifest and SASS ---------------------------------------------------------------------------
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
CUFILT = shutil.which("cu++filt") or "/usr/local/cuda/bin/cu++filt"
MANIFEST = os.path.join(ROOT, "tests", "mesh_kernel_manifest.txt")


def mesh_resources():
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not found")
    from dreamgaussian_b200 import build
    path = build.build_mesh()
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


def test_mesh_manifest_lists_exactly_the_compiled_kernels_and_names_cells():
    import kernel_names as KN
    import test_mesh_kernel_coverage_gpu as cov
    if not os.path.exists(CUFILT):
        pytest.skip("cu++filt not found")
    _, res = mesh_resources()
    dem = subprocess.run([CUFILT], input="\n".join(sorted(res)) + "\n", stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=60)
    have = {KN.normalize(l) for l in dem.stdout.splitlines() if l.strip()}
    assert len(have) == len(res) == 11, sorted(have)
    listed = KN.read_manifest(MANIFEST)
    assert set(listed) == have, (sorted(have - set(listed)), sorted(set(listed) - have))
    for name, (ids, reason) in listed.items():
        assert ids and reason is None, name
        assert all(c in cov.CELLS for c in ids), (name, ids)


def test_kernels_no_spills_no_local_memory_no_float_atomics():
    path, res = mesh_resources()
    assert len(res) == 11
    for name, r in res.items():
        assert r["stack"] == 0, (name, r)
        out = subprocess.run([CUOBJDUMP, "-sass", "-fun", name, path], stdout=-1, stderr=-1, text=True, timeout=300)
        ops = re.findall(r"/\*[0-9a-f]{4,6}\*/\s+(?:@!?U?P\d\s+)?([A-Z0-9_.]+)", out.stdout)
        assert ops and not any(op.startswith(("STL", "LDL")) for op in ops), name
        assert not any(re.match(r"(RED|REDG|ATOM|ATOMG)\.E\.(ADD|MIN|MAX)\.(F|FTZ)", op) for op in ops), (name, "float atomic")


# ---- the mesh PLY -----------------------------------------------------------------------------------------------------------------
def read_mesh_ply(path):
    """A tiny reader of the layout save_mesh_ply writes."""
    with open(path, "rb") as f:
        data = f.read()
    head, _, body = data.partition(b"end_header\n")
    lines = head.decode("ascii").splitlines()
    nv = int(next(l for l in lines if l.startswith("element vertex")).split()[2])
    nf = int(next(l for l in lines if l.startswith("element face")).split()[2])
    v = np.frombuffer(body[:12 * nv], "<f4").reshape(nv, 3)
    rec = np.frombuffer(body[12 * nv:], np.dtype([("n", "u1"), ("i", "<i4", (3,))]), count=nf)
    assert (rec["n"] == 3).all() and len(body) == 12 * nv + 13 * nf
    return v, rec["i"]


def test_mesh_ply_header_layout_and_round_trip(tmp_path):
    rng = np.random.default_rng(0)
    v = rng.normal(size=(7, 3)).astype(np.float32)
    f = rng.integers(0, 7, (5, 3)).astype(np.int32)
    path = str(tmp_path / "sub" / "mesh.ply")
    ply.save_mesh_ply(path, torch.tensor(v), torch.tensor(f))
    with open(path, "rb") as fh:
        data = fh.read()
    header = (b"ply\nformat binary_little_endian 1.0\nelement vertex 7\nproperty float x\nproperty float y\nproperty float z\n"
              b"element face 5\nproperty list uchar int vertex_indices\nend_header\n")
    assert data.startswith(header) and len(data) == len(header) + 7 * 12 + 5 * 13
    assert data[len(header) + 84] == 3 and data[len(header):len(header) + 12] == v[0].tobytes()
    rv, rf = read_mesh_ply(path)
    assert np.array_equal(rv, v) and np.array_equal(rf, f)
    ply.save_mesh_ply(path, np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32))
    rv, rf = read_mesh_ply(path)
    assert rv.shape == (0, 3) and rf.shape == (0, 3)
