"""Mesh export on the GPU (include/dgr_mesh.h, libdgr_mesh.so): marching cubes against tests/mesh_oracle.py on non-cubic grids
(faces identical, vertices within a few float32 ulps), the surface properties of closed level sets, small-component removal against
the oracle, the end-to-end export of two models with its PLY, determinism, and a default stage-1 run that never loads the library."""
import os

import numpy as np
import pytest
import torch

import helpers  # noqa: F401
import mesh_oracle as O
from dreamgaussian_b200 import _lib, fields, meshing, ply, scene, stage1

pytestmark = pytest.mark.gpu
EPS32 = float(np.finfo(np.float32).eps)


def grid(shape, fn):
    ii = np.meshgrid(*[np.arange(s, dtype=np.float64) for s in shape], indexing="ij")
    return fn(*ii).astype(np.float32)


def _dist(x, y, z, c):
    return np.sqrt((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2)


def _torus(x, y, z, c, R, r):
    return r - np.sqrt((np.sqrt((x - c[0]) ** 2 + (y - c[1]) ** 2) - R) ** 2 + (z - c[2]) ** 2)


SHAPE = (37, 45, 53)
FIELDS = {
    "sphere": lambda: grid(SHAPE, lambda x, y, z: 14.0 - _dist(x, y, z, (18.2, 21.7, 25.9))),
    "torus": lambda: grid(SHAPE, lambda x, y, z: _torus(x, y, z, (18.3, 22.1, 26.4), 11.0, 4.5)),
    "genus2": lambda: grid((37, 53, 29), lambda x, y, z: np.maximum(_torus(x, y, z, (18.4, 16.2, 14.3), 9.0, 3.6),
                                                                     _torus(x, y, z, (18.4, 36.1, 14.3), 9.0, 3.6))),
    "shells": lambda: grid(SHAPE, lambda x, y, z: np.minimum(16.0 - _dist(x, y, z, (18.1, 22.3, 26.2)),
                                                             _dist(x, y, z, (18.1, 22.3, 26.2)) - 8.0)),
    "quantised": lambda: np.round(grid(SHAPE, lambda x, y, z: 14.0 - _dist(x, y, z, (18.2, 21.7, 25.9))) * 2) / 2,
    "noise": lambda: np.random.default_rng(3).random(SHAPE).astype(np.float32),
    "empty": lambda: np.zeros(SHAPE, np.float32),
    "full": lambda: np.ones(SHAPE, np.float32),
}
THR = {"noise": 0.5, "empty": 0.5, "full": 0.5}
EULER = {"sphere": 2, "torus": 0, "genus2": -2, "shells": 4}


def run_mc(occ, thr):
    v, f = meshing.marching_cubes(torch.tensor(occ, device="cuda"), thr)
    return v.cpu().numpy(), f.cpu().numpy()


def assert_matches_oracle(occ, thr, got=None):
    v, f = got if got is not None else run_mc(occ, thr)
    wv, wf = O.marching_cubes(occ, thr)
    assert v.dtype == np.float32 and f.dtype == np.int32 and v.shape == wv.shape and f.shape == wf.shape
    assert np.array_equal(f, wf)
    assert (np.abs(v - wv) <= 4 * EPS32 * np.maximum(1.0, np.abs(wv))).all()
    return v, f


def check_field(name):
    occ = FIELDS[name]()
    thr = THR.get(name, 0.0)
    v, f = assert_matches_oracle(occ, thr)
    if name == "empty" or name == "full":
        assert v.shape == (0, 3) and f.shape == (0, 3)
    if name in EULER:
        assert O.closed_edge_violations(f) == 0, name
        assert O.euler_characteristic(v, f) == EULER[name], name
        assert O.signed_volume(v, f) > 0, name
    if name == "shells":                                        # the inner sphere faces inward: the shell's volume
        want = 4 / 3 * np.pi * (16.0 ** 3 - 8.0 ** 3)
        assert abs(O.signed_volume(v, f) / want - 1) < 0.02
    if name == "noise":
        keep = (v > 0.5).all(1) & (v < np.array(SHAPE) - 1.5).all(1)
        assert len(f) > 10000 and O.closed_edge_violations(f, keep) == 0
    return v, f


@pytest.mark.parametrize("name", list(FIELDS))
def test_marching_cubes_matches_the_oracle(name):
    check_field(name)


def test_all_256_cases_on_a_2x2x2_grid():
    for case in range(256):
        occ = np.array([(case >> (i | (j << 1) | (k << 2))) & 1 for i in range(2) for j in range(2) for k in range(2)],
                       np.float32).reshape(2, 2, 2) * 0.8 + 0.1
        v, f = assert_matches_oracle(occ, 0.5)
        assert len(f) == O.TRI_COUNT[case]


@pytest.mark.parametrize("R", [20.0, 23.5])
def test_sphere_volume_within_one_percent(R):
    c = (R + 2.3, R + 3.1, R + 1.7)
    shape = (int(2 * R + 6), int(2 * R + 8), int(2 * R + 5))
    occ = grid(shape, lambda x, y, z: R - _dist(x, y, z, c))
    v, f = assert_matches_oracle(occ, 0.0)
    vol = O.signed_volume(v, f)
    assert vol > 0 and abs(vol / (4 / 3 * np.pi * R ** 3) - 1) < 0.01
    assert O.closed_edge_violations(f) == 0 and O.euler_characteristic(v, f) == 2


def test_non_finite_grid_is_refused():
    occ = FIELDS["sphere"]()
    for bad in (np.nan, np.inf, -np.inf):
        o = occ.copy()
        o[3, 4, 5] = bad
        with pytest.raises(RuntimeError, match="non-finite"):
            run_mc(o, 0.0)


# ---- small-component removal ------------------------------------------------------------------------------------------------------
def check_components(seed=2, min_faces=64, min_diag_pct=20.0):
    occ = np.random.default_rng(seed).random((30, 33, 35)).astype(np.float32)
    # a big sphere and noise floaters around it
    occ = np.maximum(grid(occ.shape, lambda x, y, z: 12.0 - _dist(x, y, z, (15.2, 16.1, 17.3))) / 12.0, occ * 0.8)
    v, f = meshing.marching_cubes(torch.tensor(occ, device="cuda"), 0.7)
    vk, fk = meshing.remove_small_components(v, f, min_faces, min_diag_pct)
    wv, wf = O.remove_small_components(v.cpu().numpy(), f.cpu().numpy(), min_faces, min_diag_pct)
    assert np.array_equal(vk.cpu().numpy(), wv) and np.array_equal(fk.cpu().numpy(), wf)
    return len(f), len(wf)


@pytest.mark.parametrize("min_faces,min_diag_pct", [(64, 20.0), (0, 20.0), (64, 0.0), (5, 0.0), (0, 0.0)])
def test_component_removal_matches_the_oracle(min_faces, min_diag_pct):
    n, kept = check_components(2, min_faces, min_diag_pct)
    if min_faces or min_diag_pct:
        assert 0 < kept < n
    else:
        assert kept == n


def test_component_removal_refuses_bad_indices():
    v = torch.zeros(4, 3, device="cuda")
    with pytest.raises(RuntimeError, match="outside"):
        meshing.remove_small_components(v, torch.tensor([[0, 1, 4]], dtype=torch.int32, device="cuda"))


# ---- end to end ---------------------------------------------------------------------------------------------------------------------
class _Model:
    pass


def _cloud_model(P=100000):
    raw = scene.to_raw_parameters(scene.make_cloud(P, 0, seed=4, sigma=0.0128))
    g = _Model()
    g._xyz, g._opacity, g._scaling, g._rotation = (torch.tensor(raw[k], device="cuda") for k in ("xyz", "opacity", "scaling", "rotation"))
    return g


def _trained_model():
    tr = stage1.Stage1Trainer(stage1.Stage1Config(iters=500))
    tr.train(500)
    return tr


def _end_to_end(g, res, thr, tmp_path):
    occ = fields.extract_fields_of_model(g, res)
    o = occ.cpu().numpy()
    v, f = meshing.marching_cubes(occ, thr)
    assert_matches_oracle(o, thr, (v.cpu().numpy(), f.cpu().numpy()))
    w = meshing.to_world(v, res, g.center, g.scale)
    vk, fk = meshing.remove_small_components(w, f)
    wv, wf = O.remove_small_components(w.cpu().numpy(), f.cpu().numpy())
    assert np.array_equal(vk.cpu().numpy(), wv) and np.array_equal(fk.cpu().numpy(), wf)
    # the whole path in one call (extract_fields sums a voxel's Gaussians in an order integer atomics set, so its grid may differ
    # from the one above in the last bits)
    ev, ef = meshing.extract_mesh_of_model(g, thr, res)
    assert ev.dtype == torch.float32 and ef.dtype == torch.int32 and abs(len(ef) - len(fk)) <= 0.01 * len(fk) + 8
    assert len(ef) == 0 or (int(ef.min()) >= 0 and int(ef.max()) < len(ev))
    path = str(tmp_path / "mesh.ply")
    ply.save_mesh_ply(path, ev, ef)
    import test_mesh_cpu
    rv, rf = test_mesh_cpu.read_mesh_ply(path)
    assert np.array_equal(rv, ev.cpu().numpy()) and np.array_equal(rf, ef.cpu().numpy())
    return len(f), len(fk), float(o.max())


def test_end_to_end_model_like_cloud(tmp_path):
    g = _cloud_model()
    occ = fields.extract_fields_of_model(g, 128)
    peak = float(occ.max())
    n1, _, _ = _end_to_end(g, 128, 1.0, tmp_path)              # the reference's density_thresh
    n, kept, _ = _end_to_end(g, 128, 0.3 * peak, tmp_path)      # a level the cloud certainly crosses
    assert n > 1000 and kept > 0


def test_end_to_end_stage1_model_and_save_mesh(tmp_path):
    tr = _trained_model()
    n, kept, _ = _end_to_end(tr.gaussians, 128, 1.0, tmp_path)   # the reference's density_thresh
    assert n > 100 and kept > 0
    path = str(tmp_path / "out" / "model.ply")
    v, f = tr.save_mesh(path)
    import test_mesh_cpu
    rv, rf = test_mesh_cpu.read_mesh_ply(path)
    assert len(f) > 0 and np.array_equal(rv, v.cpu().numpy()) and np.array_equal(rf, f.cpu().numpy())


def test_bit_reproducible():
    occ = torch.tensor(FIELDS["noise"](), device="cuda")
    a = meshing.marching_cubes(occ, 0.5)
    b = meshing.marching_cubes(occ, 0.5)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    ca = meshing.remove_small_components(*a, 8, 10.0)
    cb = meshing.remove_small_components(*b, 8, 10.0)
    assert torch.equal(ca[0], cb[0]) and torch.equal(ca[1], cb[1])


def test_default_stage1_run_never_loads_the_mesh_library():
    class Untouchable:
        def __getattr__(self, name):
            raise AssertionError("a default stage-1 run called libdgr_mesh.so (%s)" % name)
    tr = stage1.Stage1Trainer(stage1.Stage1Config(iters=40, num_pts=1500, ref_size=96, density_start_iter=4, densification_interval=4))
    saved, _lib._mesh = _lib._mesh, Untouchable()
    try:
        tr.train(8)
    finally:
        _lib._mesh = saved
