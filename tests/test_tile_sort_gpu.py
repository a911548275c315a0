"""GPU tests of the per-tile sort (dgr_binning.cuh): every tile's sorted ids are exactly the (depth bits, id) order of its keys,
and the sorted record copy holds the records in that order.

The scene puts an exact number of sub-pixel Gaussians into every tile, so the tile populations sit on both sides of the warp
width (the record copy moves a warp's 32 records together), of every bucket-count step and of the 4096 limit above which the
big-tile kernel takes a tile; two tiles hold Gaussians at one and the same depth (the ranking then runs over a single bucket).
The binning buffers are read back through the ctypes host layer, which keeps them in its forward state.
"""
import numpy as np
import pytest
import torch

import helpers as h
import trained_scenes as ts
from dreamgaussian_b200 import rasterizer as R

pytestmark = pytest.mark.gpu

SORTED, BY_ID = 1 << 22, 2 << 22          # dgr_set_tuning bits 22-23: record staging
W = H = 640                               # 40 x 40 tiles: more tiles than the sort kernel has CTAs
TILE = 16
# populations around 1, the warp width, the bucket-count steps (128 ... 2048) and the 4096 small / big-tile split
EDGE_POPS = (1, 31, 32, 33, 127, 128, 129, 511, 512, 513, 1023, 1024, 1025, 2047, 2048, 4095, 4096, 4097, 5000)
PLANAR_POPS = (700, 1500)                 # tiles whose Gaussians all share one depth


def _populations():
    tiles = (W // TILE) * (H // TILE)
    pops = np.array([0 if t % 7 == 3 else 1 + (t * 37) % 90 for t in range(tiles)], np.int64)   # every 7th tile empty
    pops[:len(EDGE_POPS)] = EDGE_POPS
    planar = np.arange(len(EDGE_POPS), len(EDGE_POPS) + len(PLANAR_POPS))
    pops[planar] = PLANAR_POPS
    return pops, planar


def _scene(seed=0):
    """(settings, inputs, populations, planar tiles): pops[t] Gaussians of 0.3 px inside tile t, well clear of its edges."""
    rng = np.random.default_rng(seed)
    pops, planar = _populations()
    cam = ts.camera(W, H)
    tile = np.repeat(np.arange(len(pops)), pops)
    n = len(tile)
    px = (tile % (W // TILE)) * TILE + rng.uniform(5.0, 10.0, n)
    py = (tile // (W // TILE)) * TILE + rng.uniform(5.0, 10.0, n)
    z = rng.uniform(1.5, 2.5, n)
    flat = np.isin(tile, planar)
    px[flat], py[flat], z[flat] = 8.0 + (tile[flat] % (W // TILE)) * TILE, 8.0 + (tile[flat] // (W // TILE)) * TILE, 2.0
    view = ts.view_of_pixel(cam, px, py, z)
    g = ts.gaussians(cam, rng, view, np.full((n, 3), 0.3), np.broadcast_to(np.eye(3), (n, 3, 3)), np.full(n, 0.5),
                     rng.uniform(0.1, 0.9, (n, 3)), 0)
    return ts.settings_of(cam, 0), ts.as_inputs(g), pops, planar


def _al(v):
    return (v + 255) // 256 * 256


def _binning(geom, binning, image, n_inst, cap, tiles, records):
    """ranges [tiles, 2], keys / ids / sorted records of the n_inst instances, the records by id (layouts of dgr_common.cuh
    GeomLayout / ImageLayout and dgr_binning.cuh BinningLayout)."""
    img, bb, gm = image.cpu().numpy(), binning.cpu().numpy(), geom.cpu().numpy()
    off_ranges = 256 + _al(tiles * 4) + _al(tiles * 32)
    ranges = img[off_ranges: off_ranges + tiles * 8].view(np.uint32).reshape(tiles, 2).astype(np.int64)
    keys = bb[: n_inst * 8].view(np.uint64)
    off_ids = _al(cap * 8)
    ids = bb[off_ids: off_ids + n_inst * 4].view(np.uint32)
    off_rec = off_ids + _al(cap * 4)
    rec_sorted = bb[off_rec: off_rec + n_inst * 48].view(np.uint32).reshape(n_inst, 12)
    rec = gm[256: 256 + records * 48].view(np.uint32).reshape(records, 12)
    return ranges, keys, ids, rec_sorted, rec


def _check(state_bufs, n_inst, cap, tiles, records, gathered, expect_pops=None, planar=()):
    ranges, keys, ids, rec_sorted, rec = _binning(*state_bufs, n_inst, cap, tiles, records)
    cnt = ranges[:, 1] - ranges[:, 0]
    assert ranges[0, 0] == 0 and (ranges[1:, 0] == ranges[:-1, 1]).all() and int(cnt.sum()) == n_inst
    if expect_pops is not None:
        np.testing.assert_array_equal(cnt, expect_pops)
    tile_of = np.repeat(np.arange(tiles), cnt)
    want = keys[np.lexsort((keys, tile_of))]                # per tile: (depth bits << 32 | id) ascending
    bad = np.flatnonzero(ids != (want & 0xffffffff).astype(np.uint32))
    assert bad.size == 0, "tile %d: %d of %d ids out of (depth, id) order" % (tile_of[bad[0]], bad.size, n_inst)
    for t in planar:                                       # the planar tiles really are one depth
        assert len(np.unique(keys[ranges[t, 0]: ranges[t, 1]] >> np.uint64(32))) == 1, t
    if gathered:                                           # the sorted record copy is the records in that order
        np.testing.assert_array_equal(rec_sorted, rec[ids])


@pytest.fixture(autouse=True)
def _ctypes_layer_and_default_tuning():
    R.set_fast_host(False)
    yield
    h.set_tuning(h.DEFAULT_TUNING)
    R.set_fast_host(True)


def _rs(s):
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda")
    return R.GaussianRasterizationSettings(
        image_height=s["image_height"], image_width=s["image_width"], tanfovx=s["tanfovx"], tanfovy=s["tanfovy"], bg=t(s["bg"]),
        scale_modifier=1.0, viewmatrix=t(s["viewmatrix"]), projmatrix=t(s["projmatrix"]), sh_degree=s["sh_degree"],
        campos=t(s["campos"]), prefiltered=False, debug=False)


def _tensors(i):
    return {k: torch.tensor(v, device="cuda") for k, v in i.items()}


@pytest.mark.parametrize("staging", ["sorted", "by_id"])
@pytest.mark.parametrize("low_capacity", [False, True])
def test_every_tile_is_in_depth_then_id_order(staging, low_capacity):
    s, i, pops, planar = _scene()
    P = len(i["means3D"])
    h.set_tuning((1, 1, 1 | (SORTED if staging == "sorted" else BY_ID)))
    if low_capacity:                                       # the first stage-2 run clips its ranges and is run again
        R.set_capacity_hint(torch.cuda.current_device(), P, H, W, 4096, False)
    x = _tensors(i)
    color, radii, depth, alpha, st = R.forward_impl(_rs(s), x["means3D"], x["shs"], None, x["opacities"], x["scales"], x["rotations"], None)
    torch.cuda.synchronize()
    assert st.num_rendered == int(pops.sum()) and (radii.cpu().numpy() > 0).all()
    tiles = len(pops)
    _check((st.geom, st.binning, st.image), st.num_rendered, st.capacity, tiles, P, staging == "sorted", pops, planar)


def test_batched_views_sort_every_tile_of_every_view():
    s, i, pops, planar = _scene(seed=1)
    P, V = len(i["means3D"]), 3
    h.set_tuning((1, 1, 1 | SORTED))
    x = _tensors(i)
    color, radii, depth, alpha, st = R.views_forward_impl([_rs(s)] * V, x["means3D"], x["shs"], x["opacities"], x["scales"], x["rotations"])
    torch.cuda.synchronize()
    tiles = V * len(pops)
    assert st.num_rendered == V * int(pops.sum())
    _check((st.geom, st.binning, st.image), st.num_rendered, st.capacity, tiles, V * P, True, np.tile(pops, V),
           [v * len(pops) + t for v in range(V) for t in planar])
