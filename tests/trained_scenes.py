"""Scenes in the parameter regimes of a trained model, for the rasterizer's parity tests.

``scene.make_cloud`` models a cloud early in training: opacities in (0.05, 0.95), colours in (0, 1), mildly anisotropic
scales.  A model that has trained for a while is full of what it never draws: saturated opacities, dark (clamped) and
over-bright colours, needle and disc Gaussians, opacities at or below 1/255, sub-pixel Gaussians, and Gaussians at the
near plane or beyond the edge of the frustum.  Every builder here returns ``(settings, inputs)`` in the shape of
``helpers.make_case``, is deterministic for its seed, and places the values that matter by construction.

All scenes are seen by the same orbit camera at (0, 0, 2) looking at the origin.  Gaussians are placed in view space
(pixel position, view depth, orientation relative to the image plane) and mapped to world space through the inverse of
``world_view_transform`` (``p_view = [p, 1] @ V``).
"""
import numpy as np
from scipy.spatial.transform import Rotation

import helpers  # noqa: F401  (puts the repository root on sys.path)
from dreamgaussian_b200 import scene

SH_C0 = scene.SH_C0
ALPHA_MIN = 1.0 / 255.0
FAINT_OPACITIES = (0.0, 1e-6, ALPHA_MIN * (1 - 1e-3), ALPHA_MIN * (1 + 1e-3), 0.0045)
NEAR = 0.2                      # DGR_NEAR_CULL_Z
FOV_CLAMP = 1.3                 # DGR_FOV_CLAMP


def camera(W, H, fovy_deg=49.1):
    return scene.orbit_camera(0.0, 0.0, 2.0, W, H, fovy_deg=fovy_deg)


def settings_of(cam, deg, bg=(1.0, 1.0, 1.0)):
    return dict(image_height=cam.image_height, image_width=cam.image_width, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy,
                bg=np.asarray(bg, np.float32), scale_modifier=1.0, viewmatrix=cam.world_view_transform,
                projmatrix=cam.full_proj_transform, sh_degree=deg, campos=cam.camera_center)


def focal(cam):
    """Pixels per unit of x / z (and y / z)."""
    return cam.image_width / (2.0 * cam.tanfovx), cam.image_height / (2.0 * cam.tanfovy)


def view_of_pixel(cam, px, py, z):
    """View-space points that project to pixel coordinates (px, py) (pixel centres at integers) at view depth z."""
    px, py, z = np.broadcast_arrays(np.asarray(px, np.float64), np.asarray(py, np.float64), np.asarray(z, np.float64))
    x = ((2.0 * px + 1.0) / cam.image_width - 1.0) * z * cam.tanfovx
    y = ((2.0 * py + 1.0) / cam.image_height - 1.0) * z * cam.tanfovy
    return np.stack([x, y, z], 1)


def view_to_world(cam, v):
    V = cam.world_view_transform.astype(np.float64)
    return (np.concatenate([v, np.ones((v.shape[0], 1))], 1) @ np.linalg.inv(V))[:, :3]


def world_to_view(cam, p):
    V = cam.world_view_transform.astype(np.float64)
    return np.concatenate([np.asarray(p, np.float64), np.ones((len(p), 1))], 1) @ V[:, :3]


def quat_of_view_axes(cam, Rv):
    """Unit quaternions (r, x, y, z) whose rotation puts the scale axes along the columns of the VIEW-space matrices Rv."""
    A = cam.world_view_transform.astype(np.float64)[:3, :3]          # world -> view is v = A^T w
    q = Rotation.from_matrix(np.einsum("ij,njk->nik", A, Rv)).as_quat()       # (x, y, z, w)
    return np.concatenate([q[:, 3:], q[:, :3]], 1)


def axes_in_image_plane(theta):
    """View-space rotations whose first axis lies in the image plane at angle theta (radians, from +x towards +y)."""
    c, s = np.cos(theta), np.sin(theta)
    z, o = np.zeros_like(c), np.ones_like(c)
    return np.stack([np.stack([c, s, z], 1), np.stack([-s, c, z], 1), np.stack([z, z, o], 1)], 2)


def shs_of_rgb(rgb, deg, rng, rest_sigma=0.05):
    """SH rows whose DC term alone gives colour rgb (SH_C0 dc + 0.5 = rgb), plus small higher-order terms."""
    M = (deg + 1) ** 2
    shs = np.zeros((rgb.shape[0], M, 3))
    shs[:, 0] = (rgb - 0.5) / SH_C0
    if M > 1:
        shs[:, 1:] = rng.normal(0.0, rest_sigma, (rgb.shape[0], M - 1, 3))
    return shs


def gaussians(cam, rng, view, sigma_px, Rv, opacity, rgb, deg):
    """Float64 arrays of Gaussians at view-space centres `view` with per-axis pixel sigmas sigma_px [N,3] (at their own depth)
    along the columns of the view-space rotations Rv."""
    fx, _ = focal(cam)
    return dict(means3D=view_to_world(cam, view), scales=sigma_px * view[:, 2:3] / fx, rotations=quat_of_view_axes(cam, Rv),
                opacities=np.asarray(opacity, np.float64).reshape(-1, 1), shs=shs_of_rgb(rgb, deg, rng))


def concat(*parts):
    return {k: np.concatenate([p[k] for p in parts], 0) for k in parts[0]}


def as_inputs(g):
    f32 = lambda a: np.ascontiguousarray(np.asarray(a, np.float64).astype(np.float32))
    return {k: f32(g[k]) for k in ("means3D", "opacities", "shs", "scales", "rotations")}


def _background(cam, rng, n, deg, z=(1.6, 2.6), sigma=(3.0, 8.0), opacity=None, rgb=None):
    """Ordinary Gaussians over the image (a little past its edges), anisotropic up to 2:1, random orientation."""
    W, H = cam.image_width, cam.image_height
    view = view_of_pixel(cam, rng.uniform(-10, W + 10, n), rng.uniform(-10, H + 10, n), rng.uniform(*z, n))
    s = rng.uniform(*sigma, (n, 1)) * rng.uniform(0.5, 1.0, (n, 3))
    op = rng.uniform(0.2, 0.9, n) if opacity is None else opacity
    col = rng.uniform(0.05, 0.95, (n, 3)) if rgb is None else rgb
    return gaussians(cam, rng, view, s, Rotation.random(n, random_state=rng).as_matrix(), op, col, deg)


# ---------------------------------------------------------------------------------------------------------------------------
# the regimes
# ---------------------------------------------------------------------------------------------------------------------------
def _saturated(cam, rng, n, deg, pairs=True, band=0.4):
    """Opacities from sigmoid(N(4, 3)), a quarter of them exactly 1 and a fifth in [0.99, 1); and, in front of everything,
    PAIRS of opacity-1 Gaussians (same centre, depths 0.1% apart): every pixel where both have o G >= 0.99 and nothing lies
    in front sees two alpha = 0.99 clamps in a row first, T = (1 - 0.99f)^2 = 9.99998e-5, just under the T-stop 1e-4.
      * large pairs (sigma 12 px) on a lattice whose footprints do not overlap: their core (o G >= 0.99, radius 0.142 sigma)
        is 1/550 of their footprint, so they reach few pixels;
      * in the bottom `band` of the image (a fraction of its height), nearer still, sub-pixel pairs (cov2D = 0.3 I) 0.05 px off every second pixel centre
        on both axes: G = 0.992 at that pixel, and a neighbouring pair 2 px away stays below 1/255 there, so a quarter of the
        band's pixels are on the knife edge."""
    op = 1.0 / (1.0 + np.exp(-rng.normal(4.0, 3.0, n)))
    k = rng.permutation(n)
    op[k[: n // 4]] = 1.0
    op[k[n // 4: n // 4 + n // 5]] = rng.uniform(0.99, 1.0, n // 5)
    parts = [_background(cam, rng, n, deg, sigma=(4.0, 10.0), opacity=op)]
    if pairs:
        W, H = cam.image_width, cam.image_height
        sig = 12.0
        step = 3.6 * sig
        cx, cy = np.meshgrid(np.arange(step / 2, W - sig, step), np.arange(step / 2, H - sig, step), indexing="ij")
        cx, cy = cx.ravel() + rng.uniform(-0.5, 0.5, cx.size), cy.ravel() + rng.uniform(-0.5, 0.5, cx.size)
        m = cx.size
        z = 1.0 + 0.3 * rng.random(m)
        rgb = rng.uniform(0.05, 0.95, (m, 3))
        for dz in (0.0, 1e-3):
            view = view_of_pixel(cam, cx, cy, z * (1.0 + dz))
            parts.append(gaussians(cam, rng, view, np.full((m, 3), sig), axes_in_image_plane(rng.uniform(0, np.pi, m)),
                                   np.ones(m), rgb if dz == 0.0 else rng.uniform(0.05, 0.95, (m, 3)), deg))
        cx, cy = np.meshgrid(np.arange(0, W, 2.0), np.arange(2 * int(0.5 * (1.0 - band) * H), H, 2.0), indexing="ij")
        cx, cy = cx.ravel() + 0.03, cy.ravel() + 0.04
        m = cx.size
        z = 0.8 + 0.1 * rng.random(m)
        for dz in (0.0, 1e-3):
            parts.append(gaussians(cam, rng, view_of_pixel(cam, cx, cy, z * (1.0 + dz)), np.full((m, 3), 1e-4),
                                   axes_in_image_plane(np.zeros(m)), np.ones(m), rng.uniform(0.05, 0.95, (m, 3)), deg))
    return concat(*parts)


def _dark(cam, rng, n, deg):
    """DC terms giving rgb < 0 (clamped) for a third of the (Gaussian, channel) pairs, rgb in (0, 1) for a third and rgb > 1
    (never clamped from above) for the rest; no DC-only value within 0.05 of the clamp."""
    band = rng.integers(0, 3, (n, 3))
    rgb = np.choose(band, [rng.uniform(-1.0, -0.05, (n, 3)), rng.uniform(0.05, 0.95, (n, 3)), rng.uniform(1.05, 2.0, (n, 3))])
    return _background(cam, rng, n, deg, sigma=(2.0, 6.0), rgb=rgb)


def _needles(cam, rng, n, deg, constructed=96, long_px=(20.0, 400.0), log_ratio=(1.0, 3.0)):
    """Random needles (one long axis, two short) and discs (two long, one short) with axis ratios 10..1000 in random
    orientations; and `constructed` screen-space needles in the image plane at 45 or 135 degrees, sigma log-uniform in
    long_px along the long axis and 1e-3 px across (the low-pass filter dominates), centred on tile and sub-tile corners."""
    W, H = cam.image_width, cam.image_height
    view = view_of_pixel(cam, rng.uniform(0, W, n), rng.uniform(0, H, n), rng.uniform(1.6, 2.6, n))
    L = rng.uniform(5.0, 60.0, n)
    short = L / 10.0 ** rng.uniform(*log_ratio, n)
    disc = rng.random(n) < 0.5
    s = np.stack([L, np.where(disc, L * rng.uniform(0.3, 1.0, n), short), short * rng.uniform(0.5, 1.0, n)], 1)
    parts = [gaussians(cam, rng, view, s, Rotation.random(n, random_state=rng).as_matrix(), rng.uniform(0.2, 0.95, n),
                       rng.uniform(0.05, 0.95, (n, 3)), deg)]
    if constructed:
        m = constructed
        # pixel centres at integers: a 16-pixel tile corner is at 16 i - 0.5, an 8 x 4 / 8 x 8 sub-tile corner at 8 i - 0.5, 4 j - 0.5
        cx = 8.0 * rng.integers(1, max(2, W // 8), m) - 0.5
        cy = 4.0 * rng.integers(1, max(2, H // 4), m) - 0.5
        theta = np.where(rng.random(m) < 0.5, np.pi / 4, 3 * np.pi / 4)
        sig = np.stack([np.exp(rng.uniform(np.log(long_px[0]), np.log(long_px[1]), m)), np.full(m, 1e-3), np.full(m, 1e-3)], 1)
        parts.append(gaussians(cam, rng, view_of_pixel(cam, cx, cy, rng.uniform(1.6, 2.6, m)), sig, axes_in_image_plane(theta),
                               rng.uniform(0.3, 0.99, m), rng.uniform(0.05, 0.95, (m, 3)), deg))
    return concat(*parts)


def _faint(cam, rng, n, deg):
    """Two fifths of the opacities from FAINT_OPACITIES (0, 1e-6, 1/255 (1 -+ 1e-3), 0.0045), the rest ordinary."""
    op = rng.uniform(0.2, 0.9, n)
    k = rng.permutation(n)[: 2 * n // 5]
    op[k] = np.asarray(FAINT_OPACITIES)[np.arange(k.size) % len(FAINT_OPACITIES)]
    return _background(cam, rng, n, deg, sigma=(2.0, 8.0), opacity=op)


SUBPIXEL_OFFSETS = (0.5, 3.0, 7.5, 14.0, 15.5)          # within a 16-pixel tile


def _subpixel(cam, rng, deg, keep=1.0):
    """Sub-pixel Gaussians (scales 1e-4 of a pixel: cov2D = 0.3 I from the low-pass, radius 3) at SUBPIXEL_OFFSETS on both
    axes of every tile: half-integer positions, 16-pixel tile borders (15.5 | 16.5) and centres where mx -+ radius lands on a
    tile edge (3 - 3 = 0, 14 + 3 + 15 = 32); keep: the fraction of them kept (at random)."""
    W, H = cam.image_width, cam.image_height
    off = np.asarray(SUBPIXEL_OFFSETS)
    xs = (16.0 * np.arange((W + 15) // 16)[:, None] + off[None]).ravel()
    ys = (16.0 * np.arange((H + 15) // 16)[:, None] + off[None]).ravel()
    cx, cy = np.meshgrid(xs[xs < W], ys[ys < H], indexing="ij")
    cx, cy = cx.ravel(), cy.ravel()
    if keep < 1.0:
        k = rng.random(cx.size) < keep
        cx, cy = cx[k], cy[k]
    m = cx.size
    view = view_of_pixel(cam, cx, cy, rng.uniform(1.6, 2.6, m))
    return gaussians(cam, rng, view, 1e-4 * rng.uniform(0.5, 1.0, (m, 3)), Rotation.random(m, random_state=rng).as_matrix(),
                     rng.uniform(0.3, 1.0, m), rng.uniform(0.05, 0.95, (m, 3)), deg)


def _frustum_edge(cam, rng, n_near, n_edge, deg):
    """n_near Gaussians with view depths in [0.15, 0.25] (never within 2e-4 of the near plane 0.2) inside the field of view;
    n_edge per (axis, sign) with x/z (or y/z) at (1.1 .. 1.6) tan(fov / 2) and the other coordinate inside the view, and
    n_edge / 2 per corner with both beyond: every (axis, sign) of the J clamp at 1.3 tan(fov / 2) (never within 1e-3 of it)."""
    tx, ty = cam.tanfovx, cam.tanfovy
    fx, _ = focal(cam)
    z = rng.uniform(0.15, 0.25, n_near)
    z = np.where(np.abs(z - NEAR) < 2e-4, z + 5e-4, z)
    near = np.stack([rng.uniform(-0.8, 0.8, n_near) * tx * z, rng.uniform(-0.8, 0.8, n_near) * ty * z, z], 1)
    near_s = rng.uniform(2.0, 8.0, (n_near, 1)) * rng.uniform(0.5, 1.0, (n_near, 3))

    def beyond(m):
        r = rng.uniform(1.1, 1.6, m)
        return np.where(np.abs(r - FOV_CLAMP) < 1e-3, r + 2e-3, r)
    views = []
    for axis in (0, 1):
        for sign in (-1.0, 1.0):
            z = rng.uniform(1.0, 3.0, n_edge)
            r = np.stack([rng.uniform(-0.8, 0.8, n_edge) * tx, rng.uniform(-0.8, 0.8, n_edge) * ty], 1)
            r[:, axis] = sign * beyond(n_edge) * (tx, ty)[axis]
            views.append(np.stack([r[:, 0] * z, r[:, 1] * z, z], 1))
    for sx in (-1.0, 1.0):
        for sy in (-1.0, 1.0):
            m = n_edge // 2
            z = rng.uniform(1.0, 3.0, m)
            views.append(np.stack([sx * beyond(m) * tx * z, sy * beyond(m) * ty * z, z], 1))
    edge = np.concatenate(views, 0)
    m = edge.shape[0]
    # big enough (3 sigma > ~40 px) for most of them to reach into the image from beyond its edge
    edge_s = rng.uniform(12.0, 30.0, (m, 1)) * rng.uniform(0.6, 1.0, (m, 3))
    view = np.concatenate([near, edge], 0)
    s = np.concatenate([near_s, edge_s], 0)
    N = view.shape[0]
    return gaussians(cam, rng, view, s, Rotation.random(N, random_state=rng).as_matrix(), rng.uniform(0.3, 0.95, N),
                     rng.uniform(0.05, 0.95, (N, 3)), deg)


# ---------------------------------------------------------------------------------------------------------------------------
# public builders: (settings, inputs) like helpers.make_case
# ---------------------------------------------------------------------------------------------------------------------------
def saturated(seed=0, W=256, H=256, deg=1, n=6000):
    cam, rng = camera(W, H), np.random.default_rng(1000 + seed)
    return settings_of(cam, deg), as_inputs(_saturated(cam, rng, n, deg))


def dark(seed=0, W=128, H=128, deg=0, n=3000):
    cam, rng = camera(W, H), np.random.default_rng(2000 + seed)
    return settings_of(cam, deg, bg=(0.0, 0.0, 0.0)), as_inputs(_dark(cam, rng, n, deg))


def needles(seed=0, W=256, H=256, deg=1, n=1500, constructed=96, max_ratio=1000.0):
    cam, rng = camera(W, H), np.random.default_rng(3000 + seed)
    return settings_of(cam, deg), as_inputs(_needles(cam, rng, n, deg, constructed=constructed, log_ratio=(1.0, np.log10(max_ratio))))


def faint(seed=0, W=128, H=128, deg=1, n=2000):
    cam, rng = camera(W, H), np.random.default_rng(4000 + seed)
    return settings_of(cam, deg), as_inputs(_faint(cam, rng, n, deg))


def subpixel(seed=0, W=128, H=128, deg=1):
    cam, rng = camera(W, H), np.random.default_rng(5000 + seed)
    return settings_of(cam, deg), as_inputs(_subpixel(cam, rng, deg))


def frustum_edge(seed=0, W=128, H=96, deg=1, n_near=400, n_edge=60):
    cam, rng = camera(W, H), np.random.default_rng(6000 + seed)
    return settings_of(cam, deg), as_inputs(_frustum_edge(cam, rng, n_near, n_edge, deg))


def trained_mix(seed=0, W=512, H=512, deg=3):
    """Every regime above in one cloud of ~50k Gaussians (in random order), the ordinary ones included."""
    cam, rng = camera(W, H), np.random.default_rng(7000 + seed)
    g = concat(_background(cam, rng, 8000, deg), _saturated(cam, rng, 10000, deg, band=0.05), _dark(cam, rng, 8000, deg),
               _needles(cam, rng, 8000, deg, constructed=0, log_ratio=(1.0, 2.0)), _faint(cam, rng, 6000, deg), _subpixel(cam, rng, deg, keep=0.3),
               _frustum_edge(cam, rng, 400, 80, deg))
    perm = rng.permutation(g["means3D"].shape[0])
    return settings_of(cam, deg), as_inputs({k: v[perm] for k, v in g.items()})


def compact_mix(P, seed=0, W=72, H=56, deg=1):
    """Exactly P Gaussians drawn (in random order) from a small mix of the regimes above: ordinary, saturated (no pairs,
    trained_mix's band), needles with axis ratios 10-30 (the ratios test_trained_regimes_gpu.py holds to the suite's rules),
    clamped colours, and near-plane / frustum-edge Gaussians.  tests/test_kernel_coverage_gpu.py builds its scenes with it."""
    cam, rng = camera(W, H), np.random.default_rng(seed)
    g = concat(_background(cam, rng, P // 2, deg), _saturated(cam, rng, P // 3, deg, pairs=False, band=0.05),
               _needles(cam, rng, P // 12, deg, constructed=0, log_ratio=(1.0, np.log10(30.0))), _dark(cam, rng, P // 8, deg),
               _frustum_edge(cam, rng, P // 16, max(2, P // 80), deg))
    n = g["means3D"].shape[0]
    assert n >= P, (n, P)
    idx = rng.permutation(n)[:P]
    return settings_of(cam, deg), as_inputs({k: v[idx] for k, v in g.items()})


def raw_of(inputs, seed=0, extremes=False):
    """scene.to_raw_parameters of the inputs; extremes: on disjoint 2% slices, opacity logits in +-12, log-scales moved to
    within +-6 of the cloud's mean on Gaussians with axis ratios below 3 (one shift per Gaussian), and quaternion lengths from 1e-3 to 1e3."""
    raw = scene.to_raw_parameters(inputs, seed=seed)
    if extremes:
        rng = np.random.default_rng(8000 + seed)
        P = raw["xyz"].shape[0]
        ls = raw["scaling"].astype(np.float64)
        # scale extremes on Gaussians with axis ratios below 3: a needle grown 400-fold has a cov2D condition number (~1e10)
        # whose float32 cancellation no oracle bound covers
        k = np.concatenate([rng.permutation(np.nonzero(ls.max(1) - ls.min(1) < np.log(3.0))[0]), rng.permutation(P)])
        m = P // 50
        b = k[:m]
        rest = np.setdiff1d(np.arange(P), b)
        rest = rng.permutation(rest)
        a, c = rest[:m], rest[m: 2 * m]
        raw["opacity"][a] = rng.uniform(-12.0, 12.0, (m, 1)).astype(np.float32)
        raw["scaling"][b] = (ls[b] - ls[b].mean(axis=1, keepdims=True) + ls.mean() + rng.uniform(-6.0, 6.0, (m, 1))).astype(np.float32)
        q = raw["rotation"][c].astype(np.float64)
        raw["rotation"][c] = (q / np.linalg.norm(q, axis=1, keepdims=True) * 10.0 ** rng.uniform(-3.0, 3.0, (m, 1))).astype(np.float32)
    return raw


# ---------------------------------------------------------------------------------------------------------------------------
# isolated Gaussians: no pixel has more than one candidate, so each pixel's alpha belongs to exactly one Gaussian
# ---------------------------------------------------------------------------------------------------------------------------
def isolated_needles(seed=0, theta=np.pi / 4, n=36, W=1024, H=1024):
    """A comb of parallel screen-space needles at angle theta through the image centre: long-axis sigma log-uniform in 20..110
    px, 1e-3 px across, centres on 8 x 8 sub-tile corners 8 px apart across the needles (perpendicular gap 11.3 px > the
    3.7 px the low-pass makes their alpha >= 1/255 width)."""
    cam, rng = camera(W, H), np.random.default_rng(9000 + seed)
    k = np.arange(n) - n // 2
    d = np.array([np.cos(theta), np.sin(theta)])
    perp = np.sign(np.array([-d[1], d[0]])).astype(np.float64)        # (-1, 1) or (-1, -1): along the sub-tile lattice
    cx = W / 2 + 8.0 * k * perp[0] - 0.5
    cy = H / 2 + 8.0 * k * perp[1] - 0.5
    sig = np.stack([np.exp(rng.uniform(np.log(20.0), np.log(110.0), n)), np.full(n, 1e-3), np.full(n, 1e-3)], 1)
    g = gaussians(cam, rng, view_of_pixel(cam, cx, cy, rng.uniform(1.6, 2.6, n)), sig, axes_in_image_plane(np.full(n, theta)),
                  rng.uniform(0.3, 1.0, n), rng.uniform(0.05, 0.95, (n, 3)), 0)
    return settings_of(cam, 0), as_inputs(g)


def isolated_small(seed=0, W=960, H=960, cell=96):
    """One Gaussian per cell x cell block, at a random position near the block's centre: saturated (opacity 1 or in
    [0.99, 1)), faint (FAINT_OPACITIES) and needles up to 12 px long-axis sigma (footprint radius < 42 px) in random 3-D
    orientations, with ratios up to 1000."""
    cam, rng = camera(W, H), np.random.default_rng(9500 + seed)
    cx, cy = np.meshgrid(np.arange(cell / 2, W - cell / 2 + 1, cell), np.arange(cell / 2, H - cell / 2 + 1, cell), indexing="ij")
    cx, cy = cx.ravel() + rng.uniform(-2, 2, cx.size), cy.ravel() + rng.uniform(-2, 2, cx.size)
    m = cx.size
    kind = np.arange(m) % 3                                 # 0 saturated, 1 faint, 2 needle
    op = np.where(rng.random(m) < 0.5, 1.0, rng.uniform(0.99, 1.0, m))
    op = np.where(kind == 1, np.asarray(FAINT_OPACITIES)[rng.integers(0, len(FAINT_OPACITIES), m)], op)
    op = np.where(kind == 2, rng.uniform(0.3, 1.0, m), op)
    L = np.where(kind == 2, rng.uniform(4.0, 12.0, m), rng.uniform(2.0, 8.0, m))
    s = np.stack([L, np.where(kind == 2, L / 10.0 ** rng.uniform(1, 3, m), L * rng.uniform(0.5, 1.0, m)),
                  L * rng.uniform(0.001, 1.0, m)], 1)
    g = gaussians(cam, rng, view_of_pixel(cam, cx, cy, rng.uniform(1.6, 2.6, m)), s, Rotation.random(m, random_state=rng).as_matrix(),
                  op, rng.uniform(0.05, 0.95, (m, 3)), 0)
    return settings_of(cam, 0), as_inputs(g)


def clamped_stacks(seed=0, n=24):
    """1 x 1 images, each seen through a stack of three Gaussians centred within 0.05 px of the pixel: in front one of
    opacity 1 or in [0.995, 1) (alpha clamped to 0.99), then alpha ~0.5, then another clamped one (T-stop at 5e-5, far from
    the knife edge).  The front Gaussian's only hit is clamped, so its opacity and means2D gradients are all straight-through
    terms (they use the unclamped o G).  Returns a list of (settings, inputs)."""
    rng = np.random.default_rng(9900 + seed)
    cam = camera(1, 1, fovy_deg=2.0)                        # 1 px = 0.035 units of x / z: sigma of a few pixels
    cases = []
    for _ in range(n):
        off = rng.uniform(-0.05, 0.05, (3, 2))
        view = view_of_pixel(cam, off[:, 0], off[:, 1], np.array([1.5, 1.7, 1.9]) + rng.uniform(0, 0.05, 3))
        op = np.array([1.0 if rng.random() < 0.5 else rng.uniform(0.995, 1.0), rng.uniform(0.45, 0.55), 1.0])
        s = rng.uniform(3.0, 6.0, (3, 3))
        g = gaussians(cam, rng, view, s, Rotation.random(3, random_state=rng).as_matrix(), op, rng.uniform(0.05, 0.95, (3, 3)), 1)
        cases.append((settings_of(cam, 1, bg=(0.3, 0.6, 0.9)), as_inputs(g)))
    return cases
