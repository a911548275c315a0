"""Synthetic DreamGaussian-like inputs for the rasterizer path: Gaussian clouds and orbit cameras.

Host-side only (numpy); nothing here is on the GPU hot path.  It restates, from the maths, the conventions of the
caller either side of the op so that benchmarks and parity tests feed the rasterizer exactly what
``Renderer.render`` would:

* camera: ``orbit_camera`` (/root/reference/cam_utils.py:45-62, look-at :24-41) and ``MiniCam``
  (/root/reference/gs_renderer.py:645-671: w2c rectification, row-vector view / full-projection matrices,
  ``camera_center = -c2w[:3, 3]``), projection matrix (/root/reference/gs_renderer.py:629-642);
* cloud: uniform-in-ball initialisation (/root/reference/gs_renderer.py:694-702), isotropic scales from the mean
  squared distance to the 3 nearest neighbours (/root/reference/gs_renderer.py:341-342 via simple-knn), identity
  quaternions, opacity 0.1 (/root/reference/gs_renderer.py:343-346), SH DC from RGB2SH (/root/reference/sh_utils.py:114-115).

SURVEY.md §8(d) fixes the distributions used by bench.py ("init" and "trained-like" opacity variants).
"""
import math
from typing import NamedTuple, Optional

import numpy as np

SH_C0 = 0.28209479177387814  # sh_utils.py:26


class Camera(NamedTuple):
    """What MiniCam exposes to Renderer.render (gs_renderer.py:645-671), as float32 numpy."""
    image_height: int
    image_width: int
    fovy: float
    fovx: float
    tanfovx: float
    tanfovy: float
    world_view_transform: np.ndarray  # [4,4]  = w2c^T   (p_view = [p,1] @ V)
    full_proj_transform: np.ndarray   # [4,4]  = V @ P^T
    camera_center: np.ndarray         # [3]    = -c2w[:3,3]  (sign quirk of the caller, consumed as given)


def _unit(v, eps=1e-20):
    return v / np.sqrt(max(float(np.dot(v, v)), eps))


def orbit_pose(elevation_deg: float, azimuth_deg: float, radius: float = 1.0) -> np.ndarray:
    """Camera-to-world pose looking at the origin (OpenGL convention, forward = +z of the camera frame)."""
    el, az = math.radians(elevation_deg), math.radians(azimuth_deg)
    eye = np.array([radius * math.cos(el) * math.sin(az), -radius * math.sin(el), radius * math.cos(el) * math.cos(az)])
    fwd = _unit(eye)                                   # campos - target, target = 0
    right = _unit(np.cross(np.array([0.0, 1.0, 0.0]), fwd))
    up = _unit(np.cross(fwd, right))
    pose = np.eye(4, dtype=np.float32)
    pose[:3, 0], pose[:3, 1], pose[:3, 2], pose[:3, 3] = right, up, fwd, eye
    return pose


def projection_matrix(znear: float, zfar: float, fovx: float, fovy: float) -> np.ndarray:
    P = np.zeros((4, 4), dtype=np.float32)
    P[0, 0] = 1.0 / math.tan(fovx / 2)
    P[1, 1] = 1.0 / math.tan(fovy / 2)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


def make_camera(pose: np.ndarray, width: int, height: int, fovy_deg: float = 49.1,
                znear: float = 0.01, zfar: float = 100.0) -> Camera:
    fovy = math.radians(fovy_deg)
    fovx = 2 * math.atan(math.tan(fovy / 2) * width / height)      # cam_utils.py:77-79
    w2c = np.linalg.inv(pose.astype(np.float32))
    w2c[1:3, :3] *= -1
    w2c[:3, 3] *= -1
    V = np.ascontiguousarray(w2c.T.astype(np.float32))
    Pt = projection_matrix(znear, zfar, fovx, fovy).T
    return Camera(int(height), int(width), fovy, fovx, math.tan(fovx * 0.5), math.tan(fovy * 0.5),
                  V, np.ascontiguousarray((V @ Pt).astype(np.float32)), (-pose[:3, 3]).astype(np.float32))


def orbit_camera(elevation_deg, azimuth_deg, radius=2.0, width=800, height=800, fovy_deg=49.1) -> Camera:
    return make_camera(orbit_pose(elevation_deg, azimuth_deg, radius), width, height, fovy_deg)


def knn3_mean_sqdist(xyz: np.ndarray) -> np.ndarray:
    """Mean squared distance to the 3 nearest neighbours (what simple-knn's distCUDA2 returns)."""
    from scipy.spatial import cKDTree
    d, _ = cKDTree(xyz).query(xyz, k=4)
    return (d[:, 1:] ** 2).mean(axis=1)


def make_cloud(num_pts: int, sh_degree: int = 3, seed: int = 0, radius: float = 0.5,
               opacity: str = "trained", anisotropic: bool = True, sigma: Optional[float] = None) -> dict:
    """Gaussian cloud as the op's float32 inputs: means3D, scales, rotations, opacities [P,1], shs [P,M,3].

    It models a cloud at initialisation or early in training.  Saturated opacities, clamped and over-bright colours,
    needle Gaussians, opacities at or below 1/255, sub-pixel Gaussians and Gaussians at the near plane or the frustum edge
    (what a trained model is full of) come from the builders in tests/trained_scenes.py.

    opacity: "init" -> 0.1 everywhere (reference init); "trained" -> U(0.05, 0.95).
    anisotropic: per-axis sigma * exp(N(0, 0.3^2)) and random unit quaternions (else isotropic, identity).
    sigma: override the 3-NN derived isotropic scale (used by tests to avoid the kd-tree).
    """
    rng = np.random.default_rng(seed)
    phis = rng.random(num_pts) * 2 * np.pi
    costheta = rng.random(num_pts) * 2 - 1
    thetas = np.arccos(costheta)
    r = radius * np.cbrt(rng.random(num_pts))
    xyz = np.stack((r * np.sin(thetas) * np.cos(phis), r * np.sin(thetas) * np.sin(phis), r * np.cos(thetas)), axis=1)
    if sigma is None:
        s = np.sqrt(np.clip(knn3_mean_sqdist(xyz), 1e-7, None))
    else:
        s = np.full((num_pts,), float(sigma))
    scales = np.repeat(s[:, None], 3, axis=1)
    rots = np.zeros((num_pts, 4)); rots[:, 0] = 1
    if anisotropic:
        scales = scales * np.exp(rng.normal(0, 0.3, (num_pts, 3)))
        q = rng.normal(0, 1, (num_pts, 4))
        rots = q / np.linalg.norm(q, axis=1, keepdims=True)
    if opacity == "init":
        op = np.full((num_pts, 1), 0.1)
    elif opacity == "trained":
        op = rng.uniform(0.05, 0.95, (num_pts, 1))
    else:
        raise ValueError(opacity)
    M = (sh_degree + 1) ** 2
    shs = np.zeros((num_pts, M, 3))
    shs[:, 0, :] = (rng.random((num_pts, 3)) - 0.5) / SH_C0
    if M > 1:
        shs[:, 1:, :] = rng.normal(0, 0.1, (num_pts, M - 1, 3))
    f32 = lambda a: np.ascontiguousarray(a.astype(np.float32))
    return dict(means3D=f32(xyz), scales=f32(scales), rotations=f32(rots), opacities=f32(op), shs=f32(shs))


def to_raw_parameters(cloud: dict, seed: int = 0) -> dict:
    """The same cloud as GaussianModel's RAW parameters (gs_renderer.py:140-160, inverse of the activations at :127-138):
    _xyz, _features_dc [P,1,3], _features_rest [P,M-1,3], _opacity = logit, _scaling = log, _rotation = unit quaternion
    times a random positive length (F.normalize must undo it)."""
    rng = np.random.default_rng(seed + 7919)
    op = np.clip(cloud["opacities"].astype(np.float64), 1e-6, 1 - 1e-6)
    length = rng.uniform(0.5, 2.0, (cloud["rotations"].shape[0], 1))
    f32 = lambda a: np.ascontiguousarray(np.asarray(a, np.float64).astype(np.float32))
    return dict(xyz=f32(cloud["means3D"]), features_dc=f32(cloud["shs"][:, :1]), features_rest=f32(cloud["shs"][:, 1:]),
                opacity=f32(np.log(op / (1 - op))), scaling=f32(np.log(cloud["scales"].astype(np.float64))),
                rotation=f32(cloud["rotations"].astype(np.float64) * length))


def bench_views(n: int, width: int, height: int, radius: float = 2.0):
    """The fixed benchmark camera set of SURVEY.md §8(d): orbit(0, 0) then 45-degree azimuth steps; beyond 8 views further
    rings of 8 at other elevations (the reference samples elevation in [-30, 30], main.py:213-216), each ring turned a bit."""
    elev = (0.0, 15.0, -15.0, 30.0, -30.0, 7.5, -7.5, 22.5)
    cams = []
    for i in range(n):
        ring = i // 8
        az = (45.0 * i + 5.625 * ring) % 360.0
        cams.append(orbit_camera(elev[ring % 8], az - (360.0 if az >= 180.0 else 0.0), radius, width, height))
    return cams
