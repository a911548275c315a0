"""Drop-in import name: /root/reference/gs_renderer.py:10-13 does
``from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer``.
Everything is implemented in dreamgaussian_b200 (sm_90a CUDA behind the C ABI of include/dgr_b200.h)."""
from dreamgaussian_b200.rasterizer import (  # noqa: F401
    GaussianRasterizationSettings,
    GaussianRasterizer,
    rasterize_gaussians,
    _RasterizeGaussians,
)

__all__ = ["GaussianRasterizationSettings", "GaussianRasterizer", "rasterize_gaussians"]
