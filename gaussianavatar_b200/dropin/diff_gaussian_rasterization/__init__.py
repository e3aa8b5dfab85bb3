"""Drop-in `diff_gaussian_rasterization` package: put `<repo>/gaussianavatar_b200/dropin` (and `<repo>`) on PYTHONPATH and the
reference's `from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer`
(/root/reference gaussian_renderer/__init__.py:6) resolves to the sm_90a implementation."""
from gaussianavatar_b200.rasterizer import (GaussianRasterizationSettings, GaussianRasterizer,  # noqa: F401
                                             rasterize_gaussians)

__all__ = ["GaussianRasterizationSettings", "GaussianRasterizer", "rasterize_gaussians"]
