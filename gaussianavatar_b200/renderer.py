"""`gaussian_renderer.render_batch` drop-in (reference: /root/reference gaussian_renderer/__init__.py:8-50)."""
from __future__ import annotations

import math

import torch

from .rasterizer import GaussianRasterizationSettings, GaussianRasterizer


def render_batch(points, shs, colors_precomp, rotations, scales, opacity, FovX, FovY, height, width, bg_color,
                 world_view_transform, full_proj_transform, active_sh_degree, camera_center, antialiasing=False):
    """Same signature, argument meaning and return value ([3,H,W] image; radii dropped) as the reference, plus the rasterizer's
    `antialiasing` setting (default off, as the reference renders)."""
    # the reference allocates a zero screen-space leaf only so that its .grad could be read (gaussian_renderer/
    # __init__.py:11-15); it is a local that is never returned, so nothing can read it: pass a plain placeholder and
    # skip producing that gradient
    screenspace_points = torch.zeros(0, dtype=points.dtype, device=points.device)
    raster_settings = GaussianRasterizationSettings(
        image_height=int(height), image_width=int(width), tanfovx=math.tan(float(FovX) * 0.5),
        tanfovy=math.tan(float(FovY) * 0.5), bg=bg_color, scale_modifier=1.0, viewmatrix=world_view_transform,
        projmatrix=full_proj_transform, sh_degree=active_sh_degree, campos=camera_center, prefiltered=False, debug=False,
        antialiasing=bool(antialiasing))
    rasterizer = GaussianRasterizer(raster_settings=raster_settings)
    rendered_image, _ = rasterizer(means3D=points, means2D=screenspace_points, shs=shs, colors_precomp=colors_precomp,
                                   opacities=opacity, scales=scales, rotations=rotations, cov3D_precomp=None)
    return rendered_image
