"""ORACLE — TEST INFRASTRUCTURE ONLY.

The fp64 autograd twin (``raster_twin.twin_forward``) with upstream's other inputs, so that torch.autograd cross-checks the
hand-derived SH-colour and ``d_cov3D`` backward of the C oracle and the CUDA kernels:
  * SH colours by plain torch ops with ``clamp(min=0)`` (the true derivative: zero on clamped channels, the direction term through
    the normalisation), passed to the twin as its colours;
  * a precomputed Sigma built symmetrically from its six values, passed to the twin through its covariance factorisation: with
    unit scales the twin forms ``Rq Rq^T``, so the twin's rotation builder is given the Cholesky factor of Sigma instead.
Small sizes only (the twin loops over Gaussians in Python).
"""
from __future__ import annotations

from unittest import mock

import torch

from . import raster_twin

SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435)


def sh_to_rgb(means3D, shs, degree, campos):
    """max(sum_k basis_k(dir) sh_k + 0.5, 0), dir = (mean - campos) / |mean - campos|, for shs [P,M,3]."""
    d = means3D - torch.as_tensor(campos, dtype=means3D.dtype).reshape(1, 3)
    d = d / d.norm(dim=1, keepdim=True)
    x, y, z = d[:, 0:1], d[:, 1:2], d[:, 2:3]
    c = SH_C0 * shs[:, 0]
    if degree >= 1:
        c = c - SH_C1 * y * shs[:, 1] + SH_C1 * z * shs[:, 2] - SH_C1 * x * shs[:, 3]
    if degree >= 2:
        xx, yy, zz = x * x, y * y, z * z
        c = (c + SH_C2[0] * x * y * shs[:, 4] + SH_C2[1] * y * z * shs[:, 5] + SH_C2[2] * (2 * zz - xx - yy) * shs[:, 6]
             + SH_C2[3] * x * z * shs[:, 7] + SH_C2[4] * (xx - yy) * shs[:, 8])
    if degree >= 3:
        c = (c + SH_C3[0] * y * (3 * xx - yy) * shs[:, 9] + SH_C3[1] * x * y * z * shs[:, 10]
             + SH_C3[2] * y * (4 * zz - xx - yy) * shs[:, 11] + SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * shs[:, 12]
             + SH_C3[4] * x * (4 * zz - xx - yy) * shs[:, 13] + SH_C3[5] * z * (xx - yy) * shs[:, 14]
             + SH_C3[6] * x * (xx - 3 * yy) * shs[:, 15])
    return (c + 0.5).clamp(min=0.0)


def sigma_matrix(cov6):
    """[P,6] (xx, xy, xz, yy, yz, zz) -> symmetric [P,3,3]: an off-diagonal value stands for both entries."""
    v = cov6
    return torch.stack([v[:, 0], v[:, 1], v[:, 2], v[:, 1], v[:, 3], v[:, 4], v[:, 2], v[:, 4], v[:, 5]], -1).reshape(-1, 3, 3)


def twin_forward_ex(means3D, colors, opacities, scales, rotations, bg, viewmatrix, projmatrix, tanfovx, tanfovy, H, W,
                    scale_modifier=1.0, return_aux=False, shs=None, sh_degree=0, campos=None, cov3D_precomp=None):
    """raster_twin.twin_forward; shs [P,M,3] (with sh_degree, campos) replace colors, cov3D_precomp [P,6] replaces scales /
    rotations / scale_modifier."""
    dt = torch.float64
    if shs is not None:
        colors = sh_to_rgb(means3D.to(dt), shs.to(dt), sh_degree, campos)
    if cov3D_precomp is None:
        return raster_twin.twin_forward(means3D, colors, opacities, scales, rotations, bg, viewmatrix, projmatrix, tanfovx, tanfovy,
                                        H, W, scale_modifier=scale_modifier, return_aux=return_aux)
    L = torch.linalg.cholesky(sigma_matrix(cov3D_precomp.to(dt)))          # Sigma = L L^T = "Rq diag(1) Rq^T"
    ones = torch.ones(L.shape[0], 3, dtype=dt)
    with mock.patch.object(raster_twin, "quat_to_rot", lambda q: q):
        return raster_twin.twin_forward(means3D, colors, opacities, ones, L, bg, viewmatrix, projmatrix, tanfovx, tanfovy, H, W,
                                        scale_modifier=1.0, return_aux=return_aux)
