"""Seeded SH coefficients and precomputed covariances for the rasterizer's other input modes (test helper, not product)."""
import torch

from oracle.raster_twin import quat_to_rot
from oracle.raster_twin_ex import SH_C0, sh_to_rgb


def pre_clamp(means3D, shs, degree, campos):
    """sum_k basis_k(dir) sh_k + 0.5 before the clamp at 0, in fp64 (a large sh_0 shift keeps the clamp inactive)."""
    big = 100.0
    shifted = torch.as_tensor(shs, dtype=torch.float64).clone()
    shifted[:, 0] += big
    return sh_to_rgb(torch.as_tensor(means3D, dtype=torch.float64), shifted, degree, campos) - SH_C0 * big


def random_shs(sc, degree, M, seed=0, clamp_frac=0.1, margin=1e-3):
    """[P, M, 3] fp32 coefficients for scene `sc` seen from its camera centre: no channel's pre-clamp value lies within `margin`
    of 0, except that channel 0 of the first clamp_frac of the Gaussians is pushed to -0.2 (deliberately clamped)."""
    g = torch.Generator().manual_seed(seed)
    P = sc["means3D"].shape[0]
    shs = (0.3 * torch.randn(P, M, 3, generator=g, dtype=torch.float64))
    campos = sc["cam"].camera_center.double()
    pre = pre_clamp(sc["means3D"], shs, degree, campos)
    # move every channel at least `margin` away from 0 through sh_0 (basis_0 is the constant C0)
    near = pre.abs() < margin
    shs[:, 0][near] += (2 * margin / SH_C0) * torch.where(pre[near] < 0, -1.0, 1.0)
    nclamp = int(clamp_frac * P)
    if nclamp:
        pre = pre_clamp(sc["means3D"], shs, degree, campos)
        shs[:nclamp, 0, 0] -= (pre[:nclamp, 0] + 0.2) / SH_C0
    return shs.float().contiguous()


def sigma_of(scales, rotations, scale_modifier=1.0):
    """[P, 6] (xx, xy, xz, yy, yz, zz) of R S^2 R^T, computed in fp64 and rounded to fp32."""
    R = quat_to_rot(torch.as_tensor(rotations, dtype=torch.float64))
    s = scale_modifier * torch.as_tensor(scales, dtype=torch.float64)
    S = R @ torch.diag_embed(s * s) @ R.transpose(1, 2)
    return torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], -1).float().contiguous()

