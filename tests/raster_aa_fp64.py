"""fp64 restatement of the rasterizer's antialiasing (upstream's `antialiasing` setting) with running error bounds (test helper).

K1 with the filter stores conic_opacity.w = o rho, rho = sqrt(max(2.5e-5, r)), r = det0 / det1, det0 = a0 c0 - b^2 the determinant
of the projected 2D covariance and det1 = (a0 + 0.3)(c0 + 0.3) - b^2 that of the dilated one (include/gavatar.h).  The backward
(preprocess_bwd_kernel<..., kAA>) writes dL/do = gO rho and, where r > 2.5e-5, adds dL/drho drho/dr dr/d(a0, b, c0) to dL/d(a, b, c)
before they are pulled back through J W, with o = conic_opacity.w / rho and rho recomputed from its own covariance.

`forward_opacity` restates K1's stored opacity from the kernel's own inputs: the staged cov3d, the camera and the opacities.  It
follows preprocess_one's operation order, tracked with the (value, bound) arithmetic of tests/raster_fp64.py.  Every K1 operation is
round-to-nearest without contraction, and the bound counts each of them.

`preprocess_backward` is raster_fp64.preprocess_backward with the antialiasing terms (its `aa` argument) added where the kernel adds
them, right after dL/d(a, b, c), so the restatement of everything around the new terms stays the one the existing tests maintain.  Bug
switches for the self-checks: no_rho_dopac (dL/do without the rho factor), no_drho (the dL/drho term dropped), dilated_num (det1
used as r's numerator), clamp_grad (the rho term also where the clamp is active).
"""
import math

import torch

import raster_fp64 as rf
from raster_fp64 import C03, R_MIN, add, cf32, clamp_min, div, lsum, mul, sqrt_, sub


def rho_of(a0, b, c0, dilated_num=False):
    """(r, rho, det0, det1) of tracked a0, b, c0 in the kernels' operation order."""
    a, c = add(a0, C03), add(c0, C03)
    det1 = sub(mul(a, c), mul(b, b))
    det0 = det1 if dilated_num else sub(mul(a0, c0), mul(b, b))
    r = div(det0, det1)
    return r, sqrt_(clamp_min(r, R_MIN)), det0, det1


def forward_opacity(cov3d, means, view, tanfovx, tanfovy, H, W, opacities, bug=()):
    """K1's stored opacity for P Gaussians of one frame (tensors of fp32 values, computed in float64): (value, bound) [P].
    Only meaningful where the Gaussian is visible."""
    dev = means.device
    f = lambda t: torch.as_tensor(t).to(device=dev, dtype=torch.float64)
    means, view, cov3d, o = f(means), f(view).reshape(16), f(cov3d), f(opacities).reshape(-1)
    px, py, pz = means[:, 0], means[:, 1], means[:, 2]
    tvx, tvy, tvz = (rf.xf_row32(view, r, px, py, pz) for r in range(3))
    tanx, tany = cf32(tanfovx), cf32(tanfovy)
    fx = div(float(W), (torch.tensor(2.0 * tanx, dtype=torch.float64, device=dev), 0.0))      # 2 tan: exact in fp32
    fy = div(float(H), (torch.tensor(2.0 * tany, dtype=torch.float64, device=dev), 0.0))
    limx, limy = cf32(cf32(1.3) * tanx), cf32(cf32(1.3) * tany)
    tx = rf.f32(rf.f32(tvx / tvz).clamp(-limx, limx) * tvz)
    ty = rf.f32(rf.f32(tvy / tvz).clamp(-limy, limy) * tvz)
    tz2 = rf.f32(tvz * tvz)
    tv = (tvz, 0.0)
    J00, J02 = div(fx, tv), div(rf.neg(mul(fx, (tx, 0.0))), (tz2, 0.0))
    J11, J12 = div(fy, tv), div(rf.neg(mul(fy, (ty, 0.0))), (tz2, 0.0))
    V = lambda k: (view[k], 0.0)
    m0 = [add(mul(V(k * 4 + 0), J00), mul(V(k * 4 + 2), J02)) for k in range(3)]
    m1 = [add(mul(V(k * 4 + 1), J11), mul(V(k * 4 + 2), J12)) for k in range(3)]
    c3 = [(cov3d[:, k], 0.0) for k in range(6)]
    S = [[c3[0], c3[1], c3[2]], [c3[1], c3[3], c3[4]], [c3[2], c3[4], c3[5]]]
    v0 = [lsum(*[mul(S[j][k], m0[k]) for k in range(3)]) for j in range(3)]
    v1 = [lsum(*[mul(S[j][k], m1[k]) for k in range(3)]) for j in range(3)]
    a0 = lsum(*[mul(m0[k], v0[k]) for k in range(3)])
    b = lsum(*[mul(m0[k], v1[k]) for k in range(3)])
    c0 = lsum(*[mul(m1[k], v1[k]) for k in range(3)])
    r, rho, _, _ = rho_of(a0, b, c0, dilated_num="dilated_num" in bug)
    return mul((o, 0.0), rho), dict(a0=a0, b=b, c0=c0, r=r, rho=rho)


def preprocess_backward(*, co_w, bug=(), **inp):
    """raster_fp64.preprocess_backward of a frame rendered with the filter: co_w [P] is the stored opacity (geom conic_opacity.w).
    Adds "d_opacities" (value, bound), "marg_clamp" (clamp decisions within the bound) and "active" (r > 2.5e-5) to its dict."""
    aa = dict(co_w=co_w, bug=tuple(bug))
    out = rf.preprocess_backward(**inp, aa=aa)
    vis = out["vis"]
    dv, de = aa["d_opacities"]
    out["d_opacities"] = (torch.where(vis, dv, 0.0), torch.where(vis, de, 0.0) if torch.is_tensor(de) else 0.0 * dv)
    out["marg_clamp"] = aa["marg_clamp"] & vis
    out["active"] = aa["active"] & vis
    return out


# ---------------------------------------------------------------------------------------------- plain fp64 (no bounds)
def rho64(a0, b, c0):
    """rho of float64 tensors (differentiable; the clamp's subgradient is 0)."""
    det0 = a0 * c0 - b * b
    det1 = (a0 + 0.3) * (c0 + 0.3) - b * b
    return torch.sqrt(torch.clamp_min(det0 / det1, 2.5e-5))


def sigma2_64(means, cov3x3, viewmatrix, tanfovx, tanfovy, H, W):
    """The projected 2D covariance (a0, b, c0) before the dilation, as K1 forms it (upstream's EWA Jacobian with the 1.3 tan
    guard band), differentiable in float64.  viewmatrix is the transposed 4x4 (p_view = [p, 1] @ V)."""
    V = viewmatrix.to(means)
    t = means @ V[:3, :3] + V[3, :3]
    tz = t[:, 2]
    fx, fy = W / (2.0 * tanfovx), H / (2.0 * tanfovy)
    limx, limy = 1.3 * tanfovx, 1.3 * tanfovy
    tx = torch.clamp(t[:, 0] / tz, -limx, limx) * tz
    ty = torch.clamp(t[:, 1] / tz, -limy, limy) * tz
    zero = torch.zeros_like(tz)
    J = torch.stack([torch.stack([fx / tz, zero, -fx * tx / (tz * tz)], -1), torch.stack([zero, fy / tz, -fy * ty / (tz * tz)], -1)], 1)
    T = J @ V[:3, :3].T                                    # [P,2,3]: J W with W the camera rotation
    S2 = T @ cov3x3 @ T.transpose(1, 2)
    return S2[:, 0, 0], S2[:, 0, 1], S2[:, 1, 1]


def truncated_gaussian_mass(o, sx, sy, thr=1.0 / 255.0):
    """Sum over an unbounded pixel grid of alpha = o exp(-q/2) where alpha >= thr, in the continuum limit, for an axis-aligned Gaussian
    of standard deviations sx, sy (px): 2 pi sx sy (o - thr) where o > thr (the mass inside the ellipse q <= 2 ln(o / thr))."""
    if o <= thr:
        return 0.0
    return 2.0 * math.pi * sx * sy * (o - thr)
