"""fp64 restatement of the rasterizer's antialiasing (upstream's `antialiasing` setting) with running error bounds (test helper).

K1 with the filter stores conic_opacity.w = o rho, rho = sqrt(max(2.5e-5, r)), r = det0 / det1, det0 = a0 c0 - b^2 the determinant
of the projected 2D covariance and det1 = (a0 + 0.3)(c0 + 0.3) - b^2 that of the dilated one (include/gavatar.h).  The backward
(preprocess_bwd_kernel<..., kAA>) writes dL/do = gO rho and, where r > 2.5e-5, adds dL/drho drho/dr dr/d(a0, b, c0) to dL/d(a, b, c)
before they are pulled back through J W, with o = conic_opacity.w / rho and rho recomputed from its own covariance.

`forward_opacity` restates K1's stored opacity from the kernel's own inputs: the staged cov3d, the camera and the opacities.  It
follows preprocess_one's operation order, tracked with the (value, bound) arithmetic of tests/raster_fp64.py.  Every K1 operation is
round-to-nearest without contraction, and the bound counts each of them.

`preprocess_backward` is raster_fp64.preprocess_backward with the antialiasing terms inserted where the kernel adds them, right after
dL/d(a, b, c).  It is built from that function's own source, so the restatement of everything around the new terms stays the one the
existing tests maintain.  Bug switches for the self-checks: no_rho_dopac (dL/do without the rho factor), no_drho (the dL/drho term
dropped), dilated_num (det1 used as r's numerator), clamp_grad (the rho term also where the clamp is active).
"""
import inspect
import math

import torch

import raster_fp64 as rf
from raster_fp64 import add, cf32, div, lsum, mul, sqrt_, sub

R_MIN = cf32(2.5e-5)
C03, C009 = cf32(0.3), cf32(0.09)


def _clamp_min(a, t):
    """fmaxf(t, a) of a tracked value: 1-Lipschitz, so the bound carries over."""
    return a[0].clamp_min(t), a[1]


def rho_of(a0, b, c0, dilated_num=False):
    """(r, rho, det0, det1) of tracked a0, b, c0 in the kernels' operation order."""
    a, c = add(a0, C03), add(c0, C03)
    det1 = sub(mul(a, c), mul(b, b))
    det0 = det1 if dilated_num else sub(mul(a0, c0), mul(b, b))
    r = div(det0, det1)
    return r, sqrt_(_clamp_min(r, R_MIN)), det0, det1


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


def _aa_terms(loc, aa):
    """The kernel's kAA block on the restatement's locals: returns the new dL/d(a, b, c) and records d_opacities and the clamp
    decisions in aa."""
    m0, m1, v0, v1, b, denom = loc["m0"], loc["m1"], loc["v0"], loc["v1"], loc["b"], loc["denom"]
    bug = aa.get("bug", ())
    gO = (loc["d_conic_op"][:, 3], 0.0)
    a0 = lsum(*[mul(m0[k], v0[k]) for k in range(3)])
    c0 = lsum(*[mul(m1[k], v1[k]) for k in range(3)])
    det0 = denom if "dilated_num" in bug else sub(mul(a0, c0), mul(b, b))
    r = div(det0, denom)
    rho = sqrt_(_clamp_min(r, R_MIN))
    aa["d_opacities"] = gO if "no_rho_dopac" in bug else mul(gO, rho)
    active = r[0] > R_MIN
    aa["marg_clamp"] = (r[0] - R_MIN).abs() <= r[1]
    aa["active"] = active
    if "clamp_grad" in bug:
        active = torch.ones_like(active)
    da, db, dc = loc["dL_da"], loc["dL_db"], loc["dL_dc"]
    if "no_drho" in bug:
        return da, db, dc
    co_w = (torch.as_tensor(aa["co_w"]).to(r[0]).reshape(-1), 0.0)
    o = div(co_w, rho)
    g = div(mul(mul(gO, o), 0.5), mul(mul(rho, denom), denom))
    bb = mul(b, b)
    ta = mul(g, add(mul(C03, add(mul(c0, c0), bb)), mul(C009, c0)))
    tc = mul(g, add(mul(C03, add(mul(a0, a0), bb)), mul(C009, a0)))
    tb = mul(mul(rf.scale(g, 2.0), b), add(mul(C03, add(a0, c0)), C009))
    # the terms are evaluated for every Gaussian; those of clamped ones (possibly inf) are discarded, not multiplied by 0
    keep = lambda new, old: (torch.where(active, new[0], old[0]), torch.where(active, new[1], torch.as_tensor(old[1]).to(new[1])))
    return keep(add(da, ta), da), keep(sub(db, tb), db), keep(add(dc, tc), dc)


def _build():
    src = inspect.getsource(rf.preprocess_backward)
    sig = "exact32=True, bug=()):"
    hook_after = "    dL_db = mul(scale(d2i, 2.0), lsum(sub(mul(mul(b, c), gA), mul(add(denom, mul(scale(b, 2.0), b)), gBh)), mul(mul(a, b), gC)))\n"
    assert src.count(sig) == 1 and src.count(hook_after) == 1, "raster_fp64.preprocess_backward changed: update raster_aa_fp64"
    src = src.replace(sig, "exact32=True, bug=(), aa=None):")
    src = src.replace(hook_after, hook_after + "    if aa is not None:\n        dL_da, dL_db, dL_dc = _aa_terms(locals(), aa)\n")
    ns = dict(vars(rf))
    ns["_aa_terms"] = _aa_terms
    exec(compile(src, rf.__file__, "exec"), ns)
    return ns["preprocess_backward"]


_bwd = _build()


def preprocess_backward(*, co_w, bug=(), **inp):
    """raster_fp64.preprocess_backward of a frame rendered with the filter: co_w [P] is the stored opacity (geom conic_opacity.w).
    Adds "d_opacities" (value, bound), "marg_clamp" (clamp decisions within the bound) and "active" (r > 2.5e-5) to its dict."""
    aa = dict(co_w=co_w, bug=tuple(bug))
    out = _bwd(**inp, aa=aa)
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
