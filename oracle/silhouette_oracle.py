"""fp64 restatement of the soft silhouette (csrc/silhouette.cu, DESIGN.md §2) in torch: every face against every pixel, no binning,
and the vertex gradient of the loss by autograd.  Runs on whatever device its inputs are on.

    S(p) = 1 - prod_f (1 - D_f(p)),  D_f = sigmoid(+-d_f^2 / sigma) (+ inside the projected triangle, - outside), D_f = 0 outside
    beyond d_f^2 > sigma ln(1/eps - 1), eps = 1e-4; d_f the distance from pixel centre (c, r) to the triangle.

Faces with a corner at view depth <= 0.01 or outside the 2^20-pixel guard band, and faces of zero projected area, are left out.
"""
from __future__ import annotations

import math

import torch

EPS = 1e-4
ZNEAR = 0.01
GUARD = 2.0 ** 20
LN_INV_EPS = math.log(1.0 / EPS - 1.0)


def project(verts, cams, H, W):
    """verts [B,V,3], cams [B,40] (transposed view 0..15, transposed full projection 16..31) -> (pix [B,V,2], view depth [B,V])."""
    verts, cams = verts.double(), cams.double()
    B = verts.shape[0]
    Xh = torch.cat([verts, torch.ones_like(verts[..., :1])], -1)
    view = cams[:, :16].reshape(B, 4, 4)
    proj = cams[:, 16:32].reshape(B, 4, 4)
    z = (Xh @ view)[..., 2]
    h = Xh @ proj
    p_w = 1.0 / (h[..., 3] + 1e-7)
    px = ((h[..., 0] * p_w + 1.0) * W - 1.0) * 0.5
    py = ((h[..., 1] * p_w + 1.0) * H - 1.0) * 0.5
    return torch.stack([px, py], -1), z


def face_corners(verts, faces, cams, H, W):
    """Projected corners [B,F,3,2] and which faces take part [B,F]."""
    pix, z = project(verts, cams, H, W)
    fi = torch.as_tensor(faces, dtype=torch.long, device=pix.device)
    c = pix[:, fi]                                                   # [B,F,3,2]
    ok = ((z[:, fi] > ZNEAR) & (c.abs() <= GUARD).all(-1)).all(-1)
    e1, e2 = c[:, :, 1] - c[:, :, 0], c[:, :, 2] - c[:, :, 0]
    area = e1[..., 0] * e2[..., 1] - e1[..., 1] * e2[..., 0]
    return c, ok & (area != 0) & torch.isfinite(area)


def signed_d2(c, p):
    """c [F,3,2] corners, p [P,2] points -> (d^2 [P,F] to the triangle, inside [P,F])."""
    a = c[None]                                                      # [1,F,3,2]
    b = torch.roll(c, -1, dims=1)[None]
    e = b - a
    w = p[:, None, None, :] - a                                      # [P,F,3,2]
    t = ((w * e).sum(-1) / (e * e).sum(-1)).clamp(0.0, 1.0)
    d = w - t[..., None] * e
    d2 = (d * d).sum(-1).min(-1).values
    cr = e[..., 0] * w[..., 1] - e[..., 1] * w[..., 0]
    inside = (cr >= 0).all(-1) | (cr <= 0).all(-1)
    return d2, inside


def _safe(c, ok):
    """Faces that take no part moved to a far-away unit triangle, so that no 0/0 of a degenerate edge reaches the gradient."""
    far = torch.tensor([[-1e7, -1e7], [-1e7 + 1, -1e7], [-1e7, -1e7 + 1]], dtype=c.dtype, device=c.device)
    return torch.where(ok[:, None, None], c, far)


def log_one_minus(c, ok, p, sigma):
    """L(p) = sum_f log(1 - D_f(p)) = -sum_f softplus(x_f) over the faces c [F,3,2] with ok [F], at points p [P,2] -> [P]."""
    d2, inside = signed_d2(_safe(c, ok), p)
    x = torch.where(inside, d2, -d2) / sigma
    live = ok[None] & (inside | (d2 <= sigma * LN_INV_EPS))
    sp = torch.logaddexp(torch.zeros_like(x), x)
    return -torch.where(live, sp, torch.zeros_like(sp)).sum(-1)


def marginal(c, ok, p, sigma, tol_d2):
    """[P] bool: some face's outside distance^2 lies within tol_d2 of the truncation radius^2."""
    d2, inside = signed_d2(_safe(c, ok), p)
    return (ok[None] & ~inside & ((d2 - sigma * LN_INV_EPS).abs() <= tol_d2)).any(-1)


def _pixels(H, W, rows, device):
    rows = torch.arange(H, device=device) if rows is None else torch.as_tensor(rows, device=device)
    r, cc = torch.meshgrid(rows.double(), torch.arange(W, device=device, dtype=torch.float64), indexing="ij")
    return torch.stack([cc.reshape(-1), r.reshape(-1)], -1), len(rows)


def _chunks(F, P, pairs=1 << 22):
    step = max(1, pairs // max(P, 1))
    return [(s, min(F, s + step)) for s in range(0, F, step)]


def log_one_minus_frame(c, ok, p, sigma):
    L = torch.zeros(p.shape[0], dtype=torch.float64, device=p.device)
    for s, e in _chunks(c.shape[0], p.shape[0]):
        L = L + log_one_minus(c[s:e], ok[s:e], p, sigma)
    return L


def silhouette(verts, faces, cams, H, W, sigma, rows=None, tol_d2=None):
    """S [B,len(rows),W] (all rows by default) and, with tol_d2, the marginal pixels [B,len(rows),W]."""
    with torch.no_grad():
        c, ok = face_corners(verts, faces, cams, H, W)
        p, nr = _pixels(H, W, rows, c.device)
        S, marg = [], []
        for b in range(c.shape[0]):
            S.append(-torch.expm1(log_one_minus_frame(c[b], ok[b], p, sigma)).reshape(nr, W))
            if tol_d2 is not None:
                m = torch.zeros(p.shape[0], dtype=torch.bool, device=p.device)
                for s, e in _chunks(c.shape[1], p.shape[0]):
                    m |= marginal(c[b, s:e], ok[b, s:e], p, sigma, tol_d2)
                marg.append(m.reshape(nr, W))
        S = torch.stack(S)
        return (S, torch.stack(marg)) if tol_d2 is not None else S


def loss_and_grad(verts, faces, cams, masks, H, W, sigma, w=None):
    """(loss [B] = mean_p (S - M)^2, d_verts [B,V,3] of sum_b w_b loss_b) in fp64 by autograd, M = masks >= 128.  The face sum is
    taken in chunks: L is formed without a graph, dloss/dL by autograd, then each chunk's L is rebuilt with a graph and back-propagated
    with that gradient, which is the chain rule autograd would apply to the whole sum."""
    X = verts.detach().double().clone().requires_grad_(True)
    B = X.shape[0]
    w = torch.ones(B, dtype=torch.float64, device=X.device) if w is None else torch.as_tensor(w, dtype=torch.float64, device=X.device)
    M = (torch.as_tensor(masks, device=X.device) >= 128).double().reshape(B, -1)
    p, _ = _pixels(H, W, None, X.device)
    losses = []
    for b in range(B):
        with torch.no_grad():
            c, ok = face_corners(X[b:b + 1], faces, cams[b:b + 1], H, W)
            L = log_one_minus_frame(c[0], ok[0], p, sigma)
        Lg = L.clone().requires_grad_(True)
        loss = ((-torch.expm1(Lg) - M[b]) ** 2).mean()
        gL, = torch.autograd.grad(loss * w[b], Lg)
        losses.append(loss.detach())
        for s, e in _chunks(len(faces), p.shape[0]):
            c, ok = face_corners(X[b:b + 1], faces[s:e], cams[b:b + 1], H, W)
            torch.autograd.backward(log_one_minus(c[0], ok[0], p, sigma), gL)
    return torch.stack(losses), X.grad if X.grad is not None else torch.zeros_like(X)
