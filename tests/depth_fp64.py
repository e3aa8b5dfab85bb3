"""fp64 reference of the depth backward (render_bwd_kernel<·, true>) with a running error bound, built on raster_fp64's tracked
operations and its forward walk (test helper).

The forward's D = sum w z is the red channel of the same entries with colours (z, 0, 0) and bg 0 (`indicator`), so raster_fp64's
forward of that frame gives D at every checkpoint and at the end, with its bound.  `backward` is raster_fp64.backward with the
depth as a fourth channel of the recurrence, in the kernel's expression order:
  gA      = dL/dm / (1 - T_final)                 (0 where nothing was blended)
  bg_dot  = bg . dL/dout + m gA                   (m: the kernel's plane 0, an fp32 input, error 0)
  zacc    = last_alpha lz + (1 - last_alpha) zacc (restarted as (D_final - D_ckpt) / T_ckpt)
  dL/da   = [sum_c (c - acc_c) dpix_c + (z - zacc) gA] T - T_final / (1 - a) bg_dot
  dL/dz   = a T gA
and returns d_mean2D, d_conic, d_opacity and d_z as (value, bound).  `bug` names corruptions for the self-checks: no_m_term (the
m T_final / (1 - a) term dropped), no_inv_A (g used for g / A), restart_zero (a restarted segment starts from zacc = 0).
"""
import torch

import raster_fp64 as rf
from raster_fp64 import SEG, add, cdiv, div, gam, mul, neg, scale, sub, where


def indicator(fr, z):
    """A copy of Frame `fr` whose entries have colours (z, 0, 0) and bg 0: its forward's channel 0 is D."""
    f = rf.Frame.__new__(rf.Frame)
    f.__dict__.update(fr.__dict__)
    f.colors = torch.zeros(fr.P, 3, dtype=torch.float64, device=fr.dev)
    f.colors[:, 0] = torch.as_tensor(z).to(device=fr.dev, dtype=torch.float64).reshape(-1)
    f.bg = torch.zeros(3, dtype=torch.float64, device=fr.dev)
    return f


def tile_pixels(fr, img):
    """[H,W] -> [tiles, 256] in the walk's tile order (0 outside the image)."""
    H, W = fr.H, fr.W
    pid = torch.where(fr.inside, fr.py * W + fr.px, 0)
    return torch.where(fr.inside, torch.as_tensor(img).to(device=fr.dev, dtype=torch.float64).reshape(H * W)[pid], 0.0)


def backward(fr, fw, fwz, z, dL_dout, dL_dm, m, bug=()):
    """The depth backward of frame `fr` from its forward `fw` and the indicator forward `fwz`; z [P] the entries' view depths,
    dL_dout [3,H,W], dL_dm and m [H,W]."""
    dev, P, nt = fr.dev, fr.P, fr.tiles.numel()
    H, W = fr.H, fr.W
    z = torch.as_tensor(z).to(device=dev, dtype=torch.float64).reshape(-1)
    d = torch.as_tensor(dL_dout).to(device=dev, dtype=torch.float64).reshape(3, H, W)
    dpix = [tile_pixels(fr, d[c]) for c in range(3)]
    gm, mm = tile_pixels(fr, dL_dm), tile_pixels(fr, m)
    bg = fr.bg
    bg_dot = add(add(mul(bg[0], dpix[0]), mul(bg[1], dpix[1])), mul(bg[2], dpix[2]))
    Tf, Cf, Df = fw["tile_T"], fw["tile_C"], fwz["tile_C"][0]
    last = fw["tile_last"]
    blended = last > 0
    gA = (gm, torch.zeros_like(gm)) if "no_inv_A" in bug else div((gm, 0.0), sub(1.0, Tf))
    gA = where(blended, gA, (0.0, 0.0))
    if "no_m_term" not in bug:
        bg_dot = add(bg_dot, mul((mm, 0.0), gA))
    hx, hy = 0.5 * W, 0.5 * H
    acc_v = torch.zeros(10, P, dtype=torch.float64, device=dev)
    acc_e = torch.zeros_like(acc_v)
    acc_a = torch.zeros_like(acc_v)
    active_n = torch.zeros(P, dtype=torch.int64, device=dev)
    excluded = torch.zeros(P, dtype=torch.bool, device=dev)
    tmarg = fw["tile_marg"] & fr.inside
    nseg = cdiv(int(fr.len.max()), SEG) if nt else 0
    for s in range(nseg):
        lo = s * SEG
        mt = fr.prefix(lo)
        ls = last[:mt]
        rs = ls > lo + SEG
        T = (Tf[0][:mt].clone(), Tf[1][:mt].clone())
        zero = (torch.zeros_like(T[0]), torch.zeros_like(T[0]))
        acc = [(zero[0].clone(), zero[1].clone()) for _ in range(4)]
        if rs.any():
            m1 = fr.prefix(lo + SEG)
            ck, ckz = fw["ckpts"][s + 1], fwz["ckpts"][s + 1]
            pad = lambda t, fill: torch.cat([t, torch.full((mt - m1, 256), fill, dtype=t.dtype, device=dev)])
            Tck = (pad(ck[0], 1.0), pad(ck[1], 0.0))
            inv = div(1.0, Tck)
            T = where(rs, Tck, T)
            for c in range(3):
                a = mul(sub((Cf[c][0][:mt], Cf[c][1][:mt]), (pad(ck[2][c][0], 0.0), pad(ck[2][c][1], 0.0))), inv)
                acc[c] = where(rs, a, acc[c])
            if "restart_zero" not in bug:
                a = mul(sub((Df[0][:mt], Df[1][:mt]), (pad(ckz[2][0][0], 0.0), pad(ckz[2][0][1], 0.0))), inv)
                acc[3] = where(rs, a, acc[3])
        la = (zero[0].clone(), zero[1].clone())
        lc = [torch.zeros_like(T[0]) for _ in range(4)]
        T_final = (Tf[0][:mt], Tf[1][:mt])
        for pos in range(min(lo + SEG, int(fr.len[0])) - 1, lo - 1, -1):
            mp = fr.prefix(pos)
            e = fr.entry(mp, pos)
            g = e["g"]
            touched = (e["ok"] | e["marg"]) & tmarg[:mp]
            excluded[g[touched.any(1)]] = True
            act = e["ok"] & (pos < ls[:mp])
            if not act.any():
                continue
            sl = lambda t: (t[0][:mp], t[1][:mp])
            alpha, G, dx, dy, co = e["alpha"], e["G"], e["dx"], e["dy"], e["co"]
            one_m = sub(1.0, alpha)
            Tn = div(sl(T), one_m)
            dcc = mul(alpha, Tn)
            col = torch.cat([fr.colors[g], z[g][:, None]], 1)
            new_acc = [add(mul(sl(la), lc[c][:mp]), mul(sub(1.0, sl(la)), sl(acc[c]))) for c in range(4)]
            dL_da = None
            for c in range(3):
                t = mul(sub(col[:, c:c + 1], new_acc[c]), dpix[c][:mp])
                dL_da = t if dL_da is None else add(dL_da, t)
            gAs = sl(gA)
            dL_da = add(dL_da, mul(sub(col[:, 3:4], new_acc[3]), gAs))
            v = [mul(dcc, dpix[c][:mp]) for c in range(3)]
            dL_da = mul(dL_da, Tn)
            dL_da = add(dL_da, mul(neg(div(sl(T_final), one_m)), sl(bg_dot)))
            dL_dG = mul(co[:, 3:4], dL_da)
            gdx, gdy = mul(G, dx), mul(G, dy)
            dGx = sub(neg(mul(gdx, co[:, 0:1])), mul(gdy, co[:, 1:2]))
            dGy = sub(neg(mul(gdy, co[:, 2:3])), mul(gdx, co[:, 1:2]))
            v.append(mul(mul(dL_dG, dGx), hx))
            v.append(mul(mul(dL_dG, dGy), hy))
            v.append(mul(mul(scale(gdx, -0.5), dx), dL_dG))
            v.append(mul(mul(scale(gdx, -0.5), dy), dL_dG))
            v.append(mul(mul(scale(gdy, -0.5), dy), dL_dG))
            v.append(mul(G, dL_da))
            v.append(mul(dcc, gAs))
            for q in range(10):
                val, err = where(act, v[q], (0.0, 0.0))
                acc_v[q].index_add_(0, g, val.sum(1))
                acc_e[q].index_add_(0, g, err.sum(1))
                acc_a[q].index_add_(0, g, val.abs().sum(1))
            active_n.index_add_(0, g, act.sum(1))
            for c in range(4):
                acc[c][0][:mp], acc[c][1][:mp] = where(act, new_acc[c], sl(acc[c]))
                lc[c][:mp] = torch.where(act, col[:, c:c + 1].expand_as(lc[c][:mp]), lc[c][:mp])
            T[0][:mp], T[1][:mp] = where(act, Tn, sl(T))
            la[0][:mp], la[1][:mp] = where(act, alpha, sl(la))
    bound = acc_e + gam(12 + fr.ntiles)[None].double() * (acc_a + acc_e)
    out = {}
    for name, rows in (("d_colors", [0, 1, 2]), ("d_mean2D", [3, 4]), ("d_conic", [5, 6, 7]), ("d_opacity", [8]), ("d_z", [9])):
        out[name] = (acc_v[rows].T.contiguous(), bound[rows].T.contiguous())
    out["excluded"] = excluded
    out["active"] = active_n
    return out
