"""fp64 reference of the rasterizer's compositing (K6) and its backward (K7), with a running error bound (test helper);
the fused preprocess backward (K8/K9) and K1's SH colour are restated with the same bound in the section at the end.

It starts from what the kernels themselves stage: one frame's `xy`, `conic_opacity`, per-tile sorted Gaussian list and tile
ranges, plus the colours, `bg` and dL/dout.  It returns, per pixel, the image, final_T and n_contrib, and per Gaussian d_colors,
d_mean2D (dL/d ndc, the convention K7 writes), d_conic (the kernel's half off-diagonal convention: dL/dA, dL/dB / 2, dL/dC) and
d_opacity.  The formulas are upstream's (SURVEY.md §8 a-8 / a-9), including deviation (1) of oracle/raster_twin.py: the
gradient passes the min(0.99, .) cap.  Nothing is culled: every entry of a tile's list is evaluated at all 256 pixels of the
tile, so a sub-tile cull that drops a pair the per-pixel tests would take shows up as a mismatch.

Error bound.  Every value is carried as (v, e): v is the fp64 value of the kernel's expression tree as written in
csrc/raster.cu, e bounds |fp32 result of that tree - v|.  Each operation adds u |result| to the propagated error, with
u = 2^-24 + 2^-53 (the fp32 rounding plus the fp64 one of v), and 2^-126 absolute for underflow.  Counting a multiply and an
add separately also covers a contracted FMA.  Products and quotients propagate the operand errors exactly to first order plus
their product terms, so the bound is rigorous, not first order.  Division is IEEE round-to-nearest (the library is built
without --use_fast_math).  comp_exp (raster.cu: ex2.approx.ftz.f32 of x * 1.4426950f) adds, relative to exp(x):
  * ex2.approx.f32: at most 2 ulp relative error across the full range (PTX ISA, `ex2`), i.e. <= 2^-22 relative;
  * the rounding of y = x * log2e_f: |dy| <= u |y|, a relative error of ln 2 u |y| = u |x| (ln 2 log2e = 1) in 2^y;
  * log2e_f = 1.4426950f itself, 1.93e-8 below log2 e: a relative error of 1.34e-8 |x|;
  * the error e_x of x: a relative error of e_x.
For x in [-5.6, 0] (below that alpha < 1/255 whatever the opacity) this is <= 2^-22 + 5.6 (u + 1.34e-8) = 6.5e-7 before e_x:
the "<= ~6e-7" the comment above comp_exp states, plus the 7e-8 of the rounded constant it leaves out.
Sums whose order is not fixed (K7's warp_reduce8 / warp_sum tree: 5 levels, the shared-memory atomics of 8 warps: 7, the global
atomics of the CTAs of the tiles the Gaussian is listed in: ntiles - 1) are bounded by gamma(12 + ntiles) times the sum of the
absolute values of the terms (any summation tree of depth d errs by at most gamma(d) sum |x_i|).

K7 replays each 256-entry segment from the state the kernel starts it from: a pixel whose last contributor lies past segment s
starts from forward checkpoint s + 1 with acc = (C_final - C_ckpt) / T_ckpt, so its bound carries that cancellation.

Decisions (power > 0, alpha < 1/255, test_T < 1e-4) are classified as marginal when the threshold lies within [v - e, v + e]:
the kernel may go either way there.  A pixel with a marginal decision at a point where it still composites is marginal; a
Gaussian not clearly rejected at some marginal pixel is marginal.  Only clear pixels / Gaussians are held to the bound.

Written in torch: the same code runs on the CPU (small scenes) and in fp64 on the GPU (production frames), batched over the
tiles of a frame sorted by list length, so that step k touches only the tiles whose list is longer than k.
"""
import math

import torch

U = 2.0 ** -24 + 2.0 ** -53
ETA = 2.0 ** -126
EX2_REL = 2.0 ** -22
LOG2E_F = 1.4426950216293335                 # 1.4426950408889634f
C_LN2_ERR = abs(LOG2E_F * math.log(2.0) - 1.0)
A_THR = 0.003921568859368563                 # 1.0f / 255.0f
T_THR = 9.999999747378752e-05                # 0.0001f
CAP = 0.9900000095367432                     # 0.99f
SEG = 256


def gam(n):
    return n * U / (1 - n * U)


# ---------------------------------------------------------------------------------------------- tracked fp32 operations
def _e(a):
    return a[1] if isinstance(a, tuple) else 0.0


def _v(a):
    return a[0] if isinstance(a, tuple) else a


def _round(v, d):
    return v, d + U * (v.abs() + d) + ETA


def add(a, b):
    return _round(_v(a) + _v(b), _e(a) + _e(b))


def sub(a, b):
    return _round(_v(a) - _v(b), _e(a) + _e(b))


def mul(a, b):
    av, bv, ae, be = _v(a), _v(b), _e(a), _e(b)
    v = av * bv
    if not torch.is_tensor(v):
        v = torch.tensor(v, dtype=torch.float64)
    return _round(v, abs(av) * be + abs(bv) * ae + ae * be)


def div(a, b):
    av, bv, ae, be = _v(a), _v(b), _e(a), _e(b)
    den = abs(bv) * (abs(bv) - be)
    d = torch.where(den > 0, (ae * abs(bv) + abs(av) * be) / den.clamp_min(1e-300), torch.full_like(den, math.inf))
    return _round(av / bv, d)


def neg(a):
    return -_v(a), _e(a)


def scale(a, s):
    """Multiplication by a power of two: exact."""
    return _v(a) * s, _e(a) * abs(s)


def comp_exp(x):
    xv, xe = x
    rho = xe * LOG2E_F * math.log(2.0) + (xv.abs() + xe) * (C_LN2_ERR + U * LOG2E_F * math.log(2.0))
    g = torch.exp(xv)
    return g, g * ((1 + EX2_REL) * torch.exp(rho) - 1) + ETA


def fmin(a, c):
    av, ae = a
    return torch.clamp(av, max=c), torch.where(av - ae > c, torch.zeros_like(ae), ae)


def where(m, a, b):
    return torch.where(m, _v(a), _v(b)), torch.where(m, _e(a), _e(b))


def marg_gt(a, t):
    return (a[0] - a[1] > t) != (a[0] + a[1] > t)


def marg_lt(a, t):
    return (a[0] - a[1] < t) != (a[0] + a[1] < t)


# -------------------------------------------------------------------------------------------------------------- frames
def cdiv(a, b):
    return -(-a // b)


class Frame:
    """One frame's staged inputs: xy [P,2], conic_o [P,4], colors [P,3], bg [3], ranges [T,2] (into point_list), point_list."""

    def __init__(self, xy, conic_o, colors, bg, ranges, point_list, H, W, device="cpu", thresholds=(CAP, A_THR, T_THR)):
        f = lambda t: torch.as_tensor(t).to(device=device, dtype=torch.float64)
        self.xy, self.co, self.colors, self.bg = f(xy).reshape(-1, 2), f(conic_o).reshape(-1, 4), f(colors).reshape(-1, 3), f(bg).reshape(3)
        self.P = self.xy.shape[0]
        self.ranges = torch.as_tensor(ranges).to(device=device, dtype=torch.int64).reshape(-1, 2)
        self.plist = torch.as_tensor(point_list).to(device=device, dtype=torch.int64).reshape(-1)
        self.H, self.W, self.dev = int(H), int(W), device
        self.cap, self.a_thr, self.t_thr = thresholds      # the kernels' fp32 constants; an fp64 twin uses 0.99, 1/255, 1e-4
        self.gx, self.gy = cdiv(self.W, 16), cdiv(self.H, 16)
        lens = self.ranges[:, 1] - self.ranges[:, 0]
        order = torch.argsort(lens, descending=True, stable=True)
        order = order[lens[order] > 0]
        self.tiles, self.len, self.start = order, lens[order], self.ranges[order, 0]
        k = torch.arange(256, device=device)
        self.px = (self.tiles % self.gx)[:, None] * 16 + (k % 16)[None]
        self.py = (self.tiles // self.gx)[:, None] * 16 + (k // 16)[None]
        self.inside = (self.px < self.W) & (self.py < self.H)
        # number of tiles (= K7 segment CTAs) whose list holds the Gaussian: the ranges cover the whole list
        self.ntiles = torch.bincount(self.plist, minlength=self.P)

    def prefix(self, k):
        """Number of (length-sorted) tiles whose list is longer than k."""
        return int((self.len > k).sum())

    def entry(self, m, k):
        """Entry k of the first m tiles' lists at their 256 pixels: Gaussian ids [m], dx, dy, power, G, alpha and the decisions."""
        g = self.plist[self.start[:m] + k]
        xy, co = self.xy[g], self.co[g]
        pxf, pyf = self.px[:m].double(), self.py[:m].double()
        dx = sub((xy[:, 0:1], 0.0), (pxf, 0.0))
        dy = sub((xy[:, 1:2], 0.0), (pyf, 0.0))
        cx, cy, cz, o = co[:, 0:1], co[:, 1:2], co[:, 2:3], co[:, 3:4]
        t1 = mul(mul(cx, dx), dx)
        t2 = mul(mul(cz, dy), dy)
        s = scale(add(t1, t2), -0.5)
        power = sub(s, mul(mul(cy, dx), dy))
        G = comp_exp(power)
        alpha = fmin(mul(o, G), self.cap)
        pos = power[0] > 0
        low = alpha[0] < self.a_thr
        ok = ~pos & ~low
        marg = marg_gt(power, 0.0) | (~pos & marg_lt(alpha, self.a_thr))
        return dict(g=g, dx=dx, dy=dy, power=power, G=G, alpha=alpha, ok=ok, marg=marg, co=co)


def forward(fr: Frame, stop_late=False, drop=None):
    """K6 along the kernel's path.  stop_late / drop are corruptions for the self-checks: the T stop applied to the entry after
    the one that triggers it; drop = (sorted tile, list position, pixel mask) never composited there."""
    nt, dev = fr.tiles.numel(), fr.dev
    z = torch.zeros(nt, 256, dtype=torch.float64, device=dev)
    T = (torch.ones_like(z), z.clone())
    C = [(z.clone(), z.clone()) for _ in range(3)]
    last = torch.zeros(nt, 256, dtype=torch.int64, device=dev)
    done = ~fr.inside.clone()
    marg = torch.zeros(nt, 256, dtype=torch.bool, device=dev)
    ckpts = []
    L = int(fr.len.max()) if nt else 0
    for k in range(L):
        m = fr.prefix(k)
        if k % SEG == 0:
            ckpts.append((T[0][:m].clone(), T[1][:m].clone(), [(c[0][:m].clone(), c[1][:m].clone()) for c in C]))
        e = fr.entry(m, k)
        ok = e["ok"]
        if drop is not None and drop[1] == k and drop[0] < m:
            ok = ok.clone()
            ok[drop[0]] &= ~drop[2]
        live = ~done[:m]
        alpha = e["alpha"]
        Tm = (T[0][:m], T[1][:m])
        test_T = mul(Tm, sub(1.0, alpha))
        stop = live & ok & (test_T[0] < fr.t_thr)
        take = live & ok & (~stop if not stop_late else torch.ones_like(stop))
        w = mul(alpha, Tm)
        col = fr.colors[e["g"]]
        for c in range(3):
            nc = add((C[c][0][:m], C[c][1][:m]), mul(col[:, c:c + 1], w))
            C[c][0][:m], C[c][1][:m] = where(take, nc, (C[c][0][:m], C[c][1][:m]))
        T[0][:m], T[1][:m] = where(take, test_T, Tm)
        last[:m] = torch.where(take, k + 1, last[:m])
        done[:m] |= stop
        marg[:m] |= live & (e["marg"] | (ok & marg_lt(test_T, fr.t_thr)))
    H, W = fr.H, fr.W
    img = fr.bg[:, None].expand(3, H * W).clone()
    img_e = torch.zeros(3, H * W, dtype=torch.float64, device=dev)
    fT = torch.ones(H * W, dtype=torch.float64, device=dev)
    fT_e = torch.zeros(H * W, dtype=torch.float64, device=dev)
    nc = torch.zeros(H * W, dtype=torch.int64, device=dev)
    mg = torch.zeros(H * W, dtype=torch.bool, device=dev)
    ins = fr.inside
    pid = (fr.py * W + fr.px)[ins]
    for c in range(3):
        o = add(C[c], mul(T, fr.bg[c]))
        img[c, pid], img_e[c, pid] = o[0][ins], o[1][ins]
    fT[pid], fT_e[pid], nc[pid], mg[pid] = T[0][ins], T[1][ins], last[ins], marg[ins]
    maxc = last.max(1).values if nt else last.new_zeros(0)
    return dict(image=(img.reshape(3, H, W), img_e.reshape(3, H, W)), final_T=(fT.reshape(H, W), fT_e.reshape(H, W)),
                n_contrib=nc.reshape(H, W), marginal=mg.reshape(H, W), tile_T=T, tile_C=C, tile_last=last, tile_marg=marg,
                tile_maxc=maxc, ckpts=ckpts)


def backward(fr: Frame, fw, dL_dout, restart=True, use_bg_dot=True, swap_hw=False, skip=None):
    """K7 along the kernel's path, from the forward `fw` of the same frame.  restart=False, use_bg_dot=False, swap_hw=True and
    skip = (sorted tile, segment) are corruptions for the self-checks."""
    dev, P, nt = fr.dev, fr.P, fr.tiles.numel()
    H, W = fr.H, fr.W
    d = torch.as_tensor(dL_dout).to(device=dev, dtype=torch.float64).reshape(3, H * W)
    ins = fr.inside
    pid = torch.where(ins, fr.py * W + fr.px, 0)
    dpix = [torch.where(ins, d[c][pid], 0.0) for c in range(3)]
    bg = fr.bg
    bg_dot = add(add(mul(bg[0], dpix[0]), mul(bg[1], dpix[1])), mul(bg[2], dpix[2]))
    if not use_bg_dot:
        bg_dot = (torch.zeros_like(dpix[0]), torch.zeros_like(dpix[0]))
    hx, hy = (0.5 * H, 0.5 * W) if swap_hw else (0.5 * W, 0.5 * H)
    acc_v = torch.zeros(9, P, dtype=torch.float64, device=dev)
    acc_e = torch.zeros_like(acc_v)
    acc_a = torch.zeros_like(acc_v)
    active_n = torch.zeros(P, dtype=torch.int64, device=dev)
    excluded = torch.zeros(P, dtype=torch.bool, device=dev)
    Tf = fw["tile_T"]
    Cf = fw["tile_C"]
    last = fw["tile_last"]
    tmarg = fw["tile_marg"] & ins
    nseg = cdiv(int(fr.len.max()), SEG) if nt else 0
    for s in range(nseg):
        lo = s * SEG
        m = fr.prefix(lo)
        ls = last[:m]
        rs = ls > lo + SEG if restart else torch.zeros_like(ls, dtype=torch.bool)
        T = (Tf[0][:m].clone(), Tf[1][:m].clone())
        acc = [(torch.zeros_like(T[0]), torch.zeros_like(T[0])) for _ in range(3)]
        if rs.any():
            m1 = fr.prefix(lo + SEG)                # tiles that have checkpoint s + 1; a restart needs last > lo + 256
            ck = fw["ckpts"][s + 1]
            pad = lambda t, fill: torch.cat([t, torch.full((m - m1, 256), fill, dtype=t.dtype, device=dev)])
            Tck = (pad(ck[0], 1.0), pad(ck[1], 0.0))
            inv = div(1.0, Tck)
            T = where(rs, Tck, T)
            for c in range(3):
                a = mul(sub((Cf[c][0][:m], Cf[c][1][:m]), (pad(ck[2][c][0], 0.0), pad(ck[2][c][1], 0.0))), inv)
                acc[c] = where(rs, a, acc[c])
        la = (torch.zeros_like(T[0]), torch.zeros_like(T[0]))
        lc = [torch.zeros_like(T[0]) for _ in range(3)]
        T_final = (Tf[0][:m], Tf[1][:m])
        for pos in range(min(lo + SEG, int(fr.len[0])) - 1, lo - 1, -1):
            mp = fr.prefix(pos)
            e = fr.entry(mp, pos)
            g = e["g"]
            touched = (e["ok"] | e["marg"]) & tmarg[:mp]
            excluded[g[touched.any(1)]] = True
            act = e["ok"] & (pos < ls[:mp])
            if skip is not None and skip[1] == s and skip[0] < mp:
                act = act.clone()
                act[skip[0]] = False
            if not act.any():
                continue
            sl = lambda t: (t[0][:mp], t[1][:mp])
            alpha, G, dx, dy, co = e["alpha"], e["G"], e["dx"], e["dy"], e["co"]
            one_m = sub(1.0, alpha)
            Tn = div(sl(T), one_m)
            dcc = mul(alpha, Tn)
            col = fr.colors[g]
            new_acc = [add(mul(sl(la), lc[c][:mp]), mul(sub(1.0, sl(la)), sl(acc[c]))) for c in range(3)]
            dL_da = None
            for c in range(3):
                t = mul(sub(col[:, c:c + 1], new_acc[c]), dpix[c][:mp])
                dL_da = t if dL_da is None else add(dL_da, t)
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
            for q in range(9):
                val, err = where(act, v[q], (0.0, 0.0))
                acc_v[q].index_add_(0, g, val.sum(1))
                acc_e[q].index_add_(0, g, err.sum(1))
                acc_a[q].index_add_(0, g, val.abs().sum(1))
            active_n.index_add_(0, g, act.sum(1))
            # state updates of the active pixels
            for c in range(3):
                acc[c][0][:mp], acc[c][1][:mp] = where(act, new_acc[c], sl(acc[c]))
                lc[c][:mp] = torch.where(act, col[:, c:c + 1].expand_as(lc[c][:mp]), lc[c][:mp])
            T[0][:mp], T[1][:mp] = where(act, Tn, sl(T))
            la[0][:mp], la[1][:mp] = where(act, alpha, sl(la))
    bound = acc_e + gam(12 + fr.ntiles)[None].double() * (acc_a + acc_e)
    out = {}
    for name, rows in (("d_colors", [0, 1, 2]), ("d_mean2D", [3, 4]), ("d_conic", [5, 6, 7]), ("d_opacity", [8])):
        out[name] = (acc_v[rows].T.contiguous(), bound[rows].T.contiguous())
    out["excluded"] = excluded
    out["active"] = active_n
    return out


# ============================================================================================ K8/K9: preprocess_bwd_kernel
# fp64 restatement of the fused K8/K9 (preprocess_bwd_kernel) with the same running bound, from one launch's own inputs.
#
# Inputs (`preprocess_backward`): one frame's means3D, scales, rotations, scale_modifier, view / proj matrices and tanfov, the radii
# and the STAGED cov3d K1 left in the geom buffer, the d_mean2D / d_conic_op K7 left in the backward scratch, and with SH the
# coefficients, campos, K1's clamp bits and dL/drgb (K7's d_colors).  Every input is an fp32 value, so it enters with error 0.
#
# Exact part.  K1 and K8 both evaluate tvx, tvy, tvz, hx, hy, hw with xf_row, which uses __fmul_rn / __fmaf_rn / __fadd_rn; quat_to_rot
# uses __fmul_rn / __fadd_rn / __fsub_rn; txtz = tvx / tvz and limx = 1.3f * tanfovx are single correctly rounded operations (the
# library is built without fast-math).  They are reproduced bit for bit: an fp32 +, -, *, / of fp32 operands evaluated in fp64 and
# rounded to fp32 is correctly rounded (53 >= 2 * 24 + 2, so the double rounding is innocuous), and fma32 rounds the exact a * b + c
# once (TwoSum, with the one case where the fp64 sum lands on an fp32 midpoint resolved by the sign of the residual).  So the
# guard-band gates x_grad_mul / y_grad_mul and the clamped tx / ty are the kernel's own, with no marginal band, and tvz must equal
# K1's staged depth bit for bit.
#
# Bounded part.  Everything else is ordinary fp32 that nvcc may contract: each operation is counted as one rounding (u |result|,
# the model of the K6 / K7 reference above), a contracted multiply-add as two, which bounds the FMA's single rounding.  The kernel's
# left-to-right order is restated exactly, e.g. -fx * tx * tz2 = ((-fx) tx) tz2; products of compile-time constants (6.f * kShC3_0)
# are folded in fp32 and exact here; 1.f / sqrtf(.) is a correctly rounded sqrt (sqrt_ below) and a correctly rounded division.
# The one floating decision left is denom2inv != 0 (denom^2 + 1e-7f overflowing fp32): `marg_overflow` flags a Gaussian whose
# bound reaches within a factor 2 of that overflow, and callers assert there is none.
#
# Upstream's three deviations from true autograd (oracle/raster_twin.py) are encoded as the kernel has them: a clamped tx / ty is
# constant w.r.t. tz (dL_dtz uses the clamped value, dL_dtx / dL_dty are gated), the conic backward uses 1 / (det^2 + 1e-7), and
# the off-diagonal dL/dB comes in the half convention (d_conic_op.y).  The quaternion is not normalised (as upstream).
#
# `bug` names corruptions for the self-checks: gate (dL_dtx / dL_dty ungated), tz_unclamped (dL_dtz from txtz tz), scale_mod
# (d_scales without the outer scale_modifier), full_offdiag (dL/dB taken as the full off-diagonal), no_proj_w (the proj[4k+3] mul
# terms dropped), norm_quat (d_rotations of the normalised quaternion), no_sh_dir (the SH direction term missing from d_means3D),
# no_clamp_mask (d_sh ignoring the clamp bits), sh_extra (coefficient (D+1)^2 not zeroed).
F32_MAX = 3.4028234663852886e38


def f32(x):
    return x.float().double()


def fma32(a, b, c):
    """fp32 fmaf(a, b, c) of fp32 values held in float64 tensors, rounded once."""
    p = a * b                                   # exact: 24 + 24 bits
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)             # TwoSum: p + c = s + err exactly
    r = f32(s)
    inf = torch.full_like(s, math.inf).float()
    o = torch.nextafter(r.float(), torch.where(s > r, inf, -inf)).double()
    tie = (r != s) & ((r + o) * 0.5 == s)
    hi, lo = torch.maximum(r, o), torch.minimum(r, o)
    return torch.where(tie & (err != 0), torch.where(err > 0, hi, lo), r)


def xf_row32(M, r, x, y, z):
    t = f32(M[r] * x)
    t = fma32(M[4 + r], y, t)
    t = fma32(M[8 + r], z, t)
    return f32(t + M[12 + r])


def xf_row64(M, r, x, y, z):
    return ((M[r] * x + M[4 + r] * y) + M[8 + r] * z) + M[12 + r]


def quat_to_rot32(q, rn):
    qr, qx, qy, qz = q.unbind(-1)
    m = lambda a, b: rn(a * b)
    R00 = rn(1.0 - m(2.0, rn(m(qy, qy) + m(qz, qz))))
    R01 = m(2.0, rn(m(qx, qy) - m(qr, qz)))
    R02 = m(2.0, rn(m(qx, qz) + m(qr, qy)))
    R10 = m(2.0, rn(m(qx, qy) + m(qr, qz)))
    R11 = rn(1.0 - m(2.0, rn(m(qx, qx) + m(qz, qz))))
    R12 = m(2.0, rn(m(qy, qz) - m(qr, qx)))
    R20 = m(2.0, rn(m(qx, qz) - m(qr, qy)))
    R21 = m(2.0, rn(m(qy, qz) + m(qr, qx)))
    R22 = rn(1.0 - m(2.0, rn(m(qx, qx) + m(qy, qy))))
    return [[R00, R01, R02], [R10, R11, R12], [R20, R21, R22]]


def sqrt_(a):
    """Correctly rounded sqrtf: |sqrt(v') - sqrt(v)| <= e / (sqrt(v) + sqrt(v - e)) for |v' - v| <= e."""
    av, ae = a
    v = av.clamp_min(0).sqrt()
    return _round(v, ae / (v + (av - ae).clamp_min(0).sqrt()).clamp_min(1e-300))


def lsum(*terms):
    """Left-to-right sum of tracked terms (a + b + c = (a + b) + c)."""
    s = terms[0]
    for t in terms[1:]:
        s = add(s, t)
    return s


def cf32(x):
    """A float constant as the fp32 value the kernel holds."""
    import numpy as np
    return float(np.float32(x))


SH_C64 = dict(C0=0.28209479177387814, C1=0.4886025119029199, C2_0=1.0925484305920792, C2_1=-1.0925484305920792,
            C2_2=0.31539156525252005, C2_3=-1.0925484305920792, C2_4=0.5462742152960396, C3_0=-0.5900435899266435,
            C3_1=2.890611442640554, C3_2=-0.4570457994644658, C3_3=0.3731763325901154, C3_4=-0.4570457994644658,
            C3_5=1.445305721320277, C3_6=-0.5900435899266435)
SH_C32 = {k: cf32(v) for k, v in SH_C64.items()}      # the kernel's kSh* constants; the fp64 oracle uses SH_C64


def kc(a, name, C):
    """A constant product folded at compile time (in fp32 for the kernel's constants): a * kSh<name>."""
    v = a * C[name]
    return cf32(v) if C is SH_C32 else v


def sh_dir(means, campos):
    """sh_eval / sh_color_bwd: dir = (mean - campos) * (1 / sqrtf(|v|^2)); returns (x, y, z), inv."""
    v = [sub((means[:, k], 0.0), (campos[k], 0.0)) for k in range(3)]
    n2 = lsum(mul(v[0], v[0]), mul(v[1], v[1]), mul(v[2], v[2]))
    inv = div(1.0, sqrt_(n2))
    return [mul(v[k], inv) for k in range(3)], inv


def sh_basis(x, y, z, C=SH_C32):
    xx, yy, zz = mul(x, x), mul(y, y), mul(z, z)
    one = torch.ones_like(x[0])
    b = [(C["C0"] * one, torch.zeros_like(x[0]))]
    b += [mul(-C["C1"], y), mul(C["C1"], z), mul(-C["C1"], x)]
    b += [mul(mul(C["C2_0"], x), y), mul(mul(C["C2_1"], y), z), mul(C["C2_2"], sub(sub(scale(zz, 2.0), xx), yy)),
          mul(mul(C["C2_3"], x), z), mul(C["C2_4"], sub(xx, yy))]
    b += [mul(mul(C["C3_0"], y), sub(mul(3.0, xx), yy)), mul(mul(mul(C["C3_1"], x), y), z),
          mul(mul(C["C3_2"], y), sub(sub(scale(zz, 4.0), xx), yy)),
          mul(mul(C["C3_3"], z), sub(sub(scale(zz, 2.0), mul(3.0, xx)), mul(3.0, yy))),
          mul(mul(C["C3_4"], x), sub(sub(scale(zz, 4.0), xx), yy)), mul(mul(C["C3_5"], z), sub(xx, yy)),
          mul(mul(C["C3_6"], x), sub(xx, mul(3.0, yy)))]
    return b


def sh_forward(means, shs, D, campos):
    """K1's SH colour (sh_eval) of fp32 inputs: (pre-clamp value per channel as (v, e) [P,3], rgb after the clamp)."""
    dev = means.device if torch.is_tensor(means) else "cpu"
    f = lambda t: torch.as_tensor(t).to(device=dev, dtype=torch.float64)
    means, shs, campos = f(means), f(shs), f(campos).reshape(3)
    (x, y, z), _ = sh_dir(means, campos)
    b = sh_basis(x, y, z)
    pre = []
    for ch in range(3):
        r = None
        for k in range((D + 1) ** 2):
            t = mul(b[k], (shs[:, k, ch], 0.0))
            r = t if r is None else add(r, t)
        pre.append(add(r, 0.5))
    v = torch.stack([p[0] for p in pre], 1)
    e = torch.stack([p[1] for p in pre], 1)
    return (v, e), v.clamp_min(0)


R_MIN = cf32(2.5e-5)
C03, C009 = cf32(0.3), cf32(0.09)


def clamp_min(a, t):
    """fmaxf(t, a) of a tracked value: 1-Lipschitz, so the bound carries over."""
    return a[0].clamp_min(t), a[1]


def _aa_terms(m0, m1, v0, v1, b, denom, gO, dL_da, dL_db, dL_dc, aa):
    """The kernel's kAA block: returns the new dL/d(a, b, c) and records d_opacities and the clamp decisions in aa (see
    raster_aa_fp64.preprocess_backward)."""
    bug = aa.get("bug", ())
    a0 = lsum(*[mul(m0[k], v0[k]) for k in range(3)])
    c0 = lsum(*[mul(m1[k], v1[k]) for k in range(3)])
    det0 = denom if "dilated_num" in bug else sub(mul(a0, c0), mul(b, b))
    r = div(det0, denom)
    rho = sqrt_(clamp_min(r, R_MIN))
    aa["d_opacities"] = gO if "no_rho_dopac" in bug else mul(gO, rho)
    active = r[0] > R_MIN
    aa["marg_clamp"] = (r[0] - R_MIN).abs() <= r[1]
    aa["active"] = active
    if "clamp_grad" in bug:
        active = torch.ones_like(active)
    if "no_drho" in bug:
        return dL_da, dL_db, dL_dc
    co_w = (torch.as_tensor(aa["co_w"]).to(r[0]).reshape(-1), 0.0)
    o = div(co_w, rho)
    g = div(mul(mul(gO, o), 0.5), mul(mul(rho, denom), denom))
    bb = mul(b, b)
    ta = mul(g, add(mul(C03, add(mul(c0, c0), bb)), mul(C009, c0)))
    tc = mul(g, add(mul(C03, add(mul(a0, a0), bb)), mul(C009, a0)))
    tb = mul(mul(scale(g, 2.0), b), add(mul(C03, add(a0, c0)), C009))
    # the terms are evaluated for every Gaussian; those of clamped ones (possibly inf) are discarded, not multiplied by 0
    keep = lambda new, old: (torch.where(active, new[0], old[0]), torch.where(active, new[1], torch.as_tensor(old[1]).to(new[1])))
    return keep(add(dL_da, ta), dL_da), keep(sub(dL_db, tb), dL_db), keep(add(dL_dc, tc), dL_dc)


def preprocess_backward(means, view, proj, tanfovx, tanfovy, H, W, mod, radii, cov3d, d_mean2D, d_conic_op, scales=None,
                        rots=None, depth=None, shs=None, D=0, campos=None, clamped=None, d_rgb=None, exact32=True, bug=(), aa=None):
    """preprocess_bwd_kernel for one frame's P Gaussians (tensors of fp32 values; any device, computed in float64).  Returns a
    dict of (value, bound) pairs: d_means3D [P,3], d_cov3D [P,6], and without cov mode (scales given) d_scales [P,3] and
    d_rotations [P,4]; with SH d_sh [P,M,3].  Culled Gaussians (radii <= 0) get exact zeros with bound 0.  `vis`, `xgm` / `ygm`
    (the guard-band gates), `tvz` and `marg_overflow` describe the Gaussians.  exact32=False evaluates the exact part in plain
    fp64 instead (to match the fp64 oracle).  aa: a dict (co_w, bug) for a frame rendered with antialiasing, whose terms are added
    right after dL/d(a, b, c) as the kernel adds them (raster_aa_fp64.preprocess_backward)."""
    dev = means.device
    f = lambda t: torch.as_tensor(t).to(device=dev, dtype=torch.float64)
    means, view, proj = f(means), f(view).reshape(16), f(proj).reshape(16)
    radii, cov3d, d_mean2D, d_conic_op = torch.as_tensor(radii).to(dev), f(cov3d), f(d_mean2D), f(d_conic_op)
    P = means.shape[0]
    vis = radii > 0
    rn = f32 if exact32 else (lambda t: t)
    xf = xf_row32 if exact32 else xf_row64
    px, py, pz = means[:, 0], means[:, 1], means[:, 2]
    tvx, tvy, tvz = xf(view, 0, px, py, pz), xf(view, 1, px, py, pz), xf(view, 2, px, py, pz)
    tanx, tany = cf32(tanfovx), cf32(tanfovy)
    limx, limy = rn(torch.tensor(cf32(1.3) * tanx, dtype=torch.float64)), rn(torch.tensor(cf32(1.3) * tany, dtype=torch.float64))
    limx, limy = float(limx), float(limy)
    txtz, tytz = rn(tvx / tvz), rn(tvy / tvz)
    xgm = ~((txtz < -limx) | (txtz > limx))
    ygm = ~((tytz < -limy) | (tytz > limy))
    if "gate" in bug:
        xgm, ygm = torch.ones_like(xgm), torch.ones_like(ygm)
    txc, tyc = txtz.clamp(-limx, limx), tytz.clamp(-limy, limy)
    tv = (tvz, 0.0)
    fx = div(float(W), (torch.tensor(2.0 * tanx, dtype=torch.float64, device=dev), 0.0))
    fy = div(float(H), (torch.tensor(2.0 * tany, dtype=torch.float64, device=dev), 0.0))
    tx, ty = mul((txc, 0.0), tv), mul((tyc, 0.0), tv)
    tz = div(1.0, tv)
    tz2 = mul(tz, tz)
    tz3 = mul(tz2, tz)
    J00, J02 = mul(fx, tz), mul(mul(neg(fx), tx), tz2)
    J11, J12 = mul(fy, tz), mul(mul(neg(fy), ty), tz2)
    V = lambda k: (view[k], 0.0)
    m0 = [add(mul(V(k * 4 + 0), J00), mul(V(k * 4 + 2), J02)) for k in range(3)]
    m1 = [add(mul(V(k * 4 + 1), J11), mul(V(k * 4 + 2), J12)) for k in range(3)]
    c3 = [(cov3d[:, k], 0.0) for k in range(6)]
    Sg = [[c3[0], c3[1], c3[2]], [c3[1], c3[3], c3[4]], [c3[2], c3[4], c3[5]]]
    v0 = [lsum(mul(Sg[k][0], m0[0]), mul(Sg[k][1], m0[1]), mul(Sg[k][2], m0[2])) for k in range(3)]
    v1 = [lsum(mul(Sg[k][0], m1[0]), mul(Sg[k][1], m1[1]), mul(Sg[k][2], m1[2])) for k in range(3)]
    c03 = cf32(0.3)
    a = add(lsum(mul(m0[0], v0[0]), mul(m0[1], v0[1]), mul(m0[2], v0[2])), c03)
    b = lsum(mul(m0[0], v1[0]), mul(m0[1], v1[1]), mul(m0[2], v1[2]))
    c = add(lsum(mul(m1[0], v1[0]), mul(m1[1], v1[1]), mul(m1[2], v1[2])), c03)
    gA, gBh, gC = (d_conic_op[:, 0], 0.0), (d_conic_op[:, 1], 0.0), (d_conic_op[:, 2], 0.0)
    if "full_offdiag" in bug:
        gBh = scale(gBh, 2.0)
    denom = sub(mul(a, c), mul(b, b))
    dd = add(mul(denom, denom), cf32(1e-7))
    marg_overflow = vis & (dd[0] + dd[1] >= 0.5 * F32_MAX)
    d2i = div(1.0, dd)
    ac = mul(a, c)
    dL_da = mul(d2i, lsum(mul(mul(neg(c), c), gA), mul(mul(scale(b, 2.0), c), gBh), mul(sub(denom, ac), gC)))
    dL_dc = mul(d2i, lsum(mul(mul(neg(a), a), gC), mul(mul(scale(a, 2.0), b), gBh), mul(sub(denom, ac), gA)))
    dL_db = mul(scale(d2i, 2.0), lsum(sub(mul(mul(b, c), gA), mul(add(denom, mul(scale(b, 2.0), b)), gBh)), mul(mul(a, b), gC)))
    if aa is not None:
        dL_da, dL_db, dL_dc = _aa_terms(m0, m1, v0, v1, b, denom, (d_conic_op[:, 3], 0.0), dL_da, dL_db, dL_dc, aa)
    dc = [None] * 6
    for k, (i, j) in ((0, (0, 0)), (3, (1, 1)), (5, (2, 2))):
        dc[k] = lsum(mul(mul(m0[i], m0[i]), dL_da), mul(mul(m0[i], m1[i]), dL_db), mul(mul(m1[i], m1[i]), dL_dc))
    for k, (i, j) in ((1, (0, 1)), (2, (0, 2))):
        dc[k] = lsum(mul(mul(scale(m0[i], 2.0), m0[j]), dL_da), mul(add(mul(m0[i], m1[j]), mul(m0[j], m1[i])), dL_db),
                     mul(mul(scale(m1[i], 2.0), m1[j]), dL_dc))
    dc[4] = lsum(mul(mul(scale(m0[2], 2.0), m0[1]), dL_da), mul(add(mul(m0[1], m1[2]), mul(m0[2], m1[1])), dL_db),
                 mul(mul(scale(m1[1], 2.0), m1[2]), dL_dc))
    dm0 = [add(mul(scale(v0[k], 2.0), dL_da), mul(v1[k], dL_db)) for k in range(3)]
    dm1 = [add(mul(scale(v1[k], 2.0), dL_dc), mul(v0[k], dL_db)) for k in range(3)]
    dJ00 = lsum(*[mul(V(k * 4 + 0), dm0[k]) for k in range(3)])
    dJ02 = lsum(*[mul(V(k * 4 + 2), dm0[k]) for k in range(3)])
    dJ11 = lsum(*[mul(V(k * 4 + 1), dm1[k]) for k in range(3)])
    dJ12 = lsum(*[mul(V(k * 4 + 2), dm1[k]) for k in range(3)])
    dL_dtx = mul(mul(mul((xgm.double(), 0.0), neg(fx)), tz2), dJ02)
    dL_dty = mul(mul(mul((ygm.double(), 0.0), neg(fy)), tz2), dJ12)
    txz, tyz = (tx, ty) if "tz_unclamped" not in bug else (mul((txtz, 0.0), tv), mul((tytz, 0.0), tv))
    dL_dtz = lsum(sub(mul(mul(neg(fx), tz2), dJ00), mul(mul(fy, tz2), dJ11)), mul(mul(mul(scale(fx, 2.0), txz), tz3), dJ02),
                  mul(mul(mul(scale(fy, 2.0), tyz), tz3), dJ12))
    dmean = [lsum(mul(V(k * 4 + 0), dL_dtx), mul(V(k * 4 + 1), dL_dty), mul(V(k * 4 + 2), dL_dtz)) for k in range(3)]
    hx, hy, hw = xf(proj, 0, px, py, pz), xf(proj, 1, px, py, pz), xf(proj, 3, px, py, pz)
    m_w = div(1.0, add((hw, 0.0), cf32(1e-7)))
    mul1, mul2 = mul(mul((hx, 0.0), m_w), m_w), mul(mul((hy, 0.0), m_w), m_w)
    g2x, g2y = (d_mean2D[:, 0], 0.0), (d_mean2D[:, 1], 0.0)
    Pm = lambda k: (proj[k], 0.0)
    for k in range(3):
        if "no_proj_w" in bug:
            tx_, ty_ = mul(Pm(4 * k + 0), m_w), mul(Pm(4 * k + 1), m_w)
        else:
            tx_ = sub(mul(Pm(4 * k + 0), m_w), mul(Pm(4 * k + 3), mul1))
            ty_ = sub(mul(Pm(4 * k + 1), m_w), mul(Pm(4 * k + 3), mul2))
        dmean[k] = add(dmean[k], add(mul(tx_, g2x), mul(ty_, g2y)))
    out = {}
    if shs is not None:
        shs, campos, d_rgb = f(shs), f(campos).reshape(3), f(d_rgb)
        cl = torch.as_tensor(clamped).to(dev).long()
        M = shs.shape[1]
        g = [(torch.where((cl >> ch) & 1 == 1, 0.0, d_rgb[:, ch]) if "no_clamp_mask" not in bug else d_rgb[:, ch], 0.0)
             for ch in range(3)]
        (x, y, z), inv = sh_dir(means, campos)
        C = SH_C32 if exact32 else SH_C64
        bs = sh_basis(x, y, z, C)
        nk = (D + 1) ** 2
        s = []
        for k in range(16):
            if k < nk:
                s.append(lsum(*[mul((shs[:, k, ch], 0.0), g[ch]) for ch in range(3)]))
            else:
                s.append((torch.zeros(P, dtype=torch.float64, device=dev), torch.zeros(P, dtype=torch.float64, device=dev)))
        dsh_v = torch.zeros(P, M, 3, dtype=torch.float64, device=dev)
        dsh_e = torch.zeros_like(dsh_v)
        for k in range(min(nk + (1 if "sh_extra" in bug else 0), 16, M)):
            for ch in range(3):
                dsh_v[:, k, ch], dsh_e[:, k, ch] = mul(bs[k], g[ch])
        xx, yy, zz = mul(x, x), mul(y, y), mul(z, z)
        xy, yz, xz = mul(x, y), mul(y, z), mul(x, z)
        kc_ = lambda a, n: kc(a, n, C)
        ddx = lsum(mul(-C["C1"], s[3]), mul(mul(C["C2_0"], y), s[4]))
        ddx = sub(ddx, mul(mul(kc_(2, "C2_2"), x), s[6]))
        ddx = lsum(ddx, mul(mul(C["C2_3"], z), s[7]), mul(mul(kc_(2, "C2_4"), x), s[8]), mul(mul(kc_(6, "C3_0"), xy), s[9]),
                   mul(mul(C["C3_1"], yz), s[10]))
        ddx = sub(sub(ddx, mul(mul(kc_(2, "C3_2"), xy), s[11])), mul(mul(kc_(6, "C3_3"), xz), s[12]))
        ddx = lsum(ddx, mul(mul(C["C3_4"], sub(sub(scale(zz, 4.0), mul(3.0, xx)), yy)), s[13]), mul(mul(kc_(2, "C3_5"), xz), s[14]),
                   mul(mul(kc_(3, "C3_6"), sub(xx, yy)), s[15]))
        ddy = lsum(mul(-C["C1"], s[1]), mul(mul(C["C2_0"], x), s[4]), mul(mul(C["C2_1"], z), s[5]))
        ddy = sub(sub(ddy, mul(mul(kc_(2, "C2_2"), y), s[6])), mul(mul(kc_(2, "C2_4"), y), s[8]))
        ddy = lsum(ddy, mul(mul(kc_(3, "C3_0"), sub(xx, yy)), s[9]), mul(mul(C["C3_1"], xz), s[10]),
                   mul(mul(C["C3_2"], sub(sub(scale(zz, 4.0), xx), mul(3.0, yy))), s[11]))
        ddy = sub(sub(sub(sub(ddy, mul(mul(kc_(6, "C3_3"), yz), s[12])), mul(mul(kc_(2, "C3_4"), xy), s[13])),
                      mul(mul(kc_(2, "C3_5"), yz), s[14])), mul(mul(kc_(6, "C3_6"), xy), s[15]))
        ddz = lsum(mul(C["C1"], s[2]), mul(mul(C["C2_1"], y), s[5]), mul(mul(kc_(4, "C2_2"), z), s[6]), mul(mul(C["C2_3"], x), s[7]),
                   mul(mul(C["C3_1"], xy), s[10]), mul(mul(kc_(8, "C3_2"), yz), s[11]),
                   mul(mul(C["C3_3"], sub(sub(mul(6.0, zz), mul(3.0, xx)), mul(3.0, yy))), s[12]), mul(mul(kc_(8, "C3_4"), xz), s[13]),
                   mul(mul(C["C3_5"], sub(xx, yy)), s[14]))
        dot = lsum(mul(x, ddx), mul(y, ddy), mul(z, ddz))
        if "no_sh_dir" not in bug:
            for k, (dk, ck) in enumerate(((ddx, x), (ddy, y), (ddz, z))):
                dmean[k] = add(dmean[k], mul(sub(dk, mul(ck, dot)), inv))
        out["d_sh"] = (dsh_v, dsh_e)
    out["d_means3D"] = (torch.stack([d[0] for d in dmean], 1), torch.stack([d[1] for d in dmean], 1))
    out["d_cov3D"] = (torch.stack([d[0] for d in dc], 1), torch.stack([d[1] for d in dc], 1))
    if scales is not None:
        scales, rots = f(scales), f(rots)
        modf = cf32(mod)
        sv = [mul(modf, (scales[:, k], 0.0)) for k in range(3)]
        q = rots
        if "norm_quat" in bug:
            q = rn(q / q.norm(dim=1, keepdim=True))
        Rm = quat_to_rot32(q, rn)
        Rm = [[(Rm[i][j], 0.0) for j in range(3)] for i in range(3)]
        dS = [[dc[0], scale(dc[1], 0.5), scale(dc[2], 0.5)], [scale(dc[1], 0.5), dc[3], scale(dc[4], 0.5)],
              [scale(dc[2], 0.5), scale(dc[4], 0.5), dc[5]]]
        dM = [[scale(lsum(*[mul(mul(sv[a2], Rm[j][a2]), dS[j][k]) for j in range(3)]), 2.0) for k in range(3)] for a2 in range(3)]
        dsc = []
        for a2 in range(3):
            t = lsum(*[mul(Rm[k][a2], dM[a2][k]) for k in range(3)])
            dsc.append(t if "scale_mod" in bug else mul(modf, t))
        dR = [[mul(sv[a2], dM[a2][k]) for a2 in range(3)] for k in range(3)]
        qr, qx, qy, qz = [(q[:, k], 0.0) for k in range(4)]
        m2 = lambda t: scale(t, 2.0)
        dqr = lsum(mul(neg(qz), dR[0][1]), mul(qy, dR[0][2]), mul(qz, dR[1][0]))
        dqr = add(sub(sub(dqr, mul(qx, dR[1][2])), mul(qy, dR[2][0])), mul(qx, dR[2][1]))
        dqx = lsum(mul(qy, dR[0][1]), mul(qz, dR[0][2]), mul(qy, dR[1][0]))
        dqx = add(add(sub(sub(dqx, mul(m2(qx), dR[1][1])), mul(qr, dR[1][2])), mul(qz, dR[2][0])), mul(qr, dR[2][1]))
        dqx = sub(dqx, mul(m2(qx), dR[2][2]))
        dqy = lsum(mul(neg(m2(qy)), dR[0][0]), mul(qx, dR[0][1]), mul(qr, dR[0][2]), mul(qx, dR[1][0]), mul(qz, dR[1][2]))
        dqy = sub(add(sub(dqy, mul(qr, dR[2][0])), mul(qz, dR[2][1])), mul(m2(qy), dR[2][2]))
        dqz = sub(mul(neg(m2(qz)), dR[0][0]), mul(qr, dR[0][1]))
        dqz = lsum(dqz, mul(qx, dR[0][2]), mul(qr, dR[1][0]))
        dqz = lsum(sub(dqz, mul(m2(qz), dR[1][1])), mul(qy, dR[1][2]), mul(qx, dR[2][0]), mul(qy, dR[2][1]))
        dq = [m2(t) for t in (dqr, dqx, dqy, dqz)]
        out["d_scales"] = (torch.stack([d[0] for d in dsc], 1), torch.stack([d[1] for d in dsc], 1))
        out["d_rotations"] = (torch.stack([d[0] for d in dq], 1), torch.stack([d[1] for d in dq], 1))
    for k, (v, e) in out.items():
        m = vis.reshape(-1, *([1] * (v.dim() - 1)))
        out[k] = (torch.where(m, v, 0.0), torch.where(m, e, 0.0))
    out.update(vis=vis, xgm=xgm & vis, ygm=ygm & vis, tvz=tvz, marg_overflow=marg_overflow)
    if depth is not None and exact32:
        dz = f(depth)
        assert torch.equal(tvz[vis], dz[vis]), "K8's tvz differs from K1's staged depth"
    return out
