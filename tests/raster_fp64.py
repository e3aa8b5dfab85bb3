"""fp64 reference of the rasterizer's compositing (K6) and its backward (K7), with a running error bound (test helper).

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
