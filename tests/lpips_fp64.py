"""fp64 reference of the LPIPS head launches (csrc/lpips.cu: lpips_dist1..5, lpips_sum, lpips_dnorm1..5), with error bounds (test
helper).

The head reads what the rest of the network left in the workspace: each ReLU map f, NHWC [2B, h, w, C] (frames 0..B-1 rendered,
B..2B-1 ground truth; f0, f1 below are a pixel's two channel vectors), the lin weights w [C], and in the backward the caller's
g [B] and gnext, the gradient the next slice's data gradient put on this map.  From those, in fp64:

  dist      d = sum_c w_c (f0_c / d0 - f1_c / d1)^2 per pixel, n = |f| (the channel 2-norm), d = n + 1e-10; and each CTA's
            partial sum of d over the pixels the kernel gives it: pixel px = i kDistWarps + warp + m nblk kDistWarps goes to CTA i,
            warp `warp`, with kDistWarps = 8 and nblk = min(ceil(HW / 64), kMaxPart = 128).
  sum       out[b] = sum_k (sum_{i < nblk_k} part_k[b][i]) / HW_k from the device's own partials.
  dnorm     dZ = [f0 > 0] (gnext + gh / d0 - f0 (sum_c gh_c f0_c) / (n0 d0^2)),  gh = 2 g_b / HW w (f0 / d0 - f1 / d1),
            and dZ = 0 where n0 = 0.  This is d/df0 of g_b mean_px d, times the ReLU mask, plus gnext.

Error bounds.  Every value is carried as (v, e): v the fp64 value, e a bound on |kernel result - v|, with silhouette_fp64's
arithmetic: an fp32 operation adds u (|result| + e), u = 2^-24 + 2^-53 (its rounding and that of v), plus 2^-126 for underflow;
products and quotients propagate their operands' bounds rigorously.  Counting a multiply and an add as two roundings also covers
a contracted FMA, so each bound holds whether nvcc fuses (`--fmad=true`, its default) or not: in particular the two forms of
dnorm's last step, fmaf(-f0, k2, gh / d0) and gh / d0 - f0 k2.  That difference cancels, so it is bounded by its two terms'
magnitudes, never by |dZ|.  sqrtf and the division are correctly rounded (the library is built without --use_fast_math);
sqrt propagates its argument's bound as e / (sqrt(s) + sqrt(s - e)) (sqrt(s + e) when s - e <= 0).  The constant 1e-10f is
float32(1e-10), so the reference's 1e-10 carries the difference as its bound.

Fixed-order sums add gamma(depth) sum (|term| + e_term), gamma(n) = n u / (1 - n u), plus the fp64 sum's own gamma(n, 2^-52):
  |f|^2 and the dot products: each lane's FMA chain over J = C / 32 channels, then the 5-level xor tree: depth J + 5 (the chain's
          first fmaf rounds the first product, so the terms themselves are exact).
  d:      the same, over the weighted squares (w h) h, the product w h rounded and the FMA counted as a multiply and an add.
  partial each warp's serial sum over its m pixels, then the CTA's 8-term serial sum: depth m + 8, m the CTA's busiest warp.
  sum     nblk_k serial adds per layer, the division by HW_k (exact in fp32) rounded, 5 serial adds over the layers.
Bounds use |w|, so zero or negative lin weights stay bounded.

The stored dZ is tf32_rn(v) (round to nearest, ties away, low 13 bits cleared), within 2^-11 |v| of v: the bound adds
2^-11 (|ref| + e), and every stored element is a TF32 value.  The mask f0 > 0 is read from the device's own f0, so no mask
decision is marginal; the kernel's n0 > 0 branch agrees with the reference's wherever some f0_c > 0 (no square of a TF32 value
above 2^-74 underflows), and elsewhere the mask zeroes the element anyway.

Written in torch: it runs on the CPU for small maps and in fp64 on the GPU, in chunks of pixels, for full frames.
"""
import numpy as np
import torch

from silhouette_fp64 import ETA32, F32, U64, exact, gam

EPS = 1e-10
EPS_T = (EPS, abs(float(np.float32(EPS)) - EPS))   # the kernel's 1e-10f as a tracked constant
DIST_WARPS, MAX_PART = 8, 128
TF32_U = 2.0 ** -11
CHUNK = 1 << 22                                     # pixel-channel elements per chunk


def nblk(HW):
    return min(-(-HW // 64), MAX_PART)


def _u(a):
    return a[0].unsqueeze(-1), a[1].unsqueeze(-1)


def _sum(t, depth):
    """The last axis of tracked terms summed in a fixed fp32 order whose deepest term sees `depth` roundings."""
    v, e = t
    n = v.shape[-1]
    a = (v.abs() + e).sum(-1)
    return v.sum(-1), e.sum(-1) + (gam(depth) + gam(n, U64)) * a + n * ETA32


def _sqrt(a):
    v, e = a
    r = v.sqrt()
    prop = torch.where(v - e > 0, e / (r + (v - e).clamp_min(0).sqrt()), (v + e).sqrt())
    return F32.rnd(r, prop)


def _norms(x, eps_inside=False):
    """n = sqrtf(s), d = n + 1e-10f (tracked) of channel vectors x [..., C], s summed as the kernels sum it.  eps_inside: the
    value of the wrong form sqrt(s + 1e-10), for the self-checks."""
    s = _sum(exact(x * x), x.shape[-1] // 32 + 5)
    n = _sqrt(s)
    d = F32.add(n, EPS_T)
    if eps_inside:
        d = ((s[0] + EPS).sqrt(), d[1])
    return n, d


def _chunks(HW, C):
    step = max(1, CHUNK // C)
    for p0 in range(0, HW, step):
        yield slice(p0, min(HW, p0 + step))


def _frames(f, B):
    f = f.reshape(2 * B, -1, f.shape[-1])
    return f[:B], f[B:]


def layer_distance(f, lin, B, eps_inside=False):
    """Per pixel d (v, e), each [B, HW], of the relu map f [2B, h, w, C] with lin weights [C]."""
    f0, f1 = _frames(f, B)
    C = f0.shape[-1]
    w = exact(lin.reshape(-1).to(f0.device).double())
    v = torch.empty(f0.shape[:2], dtype=torch.float64, device=f0.device)
    e = torch.empty_like(v)
    for sl in _chunks(f0.shape[1], C):
        x0, x1 = f0[:, sl].double(), f1[:, sl].double()
        _, d0 = _norms(x0, eps_inside)
        _, d1 = _norms(x1, eps_inside)
        h = F32.sub(F32.div(exact(x0), _u(d0)), F32.div(exact(x1), _u(d1)))
        v[:, sl], e[:, sl] = _sum(F32.mul(F32.mul(w, h), h), C // 32 + 5)
    return v, e


def assignment(HW, nb):
    """The CTA of each pixel in lpips_dist_kernel's grid-stride loop, and each CTA's busiest warp's pixel count."""
    px = torch.arange(HW)
    cta = (px // DIST_WARPS) % nb
    per_warp = torch.bincount(cta * DIST_WARPS + px % DIST_WARPS, minlength=nb * DIST_WARPS)
    return cta, per_warp.view(nb, DIST_WARPS).amax(1)


def partials(d, nb):
    """Each CTA's partial sum (v, e) [B, nb] of the per-pixel d (v, e) [B, HW]."""
    v, e = d
    B, HW = v.shape
    cta, m = assignment(HW, nb)
    cta, m = cta.to(v.device), m.to(v.device)
    z = lambda t: torch.zeros(B, nb, dtype=torch.float64, device=v.device).index_add_(1, cta, t)
    n = torch.bincount(cta, minlength=nb).to(v.device)
    return z(v), z(e) + (gam(m + 8) + gam(n, U64)) * z(v.abs() + e) + n * ETA32


def lpips_sum(part, nb, HW):
    """out[b] (v, e) [B] from the device's partials [5, B, >= max nb] (per layer nb[k] slots read, divided by HW[k])."""
    terms = []
    for k in range(5):
        p = part[k, :, :nb[k]].double()
        s = (p.sum(1), (gam(nb[k]) + gam(nb[k], U64)) * p.abs().sum(1) + nb[k] * ETA32)
        terms.append(F32.div(s, exact(torch.full_like(s[0], float(HW[k])))))
    return _sum((torch.stack([t[0] for t in terms], -1), torch.stack([t[1] for t in terms], -1)), 5)


def dnorm(f, lin, g, gnext, HW, drop_proj=False, mask_f1=False, eps_inside=False):
    """dZ (v, e), each [B, h*w, C], of the relu map f [2B, h, w, C], lin [C], g [B] and gnext ([B, h, w, C] or None), with HW the
    divisor of the mean (the map's h*w; the self-checks pass another).  The flags give the values of plausible wrong kernels:
    drop_proj (no projection term), mask_f1 (the ReLU mask from f1), eps_inside (d = sqrt(s + 1e-10))."""
    B = g.numel()
    f0, f1 = _frames(f, B)
    C = f0.shape[-1]
    dev = f0.device
    gn = None if gnext is None else gnext.reshape(B, -1, C)
    w = exact(lin.reshape(-1).to(dev).double())
    sc = F32.div(exact(2.0 * g.to(dev).double()), exact(torch.full((B,), float(HW), dtype=torch.float64, device=dev)))
    sc = (sc[0].view(B, 1, 1), sc[1].view(B, 1, 1))
    v = torch.zeros(f0.shape, dtype=torch.float64, device=dev)
    e = torch.zeros_like(v)
    for sl in _chunks(f0.shape[1], C):
        x0, x1 = f0[:, sl].double(), f1[:, sl].double()
        n0, d0 = _norms(x0, eps_inside)
        _, d1 = _norms(x1, eps_inside)
        q = F32.sub(F32.div(exact(x0), _u(d0)), F32.div(exact(x1), _u(d1)))
        gh = F32.mul(F32.mul(sc, w), q)
        dot = _sum(F32.mul(gh, exact(x0)), C // 32 + 5)
        k2 = F32.div(dot, F32.mul(F32.mul(n0, d0), d0))
        t = F32.div(gh, _u(d0))
        if not drop_proj:
            t = F32.sub(t, F32.mul(exact(x0), _u(k2)))
        if gn is not None:
            t = F32.add(t, exact(gn[:, sl].double()))
        live = (n0[0] > 0).unsqueeze(-1) & ((x1 if mask_f1 else x0) > 0)
        tv = torch.where(live, t[0], 0.0)
        v[:, sl] = tv
        e[:, sl] = torch.where(live, t[1] + TF32_U * (tv.abs() + t[1]), 0.0)
    return v, e


def ratio(got, ref):
    """|got - ref| / bound per element (0 where both the difference and the bound are 0)."""
    v, e = ref
    diff = (got.double().reshape(v.shape) - v).abs()
    return torch.where(diff == 0, torch.zeros_like(diff), diff / e)


def rejects(got, ref):
    """A kernel that computed `got` fails the check against `ref`: some element lies beyond its bound."""
    return bool((ratio(got, ref) > 1).any())


def is_tf32(x):
    return bool(((x.contiguous().view(torch.int32) & 0x1FFF) == 0).all())
