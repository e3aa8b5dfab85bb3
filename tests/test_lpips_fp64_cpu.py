"""CPU: the bounded fp64 LPIPS head reference (tests/lpips_fp64.py) against autograd of oracle/lpips_oracle.py's distance, its
bounds against numpy fp32 restatements of lpips_dist_kernel, lpips_sum_kernel and lpips_dnorm_kernel in their operation order
(dnorm's last step with and without a contracted FMA), and the corruptions each bound must reject."""
import numpy as np
import pytest
import torch

import lpips_fp64 as lf
from oracle import lpips_oracle as lo
from oracle.mesh_oracle import fma32

f32 = np.float32
LANE = np.arange(32)


# ---- the kernels in numpy fp32 ------------------------------------------------------------------------------------------------
def _xor_tree(s):
    for o in (16, 8, 4, 2, 1):
        s = (s + s[..., LANE ^ o]).astype(f32)
    assert (s == s[..., :1]).all()
    return s[..., 0]


def _lanes(x):
    """[..., C] -> [..., J, 32]: lane l holds channels l + 32 j."""
    return x.reshape(*x.shape[:-1], x.shape[-1] // 32, 32)


def _dot(a, b):
    """Each lane's fmaf chain over its J channels, then the xor tree."""
    a, b = _lanes(a), _lanes(b)
    s = np.zeros(a.shape[:-2] + (32,), f32)
    for j in range(a.shape[-2]):
        s = fma32(a[..., j, :], b[..., j, :], s)
    return _xor_tree(s)


def _denoms(x):
    n = np.sqrt(_dot(x, x))
    return n, (n + f32(1e-10)).astype(f32)


def emu_dist(x0, x1, w):
    """lpips_dist_kernel's per-pixel d, x0 / x1 [B, P, C] float32."""
    with np.errstate(all="ignore"):
        _, d0 = _denoms(x0)
        _, d1 = _denoms(x1)
        h = (x0 / d0[..., None] - x1 / d1[..., None]).astype(f32)
        wh = (w * h).astype(f32)
    return _dot(wh, h)


def emu_partials(d, nb):
    """The kernel's grid-stride loop: each warp's serial sum, then the CTA's over its 8 warps.  d [B, HW] -> [B, nb]."""
    B, HW = d.shape
    per = nb * lf.DIST_WARPS
    passes = -(-HW // per)
    D = np.zeros((B, passes * per), f32)
    D[:, :HW] = d                            # + 0 leaves a sum unchanged: the padding stands for the loop's missing pixels
    D = D.reshape(B, passes, nb, lf.DIST_WARPS)
    acc = np.zeros((B, nb, lf.DIST_WARPS), f32)
    for p in range(passes):
        acc = (acc + D[:, p]).astype(f32)
    s = np.zeros((B, nb), f32)
    for i in range(lf.DIST_WARPS):
        s = (s + acc[..., i]).astype(f32)
    return s


def emu_sum(part, nb, HW):
    v = np.zeros(part.shape[1], f32)
    for k in range(5):
        s = np.zeros(part.shape[1], f32)
        for i in range(nb[k]):
            s = (s + part[k, :, i]).astype(f32)
        v = (v + s / f32(HW[k])).astype(f32)
    return v


def tf32_rn(x):
    u = np.ascontiguousarray(x, f32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(f32)


def emu_dnorm(x0, x1, w, g, gn, HW, fma):
    """lpips_dnorm_kernel, x0 / x1 / gn [B, P, C], g [B]; fma: the last step contracted into fmaf(-x0, k2, gh / d0)."""
    with np.errstate(all="ignore"):
        sc = (f32(2) * g / f32(HW)).astype(f32)[:, None, None]
        n0, d0 = _denoms(x0)
        _, d1 = _denoms(x1)
        d0e, d1e = d0[..., None], d1[..., None]
        gh = ((sc * w).astype(f32) * (x0 / d0e - x1 / d1e).astype(f32)).astype(f32)
        dot = _dot(gh, x0)
        k2 = np.where(n0 > 0, dot / (n0 * d0 * d0).astype(f32), f32(0)).astype(f32)[..., None]
        a = (gh / d0e).astype(f32)
        v = fma32(-x0, np.broadcast_to(k2, x0.shape), a) if fma else (a - (x0 * k2).astype(f32)).astype(f32)
        v = np.where(n0[..., None] > 0, v, f32(0)).astype(f32)
        if gn is not None:
            v = (v + gn).astype(f32)
    return np.where(x0 > 0, tf32_rn(v), f32(0))


# ---- inputs ---------------------------------------------------------------------------------------------------------------------
def _tf32(t):
    return torch.from_numpy(tf32_rn(t.float().numpy()))


def features(kind, B, h, w, C, seed):
    """A relu map f [2B, h, w, C] of TF32 values (about half exact zeros) and lin weights [C]."""
    g = torch.Generator().manual_seed(seed)
    f = torch.relu(torch.randn(2 * B, h, w, C, generator=g)) * torch.rand(2 * B, h, w, 1, generator=g) * 3
    lin = torch.rand(C, generator=g) * (2.0 / C)
    if kind == "zero0":                                # rendered pixels whose whole vector is zero: n0 = 0
        f[:B].view(B, -1, C)[:, ::3] = 0
    elif kind == "zero1":                              # ground-truth ones: n1 = 0, d1 = 1e-10
        f[B:].view(B, -1, C)[:, ::3] = 0
    elif kind == "tiny":                               # |f| ~ 1e-11: the 1e-10 epsilon dominates d
        f = f * 1e-12
    elif kind == "linzero":                            # some lin weights exactly zero: only the projection term is left there
        lin[::3] = 0
    elif kind == "linneg":
        lin[::4] = -lin[::4]
    return _tf32(f), _tf32(lin)


KINDS = ["random", "zero0", "zero1", "tiny", "linzero", "linneg"]
SHAPES = [(1, 5, 7, 64), (3, 3, 1, 192), (2, 1, 3, 384), (3, 2, 5, 256)]


def _f(t):
    return np.ascontiguousarray(t.numpy(), f32)


# ---- the restatement against the oracle ---------------------------------------------------------------------------------------
def _oracle_layer(k, lin):
    sd = lo.random_state_dict(0)
    for j in range(5):
        sd[lo.lin_key(j)] = torch.zeros(1, lo.CHANNELS[j], 1, 1)
    sd[lo.lin_key(k)] = lin.reshape(1, -1, 1, 1)
    orc = lo.LpipsOracle(sd).double()
    orc.maps = lambda x: x                             # hand the oracle its relu maps directly
    return orc


def _nchw_list(k, t):
    """Layer k's map t [N, C, h, w] among zero maps of the other layers."""
    return [t if j == k else torch.zeros(t.shape[0], c, *t.shape[2:], dtype=t.dtype) for j, c in enumerate(lo.CHANNELS)]


@pytest.mark.parametrize("kind", ["random", "zero0", "zero1", "tiny", "linzero"])
@pytest.mark.parametrize("k", range(5))
def test_restatement_matches_oracle_autograd(k, kind):
    B, h, w, C = 2, 3, 4, lo.CHANNELS[k]
    f, lin = features(kind, B, h, w, C, seed=k + 10)
    orc = _oracle_layer(k, lin.double())
    f64 = f.double()
    # the value per pixel: each pixel a 1 x 1 frame
    px = lambda t: t.reshape(-1, C, 1, 1)
    want = orc(_nchw_list(k, px(f64[:B])), _nchw_list(k, px(f64[B:]))).reshape(B, -1)
    got, _ = lf.layer_distance(f, lin, B)
    assert torch.allclose(got, want, rtol=1e-12, atol=0)
    # d/df0 of sum_b g_b mean_px d, times the ReLU mask (at n0 = 0 autograd's NaN is dropped by that mask, as in the oracle)
    g = torch.tensor([0.75, -1.25], dtype=torch.float64)            # exact in fp32
    x0 = f64[:B].permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    out = orc(_nchw_list(k, x0), _nchw_list(k, f64[B:].permute(0, 3, 1, 2)))
    (grad,) = torch.autograd.grad((out.reshape(B) * g).sum(), x0)
    grad = grad.permute(0, 2, 3, 1).reshape(B, -1, C)
    mask = f64[:B].reshape(B, -1, C) > 0
    want = torch.where(mask, grad, 0.0)
    got, _ = lf.dnorm(f, lin, g.float(), None, h * w)
    assert torch.isfinite(want).all()
    assert torch.allclose(got, want, rtol=1e-10, atol=1e-12 * float(want.abs().max()))
    gnext = _tf32(torch.randn(B, h, w, C))
    got2, _ = lf.dnorm(f, lin, g.float(), gnext, h * w)
    assert torch.allclose(got2, torch.where(mask, want + gnext.double().reshape(B, -1, C), 0.0), rtol=1e-10,
                          atol=1e-12 * float(want.abs().max()))


# ---- the bounds against the fp32 restatements ---------------------------------------------------------------------------------
def _worst(got, ref):
    assert torch.isfinite(ref[1]).all()
    return float(lf.ratio(torch.from_numpy(np.asarray(got)), ref).max())


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("B,h,w,C", SHAPES)
def test_bounds_hold_against_fp32_restatement(kind, B, h, w, C):
    f, lin = features(kind, B, h, w, C, seed=C + h)
    x = _f(f).reshape(2 * B, -1, C)
    x0, x1, wn = x[:B], x[B:], _f(lin)
    d = lf.layer_distance(f, lin, B)
    worst = {"dist": _worst(emu_dist(x0, x1, wn), d)}
    nb = lf.nblk(h * w)
    worst["partials"] = _worst(emu_partials(emu_dist(x0, x1, wn), nb), lf.partials(d, nb))
    g = np.array([0.8, -1.7, 0.0][:B], f32)
    gn = _tf32(torch.randn(B, h, w, C) * 1e-3)
    for gnext in (None, gn):
        ref = lf.dnorm(f, lin, torch.from_numpy(g), gnext, h * w)
        for fma in (False, True):
            got = emu_dnorm(x0, x1, wn, g, None if gnext is None else _f(gnext).reshape(B, -1, C), h * w, fma)
            assert lf.is_tf32(torch.from_numpy(got))
            worst[f"dnorm fma={fma} gnext={gnext is not None}"] = _worst(got, ref)
    print(f"\n{kind} {B}x{h}x{w}x{C}: " + ", ".join(f"{n} {r:.3g}" for n, r in worst.items()))
    assert max(worst.values()) <= 1.0


@pytest.mark.parametrize("HW", [1, 37, 64, 65, 8192, 8256, 8256 + 1029])
def test_partials_and_sum_bounds(HW):
    """The partials' CTA assignment at HW = 1 (one busy warp), around one CTA, at nblk = 128 exactly and past it (a second pass of
    the grid-stride loop), with d spanning nine decades; lpips_sum over five such layers."""
    g = np.random.default_rng(HW)
    B = 2
    d = (g.random((B, HW)) * 10.0 ** g.integers(-6, 3, (B, HW))).astype(f32)
    nb = lf.nblk(HW)
    assert nb == min(-(-HW // 64), 128)
    dt = (torch.from_numpy(d).double(), torch.zeros(B, HW, dtype=torch.float64))
    part = emu_partials(d, nb)
    assert _worst(part, lf.partials(dt, nb)) <= 1.0
    cta, m = lf.assignment(HW, nb)
    assert int(cta.max()) == nb - 1 and int(m.max()) == -(-HW // (8 * nb))
    HWs = [HW, 4 * HW + 1, 5, 7, 7]
    nbs = [lf.nblk(n) for n in HWs]
    P = np.zeros((5, B, 128), f32)
    for k in range(5):
        P[k, :, :nbs[k]] = emu_partials((g.random((B, HWs[k])) * 3).astype(f32), nbs[k])
        P[k, :, nbs[k]:] = np.nan                      # slots past nblk are never read
    assert _worst(emu_sum(P, nbs, HWs), lf.lpips_sum(torch.from_numpy(P), nbs, HWs)) <= 1.0


# ---- the corruptions each bound rejects -------------------------------------------------------------------------------------
def test_bounds_reject_corruptions():
    """A kernel with one of these bugs would fail its tier: each wrong value lies beyond the right reference's bound somewhere."""
    B, h, w, C = 3, 2, 5, 64
    f, lin = features("random", B, h, w, C, seed=1)
    x = _f(f).reshape(2 * B, -1, C)
    x0, x1, wn = x[:B], x[B:], _f(lin)
    HW = h * w
    # dist: one CTA's partial zeroed
    nb = lf.nblk(HW)
    ref = lf.partials(lf.layer_distance(f, lin, B), nb)
    got = torch.from_numpy(emu_partials(emu_dist(x0, x1, wn), nb))
    assert not lf.rejects(got, ref)
    bad = got.clone(); bad[1, 0] = 0
    assert lf.rejects(bad, ref)
    # sum: one partial slot not read, a neighbouring layer's HW
    HWs, P = [HW, 37, 5, 5, 5], np.zeros((5, B, 128), f32)
    nbs = [lf.nblk(n) for n in HWs]
    for k in range(5):
        P[k, :, :nbs[k]] = np.random.default_rng(k).random((B, nbs[k])) + 0.5
    sref = lf.lpips_sum(torch.from_numpy(P), nbs, HWs)
    assert not lf.rejects(torch.from_numpy(emu_sum(P, nbs, HWs)), sref)
    short = list(nbs); short[1] -= 1
    assert lf.rejects(torch.from_numpy(emu_sum(P, short, HWs)), sref)
    assert lf.rejects(torch.from_numpy(emu_sum(P, nbs, [HWs[1]] + HWs[1:])), sref)
    # dnorm
    g = torch.tensor([0.8, -1.7, 0.4])
    gn = _tf32(torch.randn(B, h, w, C) * 1e-2)
    other = _tf32(torch.randn(B, h, w, C) * 1e-2)
    ref = lf.dnorm(f, lin, g, gn, HW)
    got = torch.from_numpy(emu_dnorm(x0, x1, wn, g.numpy(), _f(gn).reshape(B, -1, C), HW, True))
    assert not lf.rejects(got, ref)
    for name, wrong in (("projection dropped", lf.dnorm(f, lin, g, gn, HW, drop_proj=True)),
                        ("gnext not added", lf.dnorm(f, lin, g, None, HW)),
                        ("gnext of another layer", lf.dnorm(f, lin, g, other, HW)),
                        ("HW of another layer", lf.dnorm(f, lin, g, gn, 4 * HW + 1)),
                        ("mask from f1", lf.dnorm(f, lin, g, gn, HW, mask_f1=True))):
        assert lf.rejects(wrong[0], ref), name
    # the epsilon inside the square root: visible only where it is a share of |f|
    ft, lint = features("tiny", B, h, w, C, seed=2)
    for fn in (lambda **kw: lf.layer_distance(ft, lint, B, **kw), lambda **kw: lf.dnorm(ft, lint, g, None, HW, **kw)):
        assert lf.rejects(fn(eps_inside=True)[0], fn())
    assert not lf.rejects(lf.layer_distance(f, lin, B, eps_inside=True)[0], lf.layer_distance(f, lin, B))
