"""GPU: the stage-1 step's kernels outside the decoder, element by element against fp64 at the sizes the step runs.

Covered: the Gaussian skinning / attribute assembly (csrc/lbs.cu, ga_lbs_forward_ex / ga_lbs_backward_ex, SMPL 24/24 and SMPL-X
55/56 weight layouts, shared and per-frame decoder output), the fused L1 + SSIM loss (csrc/loss.cu, ga_loss_forward /
ga_loss_backward), Adam (ga_adam_step / ga_adam_step_dev) and the joint transforms (csrc/smpl.cu, ga_smpl_* / ga_smplx_*).
Each kernel is called through the C ABI with its outputs inside buffers of finite sentinels, which must be bit-identical
afterwards, and with NaN in every input element it must not read; one case per kernel also runs through the Python wrapper the
step uses, so that an argument mix-up there shows.

Every output element must satisfy |got - ref| <= bound. `ref` is fp64 math on the same fp32 inputs (the kernels' fp32
constants included: 0.02f, 1e-8f, the fp32 Gaussian taps). The bound is a-priori: gamma(c) = c u / (1 - c u), u = 2^-24, times
the same expression evaluated on absolute values, where c counts the sequential fp32 roundings of the kernel's code path (each
count is derived in the docstring of the test that uses it). Counting a multiply and an add separately also covers the fused
FMA the compiler may form instead. Where a bound propagates errors through a nonlinear formula it is first order; the factor
FO = 1.01 covers the second-order terms, every relative perturbation involved being below 1e-2 of the first-order one.
Each test also corrupts a copy of an output the way a broken code path would (a stale pipeline stage, a dropped tile, swapped
frames, a dropped Gaussian tap, ...) and asserts that the same bound rejects it.

Run with -s to print the largest error / bound ratio per kernel and tier.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24
FO = 1.01
NSM = 132                                   # H100 SXM
PAD = 300                                   # sentinel elements past every output
C02 = 0.019999999552965164                  # 0.02f, the residual scale of csrc/lbs.cu
E8F = 9.99999993922529e-09                  # 1e-8f, the Rodrigues norm shift of csrc/smpl_math.cuh
NAN = float("nan")

WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for key, (r, where) in sorted(WORST.items()):
        print(f"\nstep kernels: largest error/bound, {key}: {r:.3g} ({where})")


def _lib():
    from gaussianavatar_b200 import _lib
    return _lib


def gam(c):
    return c * U / (1 - c * U)


def cdiv(a, b):
    return -(-a // b)


def ratio(got, ref, bound):
    return ((got.double() - ref) / bound.clamp_min(1e-300)).abs().max().item()   # NaN in got -> NaN -> fails every `<= 1`


def check(key, where, got, ref, bound):
    r = ratio(got, ref, bound) if got.numel() else 0.0
    if r == r and r > WORST.get(key, (-1.0, ""))[0]:
        WORST[key] = (r, where)
    assert r <= 1.0, f"{key}, {where}: error/bound {r:.4g}"


def rejects(what, bad, ref, bound):
    assert ratio(bad, ref, bound) > 1.0, f"self-check: the bound accepts {what}"


def untouched(where, after, before, lo, hi):
    """Every element of the flat buffer outside [lo, hi) is bit-identical to `before`."""
    diff = after.view(torch.int32) != before.view(torch.int32)
    diff[lo:hi] = False
    n = int(diff.sum())
    assert n == 0, f"{where}: {n} elements outside the output changed"


def stream():
    return torch.cuda.current_stream().cuda_stream


def p(t):
    return None if t is None else t.data_ptr()


def sentinel(gen, n):
    return torch.randn(n, device=DEV, generator=gen) * 1000.0


def nan_buf(*shape):
    return torch.full(shape, NAN, device=DEV)


# ========================================================================================================================== LBS
LBS_LD = {24: 24, 55: 56}


def lbs_smem_bytes(J):
    """sizeof(LbsSmem<J, ld>) of csrc/lbs.cu: two weight stages, cano2live of 8 frames, the [256][13] backward staging, 2 mbarriers."""
    raw = 4 * (2 * 256 * LBS_LD[J] + 8 * J * 12 + 256 * 13) + 8 * 2
    return cdiv(raw, 128) * 128


def lbs_grid(J, N):
    """launch_cfg of csrc/lbs.cu: as many CTAs as fit on the SMs at once (two per SM when the shared memory allows), capped by the tiles."""
    per_sm = 2 if lbs_smem_bytes(J) <= 113 * 1024 else 1
    return min(cdiv(N, 256), per_sm * NSM)


def _round(J):
    return lbs_grid(J, 1 << 30) * 256


# N: one Gaussian, a partial tile, one past a tile, one tile past one full round of CTAs, one past three rounds (stage 0 reused
# with mbarrier parity 1), configs 3-4 and 5.
LBS_N = {J: [1, 255, 257, _round(J) + 1, 3 * _round(J) + 1, 200_000, 500_000] for J in (24, 55)}


def test_lbs_sizes_reach_three_tiles_per_cta():
    """The size list gives some CTA a second tile and, for both bodies, at least three tiles (stage 0 refilled after it flips)."""
    assert lbs_grid(24, 1 << 30) == 2 * NSM and lbs_grid(55, 1 << 30) == NSM
    for J, Ns in LBS_N.items():
        per_cta = [cdiv(cdiv(N, 256), lbs_grid(J, N)) for N in Ns]
        assert 2 in per_cta and max(per_cta) >= 3, (J, per_cta)


class LbsCase:
    """Inputs of one skinning launch, with NaN in everything the kernel must not read, and the fp64 expectations."""

    def __init__(self, J, N, B, per_frame, seed):
        self.J, self.N, self.B, self.per_frame = J, N, B, per_frame
        self.ld = LBS_LD[J]
        gen = self.gen = torch.Generator(device=DEV).manual_seed(seed)
        self.P = P = N + N // 4 + 3                                   # decoder pixels, N of them valid
        self.vidx = torch.randperm(P, device=DEV, generator=gen)[:N].sort().values.to(torch.int32)
        self.frames = F_ = B if per_frame else 1
        dec = nan_buf(F_, P, 8)                                       # rows outside valid_index and column 7: NaN
        vals = torch.randn(F_, N, 8, device=DEV, generator=gen)
        vals[..., 7] = NAN
        dec[:, self.vidx.long()] = vals
        self.dec = dec
        self.q = nan_buf(N + PAD, 3)
        self.q[:N] = 0.5 * torch.randn(N, 3, device=DEV, generator=gen)
        self.w = nan_buf(N + 256, self.ld)                            # SMPL-X pad column and rows past N: NaN
        w = torch.rand(N, J, device=DEV, generator=gen) ** 4
        self.w[:N, :J] = w / w.sum(1, keepdim=True)
        self.C = nan_buf(B + 2, J, 12)                                # frames B and B + 1: NaN
        self.C[:B] = torch.randn(B, J, 12, device=DEV, generator=gen)
        self.mul = 0.30000001192092896                               # fp32(0.3): the scale ramp at iteration 300
        self.stride = P * 8 if per_frame else 0
        self.rows = F_ * P                                            # num_pixels: decoder rows (all frames)
        self.tiles = cdiv(N, 256)
        self.grid = lbs_grid(J, N)
        self.T = cdiv(self.tiles, self.grid)
        self.where = f"J={J} N={N} B={B} {'per-frame' if per_frame else 'shared'}"

    # ---------------------------------------------------------------------------------------------------------- fp64 reference
    def forward_ref(self):
        """means = M [q + 0.02f res; 1] with M = sum_j w_j C_j, in fp64.

        Bound on means: M is a J-term FMA chain from zero (J roundings, relative to sum_j |w_j| |C_j|); the position
        q + 0.02f res is a multiply and an add (2); the affine apply is three products and three adds (6):
        gamma(J + 8) (sum_k |M|_rk (|q_k| + 0.02 |res_k|) + |M|_r3).  scales = res.w * scale_mul: one rounding. colors: copies."""
        N, B, J = self.N, self.B, self.J
        w = self.w[:N, :J].double()
        C = self.C[:B].double()
        self.M = torch.einsum("nj,bje->bne", w, C).view(B, N, 3, 4)
        self.Ma = torch.einsum("nj,bje->bne", w.abs(), C.abs()).view(B, N, 3, 4)
        o = self.dec[:, self.vidx.long()].double()                    # [frames, N, 8]
        q = self.q[:N].double()
        self.o = o
        self.c = q[None] + C02 * o[..., :3]                           # [frames, N, 3]
        self.ca = q.abs()[None] + C02 * o[..., :3].abs()
        means = (self.M[..., :3] * self.c[:, :, None, :]).sum(-1) + self.M[..., 3]
        mb = gam(J + 8) * ((self.Ma[..., :3] * self.ca[:, :, None, :]).sum(-1) + self.Ma[..., 3])
        sc = (o[..., 3] * self.mul)[..., None].expand(B, N, 3)
        col = o[..., 4:7].expand(B, N, 3)
        return {"means": (means, mb), "scales": (sc, gam(1) * sc.abs()), "colors": (col, torch.zeros_like(col))}

    def skin(self, wrows, crows, b_perm=None):
        """fp64 means of Gaussians `crows` skinned with the weight rows `wrows` (a self-check helper)."""
        C = self.C[:self.B].double()
        if b_perm is not None:
            C = C[b_perm]
        M = torch.einsum("nj,bje->bne", self.w[wrows, :self.J].double(), C).view(self.B, -1, 3, 4)
        c = self.c[:, crows]
        return (M[..., :3] * c[:, :, None, :]).sum(-1) + M[..., 3]

    def backward_ref(self, dm, ds, dc):
        """d_dec rows: 0.02f sum_b M_b^T g_b (the position), scale_mul sum_b (g_s0 + g_s1 + g_s2), sum_b g_c; other rows and column 7: 0.
        dC[b][j][4r + k] = sum_n w_nj g_r (c_k or 1).

        Bounds, summing over nf = B frames into one shared row (nf = 1 per frame): position gamma(J + 1 + 2 + nf + 1) (M's chain,
        the product, the 3-term sum, the frame accumulation, the 0.02f scale) on 0.02 sum |M| |g|; scale gamma(3 nf + 1) on
        scale_mul sum |g_s|; colour gamma(nf) on sum |g_c|.  dC: each tile is one FMA chain over its (<= 256) rows, each term
        x = g_r c_k carrying c's 2 roundings and its own 1; a CTA adds its T tiles in registers (T roundings) and then atomically adds
        into dC (at most `grid` roundings): gamma(min(N, 256) + 3 + T + grid) on sum_n |w_nj| |x|."""
        N, B, J, P = self.N, self.B, self.J, self.P
        G, Gs, Gc = dm.double(), ds.double(), dc.double()
        dpos = (self.M[..., :3] * G[..., None]).sum(2)                 # [B, N, 3]
        dpos_a = (self.Ma[..., :3] * G.abs()[..., None]).sum(2)
        nf = 1 if self.per_frame else B
        rows = torch.zeros(self.frames, N, 8, dtype=torch.float64, device=DEV)
        rb = torch.zeros_like(rows)
        if self.per_frame:
            rows[..., :3] = C02 * dpos
            rb[..., :3] = gam(J + 4 + nf) * C02 * dpos_a
            rows[..., 3] = self.mul * Gs.sum(-1)
            rb[..., 3] = gam(3 * nf + 1) * self.mul * Gs.abs().sum(-1)
            rows[..., 4:7] = Gc
            rb[..., 4:7] = gam(nf) * Gc.abs()
        else:
            rows[0, :, :3] = C02 * dpos.sum(0)
            rb[0, :, :3] = gam(J + 4 + nf) * C02 * dpos_a.sum(0)
            rows[0, :, 3] = self.mul * Gs.sum(-1).sum(0)
            rb[0, :, 3] = gam(3 * nf + 1) * self.mul * Gs.abs().sum(-1).sum(0)
            rows[0, :, 4:7] = Gc.sum(0)
            rb[0, :, 4:7] = gam(nf) * Gc.abs().sum(0)
        ddec = torch.zeros(self.frames, P, 8, dtype=torch.float64, device=DEV)
        dbnd = torch.zeros_like(ddec)
        ddec[:, self.vidx.long()] = rows
        dbnd[:, self.vidx.long()] = rb
        self.X = torch.cat([G[..., None] * self.c[:, :, None, :], G[..., None]], -1).view(B, N, 12)
        Xa = torch.cat([G.abs()[..., None] * self.ca[:, :, None, :], G.abs()[..., None]], -1).view(B, N, 12)
        w = self.w[:N, :J].double()
        dC = torch.einsum("nj,bne->bje", w, self.X)
        cb = gam(min(N, 256) + 3 + self.T + self.grid) * torch.einsum("nj,bne->bje", w.abs(), Xa)
        return {"d_dec": (ddec.view(-1, 8), dbnd.view(-1, 8)), "dC": (dC, cb)}

    def tile_rows(self, t):
        return slice(t * 256, min(self.N, t * 256 + 256))


def lbs_forward_launch(cs, gen):
    B, N = cs.B, cs.N
    outs = {k: sentinel(gen, B * N * 3 + PAD) for k in ("means", "scales", "colors")}
    before = {k: v.clone() for k, v in outs.items()}
    L = _lib()
    L.check(L.lib().ga_lbs_forward_ex(N, B, cs.J, cs.ld, cs.mul, cs.stride, p(cs.dec), p(cs.vidx), p(cs.q), p(cs.w), p(cs.C),
                                      p(outs["means"]), p(outs["scales"]), p(outs["colors"]), stream()), "ga_lbs_forward_ex")
    return outs, before


def lbs_backward_launch(cs, gen):
    B, N, J = cs.B, cs.N, cs.J
    grads = []
    for _ in range(3):
        g = nan_buf(B * N * 3 + PAD)
        g[:B * N * 3] = torch.randn(B * N * 3, device=DEV, generator=gen)
        grads.append(g)
    d_dec = sentinel(gen, (cs.rows + PAD) * 8)
    dC = sentinel(gen, B * J * 12 + PAD)
    before = (d_dec.clone(), dC.clone())
    L = _lib()
    L.check(L.lib().ga_lbs_backward_ex(N, B, J, cs.ld, cs.rows, cs.mul, cs.stride, p(cs.dec), p(cs.vidx), p(cs.q), p(cs.w), p(cs.C),
                                       p(grads[0]), p(grads[1]), p(grads[2]), p(d_dec), p(dC), stream()), "ga_lbs_backward_ex")
    return [g[:B * N * 3].view(B, N, 3) for g in grads], d_dec, dC, before


@pytest.mark.parametrize("per_frame", [False, True], ids=["shared", "per_frame"])
@pytest.mark.parametrize("B", [1, 8])
@pytest.mark.parametrize("J,N", [(J, N) for J in (24, 55) for N in LBS_N[J]])
def test_lbs_launch(J, N, B, per_frame):
    """ga_lbs_forward_ex / ga_lbs_backward_ex at one size (bounds: LbsCase.forward_ref / backward_ref).  Also: sentinels past
    B N 3 (means, scales, colours), B J 12 (dC) and num_pixels rows (d_dec) are untouched; d_dec rows outside valid_index and
    column 7 are exactly 0."""
    cs = LbsCase(J, N, B, per_frame, seed=7 * N + 3 * B + J + per_frame)
    gen = cs.gen
    outs, before = lbs_forward_launch(cs, gen)
    (dm, ds, dc), d_dec, dC, (dd0, dC0) = lbs_backward_launch(cs, gen)
    torch.cuda.synchronize()
    where = cs.where
    n3 = B * N * 3
    ref = cs.forward_ref()
    for k in ("means", "scales", "colors"):
        untouched(f"{where} {k}", outs[k], before[k], 0, n3)
        check(f"lbs forward {k}", where, outs[k][:n3].view(B, N, 3), *ref[k])
    bref = cs.backward_ref(dm, ds, dc)
    untouched(f"{where} d_dec", d_dec, dd0, 0, cs.rows * 8)
    untouched(f"{where} dC", dC, dC0, 0, B * J * 12)
    got_dd = d_dec[:cs.rows * 8].view(cs.rows, 8)
    check("lbs backward d_dec", where, got_dd, *bref["d_dec"])
    got_dC = dC[:B * J * 12].view(B, J, 12)
    check("lbs backward dC", where, got_dC, *bref["dC"])

    # self-checks
    means = outs["means"][:n3].view(B, N, 3)
    mref, mb = ref["means"]
    t = None
    for back in (2, 1):       # a tile skinned with the weights of the tile `back` iterations earlier: a stale stage / wrong parity
        if cs.tiles > back * cs.grid:
            t = back * cs.grid
            rt = cs.tile_rows(t)
            ro = slice((t - back * cs.grid) * 256, (t - back * cs.grid) * 256 + (rt.stop - rt.start))
            bad = means.double().clone()
            bad[:, rt] = cs.skin(ro, rt)
            rejects(f"{where}: tile {t} skinned with the weights of {back} iterations earlier", bad, mref, mb)
    bad = means.double().clone()
    bad[:, N - 1] = before["means"][:n3].view(B, N, 3)[:, N - 1].double()
    rejects(f"{where}: the last Gaussian of the tail tile not written", bad, mref, mb)
    if B >= 2:
        rejects(f"{where}: frames 0 and 1 of cano2live swapped", cs.skin(slice(0, N), slice(0, N), [1, 0] + list(range(2, B))), mref, mb)
    # one whole tile missing from dC: the full tile whose contribution stands out most (a 1-row tail tile may be below resolution)
    full = max(N // 256, 1)
    rows = min(N, 256)
    contrib = torch.einsum("tnj,btne->tbje", cs.w[:full * rows, :J].double().view(full, rows, J),
                           cs.X[:, :full * rows].reshape(B, full, rows, 12))
    t = int((contrib.abs() / bref["dC"][1][None]).flatten(1).max(1).values.argmax())
    rejects(f"{where}: tile {t} missing from dC", got_dC.double() - contrib[t], *bref["dC"])
    bad = got_dd.double().clone()
    last = int(cs.vidx[N - 1]) + (cs.frames - 1) * cs.P
    bad[last] = 0.0
    rejects(f"{where}: the last Gaussian's d_dec row not written", bad, *bref["d_dec"])


@pytest.mark.parametrize("per_frame", [False, True], ids=["shared", "per_frame"])
@pytest.mark.parametrize("J", [24, 55])
def test_lbs_through_wrapper(J, per_frame):
    """LbsAssemble (the autograd Function the step calls) at three rounds of CTAs plus one tile, B = 8, within the same bounds."""
    from gaussianavatar_b200.ops import LbsAssemble
    B, N = 8, 3 * _round(J) + 1
    cs = LbsCase(J, N, B, per_frame, seed=J + 11 * per_frame)
    dec = cs.dec.view(-1, 8).clone().requires_grad_(True)
    C = cs.C[:B].clone().requires_grad_(True)
    means, scales, colors = LbsAssemble.apply(dec, C, cs.vidx, cs.q[:N], cs.w[:N], cs.mul, per_frame)
    gs = [torch.randn(B, N, 3, device=DEV, generator=cs.gen) for _ in range(3)]
    torch.autograd.backward([means, scales, colors], gs)
    torch.cuda.synchronize()
    where = f"wrapper {cs.where}"
    ref = cs.forward_ref()
    for k, got in (("means", means), ("scales", scales), ("colors", colors)):
        check(f"lbs forward {k}", where, got.detach(), *ref[k])
    bref = cs.backward_ref(*gs)
    check("lbs backward d_dec", where, dec.grad, *bref["d_dec"])
    check("lbs backward dC", where, C.grad, *bref["dC"])


# ==================================================================================================================== fused loss
C1F = float((torch.tensor(0.01, dtype=torch.float32) * torch.tensor(0.01, dtype=torch.float32)).item())   # 0.01f * 0.01f
C2F = float((torch.tensor(0.03, dtype=torch.float32) * torch.tensor(0.03, dtype=torch.float32)).item())   # 0.03f * 0.03f


def gauss_taps():
    """The kernel's taps (gauss_host in csrc/loss.cu): fp32 of exp(.) in double, normalised by their sequential fp32 sum in fp32."""
    f = torch.tensor([math.exp(-((i - 5) ** 2) / (2.0 * 1.5 * 1.5)) for i in range(11)], dtype=torch.float32)
    fs = torch.zeros((), dtype=torch.float32)
    for x in f:
        fs = fs + x
    return (f / fs).double()


def oracle_window_rel():
    """Largest relative difference between the oracle's fp32 11 x 11 window and the kernel's separable taps g g^T (exact)."""
    g = torch.tensor([math.exp(-(x - 5) ** 2 / float(2 * 1.5 ** 2)) for x in range(11)])
    g = (g / g.sum()).unsqueeze(1)
    w2 = g.mm(g.t()).float().double()
    k = gauss_taps()
    kk = k[:, None] * k[None, :]
    return ((w2 - kk).abs() / kk).max().item()


def blur(x, g):
    """Zero-padded separable 11-tap blur of [P, H, W] in fp64 (the window is symmetric: it is its own adjoint)."""
    k = g.to(x.device)
    y = F.conv2d(x[:, None], k.view(1, 1, 1, 11), padding=(0, 5))
    return F.conv2d(y, k.view(1, 1, 11, 1), padding=(5, 0))[:, 0]


def tile_mask(nonuni):
    """[P, H, W] bool -> [P, H, W] bool: True where the pixel's 32 x 16 tile has no True in its staged 42 x 26 support."""
    P, H, W = nonuni.shape
    ty, tx = cdiv(H, 16), cdiv(W, 32)
    pad = torch.zeros(P, ty * 16 + 10, tx * 32 + 10, dtype=torch.float64, device=nonuni.device)
    pad[:, 5:5 + H, 5:5 + W] = nonuni.double()
    I = F.pad(pad.cumsum(1).cumsum(2), (1, 0, 1, 0))
    y0 = torch.arange(ty, device=nonuni.device) * 16
    x0 = torch.arange(tx, device=nonuni.device) * 32
    cnt = I[:, y0 + 26][:, :, x0 + 42] - I[:, y0][:, :, x0 + 42] - I[:, y0 + 26][:, :, x0] + I[:, y0][:, :, x0]
    uni = cnt == 0
    return uni.repeat_interleave(16, 1).repeat_interleave(32, 2)[:, :H, :W]


def ssim_maps(a, b, g, wrel=0.0, dc1=0.0, dc2=0.0):
    """fp64 SSIM map and the three derivative maps of the forward kernel, with first-order bounds on the kernel's fp32 values.

    Moments: a horizontal and a vertical 11-FMA pass, 22 roundings on the blur of |.|, plus one for the products a a, b b, a b;
    `wrel` adds a relative window difference, dc1 / dc2 a difference of the constants.  Each intermediate of the map formulas
    (mu1 mu2, mu^2, s = xx - mu^2 (the cancellation: its error is that of xx and of mu^2, not relative to s), A, B, C, D) carries
    the propagated error of its operands plus one rounding per fp32 operation; each map adds its own operations' roundings."""
    mu1, mu2 = blur(a, g), blur(b, g)
    xx, yy, xy = blur(a * a, g), blur(b * b, g), blur(a * b, g)
    e1 = (gam(22) + wrel) * blur(a.abs(), g)
    e2 = (gam(22) + wrel) * blur(b.abs(), g)
    exx = (gam(23) + wrel) * xx
    eyy = (gam(23) + wrel) * yy
    exy = (gam(23) + wrel) * blur((a * b).abs(), g)
    mu12, m1s, m2s = mu1 * mu2, mu1 * mu1, mu2 * mu2
    s1, s2, s12 = xx - m1s, yy - m2s, xy - mu12
    A, Bv, Cc, D = 2 * mu12 + C1F, 2 * s12 + C2F, m1s + m2s + C1F, s1 + s2 + C2F
    e12 = mu2.abs() * e1 + mu1.abs() * e2 + U * mu12.abs()
    em1, em2 = 2 * mu1.abs() * e1 + U * m1s, 2 * mu2.abs() * e2 + U * m2s
    es1, es2, es12 = exx + em1 + U * s1.abs(), eyy + em2 + U * s2.abs(), exy + e12 + U * s12.abs()
    eA = 2 * e12 + U * A.abs() + dc1
    eB = 2 * es12 + U * Bv.abs() + dc2
    eC = em1 + em2 + 2 * U * Cc + dc1
    eD = es1 + es2 + 2 * U * D.abs() + dc2
    q = Cc * D
    rq = eC / Cc + eD / D + U                                       # relative error of fl(Cc D)
    out = {}
    m12 = 2 * A / q
    out["ds12"] = (m12, 2 * eA / q + m12.abs() * (rq + U))
    ms1 = -A * Bv / (q * D)
    out["ds1"] = (ms1, (eA * Bv.abs() + A.abs() * eB) / (q * D) + ms1.abs() * (rq + eD / D + 3 * U))
    T1, T2 = 2 * mu2 * Bv / q, 2 * mu2 * A / q
    T3, T4 = 2 * mu1 * A * Bv / (Cc * q), 2 * mu1 * A * Bv / (q * D)
    eT1 = 2 * (e2 * Bv.abs() + mu2.abs() * eB) / q + T1.abs() * (rq + 2 * U)
    eT2 = 2 * (e2 * A.abs() + mu2.abs() * eA) / q + T2.abs() * (rq + 2 * U)
    num = 2 * (e1 * (A * Bv).abs() + mu1.abs() * (eA * Bv.abs() + A.abs() * eB))
    eT3 = num / (Cc * q) + T3.abs() * (rq + eC / Cc + 5 * U)
    eT4 = num / (q * D) + T4.abs() * (rq + eD / D + 5 * U)
    mmu = T1 - T2 - T3 + T4
    out["dmu1"] = (mmu, eT1 + eT2 + eT3 + eT4 + gam(3) * (T1.abs() + T2.abs() + T3.abs() + T4.abs()))
    ss = A * Bv / q
    out["ssim"] = (ss, (eA * Bv.abs() + A.abs() * eB) / q + ss.abs() * (rq + 2 * U))
    return {k: (r, FO * e) for k, (r, e) in out.items()}


def f32(x):
    return torch.tensor(x, dtype=torch.float32)


def loss_coefs(g, w_l1, w_ssim, n):
    """coef[0] = (g w_l1) (float)(1/n), coef[1] = (-g w_ssim) (float)(1/n), in fp32 in the kernel's order."""
    inv = f32(1.0 / n)
    gv = f32(1.0 if g is None else g)
    return float((gv * f32(w_l1)) * inv), float((-gv * f32(w_ssim)) * inv)


MAPS = ("dmu1", "ds1", "ds12")


class LossCase:
    def __init__(self, B, H, W, img, gt, w, g):
        self.B, self.H, self.W = B, H, W
        self.n = B * 3 * H * W
        self.img, self.gt = img, gt                                  # [B, 3, H, W] fp32
        self.w = (float(f32(w[0])), float(f32(w[1])))
        self.g = None if g is None else float(f32(g))
        self.where = f"{B}x3x{H}x{W} w=({w[0]}, {w[1]}) g={'NULL' if g is None else g}"


def loss_launch(cs, gen):
    """Forward and backward through the C ABI with image / target followed by NaN and d_image / out3 inside sentinels."""
    L = _lib().lib()
    n, B, H, W = cs.n, cs.B, cs.H, cs.W
    ib, gb = nan_buf(n + PAD), nan_buf(n + PAD)
    ib[:n], gb[:n] = cs.img.reshape(-1), cs.gt.reshape(-1)
    ws = torch.empty(L.ga_loss_workspace_bytes(B, H, W), dtype=torch.uint8, device=DEV)
    out = sentinel(gen, 3 + PAD)
    dimg = sentinel(gen, n + PAD)
    gdev = None if cs.g is None else torch.full((1,), cs.g, device=DEV)
    before = (out.clone(), dimg.clone())
    _lib().check(L.ga_loss_forward(B, H, W, p(ib), p(gb), cs.w[0], cs.w[1], p(ws), p(out), stream()), "ga_loss_forward")
    maps = ws[:3 * n * 4].view(torch.float32).view(3, B * 3, H, W).clone()
    _lib().check(L.ga_loss_backward(B, H, W, p(ib), p(gb), cs.w[0], cs.w[1], p(gdev), p(ws), p(dimg), stream()), "ga_loss_backward")
    torch.cuda.synchronize()
    untouched(f"{cs.where} out3", out, before[0], 0, 3)
    untouched(f"{cs.where} d_image", dimg, before[1], 0, n)
    return maps, out[:3], dimg[:n].view(B * 3, H, W)


def loss_tier1(cs, maps, key="loss forward maps"):
    """Forward maps against ssim_maps() on the same fp32 images; tiles whose staged support has image == target: exact zeros."""
    a, b = cs.img.reshape(-1, cs.H, cs.W).double(), cs.gt.reshape(-1, cs.H, cs.W).double()
    g = gauss_taps()
    ref = ssim_maps(a, b, g)
    uni = tile_mask(a != b)
    out = {}
    for i, k in enumerate(MAPS):
        r, e = ref[k]
        r = torch.where(uni, 0.0, r)
        e = torch.where(uni, 0.0, e)
        check(key, cs.where, maps[i], r, e)
        out[k] = (r, e)
    return out, uni, a, b, g


def loss_tier2(cs, maps, a, b, g, key="loss backward (own maps)"):
    """d_img from the kernel's own maps: coef0 sign(img - gt) + coef1 (blur M0 + 2 img blur M1 + gt blur M2).

    Bound: each blur is 22 FMAs (on the blur of |M|); the products 2 img . and gt . and the two adds, 3 more; coef1 times the sum
    and the final add: gamma(25) |coef1| (blur|M0| + 2 |img| blur|M1| + |gt| blur|M2|) + 2u |coef1 S| + u |d|.
    Tiles whose three maps vanish over their staged support take the L1-only path: bit-equal to coef0 sign(img - gt)."""
    c0, c1 = loss_coefs(cs.g, cs.w[0], cs.w[1], cs.n)
    M = [m.double() for m in maps]
    S = blur(M[0], g) + 2 * a * blur(M[1], g) + b * blur(M[2], g)
    Sa = blur(M[0].abs(), g) + 2 * a.abs() * blur(M[1].abs(), g) + b.abs() * blur(M[2].abs(), g)
    sgn = torch.sign(a - b)
    d = c0 * sgn + c1 * S
    e = FO * (gam(25) * abs(c1) * Sa + 2 * U * abs(c1) * S.abs() + U * d.abs())
    zero = tile_mask((maps[0] != 0) | (maps[1] != 0) | (maps[2] != 0))
    d = torch.where(zero, c0 * sgn, d)
    e = torch.where(zero, 0.0, e)
    return d, e, zero, (c0, c1, sgn, S)


def loss_tier3(cs, uni, a, b, g):
    """d_img and out3 against oracle.avatar_oracle's ssim / l1_loss_w under fp64 autograd.

    Bound: the tier-1 map errors, recomputed with the window difference between the oracle's fp32 11 x 11 window and the
    kernel's taps and with the fp64 constants, pushed through the backward's blur, plus the tier-2 rounding, plus the window
    difference of the backward's own blur, plus the exact differences of the kernel's fp32 coefficients from g w / n.  Pixels of
    shortcut tiles carry no map error: the true maps there are (0, -1/D, 2/D), whose blurred contribution 2/D (gt - img)
    vanishes wherever it lands, because a tile's staged support covers the window of every pixel in it.
    Scalars: per-pixel SSIM / L1 errors, then a 32-lane shuffle tree (5 roundings) and a 16-warp sequential sum (15) per
    512-pixel block before the fp64 atomics: gamma(20) on the sum of |.|; the final fp32 narrowing, one more rounding."""
    from oracle import avatar_oracle as ao
    wrel = oracle_window_rel()
    ref = ssim_maps(a, b, g, wrel=wrel, dc1=abs(C1F - 0.01 ** 2), dc2=abs(C2F - 0.03 ** 2))
    n = cs.n
    w_l1, w_ssim = cs.w
    gv = 1.0 if cs.g is None else cs.g
    x = a.view(cs.B, 3, cs.H, cs.W).cpu().requires_grad_(True)       # the oracle builds its window on the CPU
    y = b.view(cs.B, 3, cs.H, cs.W).cpu()
    ss = ao.ssim(x, y)
    l1 = ao.l1_loss_w(x, y)
    loss = w_l1 * l1 + w_ssim * (1.0 - ss)
    (gv * loss).backward()
    dref = x.grad.reshape(-1, cs.H, cs.W).to(a.device)
    c0, c1 = loss_coefs(cs.g, w_l1, w_ssim, n)
    ex0, ex1 = gv * w_l1 / n, -gv * w_ssim / n
    eM = [torch.where(uni, 0.0, ref[k][1]) for k in MAPS]
    Mz = [torch.where(uni, 0.0, ref[k][0]) for k in MAPS]
    Sa = blur(Mz[0].abs(), g) + 2 * a.abs() * blur(Mz[1].abs(), g) + b.abs() * blur(Mz[2].abs(), g)
    S = blur(Mz[0], g) + 2 * a * blur(Mz[1], g) + b * blur(Mz[2], g)
    prop = blur(eM[0], g) + 2 * a.abs() * blur(eM[1], g) + b.abs() * blur(eM[2], g)
    e = FO * (abs(c1) * (prop + (gam(25) + wrel) * Sa) + 2 * U * abs(c1) * S.abs() + U * dref.abs()
              + abs(c1 - ex1) * S.abs() + abs(c0 - ex0)) + 2.0 ** -50 * (dref.abs() + abs(ex0) + abs(ex1) * Sa)
    sv, sb = ref["ssim"]
    sv = torch.where(uni, 1.0, sv)
    sb = torch.where(uni, 0.0, sb)
    s_err = (sb.sum() + gam(20) * sv.abs().sum()).item() / n + 2.0 ** -50
    l1v = (a - b).abs()
    l_err = gam(21) * l1v.sum().item() / n + 2.0 ** -50
    s_ref, l_ref = ss.item(), l1.item()
    o_ref = w_l1 * l_ref + w_ssim * (1.0 - s_ref)
    out_ref = torch.tensor([o_ref, s_ref, l_ref], dtype=torch.float64, device=DEV)
    out_b = torch.tensor([abs(w_l1) * l_err + abs(w_ssim) * s_err + U * abs(o_ref), s_err + U * abs(s_ref), l_err + U * abs(l_ref)],
                         dtype=torch.float64, device=DEV) * FO
    return (dref.detach(), e), (out_ref, out_b)


def white_figure(B, H, W, gen, frac=0.35):
    """GaussianAvatar-like frames: white background, a figure (an ellipse) where rendering and target differ."""
    yy = torch.arange(H, device=DEV, dtype=torch.float32)[:, None] / max(H - 1, 1) - 0.5
    xx = torch.arange(W, device=DEV, dtype=torch.float32)[None, :] / max(W - 1, 1) - 0.5
    fig = ((yy / frac) ** 2 + (xx / (0.6 * frac)) ** 2 <= 1.0)
    gt = torch.ones(B, 3, H, W, device=DEV)
    body = torch.rand(B, 3, H, W, device=DEV, generator=gen)
    gt = torch.where(fig, body, gt)
    img = torch.where(fig, (gt + 0.1 * torch.randn(B, 3, H, W, device=DEV, generator=gen)).clamp(0, 1), gt)
    return img.contiguous(), gt.contiguous()


def run_loss_case(cs, gen, self_checks=True):
    maps, out3, dimg = loss_launch(cs, gen)
    t1, uni, a, b, g = loss_tier1(cs, maps)
    d2, e2, zero, (c0, c1, sgn, S) = loss_tier2(cs, maps, a, b, g)
    check("loss backward (own maps)", cs.where, dimg, d2, e2)
    (d3, e3), (o3, ob) = loss_tier3(cs, uni, a, b, g)
    check("loss end to end d_img", cs.where, dimg, d3, e3)
    check("loss end to end out3", cs.where, out3, o3, ob)
    if self_checks and not bool(uni.all()):
        # one outermost tap dropped on one side of the horizontal pass: a halo staged one column short
        g1 = g.clone()
        g1[0] = 0.0
        bad = ssim_maps(a, b, g1)
        nu = ~uni
        if cs.W > 5:
            rejects(f"{cs.where}: map ds12 with one outer tap dropped", torch.where(uni, 0.0, bad["ds12"][0]), *t1["ds12"])
        bad_d = c0 * sgn + c1 * (blur(maps[0].double(), g1) + 2 * a * blur(maps[1].double(), g1) + b * blur(maps[2].double(), g1))
        if abs(c1) > 0 and cs.W > 5 and not bool(zero.all()):
            rejects(f"{cs.where}: d_img with one outer tap dropped", torch.where(zero, d2, bad_d), d2, e2)
        # one non-uniform tile given zero maps
        idx = torch.nonzero(nu)[0]
        pl, y, x = (int(v) for v in idx)
        y0, x0 = y // 16 * 16, x // 32 * 32
        bad = maps[2].double().clone()
        bad[pl, y0:y0 + 16, x0:x0 + 32] = 0.0
        rejects(f"{cs.where}: a non-uniform tile given zero maps", bad, *t1["ds12"])
    return maps, uni


LOSS_SMALL = [(1, 1, 1), (1, 5, 7), (1, 16, 32), (1, 17, 33), (3, 37, 53)]
LOSS_WEIGHTS = [(0.8, 0.2), (1.0, 0.0), (0.0, -1.0)]         # image_loss, l1_loss_w, ssim


@pytest.mark.parametrize("g", [None, 0.37], ids=["g_null", "g_dev"])
@pytest.mark.parametrize("w", LOSS_WEIGHTS, ids=["l1_ssim", "l1", "ssim"])
@pytest.mark.parametrize("B,H,W", LOSS_SMALL)
def test_loss_small(B, H, W, w, g):
    """Random images at sizes below the 11 x 11 window, one tile, one past a tile in both directions, and several ragged tiles;
    three tiers (forward maps, backward on the kernel's maps, end to end against the oracle; bounds in ssim_maps / loss_tier2 /
    loss_tier3)."""
    gen = torch.Generator(device=DEV).manual_seed(B * 1000 + H * 10 + W)
    img = torch.rand(B, 3, H, W, device=DEV, generator=gen)
    gt = torch.rand(B, 3, H, W, device=DEV, generator=gen)
    run_loss_case(LossCase(B, H, W, img, gt, w, g), gen)


@pytest.mark.parametrize("B", [2, 8])
def test_loss_training_size(B):
    """B x 1024^2, the training size: white-background frames with a figure, so both the shortcut and the full tiles run."""
    gen = torch.Generator(device=DEV).manual_seed(B)
    img, gt = white_figure(B, 1024, 1024, gen)
    _, uni = run_loss_case(LossCase(B, 1024, 1024, img, gt, (0.8, 0.2), 0.37), gen)
    assert bool(uni.any()) and not bool(uni.all())


def test_loss_white_background_borders():
    """A frame whose figure borders uniform tiles at ragged sizes (H = 16k + 1, W = 32k + 1)."""
    gen = torch.Generator(device=DEV).manual_seed(5)
    img, gt = white_figure(1, 16 * 9 + 1, 32 * 7 + 1, gen, frac=0.3)
    _, uni = run_loss_case(LossCase(1, 16 * 9 + 1, 32 * 7 + 1, img, gt, (0.8, 0.2), None), gen)
    assert bool(uni.any()) and not bool(uni.all())


@pytest.mark.parametrize("dist", [5, 6])
def test_loss_single_pixel_at_the_halo_edge(dist):
    """One differing pixel `dist` columns left of tile (1, 1) of a 48 x 96 white frame: at 5 it is inside the tile's staged support,
    which must then take the full path (its dm_ds12 ~ 2 / D is non-zero); at 6 it is outside and the tile's maps are exact zeros."""
    gen = torch.Generator(device=DEV).manual_seed(dist)
    H, W = 48, 96
    gt = torch.ones(1, 3, H, W, device=DEV)
    img = gt.clone()
    img[0, :, 20, 32 - dist] = 0.25
    maps, uni = run_loss_case(LossCase(1, H, W, img, gt, (0.8, 0.2), None), gen, self_checks=False)
    tile = maps[:, :, 16:32, 32:64]
    if dist == 5:
        assert not bool(uni[0, 20, 40]) and bool((tile[2] != 0).all())
    else:
        assert bool(uni[0, 20, 40]) and bool((tile == 0).all())


def test_loss_through_wrapper():
    """image_loss (what the step calls) forward and backward, against the end-to-end tier."""
    from gaussianavatar_b200.losses import image_loss
    gen = torch.Generator(device=DEV).manual_seed(9)
    img, gt = white_figure(2, 37 * 3, 53 * 2, gen)
    x = img.clone().requires_grad_(True)
    loss = image_loss(x, gt, 0.2)
    (0.37 * loss).backward()
    torch.cuda.synchronize()
    cs = LossCase(2, 111, 106, img, gt, (0.8, 0.2), 0.37)
    a, b, g = img.reshape(-1, 111, 106).double(), gt.reshape(-1, 111, 106).double(), gauss_taps()
    uni = tile_mask(a != b)
    (d3, e3), (o3, ob) = loss_tier3(cs, uni, a, b, g)
    check("loss end to end d_img", f"wrapper {cs.where}", x.grad.reshape(-1, 111, 106), d3, e3)
    check("loss end to end out3", f"wrapper {cs.where}", loss.detach().reshape(1), o3[:1], ob[:1])


# ========================================================================================================================== Adam
BETA1, BETA2, EPS, LR = (float(f32(v)) for v in (0.9, 0.999, 1e-8, 1e-3))


def adam_state(n, step, gen):
    """Gradients of magnitude 10^[-10, 6] (eps-dominated through large), random signs, 1 in 16 exactly 0; state of matching scale
    (zero at step 1, as torch starts it)."""
    mag = 10.0 ** (torch.rand(n, device=DEV, generator=gen) * 16 - 10)
    g = mag * torch.sign(torch.randn(n, device=DEV, generator=gen))
    g[torch.rand(n, device=DEV, generator=gen) < 1 / 16] = 0.0
    p = torch.randn(n, device=DEV, generator=gen)
    if step == 1:
        m, v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    else:
        m = 0.3 * mag * torch.randn(n, device=DEV, generator=gen)
        v = (mag * (0.2 + torch.rand(n, device=DEV, generator=gen))) ** 2
    return p, g, m, v


def adam_ref(p, g, m, v, lr, b1, b2, eps, bc1, bc2s, gs):
    """torch.optim.Adam's update in fp64 from the fp32 state: m = b1 m + (1 - b1) g', v = b2 v + (1 - b2) g'^2, g' = g gs,
    p -= (lr / bc1) m / (sqrt(v) / bc2s + eps).

    Bounds ((1 - b) is exact in fp32 for b in [1/2, 1]): m, gamma(4) (b1 |m| + (1 - b1) |g'|) (g' gs, two products, an add);
    v, gamma(6) v (g' counts twice, three products, an add).  p: one rounding of the result, plus |step| times gamma(11): lr / bc1
    (bc1 narrowed to fp32, a division: 2), the denominator (v's 6 halved by the sqrt, the sqrt, bc2s narrowed, the division, the
    + eps: 7), m / denom and the product (2); plus m's own error through (lr / bc1) / denom."""
    p, g, m, v = (t.double() for t in (p, g, m, v))
    gr = g * gs
    m1 = b1 * m + (1 - b1) * gr
    v1 = b2 * v + (1 - b2) * gr * gr
    den = v1.sqrt() / bc2s + eps
    upd = (lr / bc1) * m1 / den
    p1 = p - upd
    am = b1 * m.abs() + (1 - b1) * gr.abs()
    return {"param": (p1, gam(1) * p1.abs() + gam(11) * upd.abs() + gam(4) * (lr / bc1) * am / den),
            "exp_avg": (m1, gam(4) * am), "exp_avg_sq": (v1, gam(6) * v1)}


def adam_bufs(n, step, gen):
    p0, g, m0, v0 = adam_state(n, step, gen)
    bufs = []
    for t in (p0, m0, v0):
        b = sentinel(gen, n + PAD)
        b[:n] = t
        bufs.append(b)
    gb = nan_buf(n + PAD)
    gb[:n] = g
    return (p0, g, m0, v0), bufs, gb


def adam_check(where, bufs, before, n, ref):
    for name, b, b0 in zip(("param", "exp_avg", "exp_avg_sq"), bufs, before):
        untouched(f"{where} {name}", b, b0, 0, n)
        check(f"adam {name}", where, b[:n], *ref[name])


def bias_corrections(step):
    """As ga_adam_step forms them: 1 - b^step in double, narrowed to fp32 (the fp64 reference uses the exact values)."""
    bc1 = 1.0 - BETA1 ** step
    bc2s = math.sqrt(1.0 - BETA2 ** step)
    return bc1, bc2s, float(f32(bc1)), float(f32(bc2s))


@pytest.mark.parametrize("gs", [1.0, 0.5])
@pytest.mark.parametrize("step", [1, 2, 10000])
@pytest.mark.parametrize("n", [1, 255, 256, 257, 493_063])
def test_adam(n, step, gs):
    """ga_adam_step (host scalars) and ga_adam_step_dev (the hyper row on the device), a zero skip word given to both."""
    gen = torch.Generator(device=DEV).manual_seed(n + step + int(gs * 10))
    L = _lib()
    skip = torch.zeros(1, dtype=torch.int32, device=DEV)
    bc1, bc2s, bc1f, bc2sf = bias_corrections(step)
    where = f"n={n} step={step} grad_scale={gs}"
    (p0, g, m0, v0), bufs, gb = adam_bufs(n, step, gen)
    before = [b.clone() for b in bufs]
    L.check(L.lib().ga_adam_step(n, p(bufs[0]), p(gb), p(bufs[1]), p(bufs[2]), LR, BETA1, BETA2, EPS, step, gs, p(skip), stream()),
            "ga_adam_step")
    torch.cuda.synchronize()
    ref = adam_ref(p0, g, m0, v0, LR, BETA1, BETA2, EPS, bc1, bc2s, gs)
    adam_check(f"host {where}", bufs, before, n, ref)
    # self-checks: the update not applied; (1 - b1) and b1 swapped
    if bool((ref["param"][0] != p0.double()).any()):
        rejects(f"{where}: param not updated", p0, *ref["param"])
    if bool((m0 != 0).any() | (g != 0).any()):
        rejects(f"{where}: exp_avg with b1 and 1 - b1 swapped", (1 - BETA1) * m0.double() + BETA1 * gs * g.double(), *ref["exp_avg"])

    hyper = torch.tensor([[LR, BETA1, BETA2, EPS, bc1f, bc2sf, gs]], dtype=torch.float32, device=DEV)
    (p0, g, m0, v0), bufs, gb = adam_bufs(n, step, gen)
    before = [b.clone() for b in bufs]
    L.check(L.lib().ga_adam_step_dev(n, p(bufs[0]), p(gb), p(bufs[1]), p(bufs[2]), p(hyper), p(skip), stream()), "ga_adam_step_dev")
    torch.cuda.synchronize()
    adam_check(f"device {where}", bufs, before, n, adam_ref(p0, g, m0, v0, LR, BETA1, BETA2, EPS, bc1f, bc2sf, gs))


@pytest.mark.parametrize("n", [257, 493_063])
def test_adam_skip_word(n):
    """A non-zero skip word (the rasterizer's overflow flag) leaves parameters and both moments bit-identical, through both entries."""
    gen = torch.Generator(device=DEV).manual_seed(n)
    L = _lib()
    skip = torch.tensor([3], dtype=torch.int32, device=DEV)
    _, bufs, gb = adam_bufs(n, 2, gen)
    before = [b.clone() for b in bufs]
    hyper = torch.tensor([LR, BETA1, BETA2, EPS, 0.19, 0.0447, 1.0], dtype=torch.float32, device=DEV)
    L.check(L.lib().ga_adam_step(n, p(bufs[0]), p(gb), p(bufs[1]), p(bufs[2]), LR, BETA1, BETA2, EPS, 2, 1.0, p(skip), stream()),
            "ga_adam_step")
    L.check(L.lib().ga_adam_step_dev(n, p(bufs[0]), p(gb), p(bufs[1]), p(bufs[2]), p(hyper), p(skip), stream()), "ga_adam_step_dev")
    torch.cuda.synchronize()
    for b, b0 in zip(bufs, before):
        assert torch.equal(b.view(torch.int32), b0.view(torch.int32))


def test_adam_dev_graph_follows_hyper_row():
    """One ga_adam_step_dev launch captured in a CUDA graph; the hyper row is rewritten (lr, step 7's bias corrections, grad_scale
    0.5) after capture, and the replay must follow the new scalars."""
    n = 70_001
    gen = torch.Generator(device=DEV).manual_seed(17)
    L = _lib()
    table = torch.tensor([[LR, BETA1, BETA2, EPS, 0.1, 0.0316, 1.0], [9.0] * 7], dtype=torch.float32, device=DEV)
    skip = torch.zeros(1, dtype=torch.int32, device=DEV)
    (p0, g, m0, v0), bufs, gb = adam_bufs(n, 7, gen)
    before = [b.clone() for b in bufs]
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        L.check(L.lib().ga_adam_step_dev(n, p(bufs[0]), p(gb), p(bufs[1]), p(bufs[2]), p(table[0]), p(skip), stream()),
                "ga_adam_step_dev")
    for b, b0 in zip(bufs, before):              # capturing ran nothing
        assert torch.equal(b, b0)
    lr2 = float(f32(5e-3))
    _, _, bc1f, bc2sf = bias_corrections(7)
    table[0] = torch.tensor([lr2, BETA1, BETA2, EPS, bc1f, bc2sf, 0.5], device=DEV)
    graph.replay()
    torch.cuda.synchronize()
    adam_check("graph replay", bufs, before, n, adam_ref(p0, g, m0, v0, lr2, BETA1, BETA2, EPS, bc1f, bc2sf, 0.5))
    ref_old = adam_ref(p0, g, m0, v0, LR, BETA1, BETA2, EPS, 0.1, 0.0316, 1.0)
    rejects("a replay with the captured scalars", ref_old["param"][0], *adam_ref(p0, g, m0, v0, lr2, BETA1, BETA2, EPS, bc1f, bc2sf, 0.5)["param"])


def test_adam_through_wrapper():
    """FusedAdam (the trainer's optimiser) for two steps with grad_scale 0.5, against the fp64 restatement step by step."""
    from gaussianavatar_b200.optim import FusedAdam
    gen = torch.Generator(device=DEV).manual_seed(23)
    n = 4099
    prm = torch.nn.Parameter(torch.randn(n, device=DEV, generator=gen))
    opt = FusedAdam([prm], lr=LR, betas=(0.9, 0.999), eps=1e-8)
    opt.grad_scale = 0.5
    m = torch.zeros(n, device=DEV)
    v = torch.zeros(n, device=DEV)
    for step in (1, 2):
        g = torch.randn(n, device=DEV, generator=gen) * 10.0 ** (torch.rand(n, device=DEV, generator=gen) * 8 - 6)
        prm.grad = g.clone()
        p_old = prm.detach().clone()
        opt.step()
        torch.cuda.synchronize()
        bc1, bc2s, _, _ = bias_corrections(step)
        ref = adam_ref(p_old, g, m, v, LR, BETA1, BETA2, EPS, bc1, bc2s, 0.5)
        st = opt.state[prm]
        check("adam param", f"FusedAdam step {step}", prm.detach(), *ref["param"])
        check("adam exp_avg", f"FusedAdam step {step}", st["exp_avg"], *ref["exp_avg"])
        check("adam exp_avg_sq", f"FusedAdam step {step}", st["exp_avg_sq"], *ref["exp_avg_sq"])
        m, v = st["exp_avg"].clone(), st["exp_avg_sq"].clone()


# ============================================================================================================= joint transforms
SMPL_PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21]
SMPLX_PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 15, 15, 15, 20, 25, 26, 20, 28, 29, 20,
                 31, 32, 20, 34, 35, 20, 37, 38, 21, 40, 41, 21, 43, 44, 21, 46, 47, 21, 49, 50, 21, 52, 53]


class Rnd:
    """First-order rounding model of a per-row fp32 code path restated in fp64: every fp32 operation is x (1 + d) with d a zero
    leaf, every input known within +-e is x + d e, and the bound on an output is sum over leaves of |d out / d d| times c u (or e).
    Rows (poses x joints) are independent, so one backward pass per output component gives every row's partial derivatives."""

    def __init__(self):
        self.leaves = []

    def __call__(self, x, c=1.0):
        d = torch.zeros_like(x, requires_grad=True)
        self.leaves.append((d, c * U))
        return x * (1 + d)

    def known(self, x, e):
        d = torch.zeros_like(x, requires_grad=True)
        self.leaves.append((d, e))
        return x + d

    def bound(self, out):
        """out [rows, k] -> [rows, k] bounds."""
        cols = []
        flat = out.reshape(out.shape[0], -1)
        for k in range(flat.shape[1]):
            grads = torch.autograd.grad(flat[:, k].sum(), [d for d, _ in self.leaves], retain_graph=True, allow_unused=True)
            acc = torch.zeros(flat.shape[0], dtype=torch.float64, device=out.device)
            for gr, (d, s) in zip(grads, self.leaves):
                if gr is not None:
                    acc = acc + (gr.abs() * s).reshape(flat.shape[0], -1).sum(1)
            cols.append(acc)
        return torch.stack(cols, 1).view(out.shape)


def rod_model(r, rnd):
    """rodrigues() of csrc/smpl_math.cuh op by op: n = r + 1e-8f (the oracle's 1e-8 as a known input difference), theta = sqrtf of
    three products and two adds, d = r / theta, sincosf (within 2 ulp: c = 4), K^2 (three products, two adds), R = I + s K + (1 - c) K^2."""
    n = rnd(rnd.known(r + 1e-8, abs(E8F - 1e-8)))
    t2 = rnd(rnd(rnd(n[:, 0] * n[:, 0]) + rnd(n[:, 1] * n[:, 1])) + rnd(n[:, 2] * n[:, 2]))
    th = rnd(t2.sqrt())
    d = rnd(r / th[:, None])
    s, c = rnd(th.sin(), 4), rnd(th.cos(), 4)
    z = torch.zeros_like(d[:, 0])
    K = torch.stack([z, -d[:, 2], d[:, 1], d[:, 2], z, -d[:, 0], -d[:, 1], d[:, 0], z], 1).view(-1, 3, 3)
    K2 = rnd(rnd(rnd(K[:, :, 0, None] * K[:, None, 0, :]) + rnd(K[:, :, 1, None] * K[:, None, 1, :])) + rnd(K[:, :, 2, None] * K[:, None, 2, :]))
    I = torch.eye(3, dtype=r.dtype, device=r.device)[None]
    omc = rnd(1 - c)
    R = rnd(rnd(I + rnd(s[:, None, None] * K)) + rnd(omc[:, None, None] * K2))
    return R, (n, th, d, s, c, K, K2)


def _rod_bwd(r, gR, rnd, pair_first):
    _, (n, th, d, s, c, K, K2) = rod_model(r, rnd)
    ds = torch.zeros_like(th)
    dcm = torch.zeros_like(th)
    gRf, Kf, K2f = gR.reshape(-1, 9), K.reshape(-1, 9), K2.reshape(-1, 9)
    for i in range(9):
        ds = rnd(ds + rnd(gRf[:, i] * Kf[:, i]))
        dcm = rnd(dcm + rnd(gRf[:, i] * K2f[:, i]))
    t = torch.zeros_like(gR)
    for k in range(3):
        a, b = gR[:, :, k, None] * K[:, None, :, k], K[:, k, :, None] * gR[:, None, k, :]
        t = rnd(t + rnd(rnd(a) + rnd(b))) if pair_first else rnd(rnd(t + rnd(a)) + rnd(b))
    dK = rnd(rnd(s[:, None, None] * gR) + rnd(rnd(1 - c)[:, None, None] * t)).reshape(-1, 9)
    dd = torch.stack([rnd(dK[:, 7] - dK[:, 5]), rnd(dK[:, 2] - dK[:, 6]), rnd(dK[:, 3] - dK[:, 1])], 1)
    dth = rnd(rnd(ds * c) + rnd(dcm * s))
    dot = rnd(rnd(rnd(dd[:, 0] * r[:, 0]) + rnd(dd[:, 1] * r[:, 1])) + rnd(dd[:, 2] * r[:, 2]))
    dth = rnd(dth - rnd(dot / rnd(th * th)))
    dr = rnd(dd / th[:, None])
    return rnd(dr + rnd(rnd(dth[:, None] * n) / th[:, None]))


def rod_bwd_model(r, gR, rnd):
    """The Rodrigues backward of smpl_bwd_kernel op by op (it recomputes theta, d, s, c, K, K^2 as the forward does)."""
    return _rod_bwd(r, gR, rnd, pair_first=False)


def rodrigues_bwd_model(r, gR, rnd):
    """rodrigues_bwd() of csrc/smpl_math.cuh op by op: as rod_bwd_model, except that the d(K^2) sum adds each pair of products
    first, t += gR K^T + K^T gR, where smpl_bwd_kernel adds them one at a time."""
    return _rod_bwd(r, gR, rnd, pair_first=True)


def aff_abs(A, B):
    """|A| |B| for 3x4 affine transforms (implicit last row 0 0 0 1), on absolute values: [.., 3, 4]."""
    out = A[..., :3] @ B
    out[..., 3] = out[..., 3] + A[..., 3]
    return out


def full_pose(kind, B, J, gen):
    """Full poses [B, 3 J] fp32 of one POSES kind (or "flat_hands": random, SMPL-X hands, jaw and eyes zero) on gen's device."""
    dev, nfull = gen.device, 3 * J
    if kind == "zero":
        full = torch.zeros(B, nfull, device=dev)
    elif kind.startswith("tiny"):
        full = torch.full((B, nfull), float(kind[4:]), device=dev)
    elif kind in ("pi", "2pi"):
        axis = torch.randn(B, J, 3, device=dev, generator=gen)
        axis = axis / axis.norm(dim=-1, keepdim=True)
        full = (axis * ((1 if kind == "pi" else 2) * math.pi - 1e-3)).view(B, nfull)
    else:
        full = 0.4 * torch.randn(B, nfull, device=dev, generator=gen)
    if J == 55 and kind == "flat_hands":
        full[:, 66:] = 0.0
    return full.float()


def chain_bounds(R, eR, Jr, parents, any_order=False):
    """The global transforms G_j = G_p L_j of rotations R [B, J, 3, 3] known within eR, and bounds on their fp32 values.

    L_j = [R_j | J_j - J_p]: R_j within eR, the offset one subtraction.  Each product is three products and two adds, three adds
    for the translation, counted as gamma(4) on |G_p| |L_j|, so G_j's error is E_p |L_j| + |G_p| dL_j + gamma(4) |G_p| |L_j|.
    That holds when the kernel forms G_j from its parent's product (smpl.cu).  With any_order, |G_p| is replaced by
    |L_root| ... |L_p|, which bounds every association of the chain, e.g. chain_product's right to left (posmap.cu).
    Returns L, dL, G, EG [B, J, 3, 4] in fp64."""
    B, J = R.shape[:2]
    rel = Jr.clone()
    rel[1:] = Jr[1:] - Jr[list(parents[1:])]
    L = torch.cat([R, rel[None, :, :, None].expand(B, J, 3, 1)], -1)
    dL = torch.cat([eR, (U * rel.abs())[None, :, :, None].expand(B, J, 3, 1)], -1)
    G = [None] * J
    E = [None] * J
    P = [None] * J                                  # |G| of the association the bound assumes
    G[0], E[0], P[0] = L[:, 0], dL[:, 0], L[:, 0].abs()
    for j in range(1, J):
        pj = parents[j]
        G[j] = G[pj][..., :3] @ L[:, j]
        G[j][..., 3] = G[j][..., 3] + G[pj][..., 3]
        Pp = P[pj] if any_order else G[pj].abs()
        absG = aff_abs(Pp, L[:, j].abs())
        E[j] = aff_abs(E[pj], L[:, j].abs()) + Pp[..., :3] @ dL[:, j] + gam(4) * absG
        P[j] = absG if any_order else None
    return L, dL, torch.stack(G, 1), torch.stack(E, 1)


def rest_relative_bwd_bounds(dA, eA, Jr):
    """dG of dA [B, J, 3, 4] through A = G - pad(G_R J_j) (rest_relative): dG_R = dA_R - dA_t J^T, two roundings; dG_t = dA_t."""
    dG = dA.clone()
    dG[..., :3] = dA[..., :3] - dA[..., 3:] * Jr[None, :, None, :]
    eG = eA.clone()
    eG[..., :3] = eA[..., :3] + eA[..., 3:] * Jr.abs()[None, :, None, :] + gam(2) * (dA[..., :3].abs() + dA[..., 3:].abs() * Jr.abs()[None, :, None, :])
    return dG, eG


def reverse_walk_bounds(G, EG, L, dL, dG, eG, parents):
    """The joint chain run backwards, leaves first, restated on error bounds: dG [B, J, 3, 4] known within eG -> (dR, edR) lists of
    [B, 3, 3], one per joint.  dL_i = G_p^T dG_i (three products, two adds) takes the forward error EG of G_p and dG_i's;
    dG_p += dG_i L_i^T (four products, three adds, one accumulate: gamma(5) and u |dG_p|) takes L_i's error dL."""
    J = len(parents)
    dG = list(dG.unbind(1))
    eG = list(eG.unbind(1))
    dLR = [None] * J
    eLR = [None] * J
    for i in range(J - 1, 0, -1):
        pj = parents[i]
        GpR, EpR = G[:, pj, :, :3], EG[:, pj, :, :3]
        dLR[i] = GpR.transpose(-1, -2) @ dG[i][..., :3]
        eLR[i] = EpR.transpose(-1, -2) @ dG[i][..., :3].abs() + GpR.abs().transpose(-1, -2) @ eG[i][..., :3] \
            + gam(3) * (GpR.abs().transpose(-1, -2) @ dG[i][..., :3].abs())
        Li, dLi = L[:, i], dL[:, i]
        add = dG[i] @ Li.transpose(-1, -2)                                    # [B,3,3]
        newR = dG[pj][..., :3] + add
        eG[pj] = eG[pj].clone()
        eG[pj][..., :3] = eG[pj][..., :3] + eG[i] @ Li.abs().transpose(-1, -2) + dG[i].abs() @ dLi.transpose(-1, -2) \
            + gam(5) * (dG[i].abs() @ Li.abs().transpose(-1, -2)) + U * newR.abs()
        newt = dG[pj][..., 3] + dG[i][..., 3]
        eG[pj][..., 3] = eG[pj][..., 3] + eG[i][..., 3] + U * newt.abs()
        dG[pj] = dG[pj].clone()
        dG[pj][..., :3], dG[pj][..., 3] = newR, newt
    dLR[0], eLR[0] = dG[0][..., :3], eG[0][..., :3]
    return dLR, eLR


class BodyCase:
    def __init__(self, body, kind, B, seed):
        from gaussianavatar_b200 import synthetic as syn
        self.body, self.kind, self.B = body, kind, B
        x = body == "smplx"
        self.J = 55 if x else 24
        self.kT = 22 if x else 24
        self.parents = SMPLX_PARENTS if x else SMPL_PARENTS
        a = syn.make_avatar_assets(16, 8, seed=0, body=body)
        self.Jr = a.rest_joints.to(DEV).contiguous()
        self.inv = torch.linalg.inv(a.cano_joint_mats.double()).float().to(DEV).contiguous()
        gen = torch.Generator(device=DEV).manual_seed(seed)
        self.full = full_pose(kind, B, self.J, gen)
        self.transl = 0.3 * torch.randn(B, 3, device=DEV, generator=gen)
        self.where = f"{body} {kind} B={B}"

    # ------------------------------------------------------------------------------------------------------------ fp64 shadow
    def forward_bounds(self):
        """Bounds on the saved G and on cano2live, derived along the kinematic tree.

        L_j = [R_j | J_j - J_p]: R_j within the Rodrigues model's bound, the offset one subtraction.  G_j = G_p L_j (aff_mul: three
        products and two adds, three adds for the translation, counted as gamma(4) on |G_p| |L_j|), so its error is
        E_p |L_j| + |G_p| dL_j + gamma(4) |G_p| |L_j|: along the chain this is (depth + c) u |L_root| ... |L_j| plus each
        joint's Rodrigues error carried through its descendants.  A_t = G_t - G_R J (gamma(4)), + transl (one rounding);
        C = A inv_cano (four products, three adds: gamma(4))."""
        B, J, P = self.B, self.J, self.parents
        r = self.full.double().view(B * J, 3)
        rnd = Rnd()
        R, _ = rod_model(r.clone(), rnd)
        eR = rnd.bound(R).detach().view(B, J, 3, 3)
        R = R.detach().view(B, J, 3, 3)
        Jr = self.Jr.double()
        self.L, self.dL, self.G, self.EG = chain_bounds(R, eR, Jr, P)
        GR, Gt = self.G[..., :3], self.G[..., 3]
        A = self.G.clone()
        GJ = (GR * Jr[None, :, None, :]).sum(-1)
        A[..., 3] = Gt - GJ + self.transl.double()[:, None, :]
        EA = self.EG.clone()
        EA[..., 3] = self.EG[..., 3] + (self.EG[..., :3] * Jr.abs()[None, :, None, :]).sum(-1) + gam(4) * (Gt.abs() + (GR.abs() * Jr.abs()[None, :, None, :]).sum(-1)) \
            + U * A[..., 3].abs()
        inv = self.inv.double()
        EC = EA @ inv.abs() + gam(4) * (A.abs() @ inv.abs())
        return FO * EC.reshape(B, J, 12), FO * self.EG.reshape(B, J, 12)

    def oracle_C(self, full, transl):
        from oracle import avatar_oracle as ao
        from oracle import avatar_oracle_smplx as aox
        A = aox.joint_transforms(self.Jr.double().cpu(), full.cpu(), transl.cpu(), self.parents)
        return ao.cano2live(A, self.inv.double().cpu()[None])[:, :, :3, :].reshape(self.B, self.J, 12).to(DEV)

    def backward_bounds(self, dC):
        """d_transl = sum_j dA_t with dA = dC inv_cano^T (four products, three adds each): gamma(J + 4) on the sum of |dC| |inv_cano|^T.
        d_pose: the reverse walk restated on error bounds.  dL_i = G_p^T dG_i (three products, two adds) takes the saved G's
        forward error and dG_i's; dG_p += dG_i L_i^T (four products, three adds, one accumulate: gamma(5) and u |dG_p|) takes
        L_i's Rodrigues error; then the Rodrigues backward runs under the rounding model with dL_j as an input known within its
        bound."""
        B, J, P = self.B, self.J, self.parents
        inv = self.inv.double()
        dC = dC.double().view(B, J, 3, 4)
        dA = dC @ inv.transpose(-1, -2)
        eA = gam(4) * (dC.abs() @ inv.abs().transpose(-1, -2))
        Jr = self.Jr.double()
        dG, eG = rest_relative_bwd_bounds(dA, eA, Jr)
        dtr = dA[..., 3].sum(1)
        etr = eA[..., 3].sum(1) + gam(J) * dA[..., 3].abs().sum(1)
        dLR, eLR = reverse_walk_bounds(self.G, self.EG, self.L, self.dL, dG, eG, P)
        kT = self.kT
        gR = torch.stack(dLR[:kT], 1).reshape(B * kT, 3, 3)
        egR = torch.stack(eLR[:kT], 1).reshape(B * kT, 3, 3)
        rnd = Rnd()
        r = self.full.double().view(B, J, 3)[:, :kT].reshape(B * kT, 3)
        dr = rod_bwd_model(r, rnd.known(gR, egR), rnd)
        edr = rnd.bound(dr).detach()
        return FO * edr.view(B, 3 * kT), FO * etr


def smpl_launch(cs, fwd=True, dC=None, gen=None):
    L = _lib().lib()
    B, J, kT = cs.B, cs.J, cs.kT
    pose = nan_buf(B + 2, 3 * kT)
    pose[:B] = cs.full[:, :3 * kT]
    rest = nan_buf(B + 2, 99)
    if J == 55:
        rest[:B] = cs.full[:, 66:]
    tr = nan_buf(B + 2, 3)
    tr[:B] = cs.transl
    if fwd:
        C = sentinel(gen, B * J * 12 + PAD)
        G = sentinel(gen, B * J * 12 + PAD)
        before = (C.clone(), G.clone())
        if J == 24:
            rc = L.ga_smpl_forward(B, p(pose), p(tr), p(cs.Jr), p(cs.inv), p(C), p(G), stream())
        else:
            rc = L.ga_smplx_forward(B, p(pose), p(rest), p(tr), p(cs.Jr), p(cs.inv), p(C), p(G), stream())
        _lib().check(rc, "ga_smpl(x)_forward")
        return C, G, before
    Gs, dCb = cs.G_saved, nan_buf(B * J * 12 + PAD)
    dCb[:B * J * 12] = dC.reshape(-1)
    dp = sentinel(gen, B * 3 * kT + PAD)
    dt = sentinel(gen, B * 3 + PAD)
    before = (dp.clone(), dt.clone())
    if J == 24:
        rc = L.ga_smpl_backward(B, p(pose), p(cs.Jr), p(cs.inv), p(Gs), p(dCb), p(dp), p(dt), stream())
    else:
        rc = L.ga_smplx_backward(B, p(pose), p(rest), p(cs.Jr), p(cs.inv), p(Gs), p(dCb), p(dp), p(dt), stream())
    _lib().check(rc, "ga_smpl(x)_backward")
    return dp, dt, before


POSES = ["zero", "tiny1e-9", "tiny1e-7", "tiny1e-4", "pi", "2pi", "random"]


@pytest.mark.parametrize("B", [1, 8, 257])
@pytest.mark.parametrize("body,kind", [("smpl", k) for k in POSES] + [("smplx", k) for k in POSES] + [("smplx", "flat_hands")])
def test_joint_transforms(body, kind, B):
    """ga_smpl_* / ga_smplx_* against the oracle (fp64, autograd for the backward), bounds in BodyCase.forward_bounds /
    backward_bounds.  Poses: zero and tiny axis-angles (where the 1e-8 shift and 1 / theta dominate), angles just below pi and
    2 pi, random; SMPL-X with its rest_pose (hands, jaw, eyes) all zero."""
    cs = BodyCase(body, kind, B, seed=B + len(kind))
    gen = torch.Generator(device=DEV).manual_seed(B + 1)
    B, J, kT = cs.B, cs.J, cs.kT
    C, G, (C0, G0) = smpl_launch(cs, gen=gen)
    torch.cuda.synchronize()
    untouched(f"{cs.where} cano2live", C, C0, 0, B * J * 12)
    untouched(f"{cs.where} saved G", G, G0, 0, B * J * 12)
    eC, eG = cs.forward_bounds()
    full = cs.full.double().requires_grad_(True)
    tr = cs.transl.double().requires_grad_(True)
    Cref = cs.oracle_C(full, tr)
    check("joint transforms cano2live", cs.where, C[:B * J * 12].view(B, J, 12), Cref.detach(), eC)
    check("joint transforms saved G", cs.where, G[:B * J * 12].view(B, J, 12), cs.G.reshape(B, J, 12), eG)
    bad = C[:B * J * 12].view(B, J, 12).double().clone()
    bad[:, J - 1, 3::4] -= cs.transl.double()                        # inv_cano's last row is (0 0 0 1): transl lands in column 3
    rejects(f"{cs.where}: the last joint's translation dropped", bad, Cref.detach(), eC)

    cs.G_saved = G
    dC = torch.randn(B, J, 12, device=DEV, generator=gen)
    dp, dt, (dp0, dt0) = smpl_launch(cs, fwd=False, dC=dC, gen=gen)
    torch.cuda.synchronize()
    untouched(f"{cs.where} d_pose", dp, dp0, 0, B * 3 * kT)
    untouched(f"{cs.where} d_transl", dt, dt0, 0, B * 3)
    (Cref * dC.double()).sum().backward()
    edp, edt = cs.backward_bounds(dC)
    check("joint transforms d_pose", cs.where, dp[:B * 3 * kT].view(B, 3 * kT), full.grad[:, :3 * kT], edp)
    check("joint transforms d_transl", cs.where, dt[:B * 3].view(B, 3), tr.grad, edt)


@pytest.mark.parametrize("body", ["smpl", "smplx"])
def test_joint_transforms_through_cano2live(body):
    """Cano2Live forward and backward at B = 8 random poses of either body, within the same bounds."""
    from gaussianavatar_b200.body import body_of
    from gaussianavatar_b200.ops import Cano2Live
    cs = BodyCase(body, "random", 8, seed=31)
    gen = torch.Generator(device=DEV).manual_seed(3)
    B, J, kT = cs.B, cs.J, cs.kT
    pose = cs.full[:, :3 * kT].clone().requires_grad_(True)
    tr = cs.transl.clone().requires_grad_(True)
    b = body_of(body)
    C = Cano2Live.apply(b, pose, b.split(cs.full)[1], tr, cs.Jr, cs.inv)
    dC = torch.randn(B, J, 12, device=DEV, generator=gen)
    (C * dC).sum().backward()
    torch.cuda.synchronize()
    eC, _ = cs.forward_bounds()
    full = cs.full.double().requires_grad_(True)
    tr64 = cs.transl.double().requires_grad_(True)
    Cref = cs.oracle_C(full, tr64)
    check("joint transforms cano2live", f"wrapper {cs.where}", C.detach(), Cref.detach(), eC)
    (Cref * dC.double()).sum().backward()
    edp, edt = cs.backward_bounds(dC)
    check("joint transforms d_pose", f"wrapper {cs.where}", pose.grad, full.grad[:, :3 * kT], edp)
    check("joint transforms d_transl", f"wrapper {cs.where}", tr.grad, tr64.grad, edt)
