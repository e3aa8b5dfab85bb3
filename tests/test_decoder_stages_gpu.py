"""GPU: every launch of ga_decoder_forward / ga_decoder_backward, checked element by element against fp64 math on the
launch's own inputs, read back through ga_decoder_views.

The decoder runs once per case through the C ABI with an explicit `flags` (tensor-core TF32 or strict FP32), on a workspace
filled with NaN and with NaN in d_dec_out[:, 7], W8 row 7 and b8[7], which nothing may read. Its outputs sit inside buffers
of finite sentinels that must come back bit-identical. Then each stage's output is compared with fp64 math applied to the
buffers that stage read, so every bound stays at one launch's rounding, and the test, not decoder.cu, says which buffer
feeds which stage.

Bounds are derived before the run (u = 2^-24, fp32 unit roundoff):
  * a fp32 sum of n terms in any order, with FMA or rounded adds: n u sum|terms|; strict-FP32 GEMMs: (k per split +
    splits) u sum|a||b|;
  * TF32 MMAs (tensor-core path): operands rounded within 2^-11 each, so 2^-10 sum|a||b| on unrounded operands; each MMA
    k-step or fp32 atomic add adds 2^-23 sum|a||b| (the accumulation may truncate). Operands that are already TF32
    values (the convs' inputs) have no 2^-10 term;
  * Softplus / Sigmoid: 2^-21 (1 + x + |y a| + |b|) covers the fp32 FMA of z, __logf (abs. error 2^-21.41 on [0.5, 2]),
    __expf ((2 + 1.173 |x|) ulp) and the ex2 / lg2.approx forms; sigmoid within (5 + 1.173 |z|) 2^-23 relative;
  * an input this test has to rebuild (a buffer a later launch overwrote) carries its bound forward as |W|^T bound
    (|W| * bound for a conv). On the tensor-core path such a bound grows too wide to resolve anything after a layer
    or two, so there the overwritten layer gradients dZ5, dZ4 and dZ3 are recomputed instead by the same launches
    (ga_tc_linear_backward_ex with the decoder's arguments, wired here), each checked against fp64 from its own input;
    these launches are free of atomics, so the replayed dZ2 must equal the decoder's surviving dZ2 bit for bit, which
    pins the decoder's own layer-6..3 data-gradient launches and their wiring.
Each tier also rejects a corrupted copy of the kernel's output that a plausible bug would give (the strict path's
`rebuilt` tiers: a zeroed row or channel), with two exceptions on the strict path, which are bounded only: s1 / s2 of
layers 3 and 4, whose rebuilt bound summed over the rows is wider than the cancelling sums themselves, and dW3, whose
input gradient is rebuilt through three layers (at S = 512 its bound exceeds every row of |dW3|).
`-s` prints the largest error / bound per tier.

Which tier checks which launch:
  transpose.*     chw_to_hwc (geo), hwc_to_chw (d_geo, d_pose per frame), round_tf32 (input, weights), chw_to_hwc_add
  conv.*          geometry convs forward / dgrad / wgrad (conv_tc or the strict im2col launch_gemm)
  sample.*        sample_feat_fwd, sample_feat_bwd (texels no query touches exactly 0: stage 2, S < Hf). The stage-1
                  scatter and sum_frames write buffers a later launch overwrites: they are checked only through the
                  conv3 gradient tiers they feed (sum_frames against fp32 adds in frame order, not bit for bit)
  bn.*            BatchNorm statistics of every layer, bn_finalize_fwd (all 1408 channels, running stats), bn_finalize_bwd
  mlp.*           every MLP layer's forward launch, data-gradient and weight-gradient launch, both paths; mlp.replay
                  (tensor cores) and the strict path's `rebuilt` tiers cover the gradients of layers 5-3 as described above
  heads.*         heads_fwd, heads_bwd (dZ7, bn7 s1/s2, dW8, db8)
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NSM = 132                                  # kNumSMs: the compile-time grids (heads kernels, strict split-K) assume an H100 SXM


def runtime_sms():
    """SM count the tensor-core launches size their grids from at run time (num_sms())."""
    return torch.cuda.get_device_properties(0).multi_processor_count
U = 2.0 ** -24
TF32_OPERANDS = 2.0 ** -10 + 2.0 ** -17    # two operands rounded to TF32 (2^-11 each) and their product
KH = 128
BN_OFF = [0, 128, 256, 384, 512, 640, 1024]
MEAN, RSTD, A, B, GA, M1, M2 = range(7)
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for key, (r, where) in sorted(WORST.items()):
        print(f"\ndecoder stages: largest error/bound, {key}: {r:.3g} ({where})")


def _lib():
    from gaussianavatar_b200 import _lib
    return _lib


def tf32(t):
    i = t.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def cdiv(a, b):
    return -(-a // b)


def c_steps(steps):
    """TF32 accumulation budget in units of 2^-23 sum|a||b| (as in test_tc_launches_gpu.py)."""
    return 2 * steps + 4


# ---------------------------------------------------------------------------------------------------------- checking tools
def ratio(got, ref, bound):
    return ((got.double() - ref) / bound.clamp_min(1e-300)).abs().max().item()


def check(tier, where, got, ref, bound):
    r = ratio(got, ref, bound)
    if r == r and r > WORST.get(tier, (-1.0, ""))[0]:
        WORST[tier] = (r, where)
    assert r <= 1.0, f"{where}: {tier} error/bound {r:.4g}"


def rejects(tier, what, bad, ref, bound):
    assert ratio(bad, ref, bound) > 1.0, f"self-check: the {tier} bound accepts {what}"


def exact(tier, where, got, ref):
    assert got.dtype == ref.dtype and got.shape == ref.shape
    n = int((got.contiguous().view(torch.int32 if got.dtype == torch.float32 else torch.int64)
             != ref.contiguous().view(torch.int32 if ref.dtype == torch.float32 else torch.int64)).sum())
    if n > WORST.get(tier, (-1.0, ""))[0]:
        WORST[tier] = (float(n), where + " (elements that differ)")
    assert n == 0, f"{where}: {tier}: {n} elements differ"


def swap_worst_cols(got, ref, bound, row=-1):
    """Copy of `got` with the two columns of one row swapped whose exchange is largest relative to the bound."""
    g = got.double()
    r = g[row]
    d = (r[:, None] - r[None, :]).abs() / torch.minimum(bound[row][:, None], bound[row][None, :]).clamp_min(1e-300)
    i, j = divmod(int(d.argmax()), r.numel())
    bad = g.clone()
    bad[row, i], bad[row, j] = g[row, j], g[row, i]
    return bad


def swap_worst_rows(got, ref, bound):
    """Copy of `got` with the two rows swapped whose exchange is largest relative to the bound."""
    g = got.double()
    best, pair = -1.0, (0, 1)
    for i in range(g.shape[0]):
        d = ((g[i][None] - g).abs() / torch.minimum(bound[i][None], bound).clamp_min(1e-300)).max(1).values
        d[i] = -1
        j = int(d.argmax())
        if d[j].item() > best:
            best, pair = d[j].item(), (i, j)
    bad = g.clone()
    bad[list(pair)] = bad[list(pair[::-1])]
    return bad


def sentinel_guard(gen, n, pad=4096):
    g = torch.randn(n + 2 * pad, device=DEV, generator=gen) * 1000.0
    return g, g[pad:pad + n], g.clone(), pad


def guard_intact(where, buf, before, pad, n):
    d = buf.view(torch.int32) != before.view(torch.int32)
    d[pad:pad + n] = False
    assert int(d.sum()) == 0, f"{where}: {int(d.sum())} sentinel elements outside the output changed"


# -------------------------------------------------------------------------------------------------------- fp64 operations
def softplus_pad(Y, a, b):
    z = Y * a + b
    X = F.softplus(z)
    return X, z, 2.0 ** -21 * (1 + X + (Y * a).abs() + b.abs())


def dsigmoid(z, X, pad):
    """Bound on |sigmoid_kernel(z) - sigmoid(z)| for a kernel-evaluated z carrying Softplus pad `pad`."""
    return torch.sigmoid(-z) * (pad + 2.0 ** -21 * (1 + X)) + 2.0 ** -22


def nchw(t, P, Hf):
    return t.view(Hf, Hf, 64).permute(2, 0, 1)[None]


def hwc(t):
    return t[0].permute(1, 2, 0).reshape(-1, 64)


def w_oihw(W):
    return W.view(5, 5, 64, 64).permute(3, 2, 0, 1)


def conv_fwd(X, W, Hf):
    return hwc(F.conv2d(nchw(X, 0, Hf), w_oihw(W), padding=2))


def conv_dgrad(dY, W, Hf):
    return hwc(F.conv_transpose2d(nchw(dY, 0, Hf), w_oihw(W), padding=2))


def conv_wgrad(X, dY, Hf):
    g = torch.nn.grad.conv2d_weight(nchw(X, 0, Hf), (64, 64, 5, 5), nchw(dY, 0, Hf), padding=2)
    return g.permute(2, 3, 1, 0).reshape(25, 64, 64)


# ------------------------------------------------------------------------------------------------------------- the run
class Run:
    """One forward + backward of the decoder, with views of every workspace buffer."""

    def __init__(self, S, Hf, frames, batch, flags, pose, seed):
        L = _lib()
        lib = L.lib()
        self.S, self.Hf, self.frames, self.batch, self.flags = S, Hf, frames, batch, flags
        self.tc = bool(flags & 1)
        self.nf = max(frames, 1)
        self.M, self.P = self.nf * S * S, Hf * Hf
        self.where = f"S={S} Hf={Hf} frames={frames} {'tc' if self.tc else 'fp32'}{' pose' if pose else ''}"
        gen = torch.Generator(device=DEV).manual_seed(seed)
        self.gen = gen
        self.desc = L.GaDecoderDesc(S, Hf, batch, 64, KH, 1e-5, 0.1, flags, frames)
        lay = L.GaDecoderLayout()
        L.check(lib.ga_decoder_layout(ctypes.byref(self.desc), ctypes.byref(lay)), "ga_decoder_layout")
        self.lay = lay
        # parameters: the layers' default init scales, random BatchNorm affines, NaN in the unused head row
        prm = torch.zeros(lay.total, device=DEV)
        u = lambda n, s: (torch.rand(n, device=DEV, generator=gen) * 2 - 1) * s
        for i in range(3):
            prm[lay.gconv[i]:lay.gconv[i] + 25 * 64 * 64] = u(25 * 64 * 64, 1 / 40)
        kdim = [72, 128, 128, 128, 200, 128, 128]
        ndim = [128] * 5 + [384, 384]
        for l in range(7):
            prm[lay.w[l]:lay.w[l] + ndim[l] * kdim[l]] = u(ndim[l] * kdim[l], kdim[l] ** -0.5)
            prm[lay.b[l]:lay.b[l] + ndim[l]] = u(ndim[l], kdim[l] ** -0.5)
            prm[lay.gamma[l]:lay.gamma[l] + ndim[l]] = 1 + 0.2 * torch.randn(ndim[l], device=DEV, generator=gen)
            prm[lay.beta[l]:lay.beta[l] + ndim[l]] = 0.2 * torch.randn(ndim[l], device=DEV, generator=gen)
        prm[lay.w8:lay.w8 + 7 * KH] = u(7 * KH, KH ** -0.5)
        prm[lay.w8 + 7 * KH:lay.w8 + 8 * KH] = float("nan")
        prm[lay.b8:lay.b8 + 7] = u(7, KH ** -0.5)
        prm[lay.b8 + 7] = float("nan")
        self.prm = prm
        self.kdim, self.ndim = kdim, ndim
        self.geo = torch.randn(64, Hf, Hf, device=DEV, generator=gen)
        self.pose = 0.5 * torch.randn(self.nf, 64, Hf, Hf, device=DEV, generator=gen) if pose else None
        nbytes = lib.ga_decoder_workspace_bytes(ctypes.byref(self.desc))
        assert nbytes > 0 and nbytes % 8 == 0
        self.ws = torch.full((nbytes // 4,), float("nan"), device=DEV)
        v = L.GaDecoderViews()
        L.check(lib.ga_decoder_views(ctypes.byref(self.desc), ctypes.c_void_p(self.ws.data_ptr()), ctypes.byref(v)), "views")
        self.v = v
        M, P = self.M, self.P
        # guarded outputs
        self.g_dec = sentinel_guard(gen, M * 8)
        self.g_run = sentinel_guard(gen, 2 * 1408)
        run0 = torch.cat([0.01 * torch.randn(1408, device=DEV, generator=gen), 0.01 * (1 + torch.rand(1408, device=DEV, generator=gen))])
        self.g_run[1].copy_(run0)
        self.g_run = (self.g_run[0], self.g_run[1], self.g_run[0].clone(), self.g_run[3])
        self.run0 = run0
        self.g_dp = sentinel_guard(gen, lay.total)
        self.g_geo = sentinel_guard(gen, 64 * P)
        self.g_pose = sentinel_guard(gen, self.nf * 64 * P) if pose else None
        self.d_dec = torch.randn(M, 8, device=DEV, generator=gen)
        self.d_dec[:, 7] = float("nan")
        st = torch.cuda.current_stream().cuda_stream
        L.check(lib.ga_decoder_forward(ctypes.byref(self.desc), prm.data_ptr(), self.geo.data_ptr(),
                                       None if self.pose is None else self.pose.data_ptr(), self.g_run[1].data_ptr(),
                                       self.ws.data_ptr(), self.g_dec[1].data_ptr(), st), "ga_decoder_forward")
        L.check(lib.ga_decoder_backward(ctypes.byref(self.desc), prm.data_ptr(), self.ws.data_ptr(), self.g_dec[1].data_ptr(),
                                        self.d_dec.data_ptr(), self.g_dp[1].data_ptr(), self.g_geo[1].data_ptr(),
                                        None if self.pose is None else self.g_pose[1].data_ptr(), st), "ga_decoder_backward")
        torch.cuda.synchronize()
        for name, g in (("dec_out", self.g_dec), ("bn_running", self.g_run), ("d_params", self.g_dp), ("d_geo", self.g_geo),
                        ("d_pose_feat", self.g_pose)):
            if g is not None:
                guard_intact(f"{self.where} {name}", g[0], g[2], g[3], g[1].numel())
        self.dec = self.g_dec[1].view(M, 8)
        self.dprm = self.g_dp[1]

    def f32(self, addr, n, shape=None):
        off = addr - self.ws.data_ptr()
        assert off % 4 == 0
        t = self.ws[off // 4:off // 4 + n]
        return t.view(*shape) if shape else t

    def f64(self, addr, n):
        off = addr - self.ws.data_ptr()
        return self.ws[off // 4:off // 4 + 2 * n].view(torch.float64)

    def p(self, off, n, shape=None):
        t = self.prm[off:off + n]
        return t.view(*shape) if shape else t

    def dp(self, off, n, shape=None):
        t = self.dprm[off:off + n]
        return t.view(*shape) if shape else t


# ---------------------------------------------------------------------------------------------------- geometry convs
def conv_r(run, mode):
    """Relative rounding budget on sum|a||b| of one conv launch (operands already TF32 on the tensor-core path)."""
    P = run.P
    if run.tc:
        if mode < 2:
            return c_steps(200) * 2.0 ** -23                       # 50 steps x 4 MMAs of k = 8 per accumulator
        nchunk = cdiv(P, 32)
        nsplit = min(nchunk, runtime_sms() // 13)
        return (c_steps(4 * cdiv(nchunk, nsplit)) + nsplit) * 2.0 ** -23
    if mode < 2:
        return 1600 * U
    kps = cdiv(cdiv(P, 24), 16) * 16
    return (kps + cdiv(P, kps)) * U


def check_convs(run):
    v, Hf, P, tc, where = run.v, run.Hf, run.P, run.tc, run.where
    Fs = [run.f32(v.F[i], P * 64, (P, 64)) for i in range(4)]
    geoT = run.geo.view(64, P).t()
    exact("transpose.round", f"{where} F0", Fs[0], tf32(geoT) if tc else geoT.contiguous())
    Wp = [run.p(run.lay.gconv[i], 25 * 64 * 64, (25, 64, 64)) for i in range(3)]
    if tc:
        wr = run.f32(v.wr, 3 * 25 * 64 * 64, (3, 25, 64, 64))
        for i in range(3):
            exact("transpose.round", f"{where} wr[{i}]", wr[i], tf32(Wp[i]))
        Wu = [wr[i] for i in range(3)]
    else:
        Wu = Wp
    # forward: F[i+1] = conv(F[i]) (TF32-rounded output for i < 2 on the tensor-core path); stage 2 frames = 1 adds pose in place
    r = conv_r(run, 0)
    for i in range(3):
        X, W = Fs[i].double(), Wu[i].double()
        ref = conv_fwd(X, W, Hf)
        bound = r * conv_fwd(X.abs(), W.abs(), Hf)
        if tc and i < 2:
            bound = bound + 2.0 ** -11 * (ref.abs() + bound)
        if i == 2 and run.pose is not None and run.nf == 1:
            pz = run.pose[0].reshape(64, P).t().double()
            ref = ref + pz
            bound = bound + U * (ref.abs() + bound)
        check("conv.fwd", f"{where} conv{i + 1}", Fs[i + 1], ref, bound)
        rejects("conv.fwd", f"{where} conv{i + 1} two channels swapped", swap_worst_cols(Fs[i + 1], ref, bound), ref, bound)
    return Fs, Wu


def check_conv_bwd(run, Fs, Wu, gu, dgu):
    """gu: the up-sampling gradient the conv chain consumed (fp64), dgu its bound."""
    v, Hf, P, tc, where = run.v, run.Hf, run.P, run.tc, run.where
    lay = run.lay
    dF = [run.f32(v.dF[i], P * 64, (P, 64)) for i in range(2)]
    rw, rd = conv_r(run, 2), conv_r(run, 1)
    g, dg = gu, dgu
    # after the chain: dF[0] = gradient w.r.t. F[1], dF[1] = gradient w.r.t. F[0]; the one w.r.t. F[2] is rebuilt
    for i in (2, 1, 0):
        X = Fs[i].double()
        dW = run.dp(lay.gconv[i], 25 * 64 * 64, (25, 64, 64))
        ref = conv_wgrad(X, g, Hf)
        bound = rw * conv_wgrad(X.abs(), g.abs(), Hf) + (conv_wgrad(X.abs(), dg, Hf) if dg is not None else 0)
        ref, bound = ref.reshape(-1, 64), bound.reshape(-1, 64)
        check("conv.wgrad", f"{where} dW conv{i + 1}", dW.view(-1, 64), ref, bound)
        rejects("conv.wgrad", "two rows swapped", swap_worst_rows(dW.view(-1, 64), ref, bound), ref, bound)
        W = Wu[i].double()
        ref = conv_dgrad(g, W, Hf)
        bound = rd * conv_dgrad(g.abs(), W.abs(), Hf) + (conv_dgrad(dg, W.abs(), Hf) if dg is not None else 0)
        if tc and i > 0:
            bound = bound + 2.0 ** -11 * (ref.abs() + bound)
        if i == 2:
            g, dg = ref, bound                                     # overwritten: carried forward with its bound
            continue
        got = dF[0] if i == 1 else dF[1]
        check("conv.dgrad", f"{where} d conv{i + 1} input", got, ref, bound)
        rejects("conv.dgrad", "two channels swapped", swap_worst_cols(got, ref, bound), ref, bound)
        g, dg = got.double(), None
    exact("transpose.round", f"{where} d_geo", run.g_geo[1].view(64, P), dF[1].t().contiguous())


# -------------------------------------------------------------------------------------------------------- up-sampling
def ratio_grid(S):
    """i / (S - 1) rounded once to fp32, as the kernel's IEEE division gives it (torch divides by a scalar through its
    reciprocal, which is not correctly rounded)."""
    return (torch.arange(S, device=DEV, dtype=torch.float64) / (S - 1)).float()


def taps(S, Hf, fma):
    """fp32 bilinear tap positions of F.grid_sample(align_corners=False) in torch's op order; fma=True: the product
    (g+1)*Hf - 1 contracted into one rounding, as a compiler may emit it."""
    u = ratio_grid(S)
    g1 = (u * 2.0 - 1.0) + 1.0
    if fma:
        t = (g1.double() * Hf - 1.0).float()
    else:
        t = g1 * float(Hf) - 1.0
    pos = t / 2.0
    f = torch.floor(pos)
    return f.long(), pos - f


def bilinear_ops(S, Hf):
    """Per (variant): list of 4 (flat texel index [S*S], weight [S*S] fp64, valid mask)."""
    out = []
    for fma in (False, True):
        x0, wx = taps(S, Hf, fma)
        taps4 = []
        for dy in (0, 1):
            for dx in (0, 1):
                y = x0[:, None] + dy
                x = x0[None, :] + dx
                wy_ = (wx if dy else 1.0 - wx)[:, None]
                wx_ = (wx if dx else 1.0 - wx)[None, :]
                w = (wx_ * wy_).double()                          # fp32 product, as the kernel forms it
                ok = (x >= 0) & (x < Hf) & (y >= 0) & (y < Hf)
                taps4.append(((y.clamp(0, Hf - 1) * Hf + x.clamp(0, Hf - 1)).reshape(-1), (w * ok).reshape(-1), ok.reshape(-1)))
        out.append(taps4)
    return out


def check_sample_fwd(run, Fsrc):
    """Fsrc: [nf][P,64] the maps the up-sampling read."""
    S, Hf, where, M = run.S, run.Hf, run.where, run.M
    feat = run.f32(run.v.feat, M * 72, (M, 72))
    ii = ratio_grid(S)
    uv = torch.stack([ii[:, None].expand(S, S), ii[None, :].expand(S, S)], -1).reshape(S * S, 2)
    for f in range(run.nf):
        rows = feat[f * S * S:(f + 1) * S * S]
        exact("sample.fwd uv", f"{where} frame {f} uv", rows[:, 64:66].contiguous(), uv)
        exact("sample.fwd uv", f"{where} frame {f} pad", rows[:, 66:72].contiguous(), torch.zeros(S * S, 6, device=DEV))
        Fm = Fsrc[f]
        if Hf == S:
            exact("sample.fwd copy", f"{where} frame {f}", rows[:, :64].contiguous(), Fm)
            continue
        refs, bounds = [], []
        for taps4 in bilinear_ops(S, Hf):
            ref = 0
            mag = 0
            for t, w, ok in taps4:
                vals = Fm[t].double() * ok[:, None]
                ref = ref + w[:, None] * vals
                mag = mag + (w[:, None] * vals).abs()
            refs.append(ref)
            bounds.append(4 * U * mag)                             # 4 FMAs into o; w is exact (the taps' own fp32 product)
        ref = refs[0]
        bound = torch.maximum(bounds[0], bounds[1]) + (refs[0] - refs[1]).abs()
        got = rows[:, :64]
        check("sample.fwd", f"{where} frame {f}", got, ref, bound)
        # one bilinear tap dropped for the pixel where it matters most
        t, w, ok = bilinear_ops(S, Hf)[0][3]
        contrib = (w[:, None] * Fm[t].double() * ok[:, None]).abs() / bound.clamp_min(1e-300)
        m = int(contrib.max(1).values.argmax())
        bad = got.double().clone()
        bad[m] -= w[m] * Fm[t[m]].double() * ok[m]
        rejects("sample.fwd", "one tap dropped", bad, ref, bound)
        # the reference's own grid (fp64 F.grid_sample on the same maps); the tap positions there are exact, ours are fp32,
        # so the difference is bounded by how far a fp32 position can move per axis (six roundings: 2^-22 (Hf + 1)) times
        # the map's slope along it (at most 2 max|F| per texel), on both axes
        from oracle.avatar_oracle import upsample_features
        ref2 = upsample_features(Fm.double().t().reshape(1, 64, Hf, Hf).cpu(), S)[0].reshape(64, -1).t().to(DEV)
        wide = bound + 2 * 2.0 ** -22 * (Hf + 1) * 2 * Fm.abs().max().double()
        check("sample.fwd grid_sample", f"{where} frame {f}", got, ref2, wide)
        rejects("sample.fwd grid_sample", "one tap dropped", bad, ref2, wide)


def scatter_ref(run, d_feat):
    """fp64 transpose of the up-sampling applied to d_feat [S*S, 64] (one frame), and its bound."""
    S, Hf, P = run.S, run.Hf, run.P
    if Hf == S:
        return d_feat.double(), torch.zeros(P, 64, dtype=torch.float64, device=DEV), None
    ops = bilinear_ops(S, Hf)
    outs, mags = [], []
    cnt = torch.zeros(P, dtype=torch.float64, device=DEV)
    for k, taps4 in enumerate(ops):
        ref = torch.zeros(P, 64, dtype=torch.float64, device=DEV)
        mag = torch.zeros(P, 64, dtype=torch.float64, device=DEV)
        for t, w, ok in taps4:
            c = w[:, None] * d_feat.double()
            ref.index_add_(0, t, c)
            mag.index_add_(0, t, c.abs())
            if k == 0:
                cnt.index_add_(0, t, ok.double())
        outs.append(ref)
        mags.append(mag)
    n = cnt.max().item()
    bound = (n + 1) * U * torch.maximum(mags[0], mags[1]) + (outs[0] - outs[1]).abs()   # product + n atomic adds
    return outs[0], bound, cnt


def check_sample_bwd(run, got, f):
    """got [P,64]: the up-sampling gradient of frame f the kernel wrote (observable)."""
    S, M = run.S, run.M
    d_feat = run.f32(run.v.d_feat, M * 72, (M, 72))[f * S * S:(f + 1) * S * S, :64]
    ref, bound, cnt = scatter_ref(run, d_feat)
    where = f"{run.where} frame {f}"
    if cnt is None:
        exact("sample.bwd copy", where, got.contiguous(), d_feat.contiguous())
        return
    check("sample.bwd", where, got, ref, bound)
    untouched = cnt == 0
    if bool(untouched.any()):
        exact("sample.bwd untouched", where, got[untouched].contiguous(), torch.zeros(int(untouched.sum()), 64, device=DEV))
    # one query's contribution dropped from the texel where it matters most
    t, w, ok = bilinear_ops(S, run.Hf)[0][0]
    c = w[:, None] * d_feat.double()
    m = int((c.abs() / bound[t].clamp_min(1e-300)).max(1).values.argmax())
    bad = got.double().clone()
    bad[t[m]] -= c[m]
    rejects("sample.bwd", "one query dropped", bad, ref, bound)


# ------------------------------------------------------------------------------------------------------------ BatchNorm
def check_bn_fwd(run):
    where, M = run.where, run.M
    stat = run.f64(run.v.stat, 4 * 1408).view(4, 1408)
    coef = run.f32(run.v.coef, 7 * 1408, (7, 1408))
    lay = run.lay
    gamma = torch.cat([run.p(lay.gamma[l], run.ndim[l]) for l in range(7)]).double()
    beta = torch.cat([run.p(lay.beta[l], run.ndim[l]) for l in range(7)]).double()
    n, cr = float(M), float(run.S * run.S * run.batch)
    mu = stat[0] / n
    var = (stat[1] / n - mu * mu).clamp_min(0)
    dvar = 2.0 ** -51 * (stat[1] / n + mu * mu)                    # double division, product and difference
    eps = float(torch.tensor(1e-5, dtype=torch.float32))
    rs = 1 / torch.sqrt(var + eps)
    mean_g, rs_g, a_g, b_g = coef[MEAN].double(), coef[RSTD].double(), coef[A].double(), coef[B].double()
    tiers = [("mean", coef[MEAN], mu, U * mu.abs() * (1 + 2.0 ** -20)),
             ("rstd", coef[RSTD], rs, U * rs * (1 + 2.0 ** -20) + 0.5 * rs * dvar / (var + eps)),
             ("a", coef[A], gamma * rs_g, U * (gamma * rs_g).abs()),
             ("b", coef[B], beta - mean_g * a_g, U * ((mean_g * a_g).abs() + (beta - mean_g * a_g).abs()))]
    c1 = float(torch.tensor(1.0 - torch.tensor(0.1, dtype=torch.float32).item(), dtype=torch.float32))
    mom = float(torch.tensor(0.1, dtype=torch.float32))
    run_g = run.g_run[1].view(2, 1408)
    rm0, rv0 = run.run0.view(2, 1408).double()
    rm_ref = c1 * rm0 + mom * mean_g
    vu = var * cr / (cr - 1)
    rv_ref = c1 * rv0 + mom * vu
    tiers.append(("running mean", run_g[0], rm_ref, U * (2 * (c1 * rm0).abs() + 2 * (mom * mean_g).abs() + rm_ref.abs())))
    rv_bound = U * (2 * (c1 * rv0).abs() + 2 * mom * vu + rv_ref.abs()) + mom * (U * vu + dvar * cr / (cr - 1))
    tiers.append(("running var", run_g[1], rv_ref, rv_bound))
    for name, got, ref, bound in tiers:
        check("bn.finalize_fwd", f"{where} {name}", got[None], ref[None], bound[None])
        c = int(((ref[:-1] - ref[1:]).abs() / torch.minimum(bound[:-1], bound[1:]).clamp_min(1e-300)).argmax())
        bad = got.double().clone()
        bad[[c, c + 1]] = bad[[c + 1, c]]
        rejects("bn.finalize_fwd", f"{name} two channels swapped", bad[None], ref[None], bound[None])
    biased = c1 * rv0 + mom * var
    rejects("bn.finalize_fwd", "running var with count_running in place of count_running - 1", biased[None], rv_ref[None], rv_bound[None])


def check_bn_bwd(run):
    where, M = run.where, run.M
    stat = run.f64(run.v.stat, 4 * 1408).view(4, 1408)
    coef = run.f32(run.v.coef, 7 * 1408, (7, 1408))
    lay = run.lay
    gamma = torch.cat([run.p(lay.gamma[l], run.ndim[l]) for l in range(7)])
    dgamma = torch.cat([run.dp(lay.gamma[l], run.ndim[l]) for l in range(7)])
    dbeta = torch.cat([run.dp(lay.beta[l], run.ndim[l]) for l in range(7)])
    exact("bn.finalize_bwd", f"{where} ga", coef[GA], gamma * coef[RSTD])
    exact("bn.finalize_bwd", f"{where} m1", coef[M1], (stat[2] / float(M)).float())
    exact("bn.finalize_bwd", f"{where} m2", coef[M2], (stat[3] / float(M)).float())
    exact("bn.finalize_bwd", f"{where} d_gamma", dgamma, stat[3].float())
    exact("bn.finalize_bwd", f"{where} d_beta", dbeta, stat[2].float())
    for l in range(7):
        z = run.dp(lay.b[l], run.ndim[l])
        assert torch.count_nonzero(z).item() == 0, f"{where}: d bias of layer {l + 1} (before BatchNorm) must be 0"


def check_stats(run, l, Yg, c0=0):
    stat = run.f64(run.v.stat, 4 * 1408).view(4, 1408)
    Y = Yg.double()
    o = BN_OFF[l] + c0
    n = Y.shape[1]
    for k, (ref, mag) in enumerate(((Y.sum(0), Y.abs().sum(0)), ((Y * Y).sum(0), (Y * Y).sum(0)))):
        bound = 2.0 ** -19 * mag + 1e-12
        check("bn.stats", f"{run.where} layer {l + 1} {'sum' if k == 0 else 'sumsq'}", stat[k, o:o + n][None], ref[None], bound[None])
        bad = stat[k, o:o + n].clone()
        bad[[0, 1]] = bad[[1, 0]]
        rejects("bn.stats", "two channels swapped", bad[None], ref[None], bound[None])


def check_s12(run, l, dZ, dZb, Yp, c0=0):
    """s1 / s2 of BatchNorm layer l (0-based) from its pre-BN gradient dZ (fp64) with per-element bound dZb (or None)."""
    stat = run.f64(run.v.stat, 4 * 1408).view(4, 1408)
    coef = run.f32(run.v.coef, 7 * 1408, (7, 1408)).double()
    o = BN_OFF[l] + c0
    n = dZ.shape[1]
    a, b, mu, rs = (coef[k, o:o + n] for k in (A, B, MEAN, RSTD))
    X, z, pad = softplus_pad(Yp.double(), a, b)
    sig = torch.sigmoid(z)
    dsig = dsigmoid(z, X, pad)
    xhat = (Yp.double() - mu) * rs
    t = dZ
    # s2: the tensor-core kernels recover xhat from the stored Softplus through lg2.approx(sigmoid) (test_tc_launches_gpu.py)
    dxh = (rs / a).abs() * (pad + dsig / sig + 2.0 ** -21 * (1 + torch.log(sig).abs() + X + b.abs() + (mu * a).abs()))
    e1 = 2.0 ** -19 * t.abs().sum(0) + 1e-12
    e2 = (t.abs() * dxh).sum(0) + 2.0 ** -19 * (t * xhat).abs().sum(0) + 1e-12
    tier = "bn.s1s2"
    if dZb is not None:
        # strict path, rebuilt gradient: the corrupted copy zeroes the channel the carried bound resolves best. For layers
        # 3 and 4 (gradient carried through two or three layers) the summed bound exceeds |s1| itself, since s1 cancels
        # over the rows: there the tier bounds the error only, with no corrupted copy
        e1 = e1 + dZb.sum(0)
        e2 = e2 + (dZb * xhat.abs()).sum(0)
        tier = "bn.s1s2 rebuilt"
    where = f"{run.where} layer {l + 1}"
    for name, got, ref, bound in (("s1", stat[2, o:o + n], t.sum(0), e1), ("s2", stat[3, o:o + n], (t * xhat).sum(0), e2)):
        check(tier, f"{where} {name}", got[None], ref[None], bound[None])
        if dZb is not None:
            if l < 4:
                continue
            bad = got.double().clone()
            bad[int((ref.abs() / bound).argmax())] = 0
            rejects(tier, f"{name} one channel zeroed", bad[None], ref[None], bound[None])
            continue
        c = int((ref - ref.roll(1)).abs().div(bound).argmax())
        bad = got.double().clone()
        bad[[c, c - 1]] = bad[[c - 1, c]]
        rejects(tier, f"{name} two channels swapped", bad[None], ref[None], bound[None])


# ------------------------------------------------------------------------------------------------------------------- MLP
def r_fwd(run, K):
    return TF32_OPERANDS + c_steps(16) * 2.0 ** -23 if run.tc else K * U


def r_wgrad(run, split):
    M = run.M
    if run.tc:
        tiles = cdiv(M, 32)
        grid = min(tiles, runtime_sms())
        return TF32_OPERANDS + (c_steps(4 * cdiv(tiles, grid)) + grid) * 2.0 ** -23
    splits = 2 * NSM // split
    kps = cdiv(cdiv(M, splits), 16) * 16
    return (kps + cdiv(M, kps)) * U


class Layers:
    """Kernel activations of the MLP and the layer inputs built from them (fp64)."""

    def __init__(self, run):
        self.run = run
        v, M = run.v, run.M
        self.feat = run.f32(v.feat, M * 72, (M, 72))
        self.Y = [run.f32(v.Y[i], M * KH, (M, KH)) for i in range(5)] + [run.f32(v.Y6, M * 384, (M, 384)),
                                                                         run.f32(v.Y7, M * 384, (M, 384))]
        self.coef = run.f32(v.coef, 7 * 1408, (7, 1408))

    def ab(self, l, c0=0, n=KH):
        o = BN_OFF[l] + c0
        return self.coef[A, o:o + n].double(), self.coef[B, o:o + n].double()

    def act(self, l, c0=0):
        """Softplus(BN(Y_l)) of layer l (0-based) columns c0..c0+128, with its evaluation pad."""
        a, b = self.ab(l, c0)
        X, z, pad = softplus_pad(self.Y[l][:, c0:c0 + KH].double(), a, b)
        return X, z, pad

    def W(self, l):
        r = self.run
        return r.p(r.lay.w[l], r.ndim[l] * r.kdim[l], (r.ndim[l], r.kdim[l])).double()

    def bias(self, l):
        r = self.run
        return r.p(r.lay.b[l], r.ndim[l]).double()


def check_mlp_fwd(run, Ls):
    where = run.where
    feat = Ls.feat.double()
    for l in range(7):
        W = Ls.W(l)
        heads = range(3) if l == 6 else [None]
        for h in heads:
            if l == 0:
                Ain, pad, part1 = feat, None, None
            elif l == 4:
                X4, _, pad4 = Ls.act(3)
                Ain = torch.cat([feat, X4], 1)
                pad = torch.cat([torch.zeros_like(feat), pad4], 1)
            elif l == 6:
                Ain, _, pad = Ls.act(5, 128 * h)
            else:
                Ain, _, pad = Ls.act(l - 1)
            Wl = W[128 * h:128 * h + 128] if h is not None else W
            bias = Ls.bias(l)[128 * h:128 * h + 128] if h is not None else Ls.bias(l)
            ref = Ain @ Wl.t() + bias
            bound = r_fwd(run, Wl.shape[1]) * (Ain.abs() @ Wl.abs().t())
            if pad is not None:
                bound = bound + 1.01 * (pad @ Wl.abs().t())
            extra = (feat @ Wl[:, :72].t()).abs() if l == 4 else 0     # layer 5's stored feature part, added once more
            bound = bound + 2.0 ** -22 * (bias.abs() + ref.abs() + extra)
            got = Ls.Y[l] if h is None else Ls.Y[l][:, 128 * h:128 * h + 128]
            name = f"{where} layer {l + 1}" + (f" head {h}" if h is not None else "")
            check("mlp.fwd", name, got, ref, bound)
            rejects("mlp.fwd", f"{name} two channels swapped", swap_worst_cols(got, ref, bound), ref, bound)
            check_stats(run, l, got, 128 * h if h is not None else 0)
            del Ain, ref, bound


def bn_grad(Ls, l, dZ, dZb, c0=0, n=KH):
    """G = BN backward of layer l applied to dZ (as the loaders do), its on-load rounding pad and propagated bound."""
    o = BN_OFF[l] + c0
    ga, m1, m2, mu, rs = (Ls.coef[k, o:o + n].double() for k in (GA, M1, M2, MEAN, RSTD))
    Y = Ls.Y[l][:, c0:c0 + n].double()
    k = rs * m2
    G = ga * (dZ - m1 - (Y - mu) * k)
    padG = 2.0 ** -21 * ((ga * dZ).abs() + (ga * k * Y).abs() + ga.abs() * ((k * mu).abs() + m1.abs()))
    dG = ga.abs() * dZb if dZb is not None else None
    return G, padG, dG


def dgrad(run, G, padG, dG, W, r):
    ref = G @ W
    bound = r * (G.abs() @ W.abs()) + 1.01 * (padG @ W.abs())
    if dG is not None:
        bound = bound + dG @ W.abs()
    return ref, bound


def through_sigmoid(Ls, lp, c0, Sref, Sb):
    a, b = Ls.ab(lp, c0)
    X, z, pad = softplus_pad(Ls.Y[lp][:, c0:c0 + KH].double(), a, b)
    sig = torch.sigmoid(z)
    return Sref * sig, Sb * sig + Sref.abs() * dsigmoid(z, X, pad) + 2.0 ** -22 * Sref.abs()


def wgrad_check(run, Ls, name, got, G, padG, dG, Xin, padX, r, teeth=True):
    ref = G.t() @ Xin
    bound = r * (G.abs().t() @ Xin.abs()) + 1.01 * (padG.t() @ Xin.abs())
    if padX is not None:
        bound = bound + 1.01 * (G.abs().t() @ padX)
    if dG is not None:                                             # strict path: input gradient rebuilt through earlier layers
        rebuilt_check("mlp.wgrad rebuilt", name, got, ref, bound + dG.t() @ Xin.abs(), teeth)
        return
    check("mlp.wgrad", name, got, ref, bound)
    rejects("mlp.wgrad", f"{name} two rows swapped", swap_worst_rows(got, ref, bound), ref, bound)


def replay_tc(run, Ls):
    """The tensor-core path's overwritten layer gradients dZ5, dZ4, dZ3 and dZ2, recomputed by the same launches
    (ga_tc_linear_backward_ex, the decoder's arguments, wired by this test) from the decoder's own dZ6 and coefficients.
    These data-gradient launches have no atomics (one CTA owns a tile; the layer-6 heads add in launch order), so the
    replay is bit-identical to what the decoder computed if the decoder wired the same buffers: dZ2 is compared bit for bit
    with the decoder's surviving copy, and each replayed launch is checked against fp64 from its own input."""
    L, M, lay = _lib(), run.M, run.lay
    lib, st = L.lib(), torch.cuda.current_stream().cuda_stream
    coef = Ls.coef

    def bc(o):
        return torch.stack([coef[k, o:o + KH] for k in (GA, M1, M2, MEAN, RSTD)]).contiguous()

    def pc(o):
        return torch.stack([coef[k, o:o + KH] for k in (A, B, MEAN, RSTD)]).contiguous()

    s12 = torch.zeros(2, KH, dtype=torch.float64, device=DEV)
    dWs = torch.zeros(KH, 200, device=DEV)                         # scratch: the weight gradients are the decoder's to check

    keep = []                                                      # coefficient copies must outlive the asynchronous launches

    def launch(dZ, ldg, Y, o, Yp, op, w_off, ldw, out, mode):
        keep.extend((bc(o), pc(op)))
        rc = lib.ga_tc_linear_backward_ex(M, dZ.data_ptr(), Y.data_ptr(), ldg, keep[-2].data_ptr(), Yp.data_ptr(), KH, keep[-1].data_ptr(),
                                          run.prm[w_off:].data_ptr(), ldw, dWs[:, 72:].data_ptr(), 200, out.data_ptr(), KH, mode, s12[0].data_ptr(), s12[1].data_ptr(), KH, 0, st)
        L.check(rc, "ga_tc_linear_backward_ex")

    dZ6 = run.f32(run.v.dZ6, M * 384, (M, 384))
    out = {}
    dZ5 = torch.full((M, KH), float("nan"), device=DEV)
    for h in range(3):                                             # layer 6 heads: modes 1, 2, 3 into one dZ5
        launch(dZ6[:, 128 * h:], 384, Ls.Y[5][:, 128 * h:], BN_OFF[5] + 128 * h, Ls.Y[4], BN_OFF[4], lay.w[5] + 128 * h * KH, KH, dZ5, h + 1)
    out[5] = dZ5
    launch(dZ5, KH, Ls.Y[4], BN_OFF[4], Ls.Y[3], BN_OFF[3], lay.w[4] + 72, 200, out.setdefault(4, torch.full((M, KH), float("nan"), device=DEV)), 0)
    for l in (3, 2):                                               # layers 4, 3: dZ4 -> dZ3 -> dZ2
        out[l] = torch.full((M, KH), float("nan"), device=DEV)
        launch(out[l + 1], KH, Ls.Y[l], BN_OFF[l], Ls.Y[l - 1], BN_OFF[l - 1], lay.w[l], KH, out[l], 0)
    torch.cuda.synchronize()
    return out


def rebuilt_check(tier, where, got, ref, bound, teeth=True):
    """A strict-FP32 output checked against a rebuilt reference: rejects a zeroed row (the one the bound resolves best)."""
    check(tier, where, got, ref, bound)
    if not teeth:
        return
    r = int((ref.abs() / bound.clamp_min(1e-300)).max(1).values.argmax())
    bad = got.double().clone()
    bad[r] = 0
    rejects(tier, f"{where} one row zeroed", bad, ref, bound)


def check_mlp_bwd(run, Ls):
    where, M, v = run.where, run.M, run.v
    lay = run.lay
    dZ7 = run.f32(v.dZ7, M * 384, (M, 384))
    dZ6 = run.f32(v.dZ6, M * 384, (M, 384))
    dZa = run.f32(v.dZa, M * KH, (M, KH))
    dZb = run.f32(v.dZb, M * KH, (M, KH))
    d_feat = run.f32(v.d_feat, M * 72, (M, 72))
    feat = Ls.feat.double()
    rd = TF32_OPERANDS + c_steps(16) * 2.0 ** -23 if run.tc else None
    rep = replay_tc(run, Ls) if run.tc else None

    def carried(n, ref, bound):
        """Layer-n gradient dZ_n (overwritten in the decoder): on the tensor-core path the replayed launch's output, checked
        against fp64 from its own input and then used as the next layer's input; on the strict path the fp64 rebuild with its
        bound carried forward."""
        if rep is None:
            return ref, bound
        check("mlp.dgrad", f"{where} dZ{n} (replayed launch)", rep[n], ref, bound)
        rejects("mlp.dgrad", "two channels swapped", swap_worst_cols(rep[n], ref, bound), ref, bound)
        return rep[n].double(), None

    # layer 7 (per head): dZ7 -> dZ6[:, h], dW7[h]
    W7 = Ls.W(6)
    dW7 = run.dp(lay.w[6], 384 * KH, (384, KH))
    for h in range(3):
        c = slice(128 * h, 128 * h + 128)
        G, padG, _ = bn_grad(Ls, 6, dZ7[:, c].double(), None, 128 * h)
        S, Sb = dgrad(run, G, padG, None, W7[c], rd or 128 * U)
        ref, bound = through_sigmoid(Ls, 5, 128 * h, S, Sb)
        check("mlp.dgrad", f"{where} dZ6 head {h}", dZ6[:, c], ref, bound)
        rejects("mlp.dgrad", "two channels swapped", swap_worst_cols(dZ6[:, c], ref, bound), ref, bound)
        X6, _, pad6 = Ls.act(5, 128 * h)
        wgrad_check(run, Ls, f"{where} dW7 head {h}", dW7[c], G, padG, None, X6, pad6, r_wgrad(run, 1))
        check_s12(run, 5, dZ6[:, c].double(), None, Ls.Y[5][:, c], 128 * h)
    # layer 6: dZ6 -> dZ5 (overwritten later), dW6
    G6, padG6, _ = bn_grad(Ls, 5, dZ6.double(), None, 0, 384)
    W6 = Ls.W(5)
    r6 = (rd + 2 * 2.0 ** -22) if run.tc else 384 * U             # tensor cores: three head launches, two reduce-adds
    S, Sb = dgrad(run, G6, padG6, None, W6, r6)
    dZ5, dZ5b = carried(5, *through_sigmoid(Ls, 4, 0, S, Sb))
    X5, _, pad5 = Ls.act(4)
    wgrad_check(run, Ls, f"{where} dW6", run.dp(lay.w[5], 384 * KH, (384, KH)), G6, padG6, None, X5, pad5, r_wgrad(run, 2))
    check_s12(run, 4, dZ5, dZ5b, Ls.Y[4])
    del G6, padG6, S, Sb
    # layer 5: dZ5 -> d_feat (feature part), dZ4 (overwritten), dW5
    W5 = Ls.W(4)
    G5, padG5, dG5 = bn_grad(Ls, 4, dZ5, dZ5b)
    Sf, Sfb = dgrad(run, G5, padG5, dG5, W5[:, :72], rd or 128 * U)
    S, Sb = dgrad(run, G5, padG5, dG5, W5[:, 72:], rd or 128 * U)
    dZ, dZbnd = carried(4, *through_sigmoid(Ls, 3, 0, S, Sb))
    X4, _, pad4 = Ls.act(3)
    Xin = torch.cat([feat, X4], 1)
    padX = torch.cat([torch.zeros_like(feat), pad4], 1)
    wgrad_check(run, Ls, f"{where} dW5", run.dp(lay.w[4], KH * 200, (KH, 200)), G5, padG5, dG5, Xin, padX, r_wgrad(run, 2))
    check_s12(run, 3, dZ, dZbnd, Ls.Y[3])
    del G5, padG5, dG5, S, Sb, Xin, padX, dZ5, dZ5b
    # layers 4, 3, 2: dZ4 -> dZ3 (overwritten) -> dZ2 (survives in dZb) -> dZ1 (survives in dZa)
    for l in (3, 2, 1):
        G, padG, dG = bn_grad(Ls, l, dZ, dZbnd)
        S, Sb = dgrad(run, G, padG, dG, Ls.W(l), rd or 128 * U)
        nref, nb = through_sigmoid(Ls, l - 1, 0, S, Sb)
        Xp, _, padp = Ls.act(l - 1)
        wgrad_check(run, Ls, f"{where} dW{l + 1}", run.dp(lay.w[l], KH * KH, (KH, KH)), G, padG, dG, Xp, padp, r_wgrad(run, 1),
                    teeth=l > 2)
        if l == 3:
            dZ, dZbnd = carried(3, nref, nb)
            check_s12(run, 2, dZ, dZbnd, Ls.Y[2])
        elif l == 2:                                               # dZ2 survives in dZb: check it, then continue from it
            if rep is not None:
                exact("mlp.replay", f"{where} dZ2 (decoder vs replayed launches)", dZb, rep[2])
                check("mlp.dgrad", f"{where} dZ2", dZb, nref, nb)
                rejects("mlp.dgrad", "two channels swapped", swap_worst_cols(dZb, nref, nb), nref, nb)
            else:
                rebuilt_check("mlp.dgrad rebuilt", f"{where} dZ2", dZb, nref, nb)
            dZ, dZbnd = dZb.double(), None
            check_s12(run, 1, dZ, None, Ls.Y[1])
        else:
            check("mlp.dgrad", f"{where} dZ1", dZa, nref, nb)
            rejects("mlp.dgrad", "two channels swapped", swap_worst_cols(dZa, nref, nb), nref, nb)
            check_s12(run, 0, dZa.double(), None, Ls.Y[0])
        del G, padG, S, Sb, Xp, padp
    del rep
    # layer 1: dZ1 -> d_feat (added to layer 5's feature part), dW1
    G1, padG1, _ = bn_grad(Ls, 0, dZa.double(), None)
    S1, S1b = dgrad(run, G1, padG1, None, Ls.W(0), rd or 128 * U)
    ref = Sf + S1
    bound = Sfb + S1b + 2.0 ** -22 * (Sf.abs() + S1.abs() + ref.abs())
    check("mlp.dgrad", f"{where} d_feat", d_feat, ref, bound)
    bad = d_feat.double().clone()
    bad[:, 64:72] = 0
    rejects("mlp.dgrad", "d_feat channels 64-71 zeroed", bad, ref, bound)
    wgrad_check(run, Ls, f"{where} dW1", run.dp(lay.w[0], KH * 72, (KH, 72)), G1, padG1, None, feat, None, r_wgrad(run, 1))


# ---------------------------------------------------------------------------------------------------------------- heads
def check_heads(run, Ls):
    where, M, lay = run.where, run.M, run.lay
    dec = run.dec
    W8 = run.p(lay.w8, 8 * KH, (8, KH)).double()[:7]
    b8 = run.p(lay.b8, 8).double()[:7]
    rows = [(0, 3), (3, 4), (4, 7)]
    a7, b7 = Ls.ab(6, 0, 384)
    Y7 = Ls.Y[6].double()
    X7, z7, pad7 = softplus_pad(Y7, a7, b7)
    # forward: 4 FMAs per lane, 5 shuffle-add levels, the bias add
    pre = torch.zeros(M, 7, dtype=torch.float64, device=DEV)
    preb = torch.zeros_like(pre)
    for h, (r0, r1) in enumerate(rows):
        c = slice(128 * h, 128 * h + 128)
        pre[:, r0:r1] = X7[:, c] @ W8[r0:r1].t()
        preb[:, r0:r1] = 10 * U * (X7[:, c].abs() @ W8[r0:r1].abs().t()) + 1.01 * (pad7[:, c] @ W8[r0:r1].abs().t())
    pre = pre + b8
    preb = preb + U * (b8.abs() + pre.abs())
    sg = torch.sigmoid(pre)
    ref = torch.cat([pre[:, :3], sg[:, 3:]], 1)
    bound = torch.cat([preb[:, :3], sg[:, 3:] * (1 - sg[:, 3:]) * preb[:, 3:] + 2.0 ** -21 * sg[:, 3:]], 1)
    check("heads.fwd", f"{where} dec", dec[:, :7], ref, bound)
    exact("heads.fwd", f"{where} dec column 7", dec[:, 7].contiguous(), torch.zeros(M, device=DEV))
    bad = dec[:, :7].double().clone()
    bad[M - 1] = 0
    rejects("heads.fwd", "the last tail pixel zeroed", bad, ref, bound)
    del pre, preb, sg, ref, bound
    # backward: dZ7, s1 / s2 of bn7, dW8, db8
    dZ7 = run.f32(run.v.dZ7, M * 384, (M, 384))
    stat = run.f64(run.v.stat, 4 * 1408).view(4, 1408)
    coef = Ls.coef.double()
    mu7, rs7 = coef[MEAN, 1024:], coef[RSTD, 1024:]
    depth = cdiv(M, 2 * NSM * 8)                                   # pixels per warp of the grid-stride loop
    sig = torch.sigmoid(z7)
    dsig = sig * (torch.sigmoid(-z7) * U * z7.abs() + 2.0 ** -23 * (5 + 1.173 * z7.abs()))
    dW8 = run.dp(lay.w8, 8 * KH, (8, KH))
    db8 = run.dp(lay.b8, 8)
    assert torch.count_nonzero(dW8[7]).item() == 0 and db8[7].item() == 0, f"{where}: dW8 / db8 row 7 written"
    for h, (r0, r1) in enumerate(rows):
        c = slice(128 * h, 128 * h + 128)
        g = run.d_dec[:, r0:r1].double()
        if h == 0:
            dp, ddp = g, torch.zeros_like(g)
        else:
            s = dec[:, r0:r1].double()
            dp = g * s * (1 - s)
            ddp = 2.0 ** -22 * dp.abs()
        Wh = W8[r0:r1]
        dx = dp @ Wh
        dxb = 3 * U * (dp.abs() @ Wh.abs()) + ddp @ Wh.abs()
        ref = dx * sig[:, c]
        bound = dxb * sig[:, c] + dx.abs() * dsig[:, c] + U * ref.abs()
        got = dZ7[:, c]
        check("heads.bwd", f"{where} dZ7 head {h}", got, ref, bound)
        bad = got.double().clone()
        bad[M - 1] = 0
        rejects("heads.bwd", "the last tail pixel zeroed", bad, ref, bound)
        nd = depth + 8 + 2 * NSM                                   # per-lane sums, 8 warps in shared memory, one atomic per CTA
        Xh = X7[:, c]
        refw = dp.t() @ Xh
        bw = nd * U * (dp.abs().t() @ Xh.abs()) + ddp.t() @ Xh.abs() + 1.01 * (dp.abs().t() @ pad7[:, c])
        check("heads.bwd dW8", f"{where} dW8 head {h}", dW8[r0:r1], refw, bw)
        rejects("heads.bwd dW8", "two channels swapped", swap_worst_cols(dW8[r0:r1], refw, bw), refw, bw)
        refb = dp.sum(0)
        bb = nd * U * dp.abs().sum(0) + ddp.sum(0)
        check("heads.bwd dW8", f"{where} db8 head {h}", db8[r0:r1][None], refb[None], bb[None])
        rejects("heads.bwd dW8", "db8 of the first pixel only", dp[0][None], refb[None], bb[None])
        t = got.double()
        xhat = (Y7[:, c] - mu7[c]) * rs7[c]
        ns = depth + 8
        for name, sv, r, bd in (("s1", stat[2, 1024 + 128 * h:1152 + 128 * h], t.sum(0), ns * U * t.abs().sum(0)),
                                ("s2", stat[3, 1024 + 128 * h:1152 + 128 * h], (t * xhat).sum(0), (ns + 2) * U * (t * xhat).abs().sum(0))):
            check("heads.bwd s1s2", f"{where} bn7 head {h} {name}", sv[None], r[None], bd[None] + 1e-12)
            bad = sv.clone()
            bad[[0, 1]] = bad[[1, 0]]
            rejects("heads.bwd s1s2", "two channels swapped", bad[None], r[None], bd[None] + 1e-12)


# ------------------------------------------------------------------------------------------------------------------ cases
def run_case(S, Hf, frames, batch, flags, pose, seed):
    run = Run(S, Hf, frames, batch, flags, pose, seed)
    v, P, nf, where = run.v, run.P, run.nf, run.where
    Fs, Wu = check_convs(run)
    # the maps the up-sampling read: conv3's output, or conv3 + each frame's pose map
    if pose and nf > 1:
        Fp = run.f32(v.Fp, nf * P * 64, (nf, P, 64))
        for f in range(nf):
            exact("transpose.add", f"{where} Fp frame {f}", Fp[f], Fs[3] + run.pose[f].reshape(64, P).t())
        bad = Fp.clone()
        bad[[0, 1]] = bad[[1, 0]]
        assert not torch.equal(bad[0], Fs[3] + run.pose[0].reshape(64, P).t()), "self-check: frame swap undetected"
        Fsrc = [Fp[f] for f in range(nf)]
    else:
        Fsrc = [Fs[3]]
    check_sample_fwd(run, Fsrc)
    Ls = Layers(run)
    check_bn_fwd(run)
    check_mlp_fwd(run, Ls)
    check_heads(run, Ls)
    check_bn_bwd(run)
    check_mlp_bwd(run, Ls)
    del Ls
    # up-sampling gradient: observable per frame in stage 2 (dFp / d_pose_feat), rebuilt from d_feat in stage 1
    if pose:
        dpose = run.g_pose[1].view(nf, 64, P)
        if nf > 1:
            dFp = run.f32(v.dFp, nf * P * 64, (nf, P, 64))
            for f in range(nf):
                exact("transpose.round", f"{where} d_pose frame {f}", dpose[f], dFp[f].t().contiguous())
            ups = [dFp[f] for f in range(nf)]
        else:
            ups = [dpose[0].t()]
        for f in range(nf):
            check_sample_bwd(run, ups[f], f)
        gsum = ups[0].clone()
        for f in range(1, nf):
            gsum = gsum + ups[f]                                   # sum_frames: fp32 adds in frame order
        gu = (tf32(gsum) if run.tc else gsum).double()
        dgu = None
        if nf > 1:                                                 # a dropped frame must not pass the conv3 weight-gradient tier
            X = Fs[2].double()
            dropped = conv_wgrad(X, (tf32(gsum - ups[-1]) if run.tc else gsum - ups[-1]).double(), Hf)
            ref = conv_wgrad(X, gu, run.Hf)
            bound = conv_r(run, 2) * conv_wgrad(X.abs(), gu.abs(), run.Hf)
            rejects("conv.wgrad", "sum_frames with the last frame dropped", dropped.reshape(-1, 64), ref.reshape(-1, 64), bound.reshape(-1, 64))
    else:
        M = run.M
        d_feat = run.f32(v.d_feat, M * 72, (M, 72))[:, :64]
        gu, dgu, cnt = scatter_ref(run, d_feat)
        if cnt is None:                                            # copy branch: the gradient is d_feat itself
            gu, dgu = (tf32(d_feat) if run.tc else d_feat).double(), None
        elif run.tc:                                               # rounded to TF32 in place before the convs read it
            dgu = dgu + 2.0 ** -11 * (gu.abs() + dgu)
    check_conv_bwd(run, Fs, Wu, gu, dgu)
    del run
    torch.cuda.empty_cache()


TC, FP32 = 1, 0
STAGE1_TC = [(512, 128, 2), (2, 1, 1), (46, 5, 1), (66, 33, 1), (92, 128, 1), (128, 128, 1)]
STAGE2_TC = [(512, 128, 2), (128, 128, 1), (92, 40, 8), (92, 128, 2)]      # the last one leaves texels no query touches
STRICT = [(512, 128, 0, 2, False), (512, 128, 2, 2, True), (66, 33, 0, 1, False), (92, 128, 0, 1, False)]


@pytest.mark.parametrize("S,Hf,batch", STAGE1_TC)
def test_stage1_tensor_cores(S, Hf, batch):
    run_case(S, Hf, 0, batch, TC, False, seed=S * 1000 + Hf)


@pytest.mark.parametrize("S,Hf,frames", STAGE2_TC)
def test_stage2_tensor_cores(S, Hf, frames):
    run_case(S, Hf, frames, frames, TC, True, seed=S * 1000 + Hf + 7 * frames)


@pytest.mark.parametrize("S,Hf,frames,batch,pose", STRICT)
def test_strict_fp32(S, Hf, frames, batch, pose):
    run_case(S, Hf, frames, batch, FP32, pose, seed=S * 1000 + Hf + 3)
