"""GPU: every tensor-core decoder-layer launch that csrc/decoder.cu makes, checked element by element against fp64.

FWD / BWD list the launches of ga_tc_linear_forward / ga_tc_linear_backward_ex with the leading dimensions, pointer offsets, modes
and input widths the decoder passes. Each runs at the pixel counts where tiling goes wrong: one row, a partial tile, exact
tiles, one row past a tile, one tile past a full round of 132 CTAs (an H100 SXM), and the config-3 decoder size.

Every output element must satisfy |got - ref| <= bound in each tier that applies:
  a-priori  ref = fp64 math on the unrounded operands, bound = 2^-10 (|A| |B|) + eps. TF32 keeps each operand within 2^-11
            relative, so a correct kernel cannot exceed it. eps covers the fp32 parts: accumulation, the kernel's own fp32
            operand transforms (BatchNorm FMAs, Softplus from ex2 / lg2.approx), sigmoid and the epilogue adds.
  tight     only where the kernel's TF32 operands are exactly tf32(input): raw X, bwd_coef NULL, x_raw.
            ref = fp64 math on tf32-rounded operands, bound = c 2^-23 (|A^| |B^|) + eps, with c = 2 per sequential
            fp32 accumulation step (wgmma k-step or atomic add) + 4.
Each output sits inside a larger buffer filled with finite sentinels, which must be bit-identical afterwards. Input elements
the kernel must not read (other heads' columns, rows at or past M) are NaN. The per-launch tests also corrupt a copy of the
output (one product term dropped, two pixels swapped, channels 64-71 zeroed) and assert that the same bounds reject it.
The chain tests enqueue launches back to back on one stream as the decoder does.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu, pytest.mark.tf32]
DEV = "cuda:0"
NSM = 132                                   # H100 SXM: the M lists below put one tile past a full round of CTAs
PAD = 70                                    # spare rows past M in every buffer (more than one tile)
FWD_M = [1, 63, 64, 65, NSM * 64 + 1]       # forward tiles are 64 pixels
BWD_M = [1, 31, 32, 33, NSM * 32 + 1]       # backward tiles are 32 pixels
BIG_M = 262144                              # config-3 decoder: ~62 tiles per CTA, the mbarrier parities wrap many times

# id: X width (ldx) and K, BatchNorm + Softplus on X, W buffer (rows, cols = ldw, first column), bias, Y width (ldy), accumulate,
# statistics.  A 384-wide X / Y, or a 384-row W, is a head buffer: the launch uses head h's 128 columns / rows, h = M % 3 (so
# that the M list reaches every head).
FWD = {
    "F1": dict(ldx=72, K=72, act=False, w=(128, 72, 0), bias=True, ldy=128, acc=False, stats=True),       # layer 1
    "F2": dict(ldx=128, K=128, act=True, w=(128, 128, 0), bias=True, ldy=128, acc=False, stats=True),     # layers 2-4
    "F3": dict(ldx=72, K=72, act=False, w=(128, 200, 0), bias=False, ldy=128, acc=False, stats=False),    # layer 5, feature part
    "F4": dict(ldx=128, K=128, act=True, w=(128, 200, 72), bias=True, ldy=128, acc=True, stats=True),     # layer 5, x4 part on top
    "F5": dict(ldx=128, K=128, act=True, w=(384, 128, 0), bias=True, ldy=384, acc=False, stats=True),     # layer 6 head h
    "F6": dict(ldx=384, K=128, act=True, w=(384, 128, 0), bias=True, ldy=384, acc=False, stats=True),     # layer 7 head h
}
# id: dZ_l / Y_l width (ldg), Y_{l-1} width (ldp), W / dW buffer (rows, cols = ldw = lddw, first column), dZ_{l-1} width (ldo),
# mode, kin, x_raw, and the head for rows whose head is fixed by the mode (layer 6: h = 0, 1, 2 run modes 1, 2, 3)
BWD = {
    "B1": dict(ldg=384, ldp=384, w=(384, 128, 0), ldo=384, mode=0, kin=128, raw=False),               # layer 7 head h
    "B2.1": dict(ldg=384, ldp=128, w=(384, 128, 0), ldo=128, mode=1, kin=128, raw=False, h=0),        # layer 6 heads
    "B2.2": dict(ldg=384, ldp=128, w=(384, 128, 0), ldo=128, mode=2, kin=128, raw=False, h=1),
    "B2.3": dict(ldg=384, ldp=128, w=(384, 128, 0), ldo=128, mode=3, kin=128, raw=False, h=2),
    "B3": dict(ldg=128, ldp=128, w=(128, 200, 72), ldo=128, mode=0, kin=128, raw=False),              # layer 5, x4 part
    "B4": dict(ldg=128, ldp=72, w=(128, 200, 0), ldo=72, mode=1, kin=72, raw=True),                   # layer 5, feature part
    "B5": dict(ldg=128, ldp=128, w=(128, 128, 0), ldo=128, mode=0, kin=128, raw=False),               # layers 4-2
    "B6": dict(ldg=128, ldp=72, w=(128, 72, 0), ldo=72, mode=2, kin=72, raw=True),                    # layer 1
}

WORST = {}                                  # tier and output kind -> (largest error / bound, where)


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for key, (r, where) in sorted(WORST.items()):
        print(f"\ntc launches: largest error/bound, {key}: {r:.3g} ({where})")


def _lib():
    from gaussianavatar_b200 import _lib
    return _lib


def tf32(t):
    """fp32 -> tf32 as the kernels round (to_tf32 adds half a TF32 ulp, the tensor cores drop the low 13 bits)."""
    i = t.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def c_steps(steps):
    """Rounding budget, in units of 2^-23 |A| |B|, of `steps` sequential fp32 accumulation steps."""
    return 2 * steps + 4


def apriori(steps):
    return 2.0 ** -10 + 2.0 ** -17 + c_steps(steps) * 2.0 ** -23


def ratio(got, ref, bound):
    return ((got.double() - ref) / bound.clamp_min(1e-300)).abs().max().item()   # NaN in got -> NaN -> fails every `<= 1`


def check(where, got, tiers):
    for tier, (ref, bound) in tiers.items():
        r = ratio(got, ref, bound)
        key = f"{tier} tier, {'dW' if 'dW' in where else 'data outputs'}"
        if r == r and r > WORST.get(key, (-1.0, ""))[0]:
            WORST[key] = (r, where)
        assert r <= 1.0, f"{where}: {tier} error/bound {r:.4g}"


def rejects(where, bad, tiers):
    for tier, (ref, bound) in tiers.items():
        assert ratio(bad, ref, bound) > 1.0, f"self-check: the {tier} bound accepts a corrupted {where}"


def untouched(where, after, before, M, c0, c1, r0=0, r1=None):
    """Every element outside rows [r0, r1 or M) x columns [c0, c1) is bit-identical to `before`."""
    diff = after.view(torch.int32) != before.view(torch.int32)
    diff[r0:(M if r1 is None else r1), c0:c1] = False
    n = int(diff.sum())
    assert n == 0, f"{where}: {n} elements outside the owned region changed"


def rand(gen, *shape):
    return torch.randn(*shape, device=DEV, generator=gen)


def nan_buf(rows, cols):
    return torch.full((rows, cols), float("nan"), device=DEV)


def sentinel(gen, rows, cols):
    return rand(gen, rows, cols) * 1000.0


def stream():
    return torch.cuda.current_stream().cuda_stream


def p(t):
    return None if t is None else t.data_ptr()


def sum_terms(tiers_list):
    """Tiers of a sum of independently bounded parts (only the tiers every part has)."""
    keys = set.intersection(*(set(t) for t in tiers_list))
    return {k: (sum(t[k][0] for t in tiers_list), sum(t[k][1] for t in tiers_list)) for k in keys}


# ---------------------------------------------------------------------------------------------------------------------- forward
def fwd_launch(M, K, X, a, b, W, ldw, bias, Y, acc, s):
    L = _lib()
    L.check(L.lib().ga_tc_linear_forward(M, K, p(X), X.stride(0), p(a), p(b), p(W), ldw, p(bias), p(Y), Y.stride(0), int(acc),
                                         p(None if s is None else s[0]), p(None if s is None else s[1]), stream()),
            "ga_tc_linear_forward")


def fwd_product(X, act, a, b, W):
    """Tiers of act(X) W^T (M x 128) plus the fp64 operands; X: [M][K] fp32, W: [128][K]."""
    X64, W64 = X.double(), W.double()
    if act:
        A = F.softplus(X64 * a.double() + b.double())
        pad = 2.0 ** -21 * (1 + A + (X64 * a.double()).abs() + b.double().abs())   # the kernel's fp32 FMA + ex2 / lg2.approx
    else:
        A, pad = X64, None
    ba = apriori(16) * (A.abs() @ W64.abs().t())
    if pad is not None:
        ba = ba + 1.01 * (pad @ W64.abs().t())
    tiers = {"a-priori": (A @ W64.t(), ba)}
    if not act:
        Ah, Wh = tf32(X).double(), tf32(W).double()
        tiers["tight"] = (Ah @ Wh.t(), c_steps(16) * 2.0 ** -23 * (Ah.abs() @ Wh.abs().t()))
    return tiers, A, W64


def with_epilogue(tiers, add, add_abs):
    """Y = product + add (bias, existing Y) with two fp32 roundings."""
    out = {}
    for k, (ref, bound) in tiers.items():
        r = ref + add
        out[k] = (r, bound + 2.0 ** -22 * (add_abs + r.abs()))
    return out


def fwd_operands(spec, M, h, gen):
    K, ldx = spec["K"], spec["ldx"]
    xo = 128 * h if ldx == 384 else 0
    Xb = nan_buf(M + PAD, ldx)
    Xb[:M, xo:xo + K] = rand(gen, M, K)
    co = xo if spec["act"] else 0
    a = (1 + 0.2 * rand(gen, 384)) if spec["act"] else None
    b = 0.3 * rand(gen, 384) if spec["act"] else None
    wr, wc, w0 = spec["w"]
    Wb = rand(gen, wr, wc) / K ** 0.5
    r0 = 128 * h if wr == 384 else 0
    return Xb, xo, (a[co:co + K] if a is not None else None), (b[co:co + K] if b is not None else None), Wb, Wb[r0:r0 + 128, w0:w0 + K]


def stats_check(where, s, Yo):
    """Per-channel fp32 partial sums of 16 pixels per thread, then fp64: within 2^-19 of the fp64 sums of the stored output."""
    Y64 = Yo.double()
    assert bool(((s[0] - Y64.sum(0)).abs() <= 2.0 ** -19 * Y64.abs().sum(0) + 1e-12).all()), f"{where}: sum"
    assert bool(((s[1] - (Y64 ** 2).sum(0)).abs() <= 2.0 ** -19 * (Y64 ** 2).sum(0) + 1e-12).all()), f"{where}: sumsq"


def drop_term(out, r, A, B, bound, scale=None):
    """Copy of `out` with the largest (relative to the bound) single product term A[r, k] B[k, j] of row r removed."""
    T = A[r][:, None] * B                                   # [K][n]
    if scale is not None:
        T = T * scale[r][None, :]
    k = T.abs().argmax(0)
    j = int((T.abs().max(0).values / bound[r]).argmax())
    bad = out.double().clone()
    bad[r, j] -= T[int(k[j]), j]
    return bad


@pytest.mark.parametrize("row,M", [(r, m) for r in FWD for m in FWD_M] + [("F1", BIG_M)])
def test_forward_launch(row, M):
    spec = FWD[row]
    h = M % 3                                               # head buffers: every head is hit across the M list
    gen = torch.Generator(device=DEV).manual_seed(1000 * M + int(row[1:]))
    Xb, xo, a, b, Wb, W = fwd_operands(spec, M, h, gen)
    K, ldy = spec["K"], spec["ldy"]
    yo = 128 * h if ldy == 384 else 0
    bias = rand(gen, 128) if spec["bias"] else None
    Yb = sentinel(gen, M + PAD, ldy)
    if spec["acc"]:
        Yb[:M, yo:yo + 128] = rand(gen, M, 128)
    Y0 = Yb[:M, yo:yo + 128].clone() if spec["acc"] else None
    before = Yb.clone()
    s = torch.zeros(2, 128, dtype=torch.float64, device=DEV) if spec["stats"] else None
    X = Xb[:M, xo:xo + K]
    fwd_launch(M, K, Xb[:, xo:], a, b, W, Wb.stride(0), bias, Yb[:, yo:], spec["acc"], s)
    torch.cuda.synchronize()

    where = f"{row} M={M} h={h}"
    untouched(where, Yb, before, M, yo, yo + 128)
    got = Yb[:M, yo:yo + 128]
    prod, A, W64 = fwd_product(X, spec["act"], a, b, W)
    add = torch.zeros((), dtype=torch.float64, device=DEV)
    add_abs = torch.zeros((), dtype=torch.float64, device=DEV)
    for t in (bias, Y0):
        if t is not None:
            add, add_abs = add + t.double(), add_abs + t.double().abs()
    tiers = with_epilogue(prod, add, add_abs)
    check(where, got, tiers)
    if spec["stats"]:
        stats_check(where, s, got)

    # the bounds see one wrong term in the last (ragged) tile, two swapped pixels
    bound_a = tiers["a-priori"][1]
    rejects(f"{where} (term dropped)", drop_term(got, M - 1, A, W64.t(), bound_a), tiers)
    if M >= 2:
        sw = got.double().clone()
        sw[[M - 1, M - 2]] = sw[[M - 2, M - 1]]
        rejects(f"{where} (pixels swapped)", sw, tiers)


@pytest.mark.parametrize("M", [1, 65, NSM * 64 + 1])
def test_forward_layer5_chain(M):
    """Layer 5 as the decoder enqueues it: K = 72 raw features, then the x4 part accumulating on top, no synchronisation between."""
    gen = torch.Generator(device=DEV).manual_seed(M + 55)
    feat = nan_buf(M + PAD, 72)
    feat[:M] = rand(gen, M, 72)
    Y4 = nan_buf(M + PAD, 128)
    Y4[:M] = rand(gen, M, 128)
    a4, b4 = 1 + 0.2 * rand(gen, 128), 0.3 * rand(gen, 128)
    W5 = rand(gen, 128, 200) / 200 ** 0.5
    b5 = rand(gen, 128)
    Y5 = sentinel(gen, M + PAD, 128)
    before = Y5.clone()
    s = torch.zeros(2, 128, dtype=torch.float64, device=DEV)
    fwd_launch(M, 72, feat, None, None, W5, 200, None, Y5, 0, None)
    fwd_launch(M, 128, Y4, a4, b4, W5[:, 72:], 200, b5, Y5, 1, s)
    torch.cuda.synchronize()

    where = f"F3+F4 M={M}"
    untouched(where, Y5, before, M, 0, 128)
    p1, _, _ = fwd_product(feat[:M], False, None, None, W5[:, :72])
    p2, _, _ = fwd_product(Y4[:M], True, a4, b4, W5[:, 72:])
    part1 = p1["a-priori"][0]
    # F3's stored Y5 is added to F4's accumulator: one more rounding of |F3 part|
    tiers = with_epilogue(sum_terms([p1, p2]), b5.double(), b5.double().abs() + part1.abs())
    check(where, Y5[:M], tiers)
    stats_check(where, s, Y5[:M])


# --------------------------------------------------------------------------------------------------------------------- backward
def bwd_launch(M, dZ, Yl, bc, Yp, pc, W, dW, O, mode, s, kin, raw):
    L = _lib()
    return L.lib().ga_tc_linear_backward_ex(M, p(dZ), p(Yl), dZ.stride(0), p(bc), p(Yp), Yp.stride(0), p(pc), p(W), W.stride(0), p(dW),
                                            dW.stride(0), p(O), O.stride(0), mode, p(None if s is None else s[0]),
                                            p(None if s is None else s[1]), kin, int(raw), stream())


def bwd_coefs(gen, bn, raw):
    bc = torch.stack([1 + 0.2 * rand(gen, 128), 0.1 * rand(gen, 128), 0.1 * rand(gen, 128), 0.1 * rand(gen, 128),
                      1 + 0.1 * torch.rand(128, device=DEV, generator=gen)]).contiguous() if bn else None
    pc = None if raw else torch.stack([1 + 0.2 * rand(gen, 128), 0.3 * rand(gen, 128), 0.1 * rand(gen, 128),
                                       1 + 0.1 * torch.rand(128, device=DEV, generator=gen)]).contiguous()
    return bc, pc


class Bwd:
    """fp64 expectations of one backward launch: dX = G W (M x kin), dW += G^T X (128 x kin), sigmoid(z) for the final modes."""

    def __init__(self, dZ, Yl, bc, Yp, pc, W, M):
        kin = W.shape[1]
        dZ64 = dZ.double()
        if bc is not None:
            ga, m1, m2, mu, rstd = bc.double()
            k = rstd * m2
            self.G = ga * (dZ64 - m1 - (Yl.double() - mu) * k)
            self.padG = 2.0 ** -21 * ((ga * dZ64).abs() + (ga * k * Yl.double()).abs() + ga.abs() * ((k * mu).abs() + m1.abs()))
        else:
            self.G, self.padG = dZ64, None
        Yp64 = Yp.double()
        if pc is None:
            self.X, self.padX, self.z = Yp64, None, None
        else:
            pa, pb, pmu, prstd = (c[:kin] for c in pc.double())
            self.z = Yp64 * pa + pb
            self.X = F.softplus(self.z)
            self.padX = 2.0 ** -21 * (1 + self.X + (Yp64 * pa).abs() + pb.abs())
            self.xhat = (Yp64 - pmu) * prstd
            self.invg = prstd / pa
            self.stat_pad = pb.abs() + (pmu * pa).abs()
        self.W = W.double()
        Gt = self.G.abs()
        tiers = {"a-priori": (self.G @ self.W, apriori(16) * (Gt @ self.W.abs()))}
        if self.padG is not None:
            tiers["a-priori"] = (tiers["a-priori"][0], tiers["a-priori"][1] + 1.01 * (self.padG @ self.W.abs()))
        else:
            Gh, Wh = tf32(dZ).double(), tf32(W).double()
            tiers["tight"] = (Gh @ Wh, c_steps(16) * 2.0 ** -23 * (Gh.abs() @ Wh.abs()))
        self.dx = tiers
        # weight gradient: 4 k-steps per tile over a CTA's tiles in registers, then one atomic add per CTA
        tiles = -(-M // 32)
        grid = min(tiles, NSM)
        cw = c_steps(4 * -(-tiles // grid)) + grid
        bw = (2.0 ** -10 + 2.0 ** -17 + cw * 2.0 ** -23) * (Gt.t() @ self.X.abs())
        if self.padG is not None:
            bw = bw + 1.01 * (self.padG.t() @ self.X.abs())
        if self.padX is not None:
            bw = bw + 1.01 * (Gt.t() @ self.padX)
        self.dw = {"a-priori": (self.G.t() @ self.X, bw)}
        if self.padG is None and self.padX is None:
            Gh, Xh = tf32(dZ).double(), tf32(Yp).double()
            self.dw["tight"] = (Gh.t() @ Xh, cw * 2.0 ** -23 * (Gh.abs().t() @ Xh.abs()))
        self.grid = grid

    def dw_tiers(self, dW0):
        e = (self.grid + 2) * 2.0 ** -23 * dW0.double().abs()
        return {k: (dW0.double() + r, b + e) for k, (r, b) in self.dw.items()}

    def sigmoid(self):
        """sigmoid(z) and the bound on the kernel's |error| (1 - ex2.approx of the kernel's fp32 x)."""
        sig = torch.sigmoid(self.z)
        dsig = torch.sigmoid(-self.z) * (self.padX + 2.0 ** -21 * (1 + self.X)) + 2.0 ** -22
        return sig, dsig


def out_tiers(dx_tiers, E, final, sig=None, dsig=None):
    """dZprev = (E + dX) [* sigmoid] with its fp32 roundings; dx_tiers may be a sum of launches."""
    out = {}
    for k, (ref, bound) in dx_tiers.items():
        S = ref + (E if E is not None else 0)
        eps = 2.0 ** -22 * (S.abs() + (E.abs() if E is not None else 0))
        if final:
            out[k] = (S * sig, bound * sig + S.abs() * dsig + eps)
        else:
            out[k] = (S, bound + eps)
    return out


def bwd_stats_check(where, s, got, e, sig, dsig, final):
    if not final:
        assert torch.count_nonzero(s).item() == 0, f"{where}: s1 / s2 written in a raw mode"
        return
    t = got.double()
    assert bool(((s[0] - t.sum(0)).abs() <= 2.0 ** -19 * t.abs().sum(0) + 1e-12).all()), f"{where}: s1"
    # the kernel recovers xhat from the stored x through lg2.approx(sigmoid): its error, per element
    dxh = e.invg.abs() * (e.padX + dsig / sig + 2.0 ** -21 * (1 + torch.log(sig).abs() + e.X + e.stat_pad))
    tol = (t.abs() * dxh).sum(0) + 2.0 ** -19 * (t * e.xhat).abs().sum(0) + 1e-12
    err = (s[1] - (t * e.xhat).sum(0)).abs()
    assert bool((err <= tol).all()), f"{where}: s2 error/bound {(err / tol).max().item():.3g}"


@pytest.mark.parametrize("bn", [True, False], ids=["bn", "nobn"])
@pytest.mark.parametrize("row,M", [(r, m) for r in BWD for m in BWD_M] + [("B6", BIG_M)])
def test_backward_launch(row, M, bn):
    spec = BWD[row]
    h = spec.get("h", M % 3)
    kin, mode, raw = spec["kin"], spec["mode"], spec["raw"]
    final = mode in (0, 3)
    gen = torch.Generator(device=DEV).manual_seed(1000 * M + 10 * int(row[1]) + mode + 7 * bn)
    ldg, ldp, ldo = spec["ldg"], spec["ldp"], spec["ldo"]
    go, po, oo = (128 * h if ld == 384 else 0 for ld in (ldg, ldp, ldo))
    dZb, Yb, Ypb = nan_buf(M + PAD, ldg), nan_buf(M + PAD, ldg), nan_buf(M + PAD, ldp)
    dZb[:M, go:go + 128] = rand(gen, M, 128)
    Yb[:M, go:go + 128] = rand(gen, M, 128)
    Ypb[:M, po:po + kin] = rand(gen, M, kin)
    wr, wc, w0 = spec["w"]
    r0 = 128 * h if wr == 384 else 0
    Wb = rand(gen, wr, wc) / 128 ** 0.5
    dWb = rand(gen, wr, wc)                                  # non-zero: dW is accumulated into
    Ob = sentinel(gen, M + PAD, ldo)
    if mode in (2, 3):
        Ob[:M, oo:oo + kin] = rand(gen, M, kin)
    E = Ob[:M, oo:oo + kin].clone() if mode in (2, 3) else None
    O0, dW0 = Ob.clone(), dWb.clone()
    bc, pc = bwd_coefs(gen, bn, raw)
    s = torch.zeros(2, 128, dtype=torch.float64, device=DEV)
    W = Wb[r0:r0 + 128, w0:w0 + kin]
    rc = bwd_launch(M, dZb[:, go:], Yb[:, go:] if bn else None, bc, Ypb[:, po:], pc, Wb[r0:, w0:], dWb[r0:, w0:], Ob[:, oo:], mode, s,
                    kin, raw)
    _lib().check(rc, "ga_tc_linear_backward_ex")
    torch.cuda.synchronize()

    where = f"{row} M={M} h={h} {'bn' if bn else 'nobn'}"
    untouched(f"{where} dZprev", Ob, O0, M, oo, oo + kin)
    untouched(f"{where} dW", dWb, dW0, M, w0, w0 + kin, r0=r0, r1=r0 + 128)
    e = Bwd(dZb[:M, go:go + 128], Yb[:M, go:go + 128], bc, Ypb[:M, po:po + kin], pc, W, M)
    sig, dsig = e.sigmoid() if final else (None, None)
    tiers = out_tiers(e.dx, E, final, sig, dsig)
    got = Ob[:M, oo:oo + kin]
    check(f"{where} dZprev", got, tiers)
    dwt = e.dw_tiers(dW0[r0:r0 + 128, w0:w0 + kin])
    gotw = dWb[r0:r0 + 128, w0:w0 + kin]
    check(f"{where} dW", gotw, dwt)
    bwd_stats_check(where, s, got, e, sig, dsig, final)

    # self-checks: one dropped term in the last (ragged) tile, two swapped pixels, channels 64-71 of a kin = 72 result
    rejects(f"{where} dZprev (term dropped)", drop_term(got, M - 1, e.G, e.W, tiers["a-priori"][1], sig), tiers)
    if M >= 2:
        sw = got.double().clone()
        sw[[M - 1, M - 2]] = sw[[M - 2, M - 1]]
        rejects(f"{where} dZprev (pixels swapped)", sw, tiers)
    if kin == 72:
        for name, t, tr in (("dZprev", got, tiers), ("dW", gotw, dwt)):
            z = t.double().clone()
            z[:, 64:72] = 0
            rejects(f"{where} {name} (channels 64-71 zeroed)", z, tr)
    # the last pixel's term in one dW element, at sizes where a single pixel's term is above the tier's resolution
    for tier in dwt:
        if M <= (NSM * 32 + 1 if tier == "tight" else 33):
            T = e.G[M - 1][:, None] * e.X[M - 1][None, :]
            o, i = divmod(int((T.abs() / dwt[tier][1]).argmax()), kin)
            bad = gotw.double().clone()
            bad[o, i] -= T[o, i]
            rejects(f"{where} dW (last pixel dropped)", bad, {tier: dwt[tier]})


@pytest.mark.parametrize("M", [1, 33, NSM * 32 + 1])
def test_backward_layer6_heads_chain(M):
    """Layer 6 as the decoder enqueues it: heads 0, 1, 2 in modes 1, 2, 3 into one dZ5, no synchronisation between."""
    gen = torch.Generator(device=DEV).manual_seed(M + 66)
    dZ6, Y6 = nan_buf(M + PAD, 384), nan_buf(M + PAD, 384)
    dZ6[:M], Y6[:M] = rand(gen, M, 384), rand(gen, M, 384)
    Y5 = nan_buf(M + PAD, 128)
    Y5[:M] = rand(gen, M, 128)
    W6 = rand(gen, 384, 128) / 128 ** 0.5
    dW6 = rand(gen, 384, 128)
    dW0 = dW6.clone()
    bcs = [bwd_coefs(gen, True, False)[0] for _ in range(3)]
    _, pc5 = bwd_coefs(gen, False, False)
    dZa = sentinel(gen, M + PAD, 128)
    before = dZa.clone()
    s = torch.zeros(2, 128, dtype=torch.float64, device=DEV)
    for h in range(3):
        c = slice(128 * h, 128 * h + 128)
        _lib().check(bwd_launch(M, dZ6[:, c], Y6[:, c], bcs[h], Y5, pc5, W6[c], dW6[c], dZa, h + 1, s, 128, False), f"head {h}")
    torch.cuda.synchronize()

    where = f"B2 chain M={M}"
    untouched(where, dZa, before, M, 0, 128)
    es = [Bwd(dZ6[:M, 128 * h:128 * h + 128], Y6[:M, 128 * h:128 * h + 128], bcs[h], Y5[:M], pc5, W6[128 * h:128 * h + 128], M)
          for h in range(3)]
    sig, dsig = es[0].sigmoid()
    dx = sum_terms([e.dx for e in es])
    # heads 0 + 1 are rounded once more by the reduce-add
    mid = es[0].dx["a-priori"][0] + es[1].dx["a-priori"][0]
    tiers = {k: (r, b + 2.0 ** -22 * mid.abs() * sig) for k, (r, b) in out_tiers(dx, None, True, sig, dsig).items()}
    check(where, dZa[:M], tiers)
    for h, e in enumerate(es):
        check(f"{where} dW6 head {h}", dW6[128 * h:128 * h + 128], e.dw_tiers(dW0[128 * h:128 * h + 128]))
    bwd_stats_check(where, s, dZa[:M], es[0], sig, dsig, True)


@pytest.mark.parametrize("M", [1, 33, NSM * 32 + 1])
def test_backward_feature_gradient_chain(M):
    """d_feat as the decoder forms it: layer 5's feature part stores (mode 1), then layer 1 reduce-adds (mode 2), no sync between."""
    gen = torch.Generator(device=DEV).manual_seed(M + 15)
    dZ5, Y5, dZ1, Y1 = (nan_buf(M + PAD, 128) for _ in range(4))
    for t in (dZ5, Y5, dZ1, Y1):
        t[:M] = rand(gen, M, 128)
    feat = nan_buf(M + PAD, 72)
    feat[:M] = rand(gen, M, 72)
    W5, W1 = rand(gen, 128, 200) / 128 ** 0.5, rand(gen, 128, 72) / 128 ** 0.5
    dW5, dW1 = rand(gen, 128, 200), rand(gen, 128, 72)
    dW5_0, dW1_0 = dW5.clone(), dW1.clone()
    bc5, bc1 = bwd_coefs(gen, True, True)[0], bwd_coefs(gen, True, True)[0]
    d_feat = sentinel(gen, M + PAD, 72)
    before = d_feat.clone()
    _lib().check(bwd_launch(M, dZ5, Y5, bc5, feat, None, W5, dW5, d_feat, 1, None, 72, True), "layer 5 feature part")
    _lib().check(bwd_launch(M, dZ1, Y1, bc1, feat, None, W1, dW1, d_feat, 2, None, 72, True), "layer 1")
    torch.cuda.synchronize()

    where = f"B4+B6 chain M={M}"
    untouched(where, d_feat, before, M, 0, 72)
    untouched(f"{where} dW5", dW5, dW5_0, 128, 0, 72)       # columns 72-199 belong to the x4 part
    e5 = Bwd(dZ5[:M], Y5[:M], bc5, feat[:M], None, W5[:, :72], M)
    e1 = Bwd(dZ1[:M], Y1[:M], bc1, feat[:M], None, W1, M)
    check(where, d_feat[:M], out_tiers(sum_terms([e5.dx, e1.dx]), None, False))
    check(f"{where} dW5", dW5[:, :72], e5.dw_tiers(dW5_0[:, :72]))
    check(f"{where} dW1", dW1, e1.dw_tiers(dW1_0))


@pytest.mark.parametrize("mode", [0, 3])
def test_backward_final_modes_need_all_channels(mode):
    """Modes 0 and 3 take s1 / s2 over all 128 channels (and mode 3 reads the existing tile): kin < 128 is refused, nothing launched."""
    M = 32
    gen = torch.Generator(device=DEV).manual_seed(mode)
    dZ, Y, Yp = rand(gen, M, 128), rand(gen, M, 128), rand(gen, M, 72)
    W, dW = rand(gen, 128, 72), torch.zeros(128, 72, device=DEV)
    O = rand(gen, M, 72)
    O0 = O.clone()
    bc, pc = bwd_coefs(gen, True, False)
    s = torch.zeros(2, 128, dtype=torch.float64, device=DEV)
    L = _lib()
    n0 = L.launch_count()
    rc = bwd_launch(M, dZ, Y, bc, Yp, pc, W, dW, O, mode, s, 72, False)
    assert rc != 0
    assert b"kin" in L.lib().ga_last_error()
    assert L.launch_count() == n0
    torch.cuda.synchronize()
    assert torch.equal(O, O0) and torch.count_nonzero(dW).item() == 0 and torch.count_nonzero(s).item() == 0
