"""GPU: the skinning kernels with each training frame's exposure (csrc/lbs.cu, ga_lbs_forward_exposure / ga_lbs_backward_exposure),
element by element against an fp64 restatement with running error bounds, as test_step_kernels_gpu.py checks the kernels without it.

frame b's colours are c' = A_b c + t_b, [A_b | t_b] = E[pose_idx[b]]; the backward's decoder colour gradient is sum_b A_b^T g_b
(A_b^T g_b per frame with a per-frame decoder output) and dE[f] = sum over the slots with pose_idx == f of sum_n g_n (x) [c_n, 1], row 0
(the gauge anchor) and untouched rows 0.  Means, scales, the position / scale part of d_dec and dC must be those of the exposure-off
call.  Each case also corrupts a copy of an output the way a broken kernel would and asserts that the bound rejects it.

Bounds (u = 2^-24, gamma(c) = c u / (1 - c u), times the same expression on absolute values):
  colours:  three chained FMAs                                              gamma(3) (|A| |c| + |t|)
  d_dec colour: three roundings per frame (A^T g) and nf frame additions     gamma(3 + nf) sum_b |A_b|^T |g_b|
  dE: one product per term, a sequential sum over the tile's rows, T tile additions per CTA, at most `grid` additions of CTA
      partials (a lane's serial sum, then the shuffle tree) and B slot additions:
                                                                            gamma(1 + min(N, 256) + T + grid + B) sum |g| |[c, 1]|
"""
import pytest
import torch

from test_step_kernels_gpu import (DEV, PAD, LbsCase, _round, check, gam, lbs_backward_launch, lbs_forward_launch, nan_buf, p,
                                   rejects, sentinel, stream, untouched)

pytestmark = pytest.mark.gpu


def _lib():
    from gaussianavatar_b200 import _lib
    return _lib


def pose_rows(B):
    """A batch's rows of the table: duplicates and the anchor (row 0) whenever B allows, rows 4 and 6 never used."""
    base = [3, 0, 5, 3, 1, 7, 5, 2]
    return base[:B] if B > 1 else [2]


class ExpCase(LbsCase):
    def __init__(self, J, N, B, per_frame, seed):
        super().__init__(J, N, B, per_frame, seed)
        self.pidx = torch.tensor(pose_rows(B), dtype=torch.int32, device=DEV)
        self.F = 9
        E = nan_buf(self.F, 3, 4)                      # rows no slot reads: NaN
        for f in set(pose_rows(B)):
            E[f, :, :3] = torch.eye(3, device=DEV) + 0.3 * torch.randn(3, 3, device=DEV, generator=self.gen)
            E[f, :, 3] = 0.2 * torch.randn(3, device=DEV, generator=self.gen)
        self.E = E.contiguous()
        self.grid_e = self.grid                        # the exposure variant's shared memory keeps the same CTAs per SM

    def colors_ref(self, transpose=False, offset=True):
        A = self.E.double()[self.pidx.long(), :, :3]   # [B,3,3]
        t = self.E.double()[self.pidx.long(), :, 3]
        if transpose:
            A = A.transpose(1, 2)
        c = self.o[..., 4:7].expand(self.B, self.N, 3)
        out = torch.einsum("brk,bnk->bnr", A, c) + (t[:, None] if offset else 0)
        bound = gam(3) * (torch.einsum("brk,bnk->bnr", A.abs(), c.abs()) + t.abs()[:, None])
        return out, bound

    def dcol_ref(self, dc, transpose=False, frames=None):
        """[frames, N, 3]: sum_b A_b^T g_b (shared) or per frame."""
        A = self.E.double()[self.pidx.long(), :, :3]
        if transpose:
            A = A.transpose(1, 2)
        G = dc.double()
        per = torch.einsum("brk,bnr->bnk", A, G)
        pa = torch.einsum("brk,bnr->bnk", A.abs(), G.abs())
        if self.per_frame:
            return per, gam(4) * pa
        sel = slice(None) if frames is None else frames
        return per[sel].sum(0, keepdim=True), gam(3 + self.B) * pa.sum(0, keepdim=True)

    def dE_ref(self, dc, by_slot=False, anchor=False):
        """[F,12]: rows pose_idx[b] += sum_n g (x) [c, 1]."""
        G = dc.double()
        c = self.o[..., 4:7].expand(self.B, self.N, 3)
        c1 = torch.cat([c, torch.ones_like(c[..., :1])], -1)            # [B,N,4]
        per = torch.einsum("bnr,bnk->brk", G, c1).reshape(self.B, 12)
        pa = torch.einsum("bnr,bnk->brk", G.abs(), c1.abs()).reshape(self.B, 12)
        out = torch.zeros(self.F, 12, dtype=torch.float64, device=DEV)
        bnd = torch.zeros_like(out)
        for b, f in enumerate(self.pidx.tolist()):
            row = b if by_slot else f
            if row == 0 and not (anchor or by_slot):
                continue
            out[row] += per[b]
            bnd[row] += pa[b]
        return out, gam(1 + min(self.N, 256) + self.T + self.grid_e + self.B) * bnd


def forward_exposure(cs, gen):
    B, N = cs.B, cs.N
    outs = {k: sentinel(gen, B * N * 3 + PAD) for k in ("means", "scales", "colors")}
    before = {k: v.clone() for k, v in outs.items()}
    L = _lib()
    L.check(L.lib().ga_lbs_forward_exposure(N, B, cs.J, cs.ld, cs.mul, cs.stride, p(cs.dec), p(cs.vidx), p(cs.q), p(cs.w), p(cs.C),
                                            cs.F, p(cs.E), p(cs.pidx), p(outs["means"]), p(outs["scales"]), p(outs["colors"]), stream()),
            "ga_lbs_forward_exposure")
    return outs, before


def backward_exposure(cs, gen, grads):
    B, N, J = cs.B, cs.N, cs.J
    d_dec = sentinel(gen, (cs.rows + PAD) * 8)
    dC = sentinel(gen, B * J * 12 + PAD)
    dE = sentinel(gen, cs.F * 12 + PAD)
    before = (d_dec.clone(), dC.clone(), dE.clone())
    L = _lib()
    nbytes = int(L.lib().ga_lbs_exposure_workspace_bytes(N, J))
    assert nbytes == 4 * 12 * 8 * cs.grid_e
    ws = torch.full((nbytes // 4 + 64,), float("nan"), device=DEV)
    L.check(L.lib().ga_lbs_backward_exposure(N, B, J, cs.ld, cs.rows, cs.mul, cs.stride, p(cs.dec), p(cs.vidx), p(cs.q), p(cs.w), p(cs.C),
                                             cs.F, p(cs.E), p(cs.pidx), p(grads[0]), p(grads[1]), p(grads[2]), p(d_dec), p(dC), p(dE),
                                             p(ws), nbytes, stream()), "ga_lbs_backward_exposure")
    return d_dec, dC, dE, before


LBS_N = {J: [1, 255, 257, _round(J) + 1, 200_000] for J in (24, 55)}


@pytest.mark.parametrize("per_frame", [False, True], ids=["shared", "per_frame"])
@pytest.mark.parametrize("B", [1, 3, 8])
@pytest.mark.parametrize("J,N", [(J, N) for J in (24, 55) for N in LBS_N[J]])
def test_lbs_exposure_launch(J, N, B, per_frame):
    cs = ExpCase(J, N, B, per_frame, seed=5 * N + 3 * B + J + per_frame)
    gen = cs.gen
    where = cs.where
    n3 = B * N * 3
    off, _ = lbs_forward_launch(cs, gen)
    outs, before = forward_exposure(cs, gen)
    (dm, ds, dc), d_off, dC_off, _ = lbs_backward_launch(cs, gen)
    grads = [t.reshape(-1) for t in (dm, ds, dc)]
    d_dec, dC, dE, (dd0, dC0, dE0) = backward_exposure(cs, gen, grads)
    d_dec2, dC2, dE2, _ = backward_exposure(cs, gen, grads)
    torch.cuda.synchronize()
    cs.forward_ref()

    # forward: means / scales are the exposure-off call's bits; colours against fp64
    for k in ("means", "scales", "colors"):
        untouched(f"{where} {k}", outs[k], before[k], 0, n3)
    for k in ("means", "scales"):
        assert torch.equal(outs[k][:n3].view(torch.int32), off[k][:n3].view(torch.int32)), f"{where}: {k} differ from the exposure-off call"
    col = outs["colors"][:n3].view(B, N, 3)
    cref, cb = cs.colors_ref()
    check("exposure forward colors", where, col, cref, cb)
    rejects(f"{where}: A transposed in the forward", cs.colors_ref(transpose=True)[0], cref, cb)
    rejects(f"{where}: t dropped", cs.colors_ref(offset=False)[0], cref, cb)

    # backward: d_dec positions / scales bit-identical to the off call, colours against fp64; dC as the off call's
    rows = cs.rows
    untouched(f"{where} d_dec", d_dec, dd0, 0, rows * 8)
    untouched(f"{where} dC", dC, dC0, 0, B * J * 12)
    untouched(f"{where} dE", dE, dE0, 0, cs.F * 12)
    got = d_dec[:rows * 8].view(cs.frames, cs.P, 8)
    ref_off = d_off[:rows * 8].view(cs.frames, cs.P, 8)
    assert torch.equal(got[..., :4].contiguous().view(torch.int32), ref_off[..., :4].contiguous().view(torch.int32)), where
    assert torch.equal(got[..., 7], torch.zeros_like(got[..., 7]))
    inval = torch.ones(cs.P, dtype=torch.bool, device=DEV)
    inval[cs.vidx.long()] = False
    assert int((got[:, inval] != 0).sum()) == 0, f"{where}: d_dec rows outside valid_index written"
    vi = cs.vidx.long()
    gc = got[:, vi, 4:7]
    dref, db = cs.dcol_ref(dc)
    check("exposure backward d_dec colour", where, gc, dref, db)
    rejects(f"{where}: A not transposed in the backward", cs.dcol_ref(dc, transpose=True)[0], dref, db)
    if not per_frame and B > 1:
        rejects(f"{where}: the frame sum missing", cs.dcol_ref(dc, frames=slice(0, 1))[0], dref, db)
    dC_got, dC_ref = dC[:B * J * 12], dC_off[:B * J * 12]
    if cs.grid == 1:
        assert torch.equal(dC_got.view(torch.int32), dC_ref.view(torch.int32)), f"{where}: dC differs from the exposure-off call"
    else:     # atomics across CTAs: the same terms in another order
        bref = cs.backward_ref(dm, ds, dc)
        check("exposure backward dC", where, dC_got.view(B, J, 12), *bref["dC"])
    Eg = dE[:cs.F * 12].view(cs.F, 12)
    eref, eb = cs.dE_ref(dc)
    check("exposure backward dE", where, Eg, eref, eb)
    assert torch.equal(Eg[0], torch.zeros(12, device=DEV)), f"{where}: anchor row not zero"
    assert torch.equal(Eg[4], torch.zeros(12, device=DEV)) and torch.equal(Eg[6], torch.zeros(12, device=DEV))
    bad = eref.clone()
    bad.view(cs.F, 3, 4)[:, :, 3] = 0.0
    rejects(f"{where}: the [c, 1] offset column dropped", bad, eref, eb)
    rejects(f"{where}: gradient written to slot b", cs.dE_ref(dc, by_slot=True)[0], eref, eb)
    if 0 in pose_rows(B):
        rejects(f"{where}: nonzero anchor row", cs.dE_ref(dc, anchor=True)[0], eref, eb)
    # two backward calls: the same bits (dE and d_dec carry no atomics)
    assert torch.equal(dE[:cs.F * 12].view(torch.int32), dE2[:cs.F * 12].view(torch.int32)), f"{where}: dE differs between two calls"
    assert torch.equal(d_dec[:rows * 8].view(torch.int32), d_dec2[:rows * 8].view(torch.int32)), where


@pytest.mark.parametrize("per_frame", [False, True], ids=["shared", "per_frame"])
@pytest.mark.parametrize("J", [24, 55])
def test_lbs_exposure_through_wrapper(J, per_frame):
    """LbsAssemble with an exposure table [F,3,4] and int64 pose_idx, B = 8: the same bounds, and the identity table gives the
    exposure-off outputs and decoder gradient bit for bit."""
    from gaussianavatar_b200.ops import LbsAssemble
    B, N = 8, _round(J) + 1
    cs = ExpCase(J, N, B, per_frame, seed=J + 17 * per_frame)
    cs.forward_ref()
    E = cs.E.nan_to_num(0.0).view(cs.F, 3, 4).clone().requires_grad_(True)
    dec = cs.dec.view(-1, 8).clone().requires_grad_(True)
    C = cs.C[:B].clone().requires_grad_(True)
    means, scales, colors = LbsAssemble.apply(dec, C, cs.vidx, cs.q[:N], cs.w[:N], cs.mul, per_frame, E, cs.pidx.long())
    gs = [torch.randn(B, N, 3, device=DEV, generator=cs.gen) for _ in range(3)]
    torch.autograd.backward([means, scales, colors], gs)
    torch.cuda.synchronize()
    where = f"wrapper {cs.where}"
    check("exposure forward colors", where, colors.detach(), *cs.colors_ref())
    check("exposure backward dE", where, E.grad.view(cs.F, 12), *cs.dE_ref(gs[2]))
    dref, db = cs.dcol_ref(gs[2])
    check("exposure backward d_dec colour", where, dec.grad.view(cs.frames, cs.P, 8)[:, cs.vidx.long(), 4:7], dref, db)

    # identity rows: the exposure-off results bit for bit
    eye = torch.eye(3, 4, device=DEV).repeat(cs.F, 1, 1).requires_grad_(True)
    outs = []
    for table in (eye, None):
        d = cs.dec.view(-1, 8).clone().requires_grad_(True)
        o = LbsAssemble.apply(d, cs.C[:B].clone(), cs.vidx, cs.q[:N], cs.w[:N], cs.mul, per_frame, table,
                              None if table is None else cs.pidx)
        torch.autograd.backward(list(o), gs)
        outs.append([t.detach() for t in o] + [d.grad])
    for a, b in zip(*outs):
        assert torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0)), where


def test_no_gaussians_zero_the_whole_table():
    """N = 0: the backward writes zeros over the whole [F,12] gradient table (the ABI's argument checks are in test_exposure_cpu.py)."""
    L = _lib()
    z = torch.zeros(1024, device=DEV)
    dE = torch.full((24,), 5.0, device=DEV)
    L.check(L.lib().ga_lbs_backward_exposure(0, 1, 24, 24, 16, 1.0, 0, None, None, None, None, None, 2, None, None, None, None, None,
                                             p(z), p(z), p(dE), None, 0, stream()), "ga_lbs_backward_exposure")
    torch.cuda.synchronize()
    assert torch.equal(dE, torch.zeros_like(dE))


def test_row_outside_the_table_gives_nan_colours():
    """A pose_idx past the table is never read: that frame's colours are NaN, the others' are finite."""
    from gaussianavatar_b200.ops import LbsAssemble
    cs = ExpCase(24, 300, 2, False, seed=3)
    E = torch.eye(3, 4, device=DEV).repeat(2, 1, 1)
    _, _, colors = LbsAssemble.apply(cs.dec.view(-1, 8), cs.C[:2], cs.vidx, cs.q[:300], cs.w[:300], 1.0, False, E,
                                     torch.tensor([1, 2], device=DEV))
    assert bool(colors[0].isfinite().all()) and bool(colors[1].isnan().all())
