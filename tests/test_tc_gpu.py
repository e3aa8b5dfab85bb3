"""GPU: the tensor-core (TF32) decoder layer against fp64 torch math, and the whole TF32 decoder against the reference fixtures."""
import os

import numpy as np
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.tf32]
DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def tc_linear(X, W, bias=None, a=None, b=None, Y0=None, stats=True):
    from gaussianavatar_b200 import _lib
    from gaussianavatar_b200._lib import ptr
    M, K = X.shape[0], W.shape[1]
    Y = Y0.clone() if Y0 is not None else torch.empty(M, 128, device=DEV)
    s = torch.zeros(2, 128, dtype=torch.float64, device=DEV) if stats else None
    _lib.check(_lib.lib().ga_tc_linear_forward(M, K, ptr(X), X.stride(0), ptr(a), ptr(b), ptr(W), W.stride(0), ptr(bias), ptr(Y), Y.stride(0),
                                               1 if Y0 is not None else 0, ptr(s[0]) if stats else None, ptr(s[1]) if stats else None,
                                               torch.cuda.current_stream().cuda_stream), "ga_tc_linear_forward")
    torch.cuda.synchronize()
    return Y, s


def tf32_trunc(t):
    """fp32 -> tf32, round-to-nearest (ties away), as cvt.rna.tf32.f32 does."""
    i = t.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


@pytest.mark.parametrize("M,K,act,acc", [(128, 128, False, False), (1024, 128, True, False), (5000, 72, False, False),
                                         (128 * 300, 128, True, True), (2304, 128, True, False),
                                         (1000, 128, True, True),      # ragged last 64-pixel tile (40 rows: the second pixel half has 8) + fan-in accumulate
                                         (40, 72, True, True), (47393, 128, False, False)])      # less than one tile; > 4 stage rounds per CTA on 132 SMs
def test_tc_linear_forward(M, K, act, acc):
    g = torch.Generator().manual_seed(M + K)
    X = torch.randn(M, K, generator=g).to(DEV)
    W = (torch.randn(128, K, generator=g) / K ** 0.5).to(DEV)
    bias = torch.randn(128, generator=g).to(DEV)
    a = (1 + 0.2 * torch.randn(K, generator=g)).to(DEV) if act else None
    b = (0.3 * torch.randn(K, generator=g)).to(DEV) if act else None
    Y0 = torch.randn(M, 128, generator=g).to(DEV) if acc else None
    Y, s = tc_linear(X, W, bias, a, b, Y0)
    Xa = torch.nn.functional.softplus(X * a + b) if act else X
    ref = Xa.double() @ W.double().t() + bias.double() + (Y0.double() if acc else 0)
    # TF32: 10-bit mantissas on both operands -> ~1e-3 relative on a K-term dot product of O(1) values
    err = (Y.double() - ref).abs().max().item()
    assert err < 6e-3 * max(1.0, ref.abs().max().item()), err
    # tight check against fp64 math on TF32-truncated operands (isolates layout / descriptor bugs from rounding)
    ref_t = tf32_trunc(Xa).double() @ tf32_trunc(W).double().t() + bias.double() + (Y0.double() if acc else 0)
    assert (Y.double() - ref_t).abs().max().item() < 2e-4 * max(1.0, ref.abs().max().item())
    assert (s[0] - Y.double().sum(0)).abs().max().item() < 1e-3 * M ** 0.5
    assert (s[1] - (Y.double() ** 2).sum(0)).abs().max().item() < 1e-3 * M


@pytest.mark.parametrize("name", ["pop_s32_in16.npz", "pop_s48_in128.npz"])
def test_decoder_tf32_forward_vs_reference_fixture(name):
    """TF32 tensor-core forward vs the reference's CPU fp32 outputs: tolerance per SURVEY App. C (rel-L2 <= 2e-3)."""
    from gaussianavatar_b200.network import POP_no_unet
    from oracle import avatar_oracle as ao
    d = np.load(os.path.join(GOLD, name))
    inp, S, B, seed = int(d["inp"]), int(d["S"]), int(d["B"]), int(d["seed"])
    net = POP_no_unet(c_geom=64, hsize=128).to(DEV)
    assert net.tensor_cores
    net.load_state_dict(ao.seeded_pop_params(seed), strict=False)
    g = torch.Generator().manual_seed(seed + 1)
    geo = (torch.randn(1, 64, inp, inp, generator=g) * 0.01).to(DEV)
    dec = net.forward_packed(geo, S, B).detach().cpu().numpy()
    for sl, key in ((slice(0, 3), "res"), (slice(3, 4), "scales"), (slice(4, 7), "shs")):
        ref = d[key][0].T
        rel = np.linalg.norm(dec[:, sl] - ref) / np.linalg.norm(ref)
        assert rel < 3e-3, (key, rel)      # 8 TF32 layers with BatchNorm in between; the strict-FP32 path holds 1e-4


@pytest.mark.parametrize("M,bn,ldg", [(64, True, 128), (1000, True, 384), (64 * 333, True, 128), (4096, False, 128)])
def test_tc_linear_backward(M, bn, ldg):
    from gaussianavatar_b200 import _lib
    from gaussianavatar_b200._lib import ptr
    g = torch.Generator().manual_seed(M)
    dZ = torch.randn(M, ldg, generator=g).to(DEV); Y = torch.randn(M, ldg, generator=g).to(DEV)
    Yp = torch.randn(M, 128, generator=g).to(DEV)
    W = (torch.randn(128, 128, generator=g) / 128 ** 0.5).to(DEV)
    bc = torch.stack([1 + 0.2 * torch.randn(128, generator=g), 0.1 * torch.randn(128, generator=g), 0.1 * torch.randn(128, generator=g),
                      0.1 * torch.randn(128, generator=g), 1 + 0.1 * torch.rand(128, generator=g)]).to(DEV).contiguous()
    pc = torch.stack([1 + 0.2 * torch.randn(128, generator=g), 0.3 * torch.randn(128, generator=g), 0.1 * torch.randn(128, generator=g),
                      1 + 0.1 * torch.rand(128, generator=g)]).to(DEV).contiguous()
    off = 128 if ldg == 384 else 0                      # operate on a 128-wide slice of a wider tensor (heads layout)
    dZs, Ys = dZ[:, off:off + 128], Y[:, off:off + 128]
    d64 = lambda t: t.double()
    G = d64(bc[0]) * (d64(dZs) - d64(bc[1]) - (d64(Ys) - d64(bc[3])) * d64(bc[4]) * d64(bc[2])) if bn else d64(dZs)
    z = d64(Yp) * d64(pc[0]) + d64(pc[1])
    X = torch.nn.functional.softplus(z)
    dW_ref = G.t() @ X
    dX_ref = G @ d64(W)
    dZp_ref = dX_ref * torch.sigmoid(z)
    xhat = (d64(Yp) - d64(pc[2])) * d64(pc[3])

    def run(mode, dZprev_init=None):
        dW = torch.zeros(128, 128, device=DEV)
        dZp = dZprev_init.clone() if dZprev_init is not None else torch.empty(M, 128, device=DEV)
        s = torch.zeros(2, 128, dtype=torch.float64, device=DEV)
        _lib.check(_lib.lib().ga_tc_linear_backward(M, dZs.data_ptr(), Ys.data_ptr(), ldg, ptr(bc) if bn else None, ptr(Yp), 128, ptr(pc), ptr(W), 128,
                                                    ptr(dW), 128, ptr(dZp), 128, mode, ptr(s[0]), ptr(s[1]), torch.cuda.current_stream().cuda_stream),
                   "ga_tc_linear_backward")
        torch.cuda.synchronize()
        return dW, dZp, s

    rel = lambda a, b: ((a.double() - b).norm() / b.norm()).item()
    dW, dZp, s = run(0)
    assert rel(dW, dW_ref) < 3e-3, rel(dW, dW_ref)
    assert rel(dZp, dZp_ref) < 3e-3, rel(dZp, dZp_ref)
    assert (s[0] - dZp.double().sum(0)).abs().max().item() < 1e-3 * M ** 0.5 + 1e-3
    assert (s[1] - (dZp.double() * xhat).sum(0)).abs().max().item() < 2e-3 * M ** 0.5 + 1e-3
    _, raw, _ = run(1)
    assert rel(raw, dX_ref) < 3e-3
    init = torch.randn(M, 128, generator=g).to(DEV)
    _, acc, _ = run(2, init)
    assert rel(acc, init.double() + dX_ref) < 3e-3
    _, fin, s3 = run(3, init)
    assert rel(fin, (init.double() + dX_ref) * torch.sigmoid(z)) < 3e-3
    assert (s3[0] - fin.double().sum(0)).abs().max().item() < 1e-3 * M ** 0.5 + 1e-3


@pytest.mark.parametrize("name", ["pop_s32_in16.npz", "pop_s48_in128.npz"])
def test_decoder_tf32_backward_vs_reference_fixture(name):
    """Weight / geo_feature gradients of the TF32 tensor-core path vs the reference's CPU fp32 autograd."""
    from gaussianavatar_b200.network import POP_no_unet
    from oracle import avatar_oracle as ao
    d = np.load(os.path.join(GOLD, name))
    inp, S, B, seed = int(d["inp"]), int(d["S"]), int(d["B"]), int(d["seed"])
    net = POP_no_unet(c_geom=64, hsize=128).to(DEV)
    net.load_state_dict(ao.seeded_pop_params(seed), strict=False)
    g = torch.Generator().manual_seed(seed + 1)
    geo = (torch.randn(1, 64, inp, inp, generator=g) * 0.01).to(DEV).requires_grad_(True)
    uv = torch.tensor(d["uv"], device=DEV)
    res, sc, shs = net(None, geo.expand(B, -1, -1, -1).contiguous(), uv[None].expand(B, -1, -1).contiguous())
    gr, gs, gc = (torch.randn(res.shape, generator=g), torch.randn(sc.shape, generator=g), torch.randn(shs.shape, generator=g))
    ((res * gr.to(DEV)).sum() + (sc * gs.to(DEV)).sum() + (shs * gc.to(DEV)).sum()).backward()
    grads = {k: v.cpu().numpy() for k, v in net.reference_grads().items()}
    worst = {}
    for k in d.files:
        if k.startswith("grad:"):
            n = k[5:]
            if n in ("decoder.conv1.bias", "decoder.conv6N.bias"):
                continue
            got = grads[n][:8, :8] if n.startswith("geom_proc") else grads[n]
            worst[n] = float(np.linalg.norm(got - d[k]) / (np.linalg.norm(d[k]) + 1e-30))
    assert max(worst.values()) < 3e-2, worst
    gg = geo.grad.cpu().numpy()
    assert abs(np.linalg.norm(gg) - float(d["geo_grad_norm"])) / float(d["geo_grad_norm"]) < 2e-2


@pytest.mark.parametrize("Hf", [16, 40, 128])
def test_tc_conv5x5_all_modes(Hf):
    """tensor-core implicit-GEMM 5x5 conv (forward, data gradient, weight gradient) vs fp64 torch conv2d on the same TF32-rounded
    operands: only the accumulation order differs, so the tolerance is fp32 round-off (rel 1e-5)."""
    import torch.nn.functional as F
    from gaussianavatar_b200 import _lib
    from gaussianavatar_b200._lib import ptr
    g = torch.Generator().manual_seed(Hf)
    P = Hf * Hf
    x = torch.randn(P, 64, generator=g).to(DEV)
    dy = torch.randn(P, 64, generator=g).to(DEV)
    w = (torch.randn(25, 64, 64, generator=g) * 0.05).to(DEV)                 # [tap][ci][co]
    st = torch.cuda.current_stream().cuda_stream
    L = _lib.lib()
    xr, dyr, wr = torch.empty_like(x), torch.empty_like(dy), torch.empty_like(w)
    for src, dst in ((x, xr), (dy, dyr), (w, wr)):
        _lib.check(L.ga_round_tf32(ptr(src), ptr(dst), src.numel(), st), "ga_round_tf32")
    assert torch.equal(xr, tf32_trunc(x)) and torch.equal(wr, tf32_trunc(w))
    y = torch.empty(P, 64, device=DEV); dx = torch.empty(P, 64, device=DEV); dw = torch.zeros(25, 64, 64, device=DEV)
    _lib.check(L.ga_tc_conv5x5(0, Hf, ptr(xr), ptr(wr), ptr(y), 0, st), "conv fwd")
    _lib.check(L.ga_tc_conv5x5(1, Hf, ptr(dyr), ptr(wr), ptr(dx), 0, st), "conv dgrad")
    _lib.check(L.ga_tc_conv5x5(2, Hf, ptr(xr), ptr(dyr), ptr(dw), 0, st), "conv wgrad")
    torch.cuda.synchronize()
    # fp64 reference through autograd on the rounded operands
    xn = xr.double().view(Hf, Hf, 64).permute(2, 0, 1)[None].requires_grad_(True)            # NCHW
    wn = wr.double().view(5, 5, 64, 64).permute(3, 2, 0, 1).contiguous().requires_grad_(True)   # [co][ci][ky][kx]
    yn = F.conv2d(xn, wn, padding=2)
    yn.backward(dyr.double().view(Hf, Hf, 64).permute(2, 0, 1)[None])
    rel = lambda a, b: ((a.double() - b).norm() / b.norm()).item()
    assert rel(y, yn[0].permute(1, 2, 0).reshape(P, 64)) < 1e-5
    assert rel(dx, xn.grad[0].permute(1, 2, 0).reshape(P, 64)) < 1e-5
    assert rel(dw, wn.grad.permute(2, 3, 1, 0).reshape(25, 64, 64)) < 1e-5
    # round_out stores the TF32-rounded result
    y2 = torch.empty_like(y)
    _lib.check(L.ga_tc_conv5x5(0, Hf, ptr(xr), ptr(wr), ptr(y2), 1, st), "conv fwd rounded")
    torch.cuda.synchronize()
    assert torch.equal(y2, tf32_trunc(y))
