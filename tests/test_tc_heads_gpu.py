"""GPU: layer 6's one-launch three-head forward (ga_tc_linear_forward_heads) against the three per-head ga_tc_linear_forward
launches it replaces, bit for bit, and against fp64.

It runs at one row, partial / exact / one-past tiles, one tile past a full round of its grid (44 tile groups per head for an
H100 SXM's 132 SMs) and the config-3 decoder size.  Outputs sit in buffers filled with finite sentinels that must stay
bit-identical outside the launch's region; rows of the input at or past M are NaN.  BatchNorm statistics are summed with
atomics, whose order moves the last bit, and are compared within a relative 1e-5.  A corrupted launch (a head given another
head's weights) must be told apart.  At one size the outputs are also held to the a-priori fp64 tier of test_tc_launches_gpu.py
(fp64 math on the unrounded operands), which must reject a dropped product term and a head's output taken from another head.
"""
import pytest
import torch

from gaussianavatar_b200 import _lib as L

pytestmark = [pytest.mark.gpu, pytest.mark.tf32]
DEV = "cuda:0"
NSM = 132
PAD = 70
SENT = 12345.0
# 64-pixel tiles over num_sms // heads tile groups
FWD_M = [1, 31, 63, 64, 65, (NSM // 3) * 64 + 1, 262144]


def p(t):
    return None if t is None else t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


def nan_rows(M, cols, valid_cols=None, scale=1.0, gen=None):
    """[M + PAD, cols] buffer: random in the first M rows (in valid_cols), NaN elsewhere."""
    t = torch.full((M + PAD, cols), float("nan"), device=DEV)
    r = torch.randn(M, cols, device=DEV, generator=gen) * scale
    if valid_cols is None:
        t[:M] = r
    else:
        t[:M, valid_cols] = r[:, valid_cols]
    return t


def assert_rel(got, want, rtol=1e-5, what=""):
    err = (got.double() - want.double()).abs().max().item()
    assert err <= rtol * want.double().abs().max().item() + 1e-12, (what, err)


# ---- layer-6 forward ------------------------------------------------------------------------------------------------

def fwd_inputs(M, gen):
    X = nan_rows(M, 128, gen=gen)
    a = torch.rand(128, device=DEV, generator=gen) + 0.5
    b = torch.randn(128, device=DEV, generator=gen) * 0.5
    W = torch.randn(384, 128, device=DEV, generator=gen) / 11.3
    bias = torch.randn(384, device=DEV, generator=gen)
    return X, a, b, W, bias


def run_fwd_single(M, X, a, b, W, bias):
    Y = torch.full((M + PAD, 384), SENT, device=DEV)
    s = torch.zeros(2, 384, dtype=torch.float64, device=DEV)
    for h in range(3):
        L.check(L.lib().ga_tc_linear_forward(M, 128, p(X), 128, p(a), p(b), p(W[h * 128:]), 128, p(bias[h * 128:]), p(Y[:, h * 128:]), 384, 0,
                                             p(s[0, h * 128:]), p(s[1, h * 128:]), stream()), "ga_tc_linear_forward")
    return Y, s


def run_fwd_heads(M, X, a, b, W, bias):
    Y = torch.full((M + PAD, 384), SENT, device=DEV)
    s = torch.zeros(2, 384, dtype=torch.float64, device=DEV)
    L.check(L.lib().ga_tc_linear_forward_heads(M, 3, 128, p(X), 128, p(a), p(b), p(W), 128, 128 * 128, p(bias), p(Y), 384, 128, 0,
                                               p(s[0]), p(s[1]), 128, stream()), "ga_tc_linear_forward_heads")
    return Y, s


@pytest.mark.parametrize("M", FWD_M)
def test_layer6_forward_heads_is_three_launches(M):
    gen = torch.Generator(device=DEV).manual_seed(M)
    X, a, b, W, bias = fwd_inputs(M, gen)
    Y1, s1 = run_fwd_single(M, X, a, b, W, bias)
    Y3, s3 = run_fwd_heads(M, X, a, b, W, bias)
    torch.cuda.synchronize()
    assert torch.equal(Y3[:M], Y1[:M])                              # every head's tile math is unchanged
    assert (Y3[M:] == SENT).all()                                   # rows >= M are never stored
    assert torch.isfinite(Y3[:M]).all()
    assert_rel(s3, s1, what="statistics")
    # a head computed with another head's weights is caught
    Wbad = W.clone()
    Wbad[256:] = W[:128]
    Yb, _ = run_fwd_heads(M, X, a, b, Wbad, bias)
    assert not torch.equal(Yb[:M, 256:], Y1[:M, 256:])


# ---- a-priori fp64 tier (the bounds of test_tc_launches_gpu.py), one size past a full round of each grid ------------------

def _tl():
    import test_tc_launches_gpu as TL          # the fp64 expectations and bounds of the per-head launches
    return TL


def test_layer6_forward_heads_fp64():
    TL = _tl()
    M = (NSM // 3) * 64 + 1
    gen = torch.Generator(device=DEV).manual_seed(7)
    X, a, b, W, bias = fwd_inputs(M, gen)
    Y, s = run_fwd_heads(M, X, a, b, W, bias)
    torch.cuda.synchronize()
    for h in range(3):
        prod, A, W64 = TL.fwd_product(X[:M], True, a, b, W[h * 128:h * 128 + 128])
        tiers = TL.with_epilogue(prod, bias[h * 128:h * 128 + 128].double(), bias[h * 128:h * 128 + 128].double().abs())
        got = Y[:M, h * 128:h * 128 + 128]
        TL.check(f"heads fwd h={h}", got, tiers)
        TL.stats_check(f"heads fwd h={h}", s[:, h * 128:h * 128 + 128], got)
        TL.rejects(f"heads fwd h={h} (term dropped)", TL.drop_term(got, M - 1, A, W64.t(), tiers["a-priori"][1]), tiers)
    bad = Y[:M].double().clone()                    # a head's output taken from another head
    bad[:, 256:] = Y[:M, :128].double()
    prod, _, _ = TL.fwd_product(X[:M], True, a, b, W[256:])
    TL.rejects("heads fwd (wrong head)", bad[:, 256:], TL.with_epilogue(prod, bias[256:].double(), bias[256:].double().abs()))
