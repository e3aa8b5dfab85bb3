"""GPU: the LPIPS network's launches (csrc/lpips.cu: the five convolutions, the two pools, the four data gradients, the two
un-pools and conv1's image gradient) against fp64 from their own inputs, the module against the fp64 oracle, its known answers,
and the trainer's LPIPS term.  The head launches (lpips_dist1..5, lpips_sum, lpips_dnorm1..5) are checked element by element from
their own inputs in test_lpips_head_gpu.py."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gaussianavatar_b200 import _lib
from gaussianavatar_b200.lpips import LPIPS
from oracle import lpips_oracle as lo

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
SENTINEL = 0x5A                  # workspace bytes before the call; every byte outside the carved regions must keep it
TILE, SMS = 128, 132


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30)


_MODULES = {}


def _module(seed=0):
    if seed not in _MODULES:
        sd = lo.random_state_dict(seed)
        _MODULES[seed] = (LPIPS(sd, device=DEV), lo.LpipsOracle(sd).double().to(DEV), sd)
    return _MODULES[seed]


def _images(B, H, W, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x0 = torch.rand(B, 3, H, W, generator=g, device=DEV) * 2 - 1
    x1 = (x0 + 0.3 * torch.randn(B, 3, H, W, generator=g, device=DEV)).clamp(-1, 1)
    return x0.contiguous(), x1.contiguous()


def _run_abi(flat, x0, x1, g, in_scale=1.0, in_shift=0.0):
    """forward + backward through the C ABI on a sentinel-filled workspace; returns (out, d_in0, ws, views as tensors)."""
    L = _lib.lib()
    B, _, H, W = x0.shape
    ws = torch.full((L.ga_lpips_workspace_bytes(B, H, W),), SENTINEL, dtype=torch.uint8, device=DEV)
    out = torch.empty(B, device=DEV)
    d = torch.full_like(x0, float("nan"))
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(L.ga_lpips_forward(B, H, W, flat.data_ptr(), x0.data_ptr(), x1.data_ptr(), in_scale, in_shift, ws.data_ptr(), out.data_ptr(), st))
    _lib.check(L.ga_lpips_backward(B, H, W, flat.data_ptr(), ws.data_ptr(), g.data_ptr(), d.data_ptr(), st))
    torch.cuda.synchronize()
    v = _lib.GaLpipsViews()
    _lib.check(L.ga_lpips_views(B, H, W, ws.data_ptr(), ctypes.byref(v)))
    return out, d, ws, v


class _Regions:
    """Typed views of workspace regions; remembers which bytes they cover."""

    def __init__(self, ws):
        self.ws, self.owned = ws, torch.zeros(ws.numel(), dtype=torch.bool, device=DEV)

    def take(self, p, n, dtype=torch.float32):
        off = p - self.ws.data_ptr()
        nb = n * torch.tensor([], dtype=dtype).element_size()
        assert 0 <= off and off + nb <= self.ws.numel()
        assert not self.owned[off:off + nb].any(), "workspace regions overlap"
        self.owned[off:off + nb] = True
        return self.ws[off:off + nb].view(dtype)


def _nchw(t, imgs, h, w, c):
    return t.view(imgs, h, w, c).permute(0, 3, 1, 2).double()


def _check_conv(got, x, w, b, stride, pad, what):
    """|got - relu?(conv(x, w) + b)| <= 2^-10 conv(|x|, |w|) (TF32 operands) + 2^-11 |ref| (TF32-rounded output) + eps."""
    ref = F.conv2d(x, w, b, stride=stride, padding=pad)
    bound = F.conv2d(x.abs(), w.abs(), None, stride=stride, padding=pad) * 2.0 ** -10
    if b is not None:
        ref = ref.clamp_min(0)
    err = (got - ref).abs() - (bound + 2.0 ** -11 * ref.abs() + 1e-6)
    assert err.max().item() <= 0, f"{what}: worst excess {err.max().item():.3e} at {np.unravel_index(int(err.argmax()), err.shape)}"


def _check_dgrad(got, dz, w, pad, what):
    ref = torch.nn.grad.conv2d_input(got.shape, w, dz, padding=pad)
    bound = torch.nn.grad.conv2d_input(got.shape, w.abs(), dz.abs(), padding=pad) * 2.0 ** -10
    err = (got - ref).abs() - (bound + 1e-9)
    assert err.max().item() <= 0, f"{what}: worst excess {err.max().item():.3e}"


def _launch_pixels(B, H, W):
    """Output pixels of the forward convolutions (2B images) and of the data gradients of conv2..conv5 (B images)."""
    ms = lo.map_shapes(H, W)
    return [2 * B * h * w for h, w in ms], [B * h * w for h, w in ms[1:]]


# 1024^2 at B = 1, 2, 3; non-square; and sizes whose launches end one pixel short of / one past a 128-pixel tile (B=1 31x2047: the
# data gradients of conv3..5 have 127 pixels; 31x351: conv2's has 129) and a pixel pair past a full round of 132 tiles (1151x1919:
# conv3..5 have 132 * 128 + 2), plus a small odd batch
SIZES = [(1, 1024, 1024), (2, 1024, 1024), (3, 1024, 1024), (2, 512, 384), (3, 67, 45), (1, 31, 2047), (1, 31, 351), (1, 1151, 1919)]


def test_edge_sizes_hit_the_tile_boundaries():
    assert _launch_pixels(1, 31, 2047)[1][1:] == [TILE - 1] * 3
    assert _launch_pixels(1, 31, 351)[1][0] == TILE + 1
    assert _launch_pixels(1, 1151, 1919)[0][2:] == [TILE * SMS + 2] * 3


@pytest.mark.parametrize("B,H,W", SIZES)
def test_each_launch_against_fp64(B, H, W):
    lp, _, sd = _module(0)
    x0, x1 = _images(B, H, W, seed=B * 7 + H)
    g = torch.rand(B, device=DEV) + 0.5
    out, d, ws, v = _run_abi(lp.flat, x0, x1, g, in_scale=2.0, in_shift=-1.0)
    assert torch.isfinite(out).all() and torch.isfinite(d).all()
    R = _Regions(ws)
    ms = lo.map_shapes(H, W)
    pools = [((ms[0][0] - 3) // 2 + 1, (ms[0][1] - 3) // 2 + 1), ((ms[1][0] - 3) // 2 + 1, (ms[1][1] - 3) // 2 + 1)]
    C = lo.CHANNELS
    relu = [_nchw(R.take(v.relu[k], 2 * B * ms[k][0] * ms[k][1] * C[k]), 2 * B, *ms[k], C[k]) for k in range(5)]
    pool, arg = [], []
    for k in range(2):
        n = 2 * B * pools[k][0] * pools[k][1] * C[k]
        pool.append(_nchw(R.take(v.pool[k], n), 2 * B, *pools[k], C[k]))
        arg.append(R.take(v.pool_arg[k], n, torch.uint8).view(2 * B, *pools[k], C[k]).permute(0, 3, 1, 2))
    R.take(v.partials, 5 * B * 128)
    R.take(v.in_scale, 1)
    dz = [_nchw(R.take(v.dz[k], B * ms[k][0] * ms[k][1] * C[k]), B, *ms[k], C[k]) for k in range(5)]
    dnext = [_nchw(R.take(v.dnext[k], B * ms[k][0] * ms[k][1] * C[k]), B, *ms[k], C[k]) for k in range(4)]
    dpool = [_nchw(R.take(v.dpool[k], B * pools[k][0] * pools[k][1] * C[k]), B, *pools[k], C[k]) for k in range(2)]
    assert (ws[~R.owned] == SENTINEL).all(), "a launch wrote outside the workspace regions"

    keys = lo.conv_keys()
    W_ = [sd[wk].double().to(DEV) for wk, _, _ in keys]
    b_ = [sd[bk].double().to(DEV) for _, bk, _ in keys]
    # conv1 from the planar images through the input affine (2x - 1, then the scaling layer)
    shift = torch.tensor(lo.SHIFT, device=DEV, dtype=torch.float64).view(1, 3, 1, 1)
    scale = torch.tensor(lo.SCALE, device=DEV, dtype=torch.float64).view(1, 3, 1, 1)
    xin = (torch.cat([x0, x1]).double() * 2 - 1 - shift) / scale
    _check_conv(relu[0], xin, W_[0], b_[0], 4, 2, "conv1")
    for k in range(2):   # max pool: values and first-maximum indices exactly as torch
        rp, ri = F.max_pool2d(relu[k].float(), 3, 2, return_indices=True)
        assert torch.equal(pool[k].float(), rp), f"pool{k + 1} values"
        Wk = relu[k].shape[-1]
        oy = torch.arange(pools[k][0], device=DEV).view(1, 1, -1, 1)
        ox = torch.arange(pools[k][1], device=DEV).view(1, 1, 1, -1)
        win = (ri // Wk - 2 * oy) * 3 + (ri % Wk - 2 * ox)
        assert torch.equal(arg[k].long(), win), f"pool{k + 1} indices"
    ins = [None, pool[0], pool[1], relu[2], relu[3]]
    for k in range(1, 5):
        _check_conv(relu[k], ins[k], W_[k], b_[k], 1, lo.KERNELS[k] // 2, f"conv{k + 1}")
    # data gradients of conv5 .. conv2 from the stored dZ, and the un-pooling
    douts = [dpool[0], dpool[1], dnext[2], dnext[3]]
    for k in range(1, 5):
        _check_dgrad(douts[k - 1], dz[k], W_[k], lo.KERNELS[k] // 2, f"dgrad{k + 1}")
    for k in range(2):   # un-pooling: the same gather order as torch's max-pool backward, so bit for bit
        _check_unpool(dnext[k], relu[k][:B], dpool[k], f"unpool{k + 1}")
    # conv1's image gradient: d_in0 = 2 / scale_c * conv1 input gradient of dZ1 (the affine's chain factor)
    ref = torch.nn.grad.conv2d_input((B, 3, H, W), W_[0], dz[0], stride=4, padding=2) * 2 / scale
    bound = torch.nn.grad.conv2d_input((B, 3, H, W), W_[0].abs(), dz[0].abs(), stride=4, padding=2) * 2 / scale * 2.0 ** -20
    assert ((d.double() - ref).abs() - bound - 1e-12).max().item() <= 0, "conv1 image gradient"


def _check_unpool(got, relu, dpool, what):
    x = relu.float().contiguous().requires_grad_(True)
    (gref,) = torch.autograd.grad(F.max_pool2d(x, 3, 2), x, dpool.float().contiguous())
    assert torch.equal(got.float(), gref), what


def test_pool_ties_are_first_maximum():
    """Piecewise-constant images through a conv1 of equal weights: relu1 is full of exact ties.  The max pool picks torch's first
    maximum, and the backward routes each gradient to it."""
    sd = lo.random_state_dict(11)
    sd["net.slice1.0.weight"] = torch.full((64, 3, 11, 11), 0.01)
    lp = LPIPS(sd, device=DEV)
    B, H, W = 2, 95, 83
    x0 = (torch.randint(0, 3, (B, 3, H // 8 + 1, W // 8 + 1), device=DEV).float() - 1).repeat_interleave(8, 2).repeat_interleave(8, 3)
    x0 = x0[:, :, :H, :W].contiguous()
    x1 = torch.zeros_like(x0)
    out, d, ws, v = _run_abi(lp.flat, x0, x1, torch.ones(B, device=DEV))
    R = _Regions(ws)
    (h1, w1) = lo.map_shapes(H, W)[0]
    p1 = ((h1 - 3) // 2 + 1, (w1 - 3) // 2 + 1)
    r1 = _nchw(R.take(v.relu[0], 2 * B * h1 * w1 * 64), 2 * B, h1, w1, 64).float().contiguous()
    pooled = _nchw(R.take(v.pool[0], 2 * B * p1[0] * p1[1] * 64), 2 * B, *p1, 64).float()
    arg = R.take(v.pool_arg[0], 2 * B * p1[0] * p1[1] * 64, torch.uint8).view(2 * B, *p1, 64).permute(0, 3, 1, 2)
    rp, ri = F.max_pool2d(r1, 3, 2, return_indices=True)
    win = (ri // w1 - 2 * torch.arange(p1[0], device=DEV).view(1, 1, -1, 1)) * 3 + \
        (ri % w1 - 2 * torch.arange(p1[1], device=DEV).view(1, 1, 1, -1))
    ties = (F.unfold(r1.reshape(-1, 1, h1, w1), 3, stride=2) == rp.reshape(-1, 1, p1[0] * p1[1])).sum(1)
    assert (ties > 1).float().mean().item() > 0.3, "not tie-heavy"
    assert torch.equal(pooled, rp) and torch.equal(arg.long(), win)
    dpool = _nchw(R.take(v.dpool[0], B * p1[0] * p1[1] * 64), B, *p1, 64)
    dnext = _nchw(R.take(v.dnext[0], B * h1 * w1 * 64), B, h1, w1, 64)
    _check_unpool(dnext, r1[:B], dpool, "unpool1 on ties")


@pytest.mark.parametrize("B,H,W", [(2, 1024, 1024), (2, 96, 70)])
def test_module_against_oracle(B, H, W):
    lp, orc, _ = _module(0)
    x0, x1 = _images(B, H, W, seed=H + W)
    a = x0.clone().requires_grad_(True)
    out = lp(a, x1)
    gw = torch.rand(B, 1, 1, 1, device=DEV) + 0.5
    (out * gw).sum().backward()
    r = x0.double().requires_grad_(True)
    ref = orc(r, x1.double())
    (ref * gw.double()).sum().backward()
    assert out.shape == (B, 1, 1, 1)
    val_rel = ((out.double() - ref).abs() / ref.abs()).max().item()
    grad_rel = _rel(a.grad.cpu(), r.grad.cpu())
    print(f"LPIPS {B}x{H}x{W}: value rel {val_rel:.2e}, d_in0 rel-L2 {grad_rel:.2e}")
    assert val_rel < 1e-3           # observed on an H100: <= 1.2e-4
    assert grad_rel < 2.5e-2        # observed: <= 1.9e-2


def test_zero_feature_vectors_on_gpu():
    """All-zero relu1 vectors (a dark patch through a positive conv1 with a negative bias): finite, and as the oracle computes."""
    from test_lpips_cpu import dark_patch_pair, zero_feature_state_dict
    sd = zero_feature_state_dict()
    lp, orc = LPIPS(sd, device=DEV), lo.LpipsOracle(sd).double().to(DEV)
    x0, x1 = (t.to(DEV) for t in dark_patch_pair(B=2, H=64, W=56))
    a = x0.float().requires_grad_(True)
    lp(a, x1.float()).sum().backward()
    r = x0.clone().requires_grad_(True)
    ref = orc(r, x1)
    ref.sum().backward()
    assert torch.isfinite(a.grad).all()
    assert (a.grad[:, :, 18:30, 18:30] == 0).all()
    assert _rel(a.grad.cpu(), r.grad.cpu()) < 3e-2


def test_known_answers():
    lp, _, _ = _module(0)
    B, H, W = 3, 160, 136
    x0, x1 = _images(B, H, W, seed=5)

    def run(a, b):
        a = a.clone().requires_grad_(True)
        out = lp(a, b)
        out.sum().backward()
        torch.cuda.synchronize()
        return out.detach().clone(), a.grad.clone()

    # identical images: exactly zero, with an exactly zero gradient; their features are bit-identical
    v, g = run(x0, x0)
    assert (v == 0).all() and (g == 0).all()
    out, d, ws, views = _run_abi(lp.flat, x0, x0.clone(), torch.ones(B, device=DEV))
    R = _Regions(ws)
    for k, (h, w) in enumerate(lo.map_shapes(H, W)):
        f = R.take(views.relu[k], 2 * B * h * w * lo.CHANNELS[k]).view(2, -1)
        assert torch.equal(f[0], f[1]), f"relu{k + 1}"
    # symmetry, bit for bit
    vab, _ = run(x0, x1)
    vba, _ = run(x1, x0)
    assert torch.equal(vab, vba)
    # frame b of a B = 3 batch equals a B = 1 call on frame b, value and gradient
    v3, g3 = run(x0, x1)
    for b in range(B):
        v1, g1 = run(x0[b:b + 1], x1[b:b + 1])
        assert torch.equal(v3[b], v1[0]) and torch.equal(g3[b], g1[0]), b
    # two runs, bit-identical
    v3b, g3b = run(x0, x1)
    assert torch.equal(v3, v3b) and torch.equal(g3, g3b)


def test_module_rejects_bad_inputs():
    lp, _, _ = _module(0)
    x = torch.zeros(1, 3, 40, 40, device=DEV)
    with pytest.raises(ValueError):
        lp(x, x.clone().requires_grad_(True))
    with pytest.raises(RuntimeError):
        lp(x.cpu(), x.cpu())
    with pytest.raises(ValueError):
        lp(torch.zeros(1, 3, 30, 40, device=DEV), torch.zeros(1, 3, 30, 40, device=DEV))


# ---- trainer --------------------------------------------------------------------------------------------------------------
def _workload():
    from gaussianavatar_b200.workload import Stage1Workload
    wl = Stage1Workload(3, 2, device=DEV, N=4000, S=64, side=128, inp_posmap_size=32)
    with torch.no_grad():
        sd = wl.model.net.state_dict(); sd["decoder.conv8N.bias"] = torch.tensor([-3.9]); wl.model.net.load_state_dict(sd, strict=False)
    wl.make_ground_truth()
    return wl


def _steps(perceptual, use_graph, epoch, n=3):
    from gaussianavatar_b200.trainer import Stage1Trainer
    wl = _workload()
    tr = Stage1Trainer(wl.model, use_graph=use_graph, perceptual_loss=perceptual)
    out = []
    for i in range(n):
        l0 = _lib.launch_count()
        loss = tr.step(wl.device_batch(wl.frame_ids(i)), 5000 + i, epoch=epoch)
        torch.cuda.synchronize()
        out.append((float(loss.detach()), wl.model.net.flat.grad.detach().clone(), wl.model.geo_feature.grad.detach().clone(), _lib.launch_count() - l0))
    tr.finish()
    return out, tr


def test_trainer_before_lpips_start_is_unchanged():
    lp, _, _ = _module(1)
    with_term, _ = _steps(lp, False, epoch=1)
    without, _ = _steps(None, False, epoch=1)
    assert [s[3] for s in with_term] == [s[3] for s in without], "LPIPS kernels launched before lpips_start_iter"
    assert abs(with_term[0][0] - without[0][0]) < 1e-5 * max(1.0, abs(without[0][0]))
    assert _rel(with_term[0][1].cpu(), without[0][1].cpu()) < 1e-3
    assert _rel(with_term[0][2].cpu(), without[0][2].cpu()) < 1e-3


def test_trainer_lpips_step_is_graphed_and_matches_eager():
    lp, _, _ = _module(1)
    eager, tr_e = _steps(lp, False, epoch=31, n=4)
    graph, tr_g = _steps(lp, True, epoch=31, n=4)
    assert tr_g._graphs and not tr_e._graphs
    assert any(k[-1] for k in tr_g._graphs), "the graph key records the active LPIPS term"
    assert abs(eager[0][0] - graph[0][0]) < 1e-5 * max(1.0, abs(eager[0][0]))
    assert _rel(graph[0][1].cpu(), eager[0][1].cpu()) < 1e-3
    assert _rel(graph[0][2].cpu(), eager[0][2].cpu()) < 1e-3
    for (le, *_), (lg, *_) in zip(eager, graph):
        assert abs(le - lg) < 2e-3 * max(1.0, abs(le))


def test_trainer_lpips_term_value():
    from gaussianavatar_b200.trainer import Stage1Trainer
    lp, orc, _ = _module(1)
    wl = _workload()
    batch = wl.device_batch(wl.frame_ids(0))
    tr = Stage1Trainer(wl.model, use_graph=False, perceptual_loss=lp)
    tr0 = Stage1Trainer(wl.model, use_graph=False, perceptual_loss=None)
    with torch.no_grad():
        loss, image = tr.loss(batch, 5000, epoch=31)
        with pytest.warns(UserWarning, match="lpips_start_iter"):
            base, _ = tr0.loss(batch, 5000, epoch=31)   # the same epoch (the offset weight decays with it), no perceptual term
        term = tr.opt.lambda_lpips * orc(image.double(), batch["original_image"].double(), normalize=True).mean()
    got = float(loss) - float(base)
    assert abs(got - float(term)) <= 5e-3 * abs(float(term)) + 1e-5, (got, float(term))
