"""GPU: the LPIPS head launches of csrc/lpips.cu (lpips_dist1..5, lpips_sum, lpips_dnorm1..5), every element against the bounded
fp64 reference of tests/lpips_fp64.py from the launch's own inputs in the workspace (derivation of the bounds in its docstring).

`ga_lpips_forward` and `ga_lpips_backward` run once per case through the C ABI on a sentinel-filled workspace, read back through
`ga_lpips_views`.  Tiers, each |got - ref| <= bound on every element:
  dist     each of the 5 B nblk_k partials from the device's own relu_k; partial slots nblk_k..127 keep the sentinel bytes.
  sum      out[b] from the device's own partials; the recorded in_scale equals the caller's bit for bit.
  dnorm    dz_k for k = 4..0 from the device's own relu_k, lin_k, g and dnext_k: exact zeros where f0 <= 0, TF32 values everywhere.
  exact    a frame with g_b = 0 has dz_k = 0 for every k and d_in0 = 0; identical images give zero partials and dz; negating g
           negates dz_5 and d_in0 (every fp32 operation on the way, tf32_rn and the tensor-core data gradients are sign-symmetric).
Each bound must also reject a corrupted copy of its reference that a plausible bug would produce.  Run with -s for the largest
error / bound per tier and the corruptions rejected.  dnorm's largest ratio sits just under 1 by construction: its bound is
dominated by the final TF32 rounding, whose half ulp reaches 2^-11 |v| for v just above a power of two, so a wrong dz shows once
it moves by about 5e-4 of |dz| plus the few fp32 ulps of the terms it is made of.
"""
import pytest
import torch

import lpips_fp64 as lf
from gaussianavatar_b200.lpips import LPIPS
from oracle import lpips_oracle as lo
from test_lpips_cpu import dark_patch_pair, zero_feature_state_dict
from test_lpips_gpu import DEV, SENTINEL, SIZES, _images, _module, _Regions, _run_abi

pytestmark = pytest.mark.gpu
WORST = {}
REJECTED = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key, (r, where) in sorted(WORST.items()):
        print(f"\nlpips head: largest error/bound, {key}: {r:.3g} ({where})")
    for key, layers in sorted(REJECTED.items()):
        print(f"lpips head: rejected {key} (layers {layers})")


def _note(tier, r, where):
    if r > WORST.get(tier, (-1.0, ""))[0]:
        WORST[tier] = (r, where)


def geometry(B, H, W):
    """Per layer: HW, nblk and each dist CTA's busiest warp's pixel count (min, max over CTAs)."""
    HW = [h * w for h, w in lo.map_shapes(H, W)]
    nb = [lf.nblk(n) for n in HW]
    m = [lf.assignment(n, b)[1] for n, b in zip(HW, nb)]
    return dict(h=[h for h, _ in lo.map_shapes(H, W)], HW=HW, nblk=nb, m=[(int(x.min()), int(x.max())) for x in m])


# (id, B, H, W, features, the launch geometry or regime the case reaches)
CASES = [(f"{B}x{H}x{W}", B, H, W, "random", "") for B, H, W in SIZES] + [
    ("nblk128", 1, 259, 515, "random", "conv1's map 64x128: HW = 8192, nblk exactly 128, every warp 8 pixels"),
    ("nblk_capped", 1, 259, 519, "random", "HW = 8256: nblk capped at 128, CTAs 0..7 take a 9th pixel per warp"),
    ("one_pixel", 2, 31, 31, "random", "HW_3..5 = 1: 7 of 8 warps of the one dist CTA idle"),
    ("zero_f0", 2, 64, 56, "zero0", "all-zero rendered relu1 vectors: n0 = 0"),
    ("zero_f1", 2, 64, 56, "zero1", "all-zero ground-truth relu1 vectors: n1 = 0, d1 = 1e-10"),
    ("tiny", 2, 96, 70, "tiny", "conv1 scaled by 1e-12: |relu1| ~ 1e-11, the 1e-10 epsilon a visible share of d"),
    ("lin_zero", 3, 96, 70, "linzero", "every third lin weight 0: only the projection term there"),
    ("identical", 3, 67, 45, "same", "identical images: partials and dz exactly 0"),
]
# the cases whose corrupted references must be rejected at every layer where the corruption changes the value
SELF_CHECK = {"2x512x384", "3x67x45", "lin_zero"}


def test_cases_reach_their_geometry():
    geo = {c[0]: geometry(*c[1:4]) for c in CASES}
    assert geo["1x31x2047"]["h"][2:] == [1, 1, 1]                           # single-row maps at conv3..5
    assert geo["nblk128"]["HW"][0] == 8192 and geo["nblk128"]["nblk"][0] == 128 and geo["nblk128"]["m"][0] == (8, 8)
    assert geo["nblk_capped"]["HW"][0] == 8256 and geo["nblk_capped"]["nblk"][0] == 128 and geo["nblk_capped"]["m"][0] == (8, 9)
    assert geo["one_pixel"]["HW"][2:] == [1, 1, 1] and geo["one_pixel"]["nblk"][2:] == [1, 1, 1]
    HW = geo["3x67x45"]["HW"][2]                                             # B = 3, odd HW: dnorm's 8-warp CTAs straddle frames
    assert HW % 2 == 1 and any(len({q // HW for q in range(8 * c, min(8 * c + 8, 3 * HW))}) > 1 for c in range(-(-3 * HW // 8)))
    assert all(g["nblk"][0] == 128 and g["m"][0][1] > 8 for k, g in geo.items() if k.endswith("1024x1024"))
    for c in CASES:
        print(f"\n{c[0]}: HW {geo[c[0]]['HW']}, nblk {geo[c[0]]['nblk']}, warp pixels {geo[c[0]]['m']} {c[5]}")


_SD = {}


def _setup(kind, B, H, W):
    """(module, state dict, x0, x1, in_scale, in_shift) of a case."""
    if kind in ("random", "same"):
        lp, _, sd = _module(0)
        x0, x1 = _images(B, H, W, seed=B * 7 + H)
        return lp, sd, x0, x0.clone() if kind == "same" else x1, 2.0, -1.0
    if kind not in _SD:
        if kind in ("zero0", "zero1"):
            sd = zero_feature_state_dict()
        else:
            sd = lo.random_state_dict(2)
            if kind == "tiny":
                sd["net.slice1.0.weight"] = sd["net.slice1.0.weight"] * 1e-12
                sd["net.slice1.0.bias"] = sd["net.slice1.0.bias"] * 1e-12
            else:
                for k in range(5):
                    sd[lo.lin_key(k)].view(-1)[::3] = 0
        _SD[kind] = (LPIPS(sd, device=DEV), sd)
    lp, sd = _SD[kind]
    if kind in ("zero0", "zero1"):
        a, b = (t.float().to(DEV).contiguous() for t in dark_patch_pair(B=B, H=H, W=W))
        x0, x1 = (a, b) if kind == "zero0" else (b, a)
        return lp, sd, x0, x1, 1.0, 0.0
    x0, x1 = _images(B, H, W, seed=H + W)
    return lp, sd, x0, x1, 0.7, 0.1


def _g(B):
    """g_out per frame: positive, negative and 0 across a batch."""
    return torch.tensor([0.75, -1.5, 0.0][:B], device=DEV)


def _views(B, H, W, ws, v):
    R = _Regions(ws)
    ms, C = lo.map_shapes(H, W), lo.CHANNELS
    relu = [R.take(v.relu[k], 2 * B * h * w * C[k]).view(2 * B, h, w, C[k]) for k, (h, w) in enumerate(ms)]
    part = R.take(v.partials, 5 * B * 128).view(5, B, 128)
    in_scale = R.take(v.in_scale, 1)
    dz = [R.take(v.dz[k], B * h * w * C[k]).view(B, h, w, C[k]) for k, (h, w) in enumerate(ms)]
    dnext = [R.take(v.dnext[k], B * h * w * C[k]).view(B, h, w, C[k]) for k, (h, w) in enumerate(ms[:4])]
    return relu, part, in_scale, dz, dnext


def _lin(sd, k):
    return sd[lo.lin_key(k)].reshape(-1).float().to(DEV)


def _flat_as(t, like):
    """t's buffer read with like's shape (zeros past its end): what a kernel handed the wrong layer's pointer would see."""
    out = torch.zeros(like.numel(), dtype=t.dtype, device=t.device)
    n = min(t.numel(), like.numel())
    out[:n] = t.reshape(-1)[:n]
    return out.view(like.shape)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_head_launches_against_fp64(case):
    name, B, H, W, kind, _ = case
    lp, sd, x0, x1, in_scale, in_shift = _setup(kind, B, H, W)
    g = _g(B)
    out, d_in0, ws, v = _run_abi(lp.flat, x0, x1, g, in_scale=in_scale, in_shift=in_shift)
    relu, part, ins, dz, dnext = _views(B, H, W, ws, v)
    geo = geometry(B, H, W)
    HW, nb = geo["HW"], geo["nblk"]
    lins = [_lin(sd, k) for k in range(5)]

    # dist: every partial the sum reads, and not one slot more
    dists = [lf.layer_distance(relu[k], lins[k], B) for k in range(5)]
    pref = [lf.partials(dists[k], nb[k]) for k in range(5)]
    pbytes = part.view(torch.uint8).view(5, B, 128, 4)
    for k in range(5):
        r = lf.ratio(part[k, :, :nb[k]], pref[k])
        _note("dist", float(r.max()), f"{name} layer {k + 1}")
        assert float(r.max()) <= 1.0, f"lpips_dist{k + 1}: error/bound {float(r.max()):.3g} at {divmod(int(r.argmax()), nb[k])}"
        assert (pbytes[k, :, nb[k]:] == SENTINEL).all(), f"lpips_dist{k + 1} wrote past its {nb[k]} partials"
    # sum
    sref = lf.lpips_sum(part, nb, HW)
    r = lf.ratio(out, sref)
    _note("sum", float(r.max()), name)
    assert float(r.max()) <= 1.0, f"lpips_sum: error/bound {float(r.max()):.3g}"
    assert ins.view(torch.int32).item() == torch.tensor([in_scale], dtype=torch.float32).view(torch.int32).item()
    # dnorm, in launch order
    drefs = {}
    for k in range(4, -1, -1):
        gn = dnext[k] if k < 4 else None
        drefs[k] = lf.dnorm(relu[k], lins[k], g, gn, HW[k])
        got = dz[k].reshape(B, -1, lo.CHANNELS[k])
        r = lf.ratio(got, drefs[k])
        _note("dnorm", float(r.max()), f"{name} layer {k + 1}")
        assert torch.isfinite(drefs[k][1]).all()
        assert float(r.max()) <= 1.0, f"lpips_dnorm{k + 1}: error/bound {float(r.max()):.3g} at {int(r.argmax())}"
        assert (got[relu[k][:B].reshape(got.shape) <= 0] == 0).all(), f"lpips_dnorm{k + 1}: nonzero where f0 <= 0"
        assert lf.is_tf32(got), f"lpips_dnorm{k + 1}: not a TF32 value"
    # known answers exact in fp32
    for b in range(B):
        if float(g[b]) == 0:
            assert all((dz[k][b] == 0).all() for k in range(5)) and (d_in0[b] == 0).all(), f"frame {b}: g = 0"
    if kind == "same":
        assert (part == 0).sum() == sum(B * n for n in nb) and all((dz[k] == 0).all() for k in range(5)) and (out == 0).all()

    if name in SELF_CHECK:
        _self_check(name, B, relu, lins, part, g, dnext, HW, nb, dists, pref, sref, drefs)
    if kind == "tiny":   # sqrt(s + eps) for sqrt(s) + eps: visible only where eps is a share of |f|
        assert lf.rejects(lf.partials(lf.layer_distance(relu[0], lins[0], B, eps_inside=True), nb[0])[0], pref[0])
        assert lf.rejects(lf.dnorm(relu[0], lins[0], g, dnext[0], HW[0], eps_inside=True)[0], drefs[0])
        REJECTED.setdefault("sqrt(s + eps) [dist, dnorm]", set()).add(1)


def _self_check(name, B, relu, lins, part, g, dnext, HW, nb, dists, pref, sref, drefs):
    def rejected(key, k, ok):
        assert ok, f"{name}: {key} not rejected at layer {k + 1}"
        REJECTED.setdefault(key, set()).add(k + 1)

    for k in range(5):
        bad = pref[k][0].clone()
        bad[0, nb[k] // 2] = 0
        rejected("one CTA's partial zeroed [dist]", k, lf.rejects(bad, pref[k]))
        short = list(nb)
        short[k] -= 1
        if short[k] > 0:
            rejected("one partial slot not read [sum]", k, lf.rejects(lf.lpips_sum(part, short, HW)[0], sref))
        for j in (k - 1, k + 1):
            if 0 <= j < 5 and HW[j] != HW[k]:
                wrong = list(HW)
                wrong[k] = HW[j]
                rejected("HW of layer k+-1 [sum]", k, lf.rejects(lf.lpips_sum(part, nb, wrong)[0], sref))
                rejected("HW of layer k+-1 [dnorm]", k, lf.rejects(
                    lf.dnorm(relu[k], lins[k], g, dnext[k] if k < 4 else None, HW[j])[0], drefs[k]))
        gn = dnext[k] if k < 4 else None
        rejected("projection term dropped [dnorm]", k, lf.rejects(lf.dnorm(relu[k], lins[k], g, gn, HW[k], drop_proj=True)[0], drefs[k]))
        rejected("mask from f1 [dnorm]", k, lf.rejects(lf.dnorm(relu[k], lins[k], g, gn, HW[k], mask_f1=True)[0], drefs[k]))
        if k < 4:
            rejected("dnext not added [dnorm]", k, lf.rejects(lf.dnorm(relu[k], lins[k], g, None, HW[k])[0], drefs[k]))
        for j in (k - 1, k + 1):
            if 0 <= j < 4:
                wrong = _flat_as(dnext[j], relu[k][:B])
                rejected("dnext of layer k+-1 [dnorm]", k, lf.rejects(lf.dnorm(relu[k], lins[k], g, wrong, HW[k])[0], drefs[k]))


@pytest.mark.parametrize("B,H,W", [(3, 67, 45), (2, 512, 384)])
def test_negated_g_negates_the_gradient(B, H, W):
    """Every fp32 operation of lpips_dnorm_kernel and tf32_rn is sign-symmetric, so -g gives -dz_5 bit for bit; the data gradients,
    un-pooling and the image gradient are sums of products with dz, so d_in0 follows (zeros of either sign compare equal)."""
    lp, _, _ = _module(0)
    x0, x1 = _images(B, H, W, seed=B + W)
    g = torch.tensor([0.75, -1.5, 1.25][:B], device=DEV)
    _, d_pos, ws_p, v_p = _run_abi(lp.flat, x0, x1, g)
    _, d_neg, ws_n, v_n = _run_abi(lp.flat, x0, x1, -g)
    dz_p, dz_n = _views(B, H, W, ws_p, v_p)[3], _views(B, H, W, ws_n, v_n)[3]
    assert (dz_p[4] != 0).any()
    assert torch.equal(-dz_p[4], dz_n[4]), "dz_5"
    same = [torch.equal(-dz_p[k], dz_n[k]) for k in range(5)]
    print(f"\nlpips head {B}x{H}x{W}: -g negates dz_1..5 {same}, d_in0 {torch.equal(-d_pos, d_neg)}")
    assert all(same) and torch.equal(-d_pos, d_neg), "d_in0"
