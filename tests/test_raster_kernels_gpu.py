"""GPU: the rasterizer's compositing forward (K6, render_fwd_kernel) and backward (K7, render_bwd_kernel) element by element
against the fp64 reference of tests/raster_fp64.py, which starts from the kernels' own staged xy / conic_opacity / sorted
lists and carries a rigorous error bound along the kernels' expression trees (derivation in its docstring).

Both APIs are called through the C ABI: ga_raster_forward_preprocess / _render / ga_raster_backward_ex (per frame) and
ga_rasterb_forward / _backward (the batched path the trainer uses).  Every output lies inside a buffer of finite sentinels that
must stay bit-identical; Gaussians with radii == 0 get NaN colours (the sort kernel must never gather them).  The backward's
d_mean2D and d_conic_op are read from the caller's scratch buffer (d_conic_op at align_up(8 B P, 256), see bwd_scratch_bytes).

Tiers, each |got - ref| <= bound on every element checked:
  K6  image, final_T (and n_contrib exactly) on every pixel without a marginal decision; empty tiles equal bg bit for bit.
  K7  d_colors, d_mean2D, d_conic (half off-diagonal), d_opacity of every Gaussian that touches no marginal pixel; Gaussians
      that never blend have exact zeros.  render_bwd_kernel<true> (d_opacities given) and <false> both run.
  decisions  forward and backward take the same entries, pixel by pixel, on a sweep of alpha across 1/255 ulp by ulp.
Each bound must also reject a corrupted copy a plausible bug would produce.  Run with -s for the largest error / bound
ratio per tier and the marginal fractions.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import raster_fp64 as rf
from scenes import random_scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PAD = 300
WORST = {}
MARG = {}
# Marginal pixels / Gaussians are excluded from the element-wise checks, so they must stay rare.  A decision is marginal when
# its threshold lies within the value's bound, a band of relative width ~1e-6 around 1/255 or 1e-4; on the random scenes
# here that is a few pixels in 10^5 at most.  1e-3 leaves room and still fails if a bound blows up.
MARG_MAX = 1e-3


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key, (r, where) in sorted(WORST.items()):
        print(f"\nraster kernels: largest error/bound, {key}: {r:.3g} ({where})")
    for key, (n, tot) in sorted(MARG.items()):
        print(f"raster kernels: marginal {key}: {n} of {tot} ({n / max(tot, 1):.2e})")


def _lib():
    from gaussianavatar_b200 import _lib
    return _lib


def stream():
    return torch.cuda.current_stream().cuda_stream


def ptr(t):
    return None if t is None else t.data_ptr()


def align_up(x, a=256):
    return (x + a - 1) // a * a


class Sent:
    """An output of n floats inside PAD finite sentinels on each side; `ok()` checks the sentinels are bit-identical."""

    def __init__(self, n, seed):
        g = torch.Generator(device=DEV).manual_seed(seed)
        self.buf = torch.randn(n + 2 * PAD, device=DEV, generator=g) * 1000.0
        self.before = self.buf.clone()
        self.t = self.buf[PAD:PAD + n]
        self.n = n

    def ok(self, where):
        d = self.buf.view(torch.int32) != self.before.view(torch.int32)
        d[PAD:PAD + self.n] = False
        assert int(d.sum()) == 0, f"{where}: sentinel words changed"


def ratio(got, ref, bound, mask=None):
    r = (got.double() - ref).abs() / bound.clamp_min(1e-300)
    r = torch.where(bound == 0, torch.where(got.double() == ref, 0.0, math.inf), r)
    r = torch.where(torch.isnan(got), math.inf, r)
    if mask is not None:
        r = r[mask.expand_as(r)]
    return float(r.max()) if r.numel() else 0.0


def check(key, where, got, ref, bound, mask=None):
    r = ratio(got, ref, bound, mask)
    if r > WORST.get(key, (-1.0, ""))[0]:
        WORST[key] = (r, where)
    assert r <= 1.0, f"{key}, {where}: error/bound {r:.4g}"


def rejects(what, bad, ref, bound, mask=None):
    assert ratio(bad, ref, bound, mask) > 1.0, f"self-check: the bound accepts {what}"


def count_marg(key, n, tot):
    a, b = MARG.get(key, (0, 0))
    MARG[key] = (a + n, b + tot)


# ------------------------------------------------------------------------------------------------------------ launches
def run_perframe(sc, bg, dL, opacity_grad=True, seed=0):
    L = _lib()
    lib = L.lib()
    P, H, W = sc["means3D"].shape[0], sc["H"], sc["W"]
    s = L.GaRasterSettings(P, H, W, float(sc["tanfovx"]), float(sc["tanfovy"]), 1.0)
    t = {k: sc[k].to(DEV).float().contiguous() for k in ("means3D", "scales", "rotations", "opacities")}
    view = sc["cam"].world_view_transform.to(DEV).float().contiguous()
    proj = sc["cam"].full_proj_transform.to(DEV).float().contiguous()
    geom = torch.empty(lib.ga_raster_geom_bytes(P), dtype=torch.uint8, device=DEV)
    img = torch.empty(lib.ga_raster_img_bytes(H, W), dtype=torch.uint8, device=DEV)
    radii = torch.empty(max(P, 1), dtype=torch.int32, device=DEV)
    n = ctypes.c_int64(0)
    L.check(lib.ga_raster_forward_preprocess(ctypes.byref(s), ptr(t["means3D"]), ptr(t["scales"]), ptr(t["rotations"]),
                                             ptr(t["opacities"]), ptr(view), ptr(proj), ptr(geom), ptr(img), ptr(radii),
                                             ctypes.byref(n), stream()), "preprocess")
    R = int(n.value)
    colors = sc["colors"].to(DEV).float().clone()
    colors[radii[:P] == 0] = float("nan")
    nb = lib.ga_raster_binning_bytes(R, H, W)
    binning = torch.empty(nb, dtype=torch.uint8, device=DEV)
    bg = bg.to(DEV).float().contiguous()
    out = Sent(3 * H * W, seed)
    L.check(lib.ga_raster_forward_render(ctypes.byref(s), ptr(colors), ptr(bg), ptr(geom), ptr(binning), nb, R, ptr(img), ptr(out.t),
                                         stream()), "render")
    from gaussianavatar_b200.rasterizer import _views
    v = _views(1, P, H, W, R, geom, binning, img, radii[:P])[0]
    scratch = torch.full((lib.ga_raster_bwd_scratch_bytes(P) // 4,), float("nan"), device=DEV)
    o = {k: Sent(c * P, seed + i + 1) for i, (k, c) in enumerate((("d_means3D", 3), ("d_colors", 3), ("d_scales", 3), ("d_rot", 4),
                                                                 ("d_opac", 1), ("d_means2D", 3)))}
    if not opacity_grad:
        o.pop("d_opac")
    dL = dL.to(DEV).float().contiguous()
    L.check(lib.ga_raster_backward_ex(ctypes.byref(s), None, ptr(t["means3D"]), ptr(colors), ptr(t["scales"]), ptr(t["rotations"]),
                                      ptr(bg), ptr(view), ptr(proj), ptr(radii), ptr(geom), ptr(binning), ptr(img), R, ptr(dL),
                                      ptr(scratch), ptr(o["d_means3D"].t), ptr(o["d_colors"].t), ptr(o["d_scales"].t), ptr(o["d_rot"].t),
                                      ptr(o["d_opac"].t) if opacity_grad else None, ptr(o["d_means2D"].t), None, None, stream()),
            "backward")
    torch.cuda.synchronize()
    out.ok("image")
    for k, b in o.items():
        b.ok(k)
    off = align_up(8 * P) // 4
    got = dict(image=out.t.view(3, H, W), final_T=v["final_T"].to(DEV), n_contrib=v["n_contrib"].to(DEV).long(),
               d_colors=o["d_colors"].t.view(P, 3), d_mean2D=scratch[:2 * P].view(P, 2), d_conic_op=scratch[off:off + 4 * P].view(P, 4),
               d_opacity=o["d_opac"].t.view(P, 1) if opacity_grad else None, d_means2D=o["d_means2D"].t.view(P, 3),
               radii=radii[:P], culled_outputs=[o[k].t.view(P, -1) for k in ("d_means3D", "d_scales", "d_rot")])
    fr = rf.Frame(v["xy"], v["conic_opacity"], colors, bg, v["ranges"].long(), v.get("vals_sorted", torch.zeros(0, dtype=torch.int32)).long(), H, W, device=DEV)
    return fr, got, v


def run_batched(scs, bg, dL, rot_pf=None, opac_pf=None, opacity_grad=True, capacity=1 << 16, seed=0):
    """B frames through ga_rasterb_*; rot_pf [B,P,4] / opac_pf [B,P] select per-frame rotations / opacities."""
    from gaussianavatar_b200.rasterizer import _views, pack_cameras
    L = _lib()
    lib = L.lib()
    B, P, H, W = len(scs), scs[0]["means3D"].shape[0], scs[0]["H"], scs[0]["W"]
    cams = pack_cameras(torch.stack([s["cam"].world_view_transform for s in scs]), torch.stack([s["cam"].full_proj_transform for s in scs]),
                        [s["tanfovx"] for s in scs], [s["tanfovy"] for s in scs], DEV)
    st = lambda k: torch.stack([s[k] for s in scs]).to(DEV).float().contiguous()
    means, scales, colors = st("means3D"), st("scales"), st("colors")
    rots = (rot_pf if rot_pf is not None else scs[0]["rotations"]).to(DEV).float().contiguous()
    opac = (opac_pf if opac_pf is not None else scs[0]["opacities"].reshape(-1)).to(DEV).float().contiguous()
    bg = bg.to(DEV).float().contiguous()
    geom = torch.empty(lib.ga_rasterb_geom_bytes(B, P), dtype=torch.uint8, device=DEV)
    img = torch.empty(lib.ga_rasterb_img_bytes(B, H, W), dtype=torch.uint8, device=DEV)
    radii = torch.empty(B, P, dtype=torch.int32, device=DEV)
    out = Sent(B * 3 * H * W, seed)
    for attempt in range(3):
        d = L.GaRasterBatchDesc(B, P, H, W, capacity, 0 if rot_pf is None else 4 * P, 0 if opac_pf is None else P, 1.0)
        binning = torch.empty(lib.ga_rasterb_binning_bytes(B, H, W, capacity), dtype=torch.uint8, device=DEV)
        fwd = lambda: L.check(lib.ga_rasterb_forward(ctypes.byref(d), ptr(cams), ptr(bg), ptr(means), ptr(colors), ptr(scales), ptr(rots),
                                                     ptr(opac), ptr(geom), ptr(img), ptr(binning), ptr(radii), ptr(out.t), stream()), "rasterb_forward")
        fwd()
        torch.cuda.synchronize()
        off = lib.ga_rasterb_status(B, H, W, ptr(img)) - img.data_ptr()
        words = img[off:off + 64].view(torch.int32).cpu()
        if int(words[1]) == 0:
            break
        capacity = int(1.5 * int(words[0])) + 1024
    colors[radii == 0] = float("nan")           # same inputs, same radii: the second forward must not gather these
    fwd()
    scratch = torch.full((lib.ga_rasterb_bwd_scratch_bytes(B, P) // 4,), float("nan"), device=DEV)
    o = {k: Sent(3 * B * P, seed + i + 1) for i, k in enumerate(("d_means3D", "d_colors", "d_scales", "d_means2D"))}
    dop = Sent(B * P, seed + 9) if opacity_grad else None
    dL = dL.to(DEV).float().contiguous()
    L.check(lib.ga_rasterb_backward(ctypes.byref(d), ptr(cams), ptr(bg), ptr(means), ptr(colors), ptr(scales), ptr(rots), ptr(radii),
                                    ptr(geom), ptr(img), ptr(binning), ptr(dL), ptr(scratch), ptr(o["d_means3D"].t), ptr(o["d_colors"].t),
                                    ptr(o["d_scales"].t), None, ptr(dop.t) if dop else None, ptr(o["d_means2D"].t), stream()), "rasterb_backward")
    torch.cuda.synchronize()
    out.ok("image")
    for k, b in o.items():
        b.ok(k)
    if dop:
        dop.ok("d_opac")
    vs = _views(B, P, H, W, capacity, geom, binning, img, radii)
    off = align_up(8 * B * P) // 4
    res = []
    for b in range(B):
        v = vs[b]
        got = dict(image=out.t.view(B, 3, H, W)[b], final_T=v["final_T"].to(DEV), n_contrib=v["n_contrib"].to(DEV).long(),
                   d_colors=o["d_colors"].t.view(B, P, 3)[b], d_mean2D=scratch[:2 * B * P].view(B, P, 2)[b],
                   d_conic_op=scratch[off:off + 4 * B * P].view(B, P, 4)[b],
                   d_opacity=dop.t.view(B, P, 1)[b] if dop else None, d_means2D=o["d_means2D"].t.view(B, P, 3)[b],
                   radii=radii[b], culled_outputs=[o[k].t.view(B, P, 3)[b] for k in ("d_means3D", "d_scales")])
        fr = rf.Frame(v["xy"], v["conic_opacity"], colors[b], bg, v["ranges"].long(), v.get("vals_sorted", torch.zeros(0, dtype=torch.int32)).long(), H, W, device=DEV)
        res.append((fr, got, v))
    return res


# ------------------------------------------------------------------------------------------------------------- checks
def check_frame(where, fr, got, dL, want_restart=False):
    """K6 and K7 tiers of one frame; returns the reference forward / backward for self-checks."""
    fw = rf.forward(fr)
    H, W = fr.H, fr.W
    clear = ~fw["marginal"]
    count_marg("pixels", int(fw["marginal"].sum()), H * W)
    assert float(fw["marginal"].float().mean()) <= MARG_MAX, where
    img, ib = fw["image"]
    check("K6 image", where, got["image"], img, ib, clear[None].expand(3, H, W))
    check("K6 final_T", where, got["final_T"], fw["final_T"][0], fw["final_T"][1], clear)
    assert torch.equal(got["n_contrib"][clear], fw["n_contrib"][clear]), f"{where}: n_contrib"
    # pixels of empty tiles: bg bit for bit
    empty = torch.ones(fr.gy * 16, fr.gx * 16, dtype=torch.bool, device=fr.dev)
    lens = fr.ranges[:, 1] - fr.ranges[:, 0]
    nonempty = (lens > 0).reshape(fr.gy, fr.gx)
    empty &= ~nonempty.repeat_interleave(16, 0).repeat_interleave(16, 1)
    empty = empty[:H, :W]
    bgf = fr.bg.float()[:, None]
    assert torch.equal(got["image"][:, empty], bgf.expand(3, int(empty.sum()))), f"{where}: empty tiles"
    if want_restart:
        assert bool((fw["tile_last"] > 256).any()), f"{where}: no pixel restarts from a checkpoint"

    bw = rf.backward(fr, fw, dL)
    keep = ~bw["excluded"]
    count_marg("Gaussians", int(bw["excluded"].sum()), int((fr.ntiles > 0).sum()))
    check("K7 d_colors", where, got["d_colors"], *bw["d_colors"], keep[:, None].expand(-1, 3))
    check("K7 d_mean2D", where, got["d_mean2D"], *bw["d_mean2D"], keep[:, None].expand(-1, 2))
    check("K7 d_mean2D out", where, got["d_means2D"][:, :2], *bw["d_mean2D"], keep[:, None].expand(-1, 2))
    assert bool((got["d_means2D"][:, 2] == 0).all())
    check("K7 d_conic", where, got["d_conic_op"][:, :3], *bw["d_conic"], keep[:, None].expand(-1, 3))
    if got["d_opacity"] is not None:
        check("K7 d_opacity", where, got["d_opacity"], *bw["d_opacity"], keep[:, None])
        check("K7 d_opacity", where, got["d_conic_op"][:, 3:], *bw["d_opacity"], keep[:, None])
    else:
        assert bool((got["d_conic_op"][:, 3] == 0).all()), f"{where}: render_bwd_kernel<false> wrote d_opacity"
    # never blended (unlisted / culled included): exact zeros
    none = keep & (bw["active"] == 0)
    for k in ("d_colors", "d_mean2D", "d_conic_op"):
        assert bool((got[k][none] == 0).all()), f"{where}: {k} of a Gaussian that never blends"
    culled = got["radii"] == 0
    for t in got["culled_outputs"] + [got["d_means2D"]] + ([got["d_opacity"]] if got["d_opacity"] is not None else []):
        assert bool((t[culled] == 0).all()), f"{where}: a gradient of a culled Gaussian is not zero"
    # the marginal exclusion must leave the case's Gaussians checked: at most a quarter of those that blend may drop out
    act = bw["active"] > 0
    kept = int((act & keep).sum())
    assert kept >= 0.75 * int(act.sum()), f"{where}: only {kept} of {int(act.sum())} blending Gaussians held to the bound"
    return fw, bw


def _dl(H, W, seed, B=None):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*(() if B is None else (B,)), 3, H, W, generator=g)


CASES = [
    dict(P=300, H=64, W=80, seed=1, scale_mean=0.03),
    dict(P=2000, H=200, W=136, seed=2, scale_mean=0.02),
    dict(P=5000, H=256, W=256, seed=3, scale_mean=0.01, aniso=False, opacity_one=True),
    dict(P=1500, H=128, W=128, seed=4, scale_mean=0.05, spread=2.5),
    dict(P=800, H=96, W=96, seed=5, scale_mean=0.02, z_extra=2.4),
] + [dict(P=60, H=h, W=w, seed=10 + i, scale_mean=0.03, spread=0.1) for i, (h, w) in
     enumerate([(1, 1), (1, 17), (17, 1), (7, 9), (16, 16), (33, 45)])]


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"P{c['P']}_{c['H']}x{c['W']}")
def test_perframe_sizes(case):
    sc = random_scene(**case)
    H, W = sc["H"], sc["W"]
    bg = torch.rand(3, generator=torch.Generator().manual_seed(case["seed"])) if case["seed"] % 2 else torch.ones(3)
    dL = _dl(H, W, case["seed"])
    fr, got, v = run_perframe(sc, bg, dL, opacity_grad=case["seed"] % 3 != 0, seed=case["seed"])
    fw, bw = check_frame(f"per-frame {H}x{W}", fr, got, dL.to(DEV))
    if case["seed"] == 3:
        # self-checks on the avatar's regime (opacity 1, T stops, bg = 1)
        bad = rf.forward(fr, stop_late=True)
        rejects("the T stop applied to the entry after the one that triggers it", bad["image"][0], *fw["image"], ~fw["marginal"])
        badb = rf.backward(fr, fw, dL.to(DEV), use_bg_dot=False)
        rejects("bg_dot omitted", badb["d_opacity"][0], *bw["d_opacity"], ~bw["excluded"][:, None])


def _one_tile_scene(n, seed, cut=None):
    """n Gaussians whose rects all cover the single tile of a 16x16 image, low opacity: pixels blend deep into the list.  With
    `cut`, the Gaussians from depth rank `cut` on get opacity 0.002 < 1/255: none of them blends, so the last contributors land
    just before list position `cut` and the segments from there on start past tile_maxc."""
    sc = random_scene(P=n, H=16, W=16, seed=seed, scale_mean=0.02, aniso=False, spread=0.05)
    g = torch.Generator().manual_seed(seed + 1)
    sc["opacities"] = (0.01 + 0.05 * torch.rand(n, 1, generator=g)).contiguous()
    if cut is not None:
        ph = torch.cat([sc["means3D"].double(), torch.ones(n, 1, dtype=torch.float64)], 1)
        tz = (ph @ sc["cam"].world_view_transform.double())[:, 2]
        sc["opacities"][torch.argsort(tz)[cut:]] = 0.002
    return sc


LIST_LENGTHS = [1, 31, 32, 33, 255, 256, 257, 512, 513, 2048, 2049, 8193]
CUTS = {512: 256, 513: 258}
# the edge each case must reach: a last contributor at 0-based list position 256 (n_contrib 257), 255 with the last segment
# starting past tile_maxc, 257 likewise; a warp that blends its last entry before half the list while others go on
LAST_AT = {257: 257, 512: 256, 513: 258}
PAST_MAXC = (512, 513)
EARLY_WARP = (8193,)


@pytest.mark.parametrize("n", LIST_LENGTHS)
def test_one_tile_list_lengths(n):
    sc = _one_tile_scene(n, 100 + n, CUTS.get(n))
    bg = torch.rand(3, generator=torch.Generator().manual_seed(n))
    dL = _dl(16, 16, n)
    fr, got, v = run_perframe(sc, bg, dL, opacity_grad=n % 2 == 1, seed=n)
    assert int(fr.len[0]) == n                                  # the tile's list really is n long
    fw, bw = check_frame(f"one tile, list {n}", fr, got, dL.to(DEV), want_restart=n > 600)
    nc = fw["n_contrib"]
    maxc = int(nc.max())
    if n in LAST_AT:
        assert bool((nc == LAST_AT[n]).any()), f"list {n}: no last contributor at 1-based position {LAST_AT[n]}"
    if n in PAST_MAXC:
        assert (n - 1) // 256 * 256 >= maxc, f"list {n}: the last segment does not start at or past tile_maxc"
    if n in EARLY_WARP:
        last = nc.reshape(4, 4, 2, 8).permute(0, 2, 1, 3).reshape(8, 32).max(1).values     # per 8x4 sub-tile (warp)
        early = (last > 0) & (last * 2 < maxc)
        assert bool(early.any()), f"list {n}: no warp blends its last entry before half the list"
    if n == 2049:
        bad = rf.backward(fr, fw, dL.to(DEV), restart=False)
        rejects("the checkpoint restart replaced by (T_final, 0)", bad["d_colors"][0], *bw["d_colors"], ~bw["excluded"][:, None])
        bad = rf.backward(fr, fw, dL.to(DEV), skip=(0, 1))
        rejects("one segment's contribution missing from d_colors", bad["d_colors"][0], *bw["d_colors"], ~bw["excluded"][:, None])


def test_eccentric_gaussians_cull_margin():
    """Gaussians with eccentricity up to 100:1 and opacities from just above 1/255 to 1: a non-conservative cull_radius2
    would drop pairs whose pixels pass; the reference does not cull.  Measures how close to the cull radius passing pixels lie."""
    P, H, W = 3000, 128, 128
    sc = random_scene(P=P, H=H, W=W, seed=71, scale_mean=0.01, aniso=True)
    g = torch.Generator().manual_seed(72)
    ecc = torch.exp(torch.rand(P, generator=g) * math.log(100.0))
    sc["scales"] = (0.004 * torch.stack([ecc, torch.ones(P), torch.ones(P)], 1)).contiguous()
    ang = torch.full((P,), math.pi / 8)                         # 45 degrees about z
    sc["rotations"] = torch.stack([torch.cos(ang), torch.zeros(P), torch.zeros(P), torch.sin(ang)], 1).contiguous()
    sc["opacities"] = torch.exp(torch.rand(P, 1, generator=g) * math.log(255.0 * 1.0) + math.log(1.0 / 255.0 * 1.02)).clamp(max=1.0)
    bg = torch.rand(3, generator=g)
    dL = _dl(H, W, 73)
    fr, got, v = run_perframe(sc, bg, dL, seed=7)
    check_frame("eccentric", fr, got, dL.to(DEV))
    # cull_radius2 restated in fp64: 2.002 (ln(255 o) + 0.01) / lmin', lmin' = lmin - 1e-5 |mid|
    co = fr.co
    mid, hd = 0.5 * (co[:, 0] + co[:, 2]), 0.5 * (co[:, 0] - co[:, 2])
    lmin = mid - torch.sqrt(hd * hd + co[:, 1] ** 2) - 1e-5 * mid.abs()
    r2 = 2.002 * (torch.log(255.0 * co[:, 3]) + 0.01) / lmin
    best, where = 0.0, None
    for k in range(int(fr.len[0])):
        m = fr.prefix(k)
        e = fr.entry(m, k)
        ok = e["ok"].reshape(m, 4, 4, 2, 8)                    # (tile, sub-row, row, sub-col, col)
        gg = e["g"]
        for sy in range(4):
            for sx in range(2):
                hit = ok[:, sy, :, sx, :].any((1, 2))
                if not hit.any():
                    continue
                x0 = (fr.tiles[:m] % fr.gx) * 16 + sx * 8
                y0 = (fr.tiles[:m] // fr.gx) * 16 + sy * 4
                c = fr.xy[gg]
                ex = torch.clamp(torch.maximum(x0 - c[:, 0], c[:, 0] - (x0 + 7)), min=0)
                ey = torch.clamp(torch.maximum(y0 - c[:, 1], c[:, 1] - (y0 + 3)), min=0)
                d2 = ex * ex + ey * ey
                q = torch.where(hit, d2 / r2[gg], -1.0)
                if float(q.max()) > best:
                    best, where = float(q.max()), (int(q.argmax()), k, sx, sy)
    print(f"\nraster kernels: passing pixels reach {math.sqrt(best):.4f} of the cull radius")
    assert best > 0.99 ** 2
    # self-check: the pair nearest the cull margin dropped, as a cull radius 1 % too small would drop it
    t, k, sx, sy = where
    sub = (fr.px[t] // 8 % 2 == sx) & (fr.py[t] // 4 % 4 == sy)
    bad = rf.forward(fr, drop=(t, k, sub))
    fw = rf.forward(fr)
    rejects("the (sub-tile, entry) pair nearest the cull margin dropped", bad["image"][0], *fw["image"], ~fw["marginal"])


def test_batched_b3_per_frame_rotations_and_opacities():
    """Three frames of one scene whose rotations and opacities differ per frame by about 1e-3 (rot_stride = 4P, opac_stride = P):
    close enough that frames swapped in the batched outputs are a fine-grained self-check."""
    scs = [random_scene(P=2500, H=120, W=152, seed=81, scale_mean=0.02) for i in range(3)]
    B, P = 3, 2500
    g = torch.Generator().manual_seed(84)
    rot = scs[0]["rotations"][None] + 1e-3 * torch.randn(B, P, 4, generator=g)
    rot = rot / rot.norm(dim=-1, keepdim=True)
    opac = (torch.rand(P, generator=g) * 0.95 + 0.05)[None] * (1 - 1e-3 * torch.rand(B, P, generator=g))
    bg = torch.rand(3, generator=g)
    dL = _dl(120, 152, 85, B=3)
    res = run_batched(scs, bg, dL, rot_pf=rot, opac_pf=opac)
    for b, (fr, got, v) in enumerate(res):
        check_frame(f"batched B=3 frame {b}", fr, got, dL[b].to(DEV))
    # self-check: frames swapped in the batched outputs
    fw0 = rf.forward(res[0][0])
    rejects("frames 0 and 1 swapped", res[1][1]["image"], *fw0["image"], ~fw0["marginal"][None].expand(3, -1, -1))


def test_batched_config3_two_frames():
    """The Gaussians the workload poses at config 3 (200k, 1024^2), B = 2 in one set of launches, opacity 1, bg 1."""
    from gaussianavatar_b200.workload import Stage1Workload
    wl = Stage1Workload(3, 1, device=DEV)
    m = wl.model
    with torch.no_grad():
        means, scales, colors, _ = m._posed_gaussians(torch.tensor([3, 9], device=DEV), 5000)
    c = wl.cam
    scs = [dict(means3D=means[b].float(), scales=scales[b].float(), colors=colors[b].float(), cam=c, H=wl.side, W=wl.side,
                tanfovx=math.tan(c.FovX / 2), tanfovy=math.tan(c.FovY / 2), rotations=m.fix_rotation.float(),
                opacities=m.fix_opacity.float()) for b in range(2)]
    dL = _dl(wl.side, wl.side, 91, B=2)
    res = run_batched(scs, m.background.float(), dL, opacity_grad=False, capacity=8 * means.shape[1])
    for b, (fr, got, v) in enumerate(res):
        assert int(fr.len[0]) > 256
        fw, bw = check_frame(f"config 3 frame {b}", fr, got, dL[b].to(DEV), want_restart=True)
    # config 3 is square, so H and W swapped in the d_mean2D scaling is checked on a non-square frame
    sc = random_scene(P=2000, H=200, W=136, seed=2, scale_mean=0.02)
    dL1 = _dl(200, 136, 2)
    fr, got, v = run_perframe(sc, torch.ones(3), dL1, seed=2)
    fw = rf.forward(fr)
    bw = rf.backward(fr, fw, dL1.to(DEV))
    bad = rf.backward(fr, fw, dL1.to(DEV), swap_hw=True)
    rejects("H and W swapped in the d_mean2D scaling", bad["d_mean2D"][0], *bw["d_mean2D"], ~bw["excluded"][:, None])


def _unproject(cam, pix, z, W, H):
    """World points at view depth z (camera looking down its axis) that project to pixel centres `pix` [n,2] (fp64)."""
    Mp = cam.full_proj_transform.double()
    Mv = cam.world_view_transform.double()
    # the cameras here have identity extrinsics: view = world up to the matrix convention; solve the affine map numerically
    def proj(X, Y):
        p = torch.stack([X, Y, torch.full_like(X, z), torch.ones_like(X)], -1)
        h = p @ Mp
        ndc = h[:, :2] / (h[:, 3:4] + 1e-7)
        return torch.stack([((ndc[:, 0] + 1) * W - 1) * 0.5, ((ndc[:, 1] + 1) * H - 1) * 0.5], -1)
    z0 = torch.zeros(1, dtype=torch.float64)
    b = proj(z0, z0)[0]
    ax = proj(z0 + 1, z0)[0] - b
    ay = proj(z0, z0 + 1)[0] - b
    A = torch.stack([ax, ay], 1)
    XY = torch.linalg.solve(A, (pix - b).T).T
    return torch.cat([XY, torch.full((pix.shape[0], 1), z, dtype=torch.float64)], 1)


def test_forward_backward_take_the_same_entries():
    """One-pixel Gaussians on a 3-pixel grid: a front Gaussian whose alpha is swept across 1/255 ulp by ulp (sub-pixel offsets,
    so power rounds) over an opaque one.  The forward took the front entry iff final_T = (1 - a_f)(1 - a_b) rather than
    1 - a_b; the backward took it iff its d_opacity is non-zero (dL/dalpha = 3 T with white front, black back, bg 0).
    They must agree on every pixel."""
    from gaussianavatar_b200.camera import make_camera
    H = W = 192
    K = np.array([[400.0, 0, W / 2], [0, 400.0, H / 2], [0, 0, 1]], dtype=np.float32)
    cam = make_camera(K, np.eye(4), H, W)
    g = torch.Generator().manual_seed(7)
    gy, gx = torch.meshgrid(torch.arange(1, H - 1, 3), torch.arange(1, W - 1, 3), indexing="ij")
    centres = torch.stack([gx.flatten(), gy.flatten()], 1).double()
    n = centres.shape[0]
    off = (0.1 + 0.35 * torch.rand(n, 2, generator=g, dtype=torch.float64)) * torch.where(torch.rand(n, 2, generator=g) < 0.5, -1.0, 1.0)
    front = _unproject(cam, centres + off, 2.0, W, H)
    back = _unproject(cam, centres - 0.3 * off, 2.5, W, H)
    P = 2 * n
    sc = dict(means3D=torch.cat([front, back]).float(), scales=torch.full((P, 3), 1e-5), rotations=torch.tensor([[1.0, 0, 0, 0]]).repeat(P, 1),
              colors=torch.cat([torch.ones(n, 3), torch.zeros(n, 3)]), opacities=torch.ones(P, 1), cam=cam, H=H, W=W,
              tanfovx=math.tan(cam.FovX / 2), tanfovy=math.tan(cam.FovY / 2))
    dL = torch.ones(3, H, W)
    fr, got, v = run_perframe(sc, torch.zeros(3), dL)
    # the kernel's own fp32 xy / conic: set the front opacities so that alpha at the own pixel sweeps 1/255 by -8 .. +8 ulp
    xy, co = v["xy"][:n].double(), v["conic_opacity"][:n].double()
    dx, dy = xy[:, 0] - centres[:, 0], xy[:, 1] - centres[:, 1]
    G = torch.exp(-0.5 * (co[:, 0] * dx * dx + co[:, 2] * dy * dy) - co[:, 1] * dx * dy)
    k = (torch.arange(n) % 17 - 8).double()
    o_f = (rf.A_THR / G * (1 + k * 2.0 ** -23)).float()
    sc["opacities"] = torch.cat([o_f[:, None], torch.ones(n, 1)])
    fr, got, v = run_perframe(sc, torch.zeros(3), dL)
    cx, cy = centres[:, 0].long(), centres[:, 1].long()
    assert bool((v["radii"] > 0).all())
    xb, cb = v["xy"][n:].double(), v["conic_opacity"][n:].double()
    dx, dy = xb[:, 0] - centres[:, 0], xb[:, 1] - centres[:, 1]
    a_b = torch.exp(-0.5 * (cb[:, 0] * dx * dx + cb[:, 2] * dy * dy) - cb[:, 1] * dx * dy).clamp(max=rf.CAP)
    T_no = (1 - a_b).to(DEV)
    fT = got["final_T"][cy.to(DEV), cx.to(DEV)].double()
    fwd_take = fT < T_no * (1 - 0.5 * rf.A_THR)
    assert bool(((fT - T_no).abs() < 1e-5 * T_no).logical_or((fT - T_no * (1 - rf.A_THR)).abs() < 1e-5 * T_no).all())   # nothing else
    fwd_take = fwd_take.cpu()
    bwd_take = (got["d_opacity"][:n, 0] != 0).cpu()
    dis = int((fwd_take != bwd_take).sum())
    print(f"\nraster kernels: front entries taken {int(fwd_take.sum())} of {n}; forward/backward disagree on {dis}")
    assert dis == 0
    assert int(fwd_take.sum()) >= 300 and int((~fwd_take).sum()) >= 300
    # the reference calls most of these decisions marginal: they really straddle the threshold
    fw = rf.forward(fr)
    nm = int(fw["marginal"][cy.to(DEV), cx.to(DEV)].sum())
    print(f"raster kernels: {nm} of these pixels are marginal for the reference")
    assert nm >= 300
