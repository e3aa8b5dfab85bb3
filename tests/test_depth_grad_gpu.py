"""GPU: training against depth, kernel by kernel, through the C ABI.

  * ga_rasterb_forward_depth_train: images, depth planes, radii, final_T, n_contrib and status equal ga_rasterb_forward_depth's bit
    for bit; the stored D (every read checkpoint and the end of each list) matches the running sum of the call's own staged
    entries (raster_fp64's walk of the colours (z, 0, 0)) within its bound.
  * ga_rasterb_backward_depth: d_mean2D, d_conic_op, d_opacity and dL/dz element by element against tests/depth_fp64.py; with
    dL/dm = 0, dL/dz is exactly 0 and every gradient agrees with ga_rasterb_backward; d_means3D against raster_fp64's preprocess
    backward plus dL/dz times the view matrix's z row.
  * Each comparison rejects a plausible bug: the m T_final / (1 - alpha) term dropped, the 1 / A factor dropped, dL/dz dropped, a
    restarted segment starting from zacc = 0.
  * The masked L1 depth loss: value, N and gradient against fp64; N = 0; two graph replays bit for bit.
Cases: B from 1 to 8, H and W not multiples of 16, tile lists past 256 entries, and the step's size (200k Gaussians, 1024^2, B = 2).
Run with -s for the largest error / bound per quantity.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import depth_fp64 as dfp
import raster_fp64 as rf
from scenes import random_scene
from test_raster_kernels_gpu import _one_tile_scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key, (r, where) in sorted(WORST.items()):
        print(f"\ndepth grad: largest error/bound, {key}: {r:.3g} ({where})")


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


def _L():
    from gaussianavatar_b200 import _lib
    return _lib


def ptr(t):
    return None if t is None else t.data_ptr()


def align_up(x, a=256):
    return (x + a - 1) // a * a


def _kernel_order():
    """Walk pixel k (row-major in the tile) -> the kernel's thread: one warp per 8x4 sub-tile."""
    k = torch.arange(256)
    lx, ly = k % 16, k // 16
    return ((ly // 4) * 2 + lx // 8) * 32 + (ly % 4) * 8 + lx % 8


# ------------------------------------------------------------------------------------------------------------ launches
def run(scs, dL, g, opacity_grad=False, capacity=None):
    """The frames through ga_rasterb_forward_depth_train + ga_rasterb_backward_depth, and through ga_rasterb_forward_depth +
    ga_rasterb_backward on a second plan.  Returns a dict of the outputs and the per-frame staged views."""
    from gaussianavatar_b200.rasterizer import RasterBatchPlan, _views, pack_cameras
    L = _L()
    lib = L.lib()
    B, P, H, W = len(scs), scs[0]["means3D"].shape[0], scs[0]["H"], scs[0]["W"]
    cams = pack_cameras(torch.stack([s["cam"].world_view_transform for s in scs]), torch.stack([s["cam"].full_proj_transform for s in scs]),
                        [s["tanfovx"] for s in scs], [s["tanfovy"] for s in scs], DEV)
    st = lambda k: torch.stack([s[k] for s in scs]).to(DEV).float().contiguous()
    means, scales, colors = st("means3D"), st("scales"), st("colors")
    rots = scs[0]["rotations"].to(DEV).float().contiguous()
    opac = scs[0]["opacities"].reshape(-1).to(DEV).float().contiguous()
    bg = scs[0].get("bg", torch.ones(3)).to(DEV).float().contiguous()
    cap = capacity or 8 * B * P
    plan, ref = RasterBatchPlan(B, P, H, W, DEV, capacity=cap), RasterBatchPlan(B, P, H, W, DEV, capacity=cap)
    plan.alloc_depth()
    plan.depth_state.view(torch.float32).fill_(float("nan"))          # a slot the backward reads must have been written
    desc = plan.desc()
    d = ctypes.byref(desc)
    img, depth = torch.empty(B, 3, H, W, device=DEV), torch.empty(B, 2, H, W, device=DEV)
    L.check(lib.ga_rasterb_forward_depth_train(d, ptr(depth), ptr(plan.depth_state), plan.depth_state.numel(), ptr(cams), ptr(bg), ptr(means),
                                               ptr(colors), ptr(scales), ptr(rots), ptr(opac), ptr(plan.geom), ptr(plan.img), ptr(plan.binning),
                                               ptr(plan.radii), ptr(img), torch.cuda.current_stream().cuda_stream), "forward_depth_train")
    img_r, depth_r = torch.empty_like(img), torch.empty_like(depth)
    L.check(lib.ga_rasterb_forward_depth(d, None, None, ptr(depth_r), ptr(cams), ptr(bg), ptr(means), ptr(colors), ptr(scales), ptr(rots),
                                         ptr(opac), ptr(ref.geom), ptr(ref.img), ptr(ref.binning), ptr(ref.radii), ptr(img_r),
                                         torch.cuda.current_stream().cuda_stream), "forward_depth")
    torch.cuda.synchronize()
    assert int(plan.status_dev[1]) == 0 and int(ref.status_dev[1]) == 0, "capacity"
    out = dict(B=B, P=P, H=H, W=W, cams=cams, means=means, scales=scales, rots=rots, img=img, depth=depth, img_r=img_r, depth_r=depth_r,
               plan=plan, ref=ref)
    dL, g = dL.to(DEV).float().contiguous(), g.to(DEV).float().contiguous()
    BP = B * P

    def bwd(gm, depth_plan):
        scratch = torch.full((plan.depth_scratch.numel() // 4,), float("nan"), device=DEV)
        o = {k: torch.empty(B, P, c, device=DEV) for k, c in (("d_means3D", 3), ("d_colors", 3), ("d_scales", 3))}
        dop = torch.empty(B, P, device=DEV) if opacity_grad else None
        if depth_plan:
            L.check(lib.ga_rasterb_backward_depth(d, ptr(cams), ptr(bg), ptr(means), ptr(colors), ptr(scales), ptr(rots), ptr(plan.radii),
                                                  ptr(plan.geom), ptr(plan.img), ptr(plan.binning), ptr(dL), ptr(gm), ptr(depth),
                                                  ptr(plan.depth_state), plan.depth_state.numel(), ptr(scratch), scratch.numel() * 4,
                                                  ptr(o["d_means3D"]), ptr(o["d_colors"]), ptr(o["d_scales"]), None, ptr(dop), None,
                                                  torch.cuda.current_stream().cuda_stream), "backward_depth")
        else:
            L.check(lib.ga_rasterb_backward(d, ptr(cams), ptr(bg), ptr(means), ptr(colors), ptr(scales), ptr(rots), ptr(ref.radii), ptr(ref.geom),
                                            ptr(ref.img), ptr(ref.binning), ptr(dL), ptr(scratch), ptr(o["d_means3D"]), ptr(o["d_colors"]),
                                            ptr(o["d_scales"]), None, ptr(dop), None, torch.cuda.current_stream().cuda_stream), "backward")
        torch.cuda.synchronize()
        off, offz = align_up(8 * BP) // 4, (align_up(8 * BP) + align_up(16 * BP)) // 4
        o.update(d_mean2D=scratch[:2 * BP].view(B, P, 2), d_conic_op=scratch[off:off + 4 * BP].view(B, P, 4), d_opacity=dop,
                 d_z=scratch[offz:offz + BP].view(B, P) if depth_plan else None)
        return o

    out["grad"] = bwd(g, True)
    out["grad0"] = bwd(torch.zeros_like(g), True)
    out["grad_ref"] = bwd(None, False)
    out["views"] = _views(B, P, H, W, cap, plan.geom, plan.binning, plan.img, plan.radii)
    out["views_r"] = _views(B, P, H, W, cap, ref.geom, ref.binning, ref.img, ref.radii)
    out["colors"], out["bg"], out["dL"], out["g"] = colors, bg, dL, g
    return out


def _state_of(o):
    """(ckpt, final) float views of the depth state, and seg_start [B*T+1] from the lists' lengths."""
    from gaussianavatar_b200 import _lib
    B, H, W = o["B"], o["H"], o["W"]
    T = ((W + 15) // 16) * ((H + 15) // 16)
    plan = o["plan"]
    st = plan.depth_state.view(torch.float32)
    lens = torch.cat([v["ranges"][:, 1].long() - v["ranges"][:, 0].long() for v in o["views"]])
    segs = (lens + 255) // 256
    seg_start = torch.cat([torch.zeros(1, dtype=torch.long), torch.cumsum(segs, 0)])
    nck = _lib.lib().ga_rasterb_depth_state_bytes(B, H, W, plan.capacity)
    maxseg = plan.capacity // 256 + B * T + 1
    ck = st[:maxseg * 256]
    fin_off = align_up(maxseg * 256 * 4) // 4
    fin = st[fin_off:fin_off + B * T * 256]
    assert fin_off * 4 + B * T * 256 * 4 <= nck
    return ck, fin, seg_start, T


# ------------------------------------------------------------------------------------------------------------- checks
def check_case(where, o, mutations=False, restarts=False):
    B, P, H, W = o["B"], o["P"], o["H"], o["W"]
    # 1. the training forward is ga_rasterb_forward_depth, bit for bit
    assert torch.equal(o["img"], o["img_r"]) and torch.equal(o["depth"], o["depth_r"]), where
    assert torch.equal(o["plan"].radii, o["ref"].radii), where
    words = [0, 1, 2, 3, 13] + list(range(4, 5 + B))
    assert torch.equal(o["plan"].status_dev[words], o["ref"].status_dev[words]), where
    ck, fin, seg_start, T = _state_of(o)
    perm = _kernel_order().to(DEV)
    any_restart = False
    for b in range(B):
        v, vr = o["views"][b], o["views_r"][b]
        assert torch.equal(v["final_T"], vr["final_T"]) and torch.equal(v["n_contrib"], vr["n_contrib"]), where
        fr = rf.Frame(v["xy"], v["conic_opacity"], o["colors"][b], o["bg"], v["ranges"].long(), v["vals_sorted"].long(), H, W, device=DEV)
        z = v["depth"].to(DEV).double()
        fw, fwz = rf.forward(fr), rf.forward(dfp.indicator(fr, z))
        clear = ~fw["tile_marg"] & fr.inside
        blk = b * T + fr.tiles
        # 2. the stored D: the end of every list, and every checkpoint the backward reads (a pixel blending past it)
        got = fin.view(B * T, 256)[blk][:, perm]
        check("D final", where, got, fwz["tile_C"][0][0], fwz["tile_C"][0][1], clear)
        for j in range(1, len(fwz["ckpts"])):
            mj = fr.prefix(j * 256)
            read = clear[:mj] & (fw["tile_last"][:mj] > j * 256)
            if not read.any():
                continue
            any_restart = True
            rows = (seg_start.to(DEV)[blk[:mj]] + j)
            got = ck.view(-1, 256)[rows][:, perm]
            check("D checkpoint", where, got, fwz["ckpts"][j][2][0][0], fwz["ckpts"][j][2][0][1], read)
        # 3. the backward against the fp64 restatement
        gr = o["grad"]
        bw = dfp.backward(fr, fw, fwz, z, o["dL"][b], o["g"][b], o["depth"][b, 0])
        keep = ~bw["excluded"]
        act = bw["active"] > 0
        assert int((act & keep).sum()) >= 0.75 * int(act.sum()), where
        check("d_mean2D", where, gr["d_mean2D"][b], *bw["d_mean2D"], keep[:, None])
        check("d_conic", where, gr["d_conic_op"][b][:, :3], *bw["d_conic"], keep[:, None])
        check("dL/dz", where, gr["d_z"][b][:, None], *bw["d_z"], keep[:, None])
        if gr["d_opacity"] is not None:
            check("d_opacity", where, gr["d_opacity"][b][:, None], *bw["d_opacity"], keep[:, None])
        else:
            assert bool((gr["d_conic_op"][b][:, 3] == 0).all())
        assert bool((gr["d_z"][b][keep & ~act] == 0).all()), f"{where}: dL/dz of a Gaussian that never blends"
        assert float(bw["d_z"][0].abs().max()) > 0, where
        # 4. dL/dm = 0: dL/dz exactly 0, the rest as ga_rasterb_backward (both within the colour-only restatement's bound)
        g0, gref = o["grad0"], o["grad_ref"]
        assert bool((g0["d_z"][b] == 0).all()), where
        bw0 = rf.backward(fr, fw, o["dL"][b])
        keep0 = ~bw0["excluded"]
        for k, r in (("d_mean2D", "d_mean2D"), ("d_conic_op", "d_conic")):
            gv = g0[k][b][:, :3] if k == "d_conic_op" else g0[k][b]
            gw = gref[k][b][:, :3] if k == "d_conic_op" else gref[k][b]
            check(f"{r} (dL/dm = 0)", where, gv, *bw0[r], keep0[:, None])
            check(f"{r} (ga_rasterb_backward)", where, gw, *bw0[r], keep0[:, None])
        # 5. d_means3D: the preprocess backward plus dL/dz times the view matrix's z row
        c = o["cams"][b]
        inp = dict(means=o["means"][b], view=c[0:16], proj=c[16:32], tanfovx=float(c[32]), tanfovy=float(c[33]), H=H, W=W, mod=1.0,
                   radii=o["plan"].radii[b], cov3d=v["cov3d"].to(DEV), d_mean2D=gr["d_mean2D"][b], d_conic_op=gr["d_conic_op"][b],
                   scales=o["scales"][b], rots=o["rots"], depth=v["depth"])
        pb = rf.preprocess_backward(**inp)
        assert not bool(pb["marg_overflow"].any())
        view = c[0:16].double()
        dz = gr["d_z"][b].double()
        dm = [rf.add((pb["d_means3D"][0][:, k], pb["d_means3D"][1][:, k]), rf.mul((view[4 * k + 2], 0.0), (dz, 0.0))) for k in range(3)]
        vis = pb["vis"][:, None]
        ref_v = torch.where(vis, torch.stack([x[0] for x in dm], 1), 0.0)
        ref_e = torch.where(vis, torch.stack([x[1] for x in dm], 1), 0.0)
        check("d_means3D", where, gr["d_means3D"][b], ref_v, ref_e)
        if mutations and b == 0:
            rejects("dL/dz times the z row missing from d_means3D", gr["d_means3D"][b], pb["d_means3D"][0], pb["d_means3D"][1],
                    vis & (dz.abs() > 0)[:, None])
        if mutations and b == 0:
            for bug in ("no_m_term", "no_inv_A"):
                bad = dfp.backward(fr, fw, fwz, z, o["dL"][b], o["g"][b], o["depth"][b, 0], bug=(bug,))
                rejects(bug, bad["d_conic"][0], *bw["d_conic"], keep[:, None])
            rejects("dL/dz dropped", torch.zeros_like(gr["d_z"][b])[:, None], *bw["d_z"], keep[:, None])
        if restarts and mutations and b == 0:
            bad = dfp.backward(fr, fw, fwz, z, o["dL"][b], o["g"][b], o["depth"][b, 0], bug=("restart_zero",))
            rejects("a restarted segment from zacc = 0", bad["d_conic"][0], *bw["d_conic"], keep[:, None])
    if restarts:
        assert any_restart, f"{where}: no pixel restarts from a checkpoint"


def _frames(B, P, H, W, seed, **kw):
    scs = [random_scene(P=P, H=H, W=W, seed=seed + b, **kw) for b in range(B)]
    for s in scs[1:]:
        s["rotations"], s["opacities"] = scs[0]["rotations"], scs[0]["opacities"]
    return scs


def _grads(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, 3, H, W, generator=g), torch.randn(B, H, W, generator=g)


CASES = [dict(B=1, P=300, H=64, W=80, seed=1, scale_mean=0.03), dict(B=3, P=2000, H=100, W=140, seed=2, scale_mean=0.02),
         dict(B=8, P=400, H=40, W=56, seed=3, scale_mean=0.03), dict(B=2, P=1500, H=97, W=33, seed=4, scale_mean=0.05)]


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"B{c['B']}_P{c['P']}_{c['H']}x{c['W']}")
def test_depth_grad_random_frames(case):
    c = dict(case)
    B, P, H, W, seed = c.pop("B"), c.pop("P"), c.pop("H"), c.pop("W"), c.pop("seed")
    scs = _frames(B, P, H, W, 10 * seed, **c)
    dL, g = _grads(B, H, W, seed)
    o = run(scs, dL, g, opacity_grad=seed % 2 == 0)
    check_case(f"B={B} {H}x{W}", o, mutations=seed == 2)


def test_depth_grad_long_lists():
    """Tile lists of 2049 entries (one tile, low opacities): the backward's segments restart from the stored D."""
    scs = [_one_tile_scene(2049, 300 + b) for b in range(2)]
    for s in scs[1:]:
        s["rotations"], s["opacities"] = scs[0]["rotations"], scs[0]["opacities"]
    dL, g = _grads(2, 16, 16, 5)
    o = run(scs, dL, g, opacity_grad=True)
    check_case("one tile, list 2049", o, mutations=True, restarts=True)


def test_depth_grad_config3():
    """The Gaussians the workload poses at config 3 (200k, 1024^2), B = 2, opacity 1, bg 1, and dL/dm the depth loss would give."""
    from gaussianavatar_b200.workload import Stage1Workload
    wl = Stage1Workload(3, 1, device=DEV)
    m = wl.model
    with torch.no_grad():
        means, scales, colors, _ = m._posed_gaussians(torch.tensor([3, 9], device=DEV), 5000)
    c = wl.cam
    scs = [dict(means3D=means[b].float(), scales=scales[b].float(), colors=colors[b].float(), cam=c, H=wl.side, W=wl.side,
                tanfovx=math.tan(c.FovX / 2), tanfovy=math.tan(c.FovY / 2), rotations=m.fix_rotation.float(), opacities=m.fix_opacity.float(),
                bg=m.background.float().cpu()) for b in range(2)]
    dL, g = _grads(2, wl.side, wl.side, 91)
    g = torch.sign(g) * 1e-6
    o = run(scs, dL, g, capacity=8 * means.shape[1])
    check_case("config 3", o, restarts=True)


# ---- the depth loss ---------------------------------------------------------------------------------------------------------------
def _loss_case(B, H, W, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    depth = torch.rand(B, 2, H, W, device=DEV, generator=g) * 3 + 0.3
    depth[:, 1][torch.rand(B, H, W, device=DEV, generator=g) < 0.3] = 0          # uncovered / less than half opaque
    depth[:, 0][depth[:, 1] == 0] *= torch.rand(int((depth[:, 1] == 0).sum()), device=DEV, generator=g)
    target = torch.rand(B, H, W, device=DEV, generator=g) * 3 + 0.3
    target[torch.rand(B, H, W, device=DEV, generator=g) < 0.2] = 0                # holes / outside the mask
    target[0].view(-1)[:7] = depth[0, 0].reshape(-1)[:7]                        # sign(0) = 0 pixels
    depth[0, 1].view(-1)[:7] = 1.0
    return depth, target


@pytest.mark.parametrize("B,H,W", [(1, 33, 47), (2, 1024, 1024), (8, 100, 140)])
def test_depth_loss_against_fp64(B, H, W):
    from gaussianavatar_b200.losses import depth_loss
    depth, target = _loss_case(B, H, W, B + H)
    lam = 0.7
    d = depth.clone().requires_grad_(True)
    loss, n = depth_loss(d, target, lam, return_count=True)
    loss.backward()
    counted = (target > 0) & (depth[:, 1] != 0)
    N = int(counted.sum())
    assert int(n) == N > 0
    diff = depth[:, 0].double() - target.double()
    want = lam * diff.abs()[counted].sum() / N
    # per-CTA float sums of <= 256 terms (8-level shuffle tree, then 8 warps), then double: gamma(16) of the absolute sum
    assert abs(float(loss) - float(want)) <= rf.gam(16) * float(want) + 2 ** -24 * float(want), (float(loss), float(want))
    coef = float(np.float32(float(np.float32(lam)) / N))
    gwant = torch.where(counted, torch.sign(diff).float() * coef, torch.zeros_like(target))
    assert torch.equal(d.grad[:, 0], gwant) and bool((d.grad[:, 1] == 0).all())
    assert bool((d.grad[:, 0][counted & (diff == 0)] == 0).all()) and int((counted & (diff == 0)).sum()) >= 1
    # self-check: the unmasked mean is a different number
    assert abs(float(diff.abs().mean() * lam) - float(loss)) > 1e-3 * float(loss)


def test_depth_loss_no_counted_pixels():
    from gaussianavatar_b200.losses import depth_loss
    depth, target = _loss_case(2, 40, 30, 3)
    d = depth.clone().requires_grad_(True)
    loss, n = depth_loss(d, torch.zeros_like(target), 1.0, return_count=True)
    loss.backward()
    assert float(loss) == 0.0 and int(n) == 0 and bool((d.grad == 0).all())
    depth[:, 1] = 0
    d = depth.clone().requires_grad_(True)
    loss = depth_loss(d, target, 1.0)
    loss.backward()
    assert float(loss) == 0.0 and bool((d.grad == 0).all())


def test_depth_loss_graph_replays_bit_for_bit():
    from gaussianavatar_b200.losses import depth_loss
    depth, target = _loss_case(2, 512, 512, 9)
    d = depth.clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            d.grad = None
            depth_loss(d, target, 1.0).backward()
    torch.cuda.current_stream().wait_stream(s)
    d.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = depth_loss(d, target, 1.0)
        loss.backward()
    out = []
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        out.append((loss.clone(), d.grad.clone()))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
    eager = depth_loss(depth, target, 1.0)
    assert torch.equal(eager, out[0][0])
