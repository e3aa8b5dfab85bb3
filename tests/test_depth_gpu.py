"""GPU: the depth pass of the batched forward (ga_rasterb_forward_depth, rasterizer.rasterize_batch_depth) and of the player.

  * Nothing else changes: with depth on, images, final T, n_contrib, radii, status and mattes equal the same call without depth.
  * Mean depth (plane 0) bit for bit against an indicator render: colours (z, 0, 0), bg 0, whose red channel is D = sum w z.
  * Median depth (plane 1) against an fp64 walk over the call's own staged buffers (tests/raster_fp64.py's entries and tracked
    operations): exact on clear pixels, one of the walk's two candidates on pixels where a T-versus-0.5 comparison is marginal.
  * Known answers: one opaque Gaussian, two layers, an opaque wall in front of an avatar.
  * The player (animate.Ensemble / Animator with depth) and tools/animate.py --depth.
Run with -s for the share of marginal pixels of the median check.
"""
import contextlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import raster_fp64 as rf
from gaussianavatar_b200 import animate as an
from gaussianavatar_b200.avatar_model import kept_state
from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, TEST_POSE_K, make_camera, scaled_intrinsics
from gaussianavatar_b200.rasterizer import (RasterBatchPlan, _views, rasterize_batch, rasterize_batch_depth, rasterize_batch_mattes,
                                            rasterize_batch_scene)
from scene_fixture import random_static, scene_of
from scenes import random_scene
from test_cast_gpu import SIDE, _camera, _close, _model, _pair, _random_first, _scene
from test_scene_gpu import _cams, _frames, _wall

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WRITTEN = [0, 1, 2, 3, 13]            # status words every forward writes: instances, overflow, segments, tiles, long tiles
MARG = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key, (n, tot) in sorted(MARG.items()):
        print(f"\ndepth: marginal pixels of the median check, {key}: {n} of {tot} ({n / max(tot, 1):.2e})")


def _dyn(scs):
    t = {k: torch.stack([s[k] for s in scs]).to(DEV) for k in ("means3D", "colors", "scales")}
    return t["means3D"], t["colors"], t["scales"], scs[0]["rotations"].to(DEV), scs[0]["opacities"].to(DEV)


def _views_of(plan):
    """Per-frame staged buffers of the plan's last forward (host copies): depth, xy, conic_opacity, ranges, vals_sorted, final_T,
    n_contrib, radii."""
    return _views(plan.B, plan.P + plan.static_P, plan.H, plan.W, plan.capacity, plan.geom, plan.binning, plan.img, plan.radii)


def _status(plan):
    return plan.status_dev[WRITTEN + list(range(4, 5 + plan.B))].cpu()


# ---- 1. nothing else changes ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("with_scene", [False, True])
@pytest.mark.parametrize("K", [None, 1, 3, 8])
def test_depth_changes_nothing_else(K, with_scene, B):
    """Images, final T, n_contrib, radii, status and (with sets) mattes of the depth call equal the same call without depth, bit for
    bit; depth is finite, >= 0, and 0 exactly where nothing was blended (plane 0) / where the final T > 0.5 (plane 1).  Ragged tiles."""
    H, W, P, Ps = 100, 140, 2000, 2500
    scs = _frames(B, H, W, P, seed=30 + 10 * (K or 0) + B)
    means, colors, scales, rot, opac = _dyn(scs)
    cams, bg = _cams(scs), scs[0]["bg"].to(DEV)
    scene = scene_of(random_static(Ps, 1, seed=41, center=(0.0, -0.2, 0.2), spread=(0.8, 1.0, 0.6))).to(DEV) if with_scene else None
    sP = Ps if with_scene else 0
    first = None if K is None else _random_first(P, K, seed=K + 5 * B, full=K != 3)
    with torch.no_grad():
        plan_d, plan = RasterBatchPlan(B, P, H, W, DEV, static_P=sP), RasterBatchPlan(B, P, H, W, DEV, static_P=sP)
        out = rasterize_batch_depth(means, colors, scales, rot, opac, cams, bg, plan_d, scene, first)
        if first is not None:
            img, mattes = rasterize_batch_mattes(means, colors, scales, rot, opac, cams, bg, plan, first, scene)
            assert len(out) == 3 and torch.equal(out[1], mattes)
        elif scene is not None:
            img = rasterize_batch_scene(means, colors, scales, rot, opac, cams, bg, plan, scene)
        else:
            img = rasterize_batch(means, colors, scales, rot, opac, cams, bg, plan)
        assert plan_d.check(wait=True) and plan.check(wait=True)
    depth = out[-1]
    assert depth.shape == (B, 2, H, W) and out[0].shape == (B, 3, H, W)
    assert torch.equal(out[0], img) and torch.equal(plan_d.radii, plan.radii) and torch.equal(_status(plan_d), _status(plan))
    vd, v = _views_of(plan_d), _views_of(plan)
    for b in range(B):
        assert torch.equal(vd[b]["final_T"], v[b]["final_T"]) and torch.equal(vd[b]["n_contrib"], v[b]["n_contrib"])
        assert torch.equal(vd[b]["vals_sorted"], v[b]["vals_sorted"])
        dp = depth[b].cpu()
        assert torch.isfinite(dp).all() and (dp >= 0).all()
        assert torch.equal(dp[0] == 0, v[b]["n_contrib"] == 0)
        assert ((dp[1] == 0) == (v[b]["final_T"] > 0.5)).all()


# ---- 2. mean depth against an indicator render ------------------------------------------------------------------------------------
def _mean_from(C0, final_T, n_contrib):
    return torch.where(n_contrib > 0, C0 / (1.0 - final_T), torch.zeros_like(C0))


@pytest.mark.parametrize("with_scene", [False, True])
def test_mean_depth_equals_indicator_render(with_scene):
    """Plane 0 is where(n_contrib > 0, C0 / (1 - final T), 0) in fp32 torch ops, C0 the red channel of a render with colours
    (z, 0, 0), bg = 0, and z the call's own view depths.  With a scene the indicator render splats [dynamic; static] as one dynamic
    set, whose point lists, staged xy / conic_o and depths are first checked to be the composite's."""
    B, H, W, P, Ps = 2, 100, 140, 2500, 3000
    scs = [random_scene(P=P, H=H, W=W, seed=70 + b, scale_mean=0.03) for b in range(B)]
    for s in scs[1:]:
        s["rotations"], s["opacities"] = scs[0]["rotations"], scs[0]["opacities"]
    means, colors, scales, rot, opac = _dyn(scs)
    cams, bg = _cams(scs), scs[0]["bg"].to(DEV)
    scene = scene_of(random_static(Ps, 0, seed=72, center=(0.0, -0.2, 0.0), spread=(0.8, 1.0, 0.8))).to(DEV) if with_scene else None
    sP = Ps if with_scene else 0
    with torch.no_grad():
        plan_d = RasterBatchPlan(B, P, H, W, DEV, static_P=sP)
        img, depth = rasterize_batch_depth(means, colors, scales, rot, opac, cams, bg, plan_d, scene)
        assert plan_d.check(wait=True)
        vd = _views_of(plan_d)
        z = torch.stack([vd[b]["depth"] for b in range(B)]).to(DEV)                                       # [B, P + Ps]
        if scene is not None:
            means = torch.cat([means, scene.means3D.expand(B, Ps, 3)], 1).contiguous()
            scales = torch.cat([scales, scene.scales.expand(B, Ps, 3)], 1).contiguous()
            rot = torch.cat([rot, scene.rotations]).contiguous()
            opac = torch.cat([opac.reshape(-1), scene.opacities.reshape(-1)]).contiguous()
        ind = torch.zeros(B, P + sP, 3, device=DEV)
        ind[..., 0] = z
        plan_i = RasterBatchPlan(B, P + sP, H, W, DEV)
        red = rasterize_batch(means, ind, scales, rot, opac, cams, torch.zeros(3, device=DEV), plan_i)[:, 0]
        assert plan_i.check(wait=True)
    vi = _views_of(plan_i)
    for b in range(B):
        assert torch.equal(vi[b]["radii"], vd[b]["radii"])
        for k in ("vals_sorted", "ranges"):
            assert torch.equal(vi[b][k], vd[b][k]), (b, k)
        seen = vd[b]["radii"] > 0                      # a culled Gaussian's staged slots are never written, nor read
        for k in ("xy", "conic_opacity", "depth"):
            assert torch.equal(vi[b][k][seen], vd[b][k][seen]), (b, k)
        assert torch.equal(vi[b]["final_T"], vd[b]["final_T"]) and torch.equal(vi[b]["n_contrib"], vd[b]["n_contrib"])
        want = _mean_from(red[b], vd[b]["final_T"].to(DEV), vd[b]["n_contrib"].to(DEV))
        assert torch.equal(depth[b, 0], want), b
        assert (vd[b]["n_contrib"] > 0).float().mean() > 0.3


# ---- 3. median depth against an fp64 walk -----------------------------------------------------------------------------------------
def median_walk(fr, z):
    """The median along the kernel's path: the z of the first blended entry after which T <= 0.5, with T carried as (value, bound)
    by raster_fp64's tracked operations.  Returns per pixel [H, W]: "lo" / "hi", the medians with T read at value - bound and value
    + bound in the two comparisons (the walk's candidates; they differ only where a comparison is marginal), "marg", whether any
    blend decision is marginal, and the corrupted medians "first" (the first blended entry's z), "last" (the last contributor's)
    and "late" (the crossing taken at T < 0.5: the first entry blended once T is already below 0.5)."""
    nt, dev = fr.tiles.numel(), fr.dev
    zero = torch.zeros(nt, 256, dtype=torch.float64, device=dev)
    T = (torch.ones_like(zero), zero.clone())
    done = ~fr.inside.clone()
    marg = torch.zeros(nt, 256, dtype=torch.bool, device=dev)
    got = {k: zero.clone() for k in ("lo", "hi", "first", "last", "late")}
    seen_first, seen_late = marg.clone(), marg.clone()
    for k in range(int(fr.len.max()) if nt else 0):
        m = fr.prefix(k)
        e = fr.entry(m, k)
        ok, alpha, live = e["ok"], e["alpha"], ~done[:m]
        Tm = (T[0][:m], T[1][:m])
        test_T = rf.mul(Tm, rf.sub(1.0, alpha))
        stop = live & ok & (test_T[0] < fr.t_thr)
        take = live & ok & ~stop
        zk = z[e["g"]][:, None].expand(m, 256)
        for key, s in (("lo", -1.0), ("hi", 1.0)):
            cross = take & (Tm[0] + s * Tm[1] > 0.5) & (test_T[0] + s * test_T[1] <= 0.5)
            got[key][:m] = torch.where(cross, zk, got[key][:m])
        got["first"][:m] = torch.where(take & ~seen_first[:m], zk, got["first"][:m])
        seen_first[:m] |= take
        got["last"][:m] = torch.where(take, zk, got["last"][:m])
        late = take & (Tm[0] < 0.5) & ~seen_late[:m]
        got["late"][:m] = torch.where(late, zk, got["late"][:m])
        seen_late[:m] |= late
        T[0][:m], T[1][:m] = rf.where(take, test_T, Tm)
        done[:m] |= stop
        marg[:m] |= live & (e["marg"] | (ok & rf.marg_lt(test_T, fr.t_thr)))
    H, W = fr.H, fr.W
    ins = fr.inside
    pid = (fr.py * W + fr.px)[ins]
    out = {}
    for key, t in list(got.items()) + [("marg", marg)]:
        img = torch.zeros(H * W, dtype=t.dtype, device=dev)
        img[pid] = t[ins]
        out[key] = img.reshape(H, W)
    return out


@pytest.mark.parametrize("with_scene", [False, True])
def test_median_depth_against_fp64_walk(with_scene):
    """Clear pixels (no marginal decision, both candidates equal) match the walk exactly; a marginal pixel equals one of the two
    candidates.  The check rejects the first blended entry's z, the last contributor's, and the crossing taken at T < 0.5."""
    B, H, W, P, Ps = 2, 100, 140, 3000, 2500
    scs = [random_scene(P=P, H=H, W=W, seed=80 + b, scale_mean=0.03) for b in range(B)]       # opacities spread over (0, 1)
    for s in scs[1:]:
        s["rotations"], s["opacities"] = scs[0]["rotations"], scs[0]["opacities"]
    means, colors, scales, rot, opac = _dyn(scs)
    cams, bg = _cams(scs), scs[0]["bg"].to(DEV)
    scene = scene_of(random_static(Ps, 1, seed=83, center=(0.0, -0.2, 0.0), spread=(0.8, 1.0, 0.8))).to(DEV) if with_scene else None
    with torch.no_grad():
        plan = RasterBatchPlan(B, P, H, W, DEV, static_P=Ps if with_scene else 0)
        _, depth = rasterize_batch_depth(means, colors, scales, rot, opac, cams, bg, plan, scene)
        assert plan.check(wait=True)
    key = "scene" if with_scene else "dynamic"
    for b, v in enumerate(_views_of(plan)):
        n = v["xy"].shape[0]
        fr = rf.Frame(v["xy"], v["conic_opacity"], torch.zeros(n, 3), torch.zeros(3), v["ranges"].long(), v["vals_sorted"].long(), H, W,
                      device=DEV)
        wk = median_walk(fr, v["depth"].to(DEV).double())
        got = depth[b, 1].double()
        marginal = wk["marg"] | (wk["lo"] != wk["hi"])
        clear = ~marginal
        MARG[key] = tuple(a + c for a, c in zip(MARG.get(key, (0, 0)), (int(marginal.sum()), H * W)))
        assert marginal.float().mean().item() <= 1e-3
        assert torch.equal(got[clear], wk["lo"][clear]), b
        assert ((got == wk["lo"]) | (got == wk["hi"]))[(wk["lo"] != wk["hi"]) & ~wk["marg"]].all(), b
        assert (wk["lo"] > 0).float().mean().item() > 0.2                      # the median is set on much of the frame
        for bad in ("first", "last", "late"):
            assert (wk[bad][clear] != wk["lo"][clear]).any(), f"self-check: the median check accepts the {bad!r} corruption"


# ---- 4. known answers -------------------------------------------------------------------------------------------------------------
def _axis_gaussians(zs, sizes, opacities, H=64, W=64):
    """Isotropic Gaussians on the reference camera's optical axis at view depths zs; the frame, and the view depths the kernels
    computed."""
    E = TEST_POSE_EXTRINSIC
    Rc, tc = E[:3, :3], E[:3, 3]
    C = -Rc.T @ tc
    xyz = np.stack([np.array([0.0, 0.0, z]) @ Rc + C for z in zs]).astype(np.float32)
    K = scaled_intrinsics(TEST_POSE_K, max(H, W))
    K[0, 2], K[1, 2] = W / 2.0, H / 2.0
    from gaussianavatar_b200.mesh_render import cameras
    cams = cameras([make_camera(K, E, H, W)]).to(DEV)
    n = len(zs)
    means = torch.from_numpy(xyz)[None].to(DEV)
    scales = torch.tensor(sizes, dtype=torch.float32)[:, None].expand(n, 3)[None].contiguous().to(DEV)
    rot = torch.tensor([[1.0, 0.0, 0.0, 0.0]] * n, device=DEV)
    opac = torch.tensor(opacities, dtype=torch.float32, device=DEV).reshape(-1, 1)
    plan = RasterBatchPlan(1, n, H, W, DEV)
    with torch.no_grad():
        img, mattes, depth = rasterize_batch_depth(means, torch.rand(1, n, 3, device=DEV), scales, rot, opac, cams, torch.ones(3, device=DEV),
                                                   plan, first=list(range(n + 1)))
        assert plan.check(wait=True)
    return mattes[0], depth[0], _views_of(plan)[0]


def test_single_opaque_gaussian():
    """A single Gaussian of opacity 0.99: where it takes T to 0.5 or below (its centre), median = z exactly and mean = z within 2
    ulp (1 - T rounds alpha by at most half an ulp of a number below 0.5); the median is 0 elsewhere.  Where it blends with a small
    alpha, 1 - T carries the rounding of 1 - alpha, up to ~2^-25 / alpha relative: the mean is z within 1e-5 relative there."""
    mattes, depth, v = _axis_gaussians([2.0], [0.15], [0.99])
    z = float(v["depth"][0])
    ulp = float(np.spacing(np.float32(z)))
    peak = v["final_T"].to(DEV) <= 0.5
    assert mattes[0].max().item() > 0.98 and peak.sum().item() >= 4
    assert (depth[1][peak] == z).all() and (depth[1][~peak] == 0).all()
    assert ((depth[0][peak] - z).abs() <= 2 * ulp).all()
    blended = v["n_contrib"].to(DEV) > 0
    assert ((depth[0][blended] - z).abs() <= 1e-5 * z).all() and (depth[0][~blended] == 0).all()


@pytest.mark.parametrize("front,which", [(0.4, "back"), (0.6, "front")])
def test_two_layers(front, which):
    """A front layer of opacity 0.4 leaves T = 0.6 > 0.5, so the opaque back layer holds the median; with 0.6 it leaves T = 0.4 and
    the front layer does.  Checked where the front layer blends at close to its opacity."""
    mattes, depth, v = _axis_gaussians([2.0, 3.0], [0.12, 0.5], [front, 0.99])
    zf, zb = float(v["depth"][0]), float(v["depth"][1])
    core = mattes[0] > front * 0.95
    assert core.sum().item() >= 4
    want = zb if which == "back" else zf
    assert (depth[1][core] == want).all()
    assert ((depth[0][core] > zf) & (depth[0][core] < zb)).all()               # the mean mixes the two


def test_wall_in_front_of_an_avatar():
    """test_scene_gpu's opaque wall between the camera and the dynamic set: the median is the wall's depth where the wall covers the
    pixel, and where there is no wall the avatar's own median, bit for bit (the same entries blend)."""
    H, W = 128, 128
    scs = _frames(1, H, W, 3000, seed=90)
    wall = _wall(24, 1.2, 0.25, seed=91).to(DEV)
    means, colors, scales, rot, opac = _dyn(scs)
    cams, bg = _cams(scs), scs[0]["bg"].to(DEV)
    with torch.no_grad():
        plan = RasterBatchPlan(1, 3000, H, W, DEV, static_P=len(wall))
        _, depth = rasterize_batch_depth(means, colors, scales, rot, opac, cams, bg, plan, wall)
        plan_a = RasterBatchPlan(1, 3000, H, W, DEV)
        _, depth_a = rasterize_batch_depth(means, colors, scales, rot, opac, cams, bg, plan_a)
        none = means[:, :0].contiguous()
        plan_w = RasterBatchPlan(1, 0, H, W, DEV, static_P=len(wall))
        _, depth_w = rasterize_batch_depth(none, colors[:, :0].contiguous(), scales[:, :0].contiguous(), rot[:0].contiguous(),
                                           opac[:0].contiguous(), cams, bg, plan_w, wall)
        assert plan.check(wait=True) and plan_a.check(wait=True) and plan_w.check(wait=True)
    T_wall = an.final_transmittance(plan_w)[0]
    T_avatar = an.final_transmittance(plan_a)[0]
    covered = T_wall < 1e-3
    assert (covered & (T_avatar < 0.5)).float().mean().item() > 0.05
    med = depth[0, 1]
    assert (med[covered] - 1.2).abs().max().item() < 1e-4
    assert torch.equal(med[covered], depth_w[0, 1][covered])
    clear = (T_wall > 0.999) & (T_avatar < 0.5)
    assert clear.float().mean().item() > 0.05
    assert torch.equal(med[clear], depth_a[0, 1][clear]) and (med[clear] > 1.3).all()


# ---- 5. the player ----------------------------------------------------------------------------------------------------------------
def _play(ens, fps):
    frames, mattes, depth = [], [], []
    for first, f, m, *d in ens.frames(fps):
        assert first == sum(x.shape[0] for x in frames)
        frames.append(f.clone())
        mattes.append(None if m is None else m.clone())
        depth.append(d[0].clone() if d else None)
    cat = lambda xs: None if xs[0] is None else torch.cat(xs)
    return cat(frames), cat(mattes), cat(depth)


def _expected_depth(actors, fps, scene=None):
    """Every frame on its own, as test_cast_gpu._expected builds it, through rasterize_batch_depth."""
    from gaussianavatar_b200.camera import Camera
    from gaussianavatar_b200.mesh_render import cameras
    steps = [a.speed * a.clip.fps / fps for a in actors]
    n = max(int(np.floor((a.clip.num_keys - 1) / st)) + 1 for a, st in zip(actors, steps))
    c = _camera()
    cam = cameras([Camera(float(c["FovX"]), float(c["FovY"]), SIDE, SIDE, torch.as_tensor(c["world_view_transform"]),
                          torch.as_tensor(c["full_proj_transform"]), torch.as_tensor(c["camera_center"]))]).to(DEV)
    sampled = []
    for a, st in zip(actors, steps):
        T = a.clip.num_keys
        times = torch.tensor([min(j * st, T - 1.0) for j in range(n)], dtype=torch.float64, device=DEV)
        align = an.IDENTITY_ALIGN if a.align_to is None else an.alignment(
            a.clip.pose[0, :3].double().numpy(), a.clip.trans[0].double().numpy(), a.model.pose.weight[a.align_to, :3].detach().double().cpu().numpy(),
            a.model.transl.weight[a.align_to].detach().double().cpu().numpy())
        sampled.append(an.motion_sample(a.clip.pose.to(DEV), a.clip.trans.to(DEV), times, torch.from_numpy(align).to(DEV)))
    first = [0] + np.cumsum([a.model._query_points.shape[0] for a in actors]).tolist()
    rot = torch.cat([a.model.fix_rotation for a in actors])
    opac = torch.cat([a.model.fix_opacity for a in actors])
    bg = actors[0].model.background
    out = []
    with torch.no_grad(), contextlib.ExitStack() as kept:
        for m in {id(a.model): a.model for a in actors}.values():
            kept.enter_context(kept_state(m))
        for i in range(n):
            parts = []
            for a, (pose, trans) in zip(actors, sampled):
                m = a.model
                p, rest = m.body.split(pose[i:i + 1])
                if int(m.model_parms.train_stage) == 2:
                    parts.append(m._stage2_from_pose(a.pose_mapper, p, trans[i:i + 1], rest, placement=a.placement)[:3])
                else:
                    parts.append(m._assemble(m._stage1_decoder(1), p, trans[i:i + 1], rest, placement=a.placement))
            means, scales, colors = (torch.cat(t, 1) for t in zip(*parts))
            plan = RasterBatchPlan(1, first[-1], SIDE, SIDE, DEV, capacity=1 << 22, static_P=0 if scene is None else len(scene))
            _, d = rasterize_batch_depth(means, colors, scales, rot, opac, cam, bg, plan, scene)
            assert plan.check(wait=True)
            out.append(d.cpu())
    return torch.cat(out)


@pytest.mark.parametrize("with_scene", [False, True])
@pytest.mark.parametrize("chunk", [1, 3, 8])
def test_player_depth(chunk, with_scene):
    """Ensemble(depth=True) yields the frames and mattes of depth=False, with graphs on and off, and depth equal to each frame built
    on its own; replaying the captured graphs gives the same depth."""
    actors = _pair()
    scene = _scene().to(DEV) if with_scene else None
    ref, ref_m, none = _play(an.Ensemble(actors, _camera(), SIDE, SIDE, chunk=chunk, channels=4, mattes=True, scene=scene), 50.0)
    assert none is None
    ens = an.Ensemble(actors, _camera(), SIDE, SIDE, chunk=chunk, channels=4, mattes=True, scene=scene, depth=True)
    got, got_m, depth = _play(ens, 50.0)
    assert torch.equal(got, ref) and torch.equal(got_m, ref_m) and ens.captures >= 1
    assert depth.shape == (9, 2, SIDE, SIDE) and depth.dtype == torch.float32
    assert torch.equal(depth, _expected_depth(actors, 50.0, scene))
    assert (depth[:, 1] > 0).float().mean() > 0.05
    again = _play(ens, 50.0)
    assert torch.equal(again[2], depth) and torch.equal(again[0], got)
    eager = _play(an.Ensemble(actors, _camera(), SIDE, SIDE, chunk=chunk, channels=4, scene=scene, depth=True, graphs=False), 50.0)
    assert torch.equal(eager[0], ref) and eager[1] is None and torch.equal(eager[2], depth)


def test_player_depth_forced_overflow():
    actors = _pair()
    ref = _play(an.Ensemble(actors, _camera(), SIDE, SIDE, chunk=4, channels=3, depth=True), 45.0)
    small = an.Ensemble(actors, _camera(), SIDE, SIDE, chunk=4, channels=3, depth=True, capacity=64)
    got = _play(small, 45.0)
    assert small.overflows >= 1 and small.recaptures >= 1
    assert torch.equal(got[0], ref[0]) and torch.equal(got[2], ref[2])
    assert torch.equal(ref[2], _expected_depth(actors, 45.0))


def test_player_depth_stage2_beside_stage1():
    """Rendered eagerly; the stage-2 decoder's BatchNorm sums use atomics in no fixed order, so frames and depth may differ from the
    independent construction in the last bits: bytes by one step, depth to 1e-4 relative on 99.5 % of the pixels."""
    actors = _pair(stage2=True)
    with torch.backends.cudnn.flags(deterministic=True):
        ref = _play(an.Ensemble(actors, _camera(), SIDE, SIDE, chunk=3, channels=4, mattes=True), 40.0)
        ens = an.Ensemble(actors, _camera(), SIDE, SIDE, chunk=3, channels=4, mattes=True, depth=True)
        got = _play(ens, 40.0)
        want = _expected_depth(actors, 40.0)
    assert ens.captures == 0
    assert _close(got[0], ref[0]) and _close(got[1], ref[1])
    near = (got[2] - want).abs() <= 1e-4 * want.abs()
    assert near.float().mean().item() > 0.995 and (want[:, 1] > 0).any()


def test_animator_depth():
    m, _ = _model("smpl")
    from test_animate_gpu import _clip
    clip = _clip("smpl")
    plain = [f.clone() for _, f in an.Animator(m, _camera(), SIDE, SIDE, chunk=3).frames(clip, 45.0, align_to=1)]
    anim = an.Animator(m, _camera(), SIDE, SIDE, chunk=3, depth=True)
    out = [(f.clone(), d.clone()) for _, f, d in anim.frames(clip, 45.0, align_to=1)]
    assert torch.equal(torch.cat(plain), torch.cat([f for f, _ in out]))
    want = _play(an.Ensemble([an.Actor(m, clip, align_to=1)], _camera(), SIDE, SIDE, chunk=3, depth=True), 45.0)[2]
    assert torch.equal(torch.cat([d for _, d in out]), want)


# ---- 6. the tool ------------------------------------------------------------------------------------------------------------------
def test_tool_depth(tmp_path):
    """tools/animate.py --depth writes one float32 [2,H,W] file per frame, equal to the player's depth in process (to 1e-5 relative:
    the decoder's atomics may move the last bits between processes); with --cast and --mattes too."""
    from dataset_fixture import write_synthetic_dataset
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams, OptimizationParams
    from gaussianavatar_b200.dataset import camera_item
    mp = write_synthetic_dataset(str(tmp_path), seed=0)
    torch.manual_seed(0)
    m = AvatarModel(mp, NetworkParams(nf=8), OptimizationParams(), train=True)
    m.training_setup()
    with torch.no_grad():
        sd = m.net.state_dict()
        sd["decoder.conv8N.bias"] = torch.tensor([-5.3])
        m.net.load_state_dict(sd, strict=False)
    m.save(7)
    clip_path = os.path.join(mp.test_folder, "smpl_parms.pth")
    smpl_model = os.path.join(mp.smpl_model_path, "SMPL_NEUTRAL.pkl")
    tool = [sys.executable, os.path.join(ROOT, "tools", "animate.py"), "--project_path", mp.project_path, "--fps", "30", "--size", "80",
            "48", "--chunk", "3"]
    out = tmp_path / "depth"
    r = subprocess.run(tool + ["-s", mp.source_path, "-m", mp.model_path, "--smpl_model", smpl_model, "--query_posmap_size",
                               str(mp.query_posmap_size), "--inp_posmap_size", str(mp.inp_posmap_size), "--epoch", "7", "--motion",
                               clip_path, "--clip_fps", "30", "--align_to", "1", "--depth", str(out)], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    n = json.loads(r.stdout.strip().splitlines()[-1])["frames"]
    assert sorted(os.listdir(out)) == ["{:05d}.npy".format(i) for i in range(n)]
    files = [np.load(out / "{:05d}.npy".format(i)) for i in range(n)]
    assert all(f.dtype == np.float32 and f.shape == (2, 48, 80) for f in files)
    mp2 = type(mp)(**{**vars(mp), "batch_size": 1})
    model = AvatarModel(mp2, NetworkParams(nf=8), OptimizationParams(), train=False)
    model.load(7)
    clip = an.MotionClip.load(clip_path, "smpl", fps=30)
    cam = np.load(os.path.join(mp.source_path, "train", "cam_parms.npz"))
    K = np.array(cam["intrinsic"], np.float32).reshape(3, 3)
    K[0, :] *= 80 / 64
    K[1, :] *= 48 / 64
    anim = an.Animator(model, camera_item(K, np.asarray(cam["extrinsic"], np.float64), 48, 80), 48, 80, chunk=3, depth=True)
    want = torch.cat([d.clone() for _, _, d in anim.frames(clip, 30.0, align_to=1)]).numpy()
    got = np.stack(files)
    assert want.shape == got.shape and (want[:, 1] > 0).any()
    near = np.abs(got - want) <= 1e-5 * np.abs(want)
    assert near.mean() > 0.995
    cast = tmp_path / "cast.json"
    common = dict(source_path=mp.source_path, model_path=mp.model_path, epoch=7, motion=clip_path, clip_fps=30, smpl_model=smpl_model,
                  query_posmap_size=mp.query_posmap_size, inp_posmap_size=mp.inp_posmap_size, nf=8)
    cast.write_text(json.dumps([dict(common, align_to=1), dict(common, speed=2.0)]))
    out2, mattes = tmp_path / "depth2", tmp_path / "mattes"
    r = subprocess.run(tool + ["--cast", str(cast), "--depth", str(out2), "--mattes", str(mattes)], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    k = json.loads(r.stdout.strip().splitlines()[-1])["frames"]
    assert sorted(os.listdir(out2)) == ["{:05d}.npy".format(i) for i in range(k)] and len(os.listdir(mattes)) == 2 * k
