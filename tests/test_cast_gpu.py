"""GPU: several avatars rendered together.  The matte variant of the batched forward (ga_rasterb_forward_mattes) against the same
call without mattes, against indicator-colour renders and against the CPU oracle with a scene; its occlusion known answer; the
ensemble player (animate.Ensemble) against an independent construction of every frame; and tools/animate.py --cast / --mattes."""
import contextlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gaussianavatar_b200 import animate as an
from gaussianavatar_b200.avatar_model import kept_state
from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, TEST_POSE_K, make_camera, scaled_intrinsics
from gaussianavatar_b200.rasterizer import RasterBatchPlan, rasterize_batch, rasterize_batch_mattes, rasterize_batch_scene
from gaussianavatar_b200.scene import Placement
from scene_fixture import random_static, scene_of
from test_animate_gpu import _avatar, _clip, _model_state, _same_state
from test_scene_gpu import _cams, _frames, _wall

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WRITTEN = [0, 1, 2, 3, 13]            # status words every forward writes: instances, overflow, segments, tiles, long tiles


# ---- the kernel -------------------------------------------------------------------------------------------------------------------
def _dyn(scs):
    t = {k: torch.stack([s[k] for s in scs]).to(DEV) for k in ("means3D", "colors", "scales")}
    return t["means3D"], t["colors"], t["scales"], scs[0]["rotations"].to(DEV), scs[0]["opacities"].to(DEV)


def _random_first(P, K, seed, full=True):
    g = np.random.default_rng(seed)
    cuts = np.sort(g.integers(0, P + 1, size=K - 1)).tolist()
    return [0] + cuts + [P if full else int(g.integers(cuts[-1] if cuts else 0, P))]


def _indicator(B, P, first, k):
    ind = torch.zeros(P, 3, device=DEV)
    ind[first[k]:first[k + 1]] = 1.0
    return ind.expand(B, P, 3).contiguous()


def _status(plan, B):
    return plan.status_dev[WRITTEN + list(range(4, 5 + B))]


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("K", [1, 2, 3, 5, 8])
def test_mattes_without_scene(K, B):
    """With mattes on, the images, final T, radii and status are those of the same call without mattes, bit for bit.  Matte k is the
    red channel of rasterize_batch with colours = the indicator of set k and bg = 0 (the same alpha and T sequence, the same adds),
    bit for bit, and the mattes sum to 1 - final T within 1e-5 where every Gaussian is in a set.  Ragged tiles: 100 x 140."""
    H, W, P = 100, 140, 2500
    scs = _frames(B, H, W, P, seed=10 * K + B)
    means, colors, scales, rot, opac = _dyn(scs)
    cams, bg = _cams(scs), scs[0]["bg"].to(DEV)
    full = K != 3                                   # K = 3 leaves the last Gaussians in no set
    first = _random_first(P, K, seed=K + 7 * B, full=full)
    with torch.no_grad():
        plan_m, plan = RasterBatchPlan(B, P, H, W, DEV), RasterBatchPlan(B, P, H, W, DEV)
        img_m, mattes = rasterize_batch_mattes(means, colors, scales, rot, opac, cams, bg, plan_m, first)
        img = rasterize_batch(means, colors, scales, rot, opac, cams, bg, plan)
        assert plan_m.check(wait=True) and plan.check(wait=True)
        assert mattes.shape == (B, K, H, W)
        assert torch.equal(img_m, img) and torch.equal(plan_m.radii, plan.radii)
        assert torch.equal(an.final_transmittance(plan_m), an.final_transmittance(plan))
        assert torch.equal(_status(plan_m, B), _status(plan, B))
        zero = torch.zeros(3, device=DEV)
        for k in range(K):
            pk = RasterBatchPlan(B, P, H, W, DEV)
            ref = rasterize_batch(means, _indicator(B, P, first, k), scales, rot, opac, cams, zero, pk)
            assert torch.equal(mattes[:, k], ref[:, 0]), k
        alpha = 1.0 - an.final_transmittance(plan)
        total = mattes.double().sum(1)
        if full:
            assert (total - alpha.double()).abs().max().item() <= 1e-5
        else:
            assert (total <= alpha.double() + 1e-5).all()
        covered = [(mattes[:, k] > 0.5).any().item() for k in range(K) if first[k + 1] - first[k] > 200]
        assert covered and all(covered)


def test_mattes_with_scene_match_oracle():
    """With a scene the images, final T, radii and status are the composite's without mattes, bit for bit, and each matte is the
    oracle's render of [dynamic; static] with indicator colours (set k's, the scene's 0) and bg 0, within the mean-L1 bound of
    test_composite_matches_oracle_per_frame (three sets at once, one per colour channel)."""
    from oracle import raster_oracle as ro
    B, Pd, Ps, H, W = 2, 1500, 2500, 136, 200
    scs = _frames(B, H, W, Pd, seed=160)
    scene = scene_of(random_static(Ps, 1, seed=171, center=(0.0, -0.2, 0.2), spread=(0.8, 1.0, 0.6)))
    means, colors, scales, rot, opac = _dyn(scs)
    cams, bg = _cams(scs), scs[0]["bg"].to(DEV)
    first = [0, 400, 1100, 1500]
    with torch.no_grad():
        plan_m, plan = RasterBatchPlan(B, Pd, H, W, DEV, static_P=Ps), RasterBatchPlan(B, Pd, H, W, DEV, static_P=Ps)
        img_m, mattes = rasterize_batch_mattes(means, colors, scales, rot, opac, cams, bg, plan_m, first, scene.to(DEV))
        img = rasterize_batch_scene(means, colors, scales, rot, opac, cams, bg, plan, scene.to(DEV))
        assert plan_m.check(wait=True) and plan.check(wait=True)
    assert torch.equal(img_m, img) and torch.equal(plan_m.radii, plan.radii)
    assert torch.equal(an.final_transmittance(plan_m), an.final_transmittance(plan))
    assert torch.equal(_status(plan_m, B), _status(plan, B))
    ind = np.zeros((Pd + Ps, 3), np.float32)
    for k in range(3):
        ind[first[k]:first[k + 1], k] = 1.0
    got = mattes.cpu().numpy().astype(np.float64)
    for b, sc in enumerate(scs):
        o = ro.forward(means3D=np.concatenate([sc["means3D"].numpy(), scene.means3D.numpy()]), colors=ind,
                       opacities=np.concatenate([sc["opacities"].numpy().reshape(-1, 1), scene.opacities.numpy().reshape(-1, 1)]),
                       scales=np.concatenate([sc["scales"].numpy(), scene.scales.numpy()]),
                       rotations=np.concatenate([sc["rotations"].numpy(), scene.rotations.numpy()]), bg=np.zeros(3, np.float32),
                       viewmatrix=sc["cam"].world_view_transform.numpy(), projmatrix=sc["cam"].full_proj_transform.numpy(),
                       tanfovx=sc["tanfovx"], tanfovy=sc["tanfovy"], H=H, W=W, precision="f32")
        assert np.abs(got[b] - o.image).mean() <= 1e-4
        assert (o.image.max(axis=(1, 2)) > 0.5).all()          # every set shows somewhere
        alpha = 1.0 - an.final_transmittance(plan)[b].double().cpu().numpy()
        assert (got[b].sum(0) <= alpha + 1e-5).all() and (alpha - got[b].sum(0)).max() > 0.5      # the scene covers the rest


def _render_walls(order, H=112, W=144):
    """Two opaque walls in front of the reference camera, a near one and a larger far one, each its own set and colour; `order`
    puts them in the index space."""
    walls = [_wall(24, 1.2, 0.25, seed=1), _wall(48, 2.4, 1.2, seed=2)]
    tint = [torch.tensor([0.9, 0.2, 0.1]), torch.tensor([0.1, 0.3, 0.8])]
    sets = [walls[i] for i in order]
    P = [len(s) for s in sets]
    cat = lambda k: torch.cat([getattr(s, k) for s in sets]).to(DEV)
    colors = torch.cat([tint[i].expand(len(walls[i]), 3) for i in order]).to(DEV)[None]
    K = scaled_intrinsics(TEST_POSE_K, max(H, W))
    K[0, 2], K[1, 2] = W / 2.0, H / 2.0
    from gaussianavatar_b200.mesh_render import cameras
    cams = cameras([make_camera(K, TEST_POSE_EXTRINSIC, H, W)]).to(DEV)
    plan = RasterBatchPlan(1, sum(P), H, W, DEV)
    with torch.no_grad():
        img, mattes = rasterize_batch_mattes(cat("means3D")[None], colors, cat("scales")[None], cat("rotations"), cat("opacities").reshape(-1, 1),
                                             cams, torch.ones(3, device=DEV), plan, [0, P[0], P[0] + P[1]])
        assert plan.check(wait=True)
    return img, mattes, plan


def test_occlusion_known_answer_and_set_order():
    """The far wall's matte is below 1/255 wherever the near wall covers the pixel, and near 1 over most of what only it reaches.
    Swapping the two sets in the index space swaps the mattes and leaves the image and final T bit for bit as they were."""
    img, mattes, plan = _render_walls([0, 1])
    near, far = mattes[0, 0], mattes[0, 1]
    covered = near >= 0.999
    assert covered.float().mean().item() > 0.05
    assert far[covered].max().item() < 1.0 / 255
    only_far = near == 0
    assert only_far.float().mean().item() > 0.05 and (far[only_far] > 0.99).float().mean().item() > 0.5
    img2, mattes2, plan2 = _render_walls([1, 0])
    assert torch.equal(mattes2[:, 0], mattes[:, 1]) and torch.equal(mattes2[:, 1], mattes[:, 0])
    assert torch.equal(img, img2) and torch.equal(an.final_transmittance(plan), an.final_transmittance(plan2))


# ---- the player -------------------------------------------------------------------------------------------------------------------
SIDE = 96
_MODELS = {}


def _model(body, stage=1):
    if (body, stage) not in _MODELS:
        _MODELS[(body, stage)] = _avatar(body, stage=stage)
    return _MODELS[(body, stage)]


def _scene():
    """A scene behind the actors (the camera looks down -z from z ~ 2.4), filling the rest of the frame."""
    return scene_of(random_static(4000, 2, seed=5, center=(0.0, -0.2, -1.2), spread=(1.5, 1.5, 0.4), scale_mean=0.08))


def _camera():
    from gaussianavatar_b200.dataset import camera_item
    return camera_item(scaled_intrinsics(TEST_POSE_K, SIDE), TEST_POSE_EXTRINSIC, SIDE, SIDE)


def _pair(same_model=False, stage2=False):
    """Actor 0: SMPL, 6 keys, identity alignment; actor 1: SMPL-X (or the same SMPL model), 4 keys, aligned to training frame 2, moved
    sideways by a placement."""
    m0, _ = _model("smpl")
    if same_model:
        m1, mp1, c1 = m0, None, _clip("smpl", T=4)
    else:
        m1, mp1 = _model("smplx", stage=2 if stage2 else 1)
        c1 = _clip("smplx", T=4)
    place = Placement.from_axis_angle(0.9, [0.0, 0.4, 0.0], [0.35, 0.0, -0.1])
    return [an.Actor(m0, _clip("smpl", T=6)), an.Actor(m1, c1, place, align_to=2, speed=1.25, pose_mapper=mp1)]


def _play(ens, fps):
    frames, mattes = [], []
    for first, f, m in ens.frames(fps):
        assert first == sum(x.shape[0] for x in frames)
        frames.append(f.clone())
        mattes.append(None if m is None else m.clone())
    return torch.cat(frames), (None if mattes[0] is None else torch.cat(mattes))


def _expected(actors, fps, channels, scene=None):
    """Every frame on its own: each actor's _assemble (or stage-2 forward) at its sampled, clamped pose, concatenated, the composite
    with mattes, frame_pack and the matte quantisation."""
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
    frames, mattes = [], []
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
            img, mt = rasterize_batch_mattes(means, colors, scales, rot, opac, cam, bg, plan, first, scene)
            assert plan.check(wait=True)
            frames.append(an.frame_pack(img, an.final_transmittance(plan), bg, channels).cpu())
            mattes.append(an.matte_pack(mt).cpu())
    return torch.cat(frames), torch.cat(mattes)


@pytest.mark.parametrize("with_scene", [False, True])
@pytest.mark.parametrize("channels", [3, 4])
@pytest.mark.parametrize("chunk", [1, 3, 8])
def test_two_actors_equal_independent_construction(chunk, channels, with_scene):
    """SMPL and SMPL-X actors on clips of different lengths (the shorter holds its last pose), one placed: every frame's bytes and
    mattes equal the frame built on its own; the models' state is unchanged; graphs were captured and replaying them gives the
    same bytes."""
    actors = _pair()
    scene = _scene().to(DEV) if with_scene else None
    before = [_model_state(a.model) for a in actors]
    ens = an.Ensemble(actors, _camera(), SIDE, SIDE, chunk=chunk, channels=channels, mattes=True, scene=scene)
    got, mattes = _play(ens, 50.0)
    assert all(_same_state(b, _model_state(a.model)) for b, a in zip(before, actors))
    want, want_m = _expected(actors, 50.0, channels, scene)
    assert got.shape == (9, SIDE, SIDE, channels) and mattes.shape == (9, 2, SIDE, SIDE)    # 6 keys at 30 fps -> 9 frames at 50
    assert torch.equal(got, want) and torch.equal(mattes, want_m)
    assert ens.captures >= 1
    for k in range(2):
        assert (mattes[:, k] > 128).any(), k                   # each actor is seen
    n = ens.captures
    again, again_m = _play(ens, 50.0)
    assert torch.equal(again, got) and torch.equal(again_m, mattes) and ens.captures == n
    if chunk == 3:                                             # mattes off: the same frames, no mattes
        plain, none = _play(an.Ensemble(actors, _camera(), SIDE, SIDE, chunk=chunk, channels=channels, scene=scene), 50.0)
        assert none is None and torch.equal(plain, got)


def test_graphs_off_and_forced_overflow():
    actors = _pair()
    ref, ref_m = _play(an.Ensemble(actors, _camera(), SIDE, SIDE, chunk=4, channels=4, mattes=True), 45.0)
    eager, eager_m = _play(an.Ensemble(actors, _camera(), SIDE, SIDE, chunk=4, channels=4, mattes=True, graphs=False), 45.0)
    assert torch.equal(eager, ref) and torch.equal(eager_m, ref_m)
    small = an.Ensemble(actors, _camera(), SIDE, SIDE, chunk=4, channels=4, mattes=True, capacity=64)
    got, got_m = _play(small, 45.0)
    assert small.overflows >= 1 and small.recaptures >= 1
    assert torch.equal(got, ref) and torch.equal(got_m, ref_m)


def test_same_model_as_two_actors():
    actors = _pair(same_model=True)
    before = _model_state(actors[0].model)
    got, mattes = _play(an.Ensemble(actors, _camera(), SIDE, SIDE, chunk=3, channels=4, mattes=True), 40.0)
    assert _same_state(before, _model_state(actors[0].model))
    want, want_m = _expected(actors, 40.0, 4)
    assert torch.equal(got, want) and torch.equal(mattes, want_m)


def _close(got, want):
    """Two stage-2 forwards of the same frame may differ in the last bits (the decoder's BatchNorm sums use atomics, in no fixed
    order); un-compositing magnifies that where alpha is small, so bytes may differ by one step (as in test_animate_gpu)."""
    d = (got.int() - want.int()).abs()
    return d.max().item() <= 1 and (d == 0).float().mean().item() > 0.995


def test_stage2_actor_with_a_stage1_actor():
    actors = _pair(stage2=True)
    before = [_model_state(a.model) for a in actors]
    with torch.backends.cudnn.flags(deterministic=True):
        ens = an.Ensemble(actors, _camera(), SIDE, SIDE, chunk=3, channels=4, mattes=True)
        got, mattes = _play(ens, 40.0)
        want, want_m = _expected(actors, 40.0, 4)
    assert ens.captures == 0                                   # rendered eagerly
    assert all(_same_state(b, _model_state(a.model)) for b, a in zip(before, actors))
    assert _close(got, want) and _close(mattes, want_m)
    assert (mattes[:, 1] > 0).any() and (mattes[:, 0] > 0).any()


@pytest.mark.parametrize("stage", [1, 2])
@pytest.mark.parametrize("with_scene", [False, True])
def test_one_actor_equals_animator(stage, with_scene):
    m, mapper = _model("smpl", stage=stage)
    clip = _clip("smpl")
    scene = _scene().to(DEV) if with_scene else None
    place = Placement.from_axis_angle(1.1, [0.0, 0.3, 0.0], [0.05, 0.02, -0.1]) if with_scene else None
    with torch.backends.cudnn.flags(deterministic=True):
        anim = an.Animator(m, _camera(), SIDE, SIDE, chunk=3, channels=4, pose_mapper=mapper, scene=scene, placement=place)
        ref = torch.cat([f.clone() for _, f in anim.frames(clip, 45.0, align_to=1)])
        ens = an.Ensemble([an.Actor(m, clip, place, align_to=1, pose_mapper=mapper)], _camera(), SIDE, SIDE, chunk=3, channels=4,
                          mattes=True, scene=scene)
        got, mattes = _play(ens, 45.0)
    if stage == 1:
        assert torch.equal(got, ref)
    else:
        assert _close(got, ref)
    if not with_scene:                                         # alone, the actor's matte is the frame's alpha
        assert _close(mattes[:, 0], got[..., 3])
    else:
        assert (mattes[:, 0].int() <= got[..., 3].int() + 1).all() and (mattes[:, 0] < got[..., 3]).any()


def test_backgrounds_must_agree():
    m0, _ = _model("smpl")
    m1 = _avatar("smpl")[0]
    m1.background = torch.zeros(3, device=DEV)
    with pytest.raises(ValueError, match="background"):
        an.Ensemble([an.Actor(m0, _clip("smpl")), an.Actor(m1, _clip("smpl"))], _camera(), SIDE, SIDE)
    with pytest.raises(ValueError, match="actor 1's avatar is 'smpl'"):
        an.Ensemble([an.Actor(m0, _clip("smpl")), an.Actor(m0, _clip("smplx"))], _camera(), SIDE, SIDE)


# ---- the tool ---------------------------------------------------------------------------------------------------------------------
def test_tool_cast_and_mattes(tmp_path):
    from PIL import Image
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from dataset_fixture import write_synthetic_dataset
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams, OptimizationParams
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
    common = dict(source_path=mp.source_path, model_path=mp.model_path, epoch=7, motion=clip_path, clip_fps=30,
                  smpl_model=os.path.join(mp.smpl_model_path, "SMPL_NEUTRAL.pkl"), query_posmap_size=mp.query_posmap_size,
                  inp_posmap_size=mp.inp_posmap_size, nf=8)
    cast = tmp_path / "cast.json"
    cast.write_text(json.dumps([dict(common, align_to=1), dict(common, speed=2.0, place=[0.8, 0, 0.5, 0, 0.3, 0, 0])]))
    png, mattes = tmp_path / "png", tmp_path / "mattes"
    tool = [sys.executable, os.path.join(ROOT, "tools", "animate.py"), "--project_path", mp.project_path, "--fps", "30", "--size", "80",
            "48", "--chunk", "3"]
    r = subprocess.run(tool + ["--cast", str(cast), "--png", str(png), "--mattes", str(mattes)], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    n = json.loads(r.stdout.strip().splitlines()[-1])["frames"]
    assert sorted(os.listdir(png)) == ["{:05d}.png".format(i) for i in range(n)]
    assert sorted(os.listdir(mattes)) == sorted("{:05d}_{}.png".format(i, k) for i in range(n) for k in range(2))
    # the same playback in process (the decoder's atomics may move the last bits between processes)
    mp2 = type(mp)(**{**vars(mp), "batch_size": 1})
    model = AvatarModel(mp2, NetworkParams(nf=8), OptimizationParams(), train=False)
    model.load(7)
    clip = an.MotionClip.load(clip_path, "smpl", fps=30)
    cam = np.load(os.path.join(mp.source_path, "train", "cam_parms.npz"))
    K = np.array(cam["intrinsic"], np.float32).reshape(3, 3)
    K[0, :] *= 80 / 64
    K[1, :] *= 48 / 64
    from gaussianavatar_b200.dataset import camera_item
    actors = [an.Actor(model, clip, align_to=1), an.Actor(model, clip, Placement.from_axis_angle(0.8, [0, 0.5, 0], [0.3, 0, 0]), speed=2.0)]
    ens = an.Ensemble(actors, camera_item(K, np.asarray(cam["extrinsic"], np.float64), 48, 80), 48, 80, chunk=3, mattes=True)
    want, want_m = _play(ens, 30.0)
    assert want.shape[0] == n
    got = torch.from_numpy(np.stack([np.array(Image.open(png / "{:05d}.png".format(i))) for i in range(n)]))
    got_m = torch.from_numpy(np.stack([[np.array(Image.open(mattes / "{:05d}_{}.png".format(i, k))) for k in range(2)] for i in range(n)]))
    assert _close(got, want) and _close(got_m, want_m)
    assert (want_m[:, 0] > 0).any() and (want_m[:, 1] > 0).any()
    # the single avatar's --mattes
    single = tmp_path / "single"
    r = subprocess.run(tool + ["-s", mp.source_path, "-m", mp.model_path, "--smpl_model", common["smpl_model"], "--query_posmap_size",
                               str(mp.query_posmap_size), "--inp_posmap_size", str(mp.inp_posmap_size), "--epoch", "7", "--motion",
                               clip_path, "--clip_fps", "30", "--mattes", str(single)], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    k = json.loads(r.stdout.strip().splitlines()[-1])["frames"]
    assert sorted(os.listdir(single)) == ["{:05d}_0.png".format(i) for i in range(k)]
