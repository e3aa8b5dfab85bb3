"""GPU: the composite forward (an avatar's dynamic Gaussians splatted with a static 3DGS scene in one sort) against the CPU oracle
frame by frame, its empty-scene and occlusion known answers, the placement, the animation player with a scene, and
tools/animate.py --scene end to end."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, TEST_POSE_K, make_camera, scaled_intrinsics
from gaussianavatar_b200.dataset import rotate_camera_by_frame_idx
from scene_fixture import random_static, scene_of, write_cameras_json, write_ply
from scenes import random_scene
from sh_scenes import pre_clamp

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _frames(B, H, W, Pd, seed):
    """B frames: isotropic opaque dynamic Gaussians that differ per frame (shared rotations / opacities, as the avatar's), each seen
    by its own camera (an orbit step around the scene's centre)."""
    scs = [random_scene(P=Pd, H=H, W=W, seed=seed + b, scale_mean=0.02, aniso=False, opacity_one=True) for b in range(B)]
    K = scaled_intrinsics(TEST_POSE_K, max(H, W))
    K[0, 2], K[1, 2] = W / 2.0, H / 2.0
    for b, s in enumerate(scs):
        s["rotations"], s["opacities"] = scs[0]["rotations"], scs[0]["opacities"]
        s["cam"] = make_camera(K, rotate_camera_by_frame_idx(TEST_POSE_EXTRINSIC, b, trans=np.array([0.0, -0.2, 0.0]), period=40), H, W)
    return scs


def _cams(scs):
    from gaussianavatar_b200.mesh_render import cameras
    return cameras([s["cam"] for s in scs]).to(DEV)


def _composite(scs, scene, capacity=None):
    from gaussianavatar_b200.rasterizer import RasterBatchPlan, rasterize_batch_scene
    B, Pd, H, W = len(scs), scs[0]["means3D"].shape[0], scs[0]["H"], scs[0]["W"]
    plan = RasterBatchPlan(B, Pd, H, W, DEV, capacity=capacity, static_P=len(scene))
    t = {k: torch.stack([s[k] for s in scs]).to(DEV) for k in ("means3D", "colors", "scales")}
    with torch.no_grad():
        img = rasterize_batch_scene(t["means3D"], t["colors"], t["scales"], scs[0]["rotations"].to(DEV), scs[0]["opacities"].to(DEV),
                                    _cams(scs), scs[0]["bg"].to(DEV), plan, scene.to(DEV))
    torch.cuda.synchronize()
    return img, plan


@pytest.mark.parametrize("degree", [0, 1, 2, 3])
def test_composite_matches_oracle_per_frame(degree):
    """Frame b's composite is the oracle's render of [dynamic_b; static] with the static colours the oracle's SH evaluation at frame b's
    camera centre: radii, sorted keys / values and ranges bit-exact, image mean-L1 <= 1e-4, the device's static rgb within 1e-6."""
    from oracle import raster_oracle as ro
    B, Pd, Ps, H, W = 3, 1500, 2500, 136, 200
    scs = _frames(B, H, W, Pd, seed=60)
    raw = random_static(Ps, degree, seed=70 + degree, center=(0.0, -0.2, 0.2), spread=(0.8, 1.0, 0.6))
    scene = scene_of(raw)
    img, plan = _composite(scs, scene)
    assert plan.check(wait=True)
    views = plan.views()
    rgb_dev = plan.scene_rgb.cpu().numpy().astype(np.float64)
    for b, sc in enumerate(scs):
        campos = sc["cam"].camera_center.double()
        rgb = pre_clamp(scene.means3D, scene.shs, degree, campos).clamp_min(0.0).numpy()
        o = ro.forward(means3D=np.concatenate([sc["means3D"].numpy(), scene.means3D.numpy()]),
                       colors=np.concatenate([sc["colors"].numpy(), rgb.astype(np.float32)]),
                       opacities=np.concatenate([sc["opacities"].numpy().reshape(-1, 1), scene.opacities.numpy().reshape(-1, 1)]),
                       scales=np.concatenate([sc["scales"].numpy(), scene.scales.numpy()]),
                       rotations=np.concatenate([sc["rotations"].numpy(), scene.rotations.numpy()]), bg=sc["bg"].numpy(),
                       viewmatrix=sc["cam"].world_view_transform.numpy(), projmatrix=sc["cam"].full_proj_transform.numpy(),
                       tanfovx=sc["tanfovx"], tanfovy=sc["tanfovy"], H=H, W=W, precision="f32")
        v = views[b]
        assert v["num_rendered"] == o.num_rendered and v["overflow"] == 0
        np.testing.assert_array_equal(v["radii"].numpy(), o.get("radii"))
        vis = o.get("radii") > 0
        assert vis[:Pd].sum() > 100 and vis[Pd:].sum() > 100
        np.testing.assert_array_equal(v["keys_sorted"].numpy().view(np.uint64), o.get("keys"))
        np.testing.assert_array_equal(v["vals_sorted"].numpy().view(np.uint32), o.get("vals"))
        np.testing.assert_array_equal(v["ranges"].numpy().view(np.uint32), o.get("ranges"))
        assert (o.get("vals") >= Pd).any() and (o.get("vals") < Pd).any()          # both sets in the lists
        vs = vis[Pd:]
        assert np.abs(rgb_dev[b][vs] - rgb[vs]).max() <= 1e-6
        assert not rgb_dev[b][~vs].any()
        assert np.abs(img[b].cpu().numpy().astype(np.float64) - o.image).mean() <= 1e-4


def test_empty_static_set_equals_rasterize_batch():
    from gaussianavatar_b200.rasterizer import RasterBatchPlan, rasterize_batch
    from gaussianavatar_b200.scene import GaussianScene
    scs = _frames(3, 96, 128, 2000, seed=80)
    z = torch.zeros(0, 3)
    empty = GaussianScene(z, z, torch.zeros(0, 4), torch.zeros(0), torch.zeros(0, 1, 3), 0)
    img, plan = _composite(scs, empty)
    ref_plan = RasterBatchPlan(3, 2000, 96, 128, DEV)
    t = {k: torch.stack([s[k] for s in scs]).to(DEV) for k in ("means3D", "colors", "scales")}
    with torch.no_grad():
        ref = rasterize_batch(t["means3D"], t["colors"], t["scales"], scs[0]["rotations"].to(DEV), scs[0]["opacities"].to(DEV),
                              _cams(scs), scs[0]["bg"].to(DEV), ref_plan)
    torch.cuda.synchronize()
    assert torch.equal(img, ref) and torch.equal(plan.radii, ref_plan.radii)
    written = [0, 1, 2, 3, 4, 5, 6, 7, 13]                # instances, overflow, segments, tiles, frame starts 4..4+B, long tiles
    assert torch.equal(plan.status_dev[written], ref_plan.status_dev[written])
    from gaussianavatar_b200.animate import final_transmittance
    assert torch.equal(final_transmittance(plan), final_transmittance(ref_plan))


def _wall(n_side, z, half, seed):
    """An opaque wall of scene Gaussians: an n_side x n_side grid in the plane at distance z in front of the reference camera."""
    E = TEST_POSE_EXTRINSIC
    Rc, tc = E[:3, :3], E[:3, 3]
    C = -Rc.T @ tc
    u = np.linspace(-half, half, n_side)
    gx, gy = np.meshgrid(u, u)
    cam_pts = np.stack([gx.ravel(), gy.ravel(), np.full(gx.size, z)], 1)
    xyz = cam_pts @ Rc + C                                # camera -> world (Rc orthonormal)
    P = xyz.shape[0]
    raw = random_static(P, 1, seed=seed)
    raw["xyz"] = xyz.astype(np.float32)
    raw["scale"] = np.full((P, 3), np.log(1.5 * 2 * half / n_side), np.float32)
    raw["opacity"] = np.full(P, 6.0, np.float32)          # sigmoid(6) = 0.9975
    return scene_of(raw)


def test_opaque_wall_hides_the_avatar():
    """Scene Gaussians between the camera and the dynamic set.  Every wall entry of a pixel's list precedes every dynamic one (the
    wall is nearer), so both walks are identical through the wall and differ only in what the remaining transmittance T of the
    scene-only render is spent on: |composite - scene-only| <= T there.  Where the wall is opaque (T < 1e-3) the dynamic set, which
    alone covers those pixels, is hidden; where there is no wall it shows."""
    from gaussianavatar_b200.animate import final_transmittance
    H, W = 128, 128
    scs = _frames(1, H, W, 3000, seed=90)
    wall = _wall(24, 1.2, 0.25, seed=91)                 # the dynamic set lies about 2.5 from the camera
    img, _ = _composite(scs, wall)
    only = dict(scs[0])
    for k in ("means3D", "colors", "scales", "rotations", "opacities"):
        only[k] = only[k][:0]
    img_scene, plan_scene = _composite([only], wall)
    behind = scene_of(random_static(1, 0, seed=0, center=(0.0, 0.0, 50.0), spread=(0.1, 0.1, 0.1)))      # behind the camera
    img_avatar, plan_avatar = _composite(scs, behind)
    T_scene = final_transmittance(plan_scene)[0]
    T_avatar = final_transmittance(plan_avatar)[0]
    d = (img[0] - img_scene[0]).abs().amax(0)
    assert (d <= T_scene + 1e-6).all()
    covered = T_scene < 1e-3
    hidden = covered & (T_avatar < 0.5)                  # pixels the dynamic set alone would cover
    assert hidden.float().mean() > 0.05
    assert d[hidden].max().item() <= 1e-3
    clear = (T_scene > 0.999) & (T_avatar < 0.5)
    assert clear.any() and (img[0] - img_avatar[0]).abs().amax(0)[clear].max().item() <= 2e-3


def test_placement_renders_the_same_image():
    """The avatar's Gaussians placed by (s, R, t) and seen through the carried camera render the unplaced image.  The placed
    camera coordinates are s x the unplaced ones up to fp32 rounding (|x| <= ~4, so ~1e-6 relative), which moves centres by
    < 1e-3 px and conics by ~1e-6: the image changes by far less than 1e-4 per pixel, except that a radius can round to the
    other side of a ceil (rect one tile larger or smaller); such a Gaussian's 3-sigma rim (alpha <= 0.011) then enters or leaves a
    few pixels.  Bound: mean-L1 <= 1e-5, pixels off by more than 1e-3 <= 0.5 %, none by more than 0.05."""
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams
    from gaussianavatar_b200.mesh_render import cameras
    from gaussianavatar_b200.rasterizer import RasterBatchPlan, rasterize_batch
    from gaussianavatar_b200.scene import Placement
    from gaussianavatar_b200 import synthetic as syn
    from gaussianavatar_b200.workload import load_poses
    a = syn.make_avatar_assets(3000, 64, seed=0, body="smpl")
    pose, transl, _ = load_poses(2)
    torch.manual_seed(0)
    m = AvatarModel.from_assets(a, [], pose, transl, batch_size=1, train=False, net_parms=NetworkParams(nf=8))
    place = Placement.from_axis_angle(1.3, [0.4, -1.1, 0.3], [1.5, -0.7, 2.2])
    H = W = 128
    K = scaled_intrinsics(TEST_POSE_K, H)
    cam = make_camera(K, TEST_POSE_EXTRINSIC, H, W)
    with torch.no_grad():
        dec = m._stage1_decoder(1)
        p, t = pose[:2].to(DEV), transl[:2].to(DEV)
        imgs = []
        for pl, c in ((None, cam), (place, place.carry(cam))):
            means, scales, colors = m._assemble(dec, p, t, placement=pl)
            plan = RasterBatchPlan(2, means.shape[1], H, W, DEV, capacity=1 << 22)
            cams = cameras([c, c]).to(DEV)
            imgs.append(rasterize_batch(means, colors, scales, m.fix_rotation, m.fix_opacity, cams, m.background, plan))
            assert plan.check(wait=True)
    d = (imgs[0] - imgs[1]).abs()
    assert (imgs[0] != m.background.view(1, 3, 1, 1)).any()
    assert d.mean().item() <= 1e-5, d.mean().item()
    assert (d > 1e-3).float().mean().item() <= 5e-3 and d.max().item() <= 0.05
    # cano2live folding agrees with placing the unplaced means on the host
    with torch.no_grad():
        m0, _, _ = m._assemble(dec, p, t)
        m1, s1, _ = m._assemble(dec, p, t, placement=place)
        s0 = m._assemble(dec, p, t)[1]
    M = torch.from_numpy(place.matrix()).to(DEV)
    want = m0.double() @ M[:, :3].T + M[:, 3]
    assert (m1.double() - want).abs().max().item() < 1e-5
    assert torch.allclose(s1, 1.3 * s0, rtol=1e-6, atol=0)


# ---- the player -------------------------------------------------------------------------------------------------------------------
SIDE = 96


def _player_setup(stage=1):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_animate_gpu import _avatar, _cameras, _clip
    m, mapper = _avatar("smpl", stage=stage)
    raw = random_static(4000, 3, seed=5, center=(0.0, -0.2, 0.3), spread=(1.0, 1.2, 1.5), scale_mean=0.08)
    return m, mapper, _clip("smpl"), _cameras, scene_of(raw)


def _play(anim, clip, fps, align_to):
    out = []
    for first, frames in anim.frames(clip, fps, align_to=align_to):
        out.append(frames.clone())
    return torch.cat(out)


def test_player_stage1_graph_replay_equals_eager_and_overflow_recovers():
    from gaussianavatar_b200 import animate as an
    from gaussianavatar_b200.scene import Placement
    m, _, clip, cams, scene = _player_setup()
    place = Placement.from_axis_angle(1.1, [0.0, 0.3, 0.0], [0.05, 0.02, -0.1])
    a = _play(an.Animator(m, cams("orbit"), SIDE, SIDE, chunk=4, channels=4, scene=scene, placement=place), clip, 45.0, 1)
    b = _play(an.Animator(m, cams("orbit"), SIDE, SIDE, chunk=4, channels=4, scene=scene, placement=place, graphs=False), clip, 45.0, 1)
    assert torch.equal(a, b)
    assert (a[..., 3] > 0).float().mean() > 0.3              # the scene fills much of the frame
    small = an.Animator(m, cams("fixed"), SIDE, SIDE, chunk=4, channels=4, scene=scene, capacity=512)
    ref = _play(an.Animator(m, cams("fixed"), SIDE, SIDE, chunk=4, channels=4, scene=scene), clip, 60.0, None)
    got = _play(small, clip, 60.0, None)
    assert small.overflows >= 1 and small.recaptures >= 1
    assert small._plans[4].capacity > 512
    assert torch.equal(got, ref)
    # the avatar is in the composite: without it the frames differ
    no_avatar = _play(an.Animator(m, cams("fixed"), SIDE, SIDE, chunk=4, channels=4), clip, 60.0, None)
    assert not torch.equal(ref, no_avatar)


def test_player_stage2_with_a_scene():
    from gaussianavatar_b200 import animate as an
    m, mapper, clip, cams, scene = _player_setup(stage=2)
    anim = an.Animator(m, cams("orbit"), SIDE, SIDE, chunk=2, channels=4, pose_mapper=mapper, scene=scene)
    got = _play(anim, clip, 30.0, 1)
    assert got.shape == (6, SIDE, SIDE, 4)
    assert (got[..., 3] == 255).any() and (got[..., :3] != 255).any()
    plain = _play(an.Animator(m, cams("orbit"), SIDE, SIDE, chunk=2, channels=4, pose_mapper=mapper), clip, 30.0, 1)
    assert (got[..., 3].int() > plain[..., 3].int()).any()      # scene Gaussians add coverage


def test_tool_with_scene(tmp_path):
    from PIL import Image
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from dataset_fixture import write_synthetic_dataset
    from gaussianavatar_b200 import animate as an
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams, OptimizationParams
    from gaussianavatar_b200.scene import GaussianScene, Placement, load_scene_cameras
    mp = write_synthetic_dataset(str(tmp_path), seed=0)
    torch.manual_seed(0)
    m = AvatarModel(mp, NetworkParams(nf=8), OptimizationParams(), train=True)
    m.training_setup()
    with torch.no_grad():
        sd = m.net.state_dict()
        sd["decoder.conv8N.bias"] = torch.tensor([-5.3])
        m.net.load_state_dict(sd, strict=False)
    m.save(7)
    room = tmp_path / "room"
    (room / "point_cloud" / "iteration_30000").mkdir(parents=True)
    ply = room / "point_cloud" / "iteration_30000" / "point_cloud.ply"
    write_ply(ply, random_static(3000, 2, seed=3, center=(0.0, 0.0, 0.5), spread=(1.5, 1.5, 1.0)), shuffle_seed=1)
    cam = np.load(os.path.join(mp.source_path, "train", "cam_parms.npz"))
    K = np.array(cam["intrinsic"], np.float32).reshape(3, 3)
    E = np.asarray(cam["extrinsic"], np.float64)
    place = Placement.from_axis_angle(1.2, [0.0, 0.2, 0.0], [0.1, 0.0, 0.3])
    write_cameras_json(room / "cameras.json", [(K, place.extrinsic(E), 64, 64)])
    clip_path = os.path.join(mp.test_folder, "smpl_parms.pth")
    png = tmp_path / "png"
    cmd = [sys.executable, os.path.join(ROOT, "tools", "animate.py"), "-s", mp.source_path, "-m", mp.model_path, "--project_path",
           mp.project_path, "--smpl_model", os.path.join(mp.smpl_model_path, "SMPL_NEUTRAL.pkl"), "--query_posmap_size", str(mp.query_posmap_size), "--inp_posmap_size", str(mp.inp_posmap_size), "--epoch", "7",
           "--stage", "1", "--motion", clip_path, "--clip_fps", "30", "--body", "smpl", "--fps", "30", "--align_to", "1",
           "--scene", str(ply), "--place", "1.2", "0", "0.2", "0", "0.1", "0", "0.3", "--camera", "scene:0", "--chunk", "2", "--png", str(png)]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    mp2 = type(mp)(**{**vars(mp), "batch_size": 1})
    model = AvatarModel(mp2, NetworkParams(nf=8), OptimizationParams(), train=False)
    model.load(7)
    clip = an.MotionClip.load(clip_path, "smpl", fps=30)
    scene = GaussianScene.load_ply(ply)
    want = _play(an.Animator(model, load_scene_cameras(room / "cameras.json")[0], 64, 64, chunk=2, scene=scene, placement=place), clip,
                 30.0, 1).numpy()
    names = sorted(os.listdir(png))
    assert names == ["{:05d}.png".format(i) for i in range(want.shape[0])]
    got = np.stack([np.array(Image.open(png / n)) for n in names])
    # as in test_animate_gpu's tool test: the decoder's atomics may move the last bits between processes
    d = np.abs(got.astype(int) - want.astype(int))
    assert d.max() <= 1 and (d == 0).mean() > 0.995
    assert (want[..., :3] != 255).any()
