"""GPU: the animation player.  ga_motion_sample and ga_frame_pack against oracle/animate_oracle.py; every frame the stage-1
Animator yields against the packed render_free_stage1 of that frame alone (SMPL and SMPL-X, chunks 1 / 3 / 8 with a partial last
chunk, fixed and orbit cameras, RGB and RGBA), a forced binning overflow, stage 2 against render_free_stage2 with the sampled pose
written into the model's table, the model's state after animating, and tools/animate.py end to end on a saved checkpoint."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gaussianavatar_b200 import animate as an
from gaussianavatar_b200 import synthetic as syn
from gaussianavatar_b200.avatar_model import AvatarModel
from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, TEST_POSE_K, scaled_intrinsics
from gaussianavatar_b200.config import NetworkParams
from gaussianavatar_b200.dataset import camera_item
from gaussianavatar_b200.workload import load_poses
from oracle import animate_oracle as ao

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIDE = 96
Rotation = pytest.importorskip("scipy.spatial.transform").Rotation


# ---- kernels ----------------------------------------------------------------------------------------------------------------------
def _clip_arrays(T, J, seed):
    g = np.random.default_rng(seed)
    aa = Rotation.random(T * J, random_state=seed).as_rotvec().reshape(T, J, 3)
    ax = g.normal(size=(J, 3))
    ax /= np.linalg.norm(ax, axis=-1, keepdims=True)
    aa[1] = ax * (np.pi - g.uniform(0, 1e-6, size=(J, 1)))          # angles near pi
    aa[2, :5] = ax[:5] * np.pi
    th = np.linalg.norm(aa[3], axis=-1, keepdims=True)
    aa[4] = -aa[3] / th * (2 * np.pi - th)                           # antipodal neighbours
    return aa.reshape(T, J * 3).astype(np.float32), g.normal(0, 1, size=(T, 3)).astype(np.float32)


@pytest.mark.parametrize("J", [24, 55])
def test_motion_sample_matches_oracle(J):
    T = 9
    pose, trans = _clip_arrays(T, J, seed=J)
    times = np.concatenate([np.arange(T, dtype=np.float64), np.linspace(-2, T + 2, 53), [0.5, 1.5, 3.5, 3.0 + 1e-9, np.nan]])
    align = np.concatenate([Rotation.random(random_state=J + 1).as_matrix().reshape(9), [0.5, -2.0, 1.25]])
    for al in (an.IDENTITY_ALIGN, align):
        n = len(times)
        pose_out = torch.full((n, J * 3), float("nan"), device=DEV)
        trans_out = torch.full((n, 3), float("nan"), device=DEV)
        an.motion_sample(torch.from_numpy(pose).to(DEV), torch.from_numpy(trans).to(DEV), torch.from_numpy(times).to(DEV),
                         torch.from_numpy(al).to(DEV), pose_out, trans_out)
        torch.cuda.synchronize()
        gp, gt = pose_out.cpu().double().numpy(), trans_out.cpu().double().numpy()
        assert np.isfinite(gp).all() and np.isfinite(gt).all()
        wp, wt = ao.motion_sample(pose, trans, times, al)
        Rg = Rotation.from_rotvec(gp.reshape(-1, 3)).as_matrix()
        Rw = Rotation.from_rotvec(wp.reshape(-1, 3)).as_matrix()
        assert np.abs(Rg - Rw).max() < 2e-6
        assert (np.abs(gt - wt) <= 1e-6 * np.maximum(np.abs(wt), 1.0)).all()
        assert (np.linalg.norm(gp.reshape(-1, 3), axis=-1) <= np.pi + 1e-6).all()


def _pack_inputs(B, H, W, seed):
    g = np.random.default_rng(seed)
    img = g.uniform(-0.05, 1.05, size=(B, 3, H, W)).astype(np.float32)
    k = g.integers(0, 256, size=img.size // 4)
    edge = ((k - 0.5) / 255.0).astype(np.float32)
    flat = img.reshape(-1)
    flat[: edge.size] = np.where(g.random(edge.size) < 0.5, np.nextafter(edge, np.float32(2)), np.nextafter(edge, np.float32(-2)))
    special = np.array([np.nan, np.inf, -np.inf, -0.0, 1.0, 0.0, 300.0], np.float32)
    m = min(special.size, flat.size - edge.size)
    flat[edge.size:edge.size + m] = special[:m]
    Tr = g.uniform(0, 1, size=(B, H, W)).astype(np.float32)
    Tf = Tr.reshape(-1)
    Tf[::3] = 1.0
    Tf[1::7] = 0.0
    Tf[2::11] = np.float32(1.0 - 1.0 / 512)
    return img, Tr


@pytest.mark.parametrize("H,W", [(1, 1), (540, 960), (1023, 1025)])
@pytest.mark.parametrize("C", [3, 4])
def test_frame_pack_bit_exact(H, W, C):
    bg = np.array([1.0, 0.25, 0.0], np.float32)
    Bs = range(1, 9) if H * W < 10 else (1, 3, 8)
    for B in Bs:
        img, Tr = _pack_inputs(B, H, W, seed=B + C)
        out = torch.full((B, H, W, C), 0xAB, dtype=torch.uint8, device=DEV)
        an.frame_pack(torch.from_numpy(img).to(DEV), torch.from_numpy(Tr).to(DEV), torch.from_numpy(bg).to(DEV), C, out)
        want = ao.frame_pack(img, Tr, bg, C)
        assert np.array_equal(out.cpu().numpy(), want), (B, H, W, C)


# ---- the player -------------------------------------------------------------------------------------------------------------------
def _avatar(body, stage=1, N=3000, S=64, inp=32):
    a = syn.make_avatar_assets(N, S, seed=0, body=body)
    pose, transl, _ = load_poses(6)
    if body == "smplx":
        pose = pose[:, :66].contiguous()
    fields = dict(train_stage=2, inp_posmap_size=inp) if stage == 2 else {}
    torch.manual_seed(0)
    m = AvatarModel.from_assets(a, [], pose, transl, batch_size=1, train=False, net_parms=NetworkParams(nf=8), **fields)
    with torch.no_grad():
        sd = m.net.state_dict()
        sd["decoder.conv8N.bias"] = torch.tensor([-5.3])
        m.net.load_state_dict(sd, strict=False)
    mapper = None
    if stage == 2:
        from gaussianavatar_b200.posmap import PoseMapper, SmplxPoseMapper
        if body == "smplx":
            t = syn.make_smplx_uv_template(0)
            mapper = SmplxPoseMapper(syn.smplx_mesh_model(a.body, t, syn.smplx_posedirs(0)), a.body.betas[0], t, inp, device=DEV)
        else:
            t = syn.make_uv_template(0)
            mapper = PoseMapper(syn.smpl_mesh_model(a.body, t), a.body.betas[0], t, inp, device=DEV)
    return m, mapper


def _clip(body, T=6):
    pose, transl, _ = load_poses(T)
    if body == "smplx":
        pose = torch.cat([pose[:, :66], syn.synthetic_smplx_poses(T, seed=0)[1]], 1)
    return an.MotionClip(pose.float().contiguous(), transl.float().contiguous(), 30.0, body)


def _cameras(kind):
    K = scaled_intrinsics(TEST_POSE_K, SIDE)
    return camera_item(K, TEST_POSE_EXTRINSIC, SIDE, SIDE) if kind == "fixed" else an.OrbitCamera(K, TEST_POSE_EXTRINSIC)


def _model_state(m):
    sd = {("net." + k): v.detach().cpu().clone() for k, v in m.net.state_dict().items()}
    if hasattr(m, "pose_encoder"):
        sd.update({("enc." + k): v.detach().cpu().clone() for k, v in m.pose_encoder.state_dict().items()})
    sd["pose"], sd["transl"] = m.pose.weight.detach().cpu().clone(), m.transl.weight.detach().cpu().clone()
    sd["geo"] = m.geo_feature.detach().cpu().clone()
    return sd


def _same_state(a, b):
    return a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)


def _play(anim, clip, fps, align_to):
    out = []
    for first, frames in anim.frames(clip, fps, align_to=align_to):
        assert first == sum(f.shape[0] for f in out)
        out.append(frames.clone())                      # the pinned buffer is reused two chunks later
    return torch.cat(out)


def _expected_stage1(m, anim, clip, fps, align_to, channels):
    sched = anim.schedule(clip, fps, align_to=align_to)
    pose, trans = anim.sample(clip, sched)
    want, alphas = [], []
    for i in range(len(sched.times)):
        batch = {"pose_data": pose[i:i + 1, :66] if m.smplx else pose[i:i + 1], "transl_data": trans[i:i + 1],
                 "_cams": sched.cams[i:i + 1].to(DEV), "height": [SIDE], "width": [SIDE]}
        if m.smplx:
            batch["rest_pose"] = pose[i:i + 1, 66:]
        with torch.no_grad():
            img = m.render_free_stage1(batch, 59400)
            Tr = an.final_transmittance(m._last_plan)
            want.append(an.frame_pack(img, Tr, m.background, channels).cpu())
            alphas.append(ao.quant8(np.float32(1.0) - Tr.cpu().numpy()))
    return torch.cat(want), np.concatenate(alphas)


@pytest.mark.parametrize("body", ["smpl", "smplx"])
@pytest.mark.parametrize("chunk,camera,channels", [(1, "fixed", 3), (3, "orbit", 4), (8, "fixed", 4), (8, "orbit", 3), (3, "fixed", 3)])
def test_stage1_frames_equal_single_frame_renders(body, chunk, camera, channels):
    m, _ = _avatar(body)
    clip = _clip(body)
    anim = an.Animator(m, _cameras(camera), SIDE, SIDE, chunk=chunk, channels=channels)
    before = _model_state(m)
    got = _play(anim, clip, 60.0, 2)                       # 6 keys at 30 fps -> 11 frames at 60 fps: partial last chunks
    assert _same_state(before, _model_state(m))
    assert got.shape == (11, SIDE, SIDE, channels) and anim.captures >= 1
    want, alpha = _expected_stage1(m, anim, clip, 60.0, 2, channels)
    assert torch.equal(got, want)
    if channels == 3:          # the body is in the frame, on the white background
        assert (got != 255).any() and (got == 255).any()
    else:
        assert (got[..., 3] > 0).any() and (got[..., 3] == 0).any()
    if channels == 4:
        assert np.array_equal(got[..., 3].numpy(), alpha)
    # a second playback of the same clip replays the captured graphs
    n = anim.captures
    assert torch.equal(_play(anim, clip, 60.0, 2), want) and anim.captures == n


def test_stage1_forced_overflow_recaptures():
    m, _ = _avatar("smpl")
    clip = _clip("smpl")
    ref = _play(an.Animator(m, _cameras("fixed"), SIDE, SIDE, chunk=4, channels=4), clip, 60.0, None)
    anim = an.Animator(m, _cameras("fixed"), SIDE, SIDE, chunk=4, channels=4, capacity=64)
    got = _play(anim, clip, 60.0, None)
    assert anim.overflows >= 1 and anim.recaptures >= 1
    assert torch.equal(got, ref)


def test_stage1_graphs_off_gives_the_same_bytes():
    m, _ = _avatar("smplx")
    clip = _clip("smplx")
    a = _play(an.Animator(m, _cameras("orbit"), SIDE, SIDE, chunk=3), clip, 45.0, 1)
    b = _play(an.Animator(m, _cameras("orbit"), SIDE, SIDE, chunk=3, graphs=False), clip, 45.0, 1)
    assert torch.equal(a, b)


@pytest.mark.parametrize("body", ["smpl", "smplx"])
def test_stage2_frames_equal_render_free_stage2(body):
    """Two stage-2 forwards of the same frame may differ in the last bits: the decoder's per-frame BatchNorm sums are accumulated
    with atomics, in no fixed order.  Un-compositing divides by alpha, which magnifies such a difference where alpha is small, so
    bytes may differ by one step; a wrong pose or map would move whole regions of the frame."""
    m, mapper = _avatar(body, stage=2)
    clip = _clip(body)
    anim = an.Animator(m, _cameras("orbit"), SIDE, SIDE, chunk=3, channels=4, pose_mapper=mapper)
    before = _model_state(m)
    with torch.backends.cudnn.flags(deterministic=True):
        got = _play(anim, clip, 45.0, 1)
    assert _same_state(before, _model_state(m))
    sched = anim.schedule(clip, 45.0, align_to=1)
    pose, trans = anim.sample(clip, sched)
    F = m.pose.weight.shape[0]
    assert got.shape[0] == len(sched.times) > F           # more frames than the training table has rows
    for i in range(got.shape[0]):
        r = i % F
        with torch.no_grad(), torch.backends.cudnn.flags(deterministic=True):
            m.pose.weight[r] = pose[i, :m.pose.weight.shape[1]]
            m.transl.weight[r] = trans[i]
            batch = {"pose_idx": torch.tensor([r], device=DEV), "_cams": sched.cams[i:i + 1].to(DEV), "height": [SIDE], "width": [SIDE]}
            if m.smplx:
                batch["rest_pose"] = pose[i:i + 1, 66:]
                batch["inp_pos_map"] = mapper(pose[i:i + 1, :66], pose[i:i + 1, 66:], trans[i:i + 1])
            else:
                batch["inp_pos_map"] = mapper(pose[i:i + 1], trans[i:i + 1])
            img = m.render_free_stage2(batch, 59400)
            want = an.frame_pack(img, an.final_transmittance(m._last_plan), m.background, 4).cpu()[0]
        d = (got[i].int() - want.int()).abs()
        opaque = want[..., 3] >= 64                              # alpha >= 1/4: at most a 4x magnification
        assert d[..., 3].max() <= 1 and d[opaque].max() <= 1, i
        assert (d == 0).float().mean() > 0.995, i
        assert (want[..., 3] > 0).any(), i


def test_tool_end_to_end(tmp_path):
    from PIL import Image
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from dataset_fixture import write_synthetic_dataset
    from gaussianavatar_b200.config import OptimizationParams
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
    png, raw = tmp_path / "png", tmp_path / "frames.rgba"
    cmd = [sys.executable, os.path.join(ROOT, "tools", "animate.py"), "-s", mp.source_path, "-m", mp.model_path, "--project_path",
           mp.project_path, "--smpl_model", os.path.join(mp.smpl_model_path, "SMPL_NEUTRAL.pkl"), "--query_posmap_size",
           str(mp.query_posmap_size), "--inp_posmap_size", str(mp.inp_posmap_size), "--epoch", "7", "--stage", "1", "--motion", clip_path, "--clip_fps", "30", "--body", "smpl",
           "--fps", "50", "--align_to", "1", "--camera", "orbit", "--size", "80", "48", "--chunk", "3", "--rgba", "--png", str(png),
           "--raw", str(raw)]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    # the same playback in process
    mp2 = type(mp)(**{**vars(mp), "batch_size": 1})
    model = AvatarModel(mp2, NetworkParams(nf=8), OptimizationParams(), train=False)
    model.load(7)
    cam = np.load(os.path.join(mp.source_path, "train", "cam_parms.npz"))
    K = np.array(cam["intrinsic"], np.float32).reshape(3, 3)
    K[0, :] *= 80 / 64
    K[1, :] *= 48 / 64
    clip = an.MotionClip.load(clip_path, "smpl", fps=30)
    want = _play(an.Animator(model, an.OrbitCamera(K, np.asarray(cam["extrinsic"])), 48, 80, chunk=3, channels=4), clip, 50.0, 1).numpy()
    n = want.shape[0]
    data = raw.read_bytes()
    assert len(data) == n * 48 * 80 * 4
    got = np.frombuffer(data, np.uint8).reshape(n, 48, 80, 4)
    names = sorted(os.listdir(png))
    assert names == ["{:05d}.png".format(i) for i in range(n)]
    for i, name in enumerate(names):
        assert np.array_equal(np.array(Image.open(png / name)), got[i])
    # The tool's process evaluates the decoder once on its own, and the decoder's BatchNorm sums use atomics: its output can
    # differ from this process's in the last bits, which un-compositing magnifies where alpha is small (as in the stage-2 test).
    d = np.abs(got.astype(int) - want.astype(int))
    assert d[..., 3].max() <= 1 and d[want[..., 3] >= 64].max() <= 1
    assert (d == 0).mean() > 0.995 and (want[..., 3] > 0).any()
