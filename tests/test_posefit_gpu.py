"""GPU: test-time pose fitting.  The new backward kernels (ga_smpl_vertices_backward, ga_smplx_vertices_backward,
ga_posmap_fill_backward) against the autograd gradients of oracle/posefit_oracle.py and their bit-reproducibility across calls and
batch compositions; the differentiable position-map mapper; PoseFitter's recovery of known poses (stage 1 and 2, SMPL and SMPL-X),
its chunk independence, overflow handling and untouched model state; and tools/fit_poses.py end to end on a saved checkpoint."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gaussianavatar_b200 import synthetic as syn
from gaussianavatar_b200.avatar_model import AvatarModel
from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, TEST_POSE_K, scaled_intrinsics
from gaussianavatar_b200.config import NetworkParams
from gaussianavatar_b200.dataset import camera_item
from gaussianavatar_b200.posefit import PoseFitter
from gaussianavatar_b200.posmap import PoseMapper, SmplxPoseMapper, vertices_backward
from gaussianavatar_b200.workload import load_poses
from oracle import posefit_oracle as pfo

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# fp32 kernels against fp64 autograd: the gradients are sums over ~10^4 vertices (and 10^5 texels) of fp32 products
REL = 1e-3


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _mapper(body, S):
    if body == "smpl":
        b, t = syn.make_body(0), syn.make_uv_template(0)
        model = syn.smpl_mesh_model(b, t)
        return PoseMapper(model, b.betas[0], t, S, device=DEV), model, b.betas[0], t
    b, t = syn.make_smplx_body(0), syn.make_smplx_uv_template(0)
    model = syn.smplx_mesh_model(b, t, syn.smplx_posedirs(0))
    return SmplxPoseMapper(model, b.betas[0], t, S, device=DEV), model, b.betas[0], t


def _poses(body, B, seed):
    if body == "smpl":
        p, t = syn.synthetic_poses(B, seed=seed)
        return p, None, t
    return syn.synthetic_smplx_poses(B, seed=seed)


# ---- kernels ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("body", ["smpl", "smplx"])
def test_vertices_backward_matches_oracle_and_is_batch_independent(body):
    mapper, model, betas, _ = _mapper(body, 32)
    ob = pfo.Body(model, betas.numpy())
    p, r, t = _poses(body, 8, seed=5)
    g = torch.randn(8, mapper.V, 3, generator=torch.Generator().manual_seed(6))
    full = p.double() if r is None else torch.cat([p.double(), r.double()], 1)
    x = torch.cat([full, t.double()], 1).requires_grad_(True)
    v = pfo.vertices(ob, x[:, :-3], x[:, -3:])
    want, = torch.autograd.grad((v * g.double()).sum(), x)
    W = p.shape[1]
    pd, rd, td, gd = p.to(DEV), (r.to(DEV) if r is not None else None), t.to(DEV), g.to(DEV)
    results = {}
    for B in (1, 2, 8):
        dp, dt = vertices_backward(mapper, pd[:B].contiguous(), rd[:B].contiguous() if rd is not None else None, gd[:B].contiguous())
        torch.cuda.synchronize()
        for b in range(B):
            assert _rel(dp[b], want[b, :W]) < REL, (B, b, _rel(dp[b], want[b, :W]))
            assert _rel(dt[b], want[b, -3:]) < REL
        results[B] = (dp, dt)
        again = vertices_backward(mapper, pd[:B].contiguous(), rd[:B].contiguous() if rd is not None else None, gd[:B].contiguous())
        assert torch.equal(again[0], dp) and torch.equal(again[1], dt)          # bit-reproducible
    for B in (1, 2):      # a frame's result does not depend on the batch it is in
        assert torch.equal(results[B][0], results[8][0][:B]) and torch.equal(results[B][1], results[8][1][:B])
    # a frame at a later position in another batch
    dp, dt = vertices_backward(mapper, pd[5:8].contiguous(), rd[5:8].contiguous() if rd is not None else None, gd[5:8].contiguous())
    assert torch.equal(dp, results[8][0][5:8]) and torch.equal(dt, results[8][1][5:8])


@pytest.mark.parametrize("S", [32, 128, 512])
@pytest.mark.parametrize("body", ["smpl", "smplx"])
def test_fill_backward_matches_oracle_and_is_batch_independent(body, S):
    mapper, _, _, t = _mapper(body, S)
    face_id, bary = mapper.face_id.cpu().numpy(), mapper.bary.cpu().numpy()
    d = torch.randn(8, 3, S, S, generator=torch.Generator().manual_seed(S))
    verts = torch.zeros(8, mapper.V, 3, dtype=torch.float64, requires_grad=True)
    want, = torch.autograd.grad((pfo.fill(verts, t[1], face_id, bary) * d.double()).sum(), verts)
    outs = {}
    for B in (1, 2, 8):
        got = mapper.fill_backward(d[:B].to(DEV))
        torch.cuda.synchronize()
        assert torch.isfinite(got).all()
        for b in range(B):
            assert _rel(got[b], want[b]) < 1e-5, (B, b)
        assert torch.equal(mapper.fill_backward(d[:B].to(DEV)), got)
        outs[B] = got
    assert torch.equal(outs[1], outs[8][:1]) and torch.equal(outs[2], outs[8][:2])
    # vertices no texel uses get exactly 0 (SMPL-X's last 25 vertices belong to no face)
    used = np.zeros(mapper.V, bool)
    used[np.asarray(t[1])[face_id[face_id >= 0]].reshape(-1)] = True
    assert (outs[8][:, torch.from_numpy(~used).to(DEV)] == 0).all()
    # the CSR: ascending entries per vertex, every (covered texel, corner) exactly once
    offsets, entries = (a.cpu().numpy() for a in mapper.vertex_csr())
    n = int(offsets[-1])
    assert n == 3 * int((face_id >= 0).sum())
    e = entries[:n]
    assert np.array_equal(np.sort(e), np.sort((3 * np.nonzero(face_id.reshape(-1) >= 0)[0][:, None] + np.arange(3)).reshape(-1)))
    for v in range(0, mapper.V, 97):
        seg = e[offsets[v]:offsets[v + 1]]
        assert (np.diff(seg) > 0).all()


@pytest.mark.parametrize("body", ["smpl", "smplx"])
def test_differentiable_mapper(body):
    mapper, model, betas, t = _mapper(body, 128)
    p, r, tr = _poses(body, 3, seed=9)
    pd, td = p.to(DEV).requires_grad_(True), tr.to(DEV).requires_grad_(True)
    rd = r.to(DEV) if r is not None else None
    args = (pd, td) if r is None else (pd, rd, td)
    live = mapper(*args)
    with torch.no_grad():
        plain = mapper(*((p.to(DEV), tr.to(DEV)) if r is None else (p.to(DEV), rd, tr.to(DEV))))
    assert torch.equal(live.detach(), plain)
    wm = torch.randn(3, 3, 128, 128, generator=torch.Generator().manual_seed(2))
    gp, gt = torch.autograd.grad((live * wm.to(DEV)).sum(), (pd, td))
    ob = pfo.Body(model, betas.numpy())
    fid, bary = mapper.face_id.cpu().numpy(), mapper.bary.cpu().numpy()
    x = torch.cat([p.double(), tr.double()], 1).requires_grad_(True)
    full = x[:, :-3] if r is None else torch.cat([x[:, :-3], r.double()], 1)
    want, = torch.autograd.grad((pfo.fill(pfo.vertices(ob, full, x[:, -3:]), t[1], fid, bary) * wm.double()).sum(), x)
    assert _rel(gp, want[:, :-3]) < REL and _rel(gt, want[:, -3:]) < REL


# ---- the fitter -------------------------------------------------------------------------------------------------------------------
SIDE = 128


def _avatar(body, stage):
    a = syn.make_avatar_assets(4000, 64, seed=0, body=body)
    pose, transl, _ = load_poses(6)
    if body == "smplx":
        pose = pose[:, :66].contiguous()
    fields = dict(train_stage=2, inp_posmap_size=32) if stage == 2 else {}
    torch.manual_seed(0)
    m = AvatarModel.from_assets(a, [], pose, transl, batch_size=1, train=False, net_parms=NetworkParams(nf=8), **fields)
    with torch.no_grad():
        sd = m.net.state_dict()
        sd["decoder.conv8N.bias"] = torch.tensor([-5.3])
        m.net.load_state_dict(sd, strict=False)
    mapper = _mapper(body, 32)[0] if stage == 2 else None
    return m, mapper


def _render(m, mapper, pose, transl, rest, cam):
    """Frames [n,3,H,W] of the avatar at the given poses, one at a time."""
    out = []
    K = {k: [cam[k]] for k in ("FovX", "FovY", "world_view_transform", "full_proj_transform")}
    with torch.no_grad():
        for i in range(pose.shape[0]):
            p, t = pose[i:i + 1].to(DEV), transl[i:i + 1].to(DEV)
            rp = rest[i:i + 1].to(DEV) if rest is not None else None
            batch = dict(K, height=[SIDE], width=[SIDE], pose_data=p, transl_data=t)
            if rp is not None:
                batch["rest_pose"] = rp
            if mapper is None:
                img = m.render_free_stage1(batch, 59400)
            else:
                batch["inp_pos_map"] = mapper(p, rp, t) if rp is not None else mapper(p, t)
                means, scales, colors, _, _ = m._stage2_gaussians(batch, pose=p, transl=t)
                img = m._render_frames(batch, means, scales, colors)
            out.append(img[0].cpu())
    return torch.stack(out)


PERTURBED = [0, 1, 2, 3, 4, 5, 6, 7, 8, 12, 13, 14, 48, 49, 50, 51, 52, 53]      # root, hips, knees, shoulders


def _problem(body, stage, n=4, seed=0):
    """(model, mapper, frames with perturbed poses, true pose, true transl)."""
    m, mapper = _avatar(body, stage)
    pose, transl, _ = load_poses(n)
    pose, transl = pose.float(), transl.float()
    rest = syn.synthetic_smplx_poses(n, seed=0)[1] if body == "smplx" else None
    if body == "smplx":
        pose = pose[:, :66].contiguous()
    cam = camera_item(scaled_intrinsics(TEST_POSE_K, SIDE), TEST_POSE_EXTRINSIC, SIDE, SIDE)
    images = _render(m, mapper, pose, transl, rest, cam)
    g = torch.Generator().manual_seed(100 + seed)
    noisy = pose.clone()
    noisy[:, PERTURBED] += torch.randn(n, len(PERTURBED), generator=g) * 0.08
    ntransl = transl + torch.randn(n, 3, generator=g) * 0.03
    frames = []
    for i in range(n):
        it = dict(cam, original_image=images[i], pose_data=noisy[i], transl_data=ntransl[i])
        if rest is not None:
            it["rest_pose"] = rest[i]
        frames.append(it)
    return m, mapper, frames, pose, transl


def _model_state(m):
    sd = {("net." + k): v.detach().cpu().clone() for k, v in m.net.state_dict().items()}
    if hasattr(m, "pose_encoder"):
        sd.update({("enc." + k): v.detach().cpu().clone() for k, v in m.pose_encoder.state_dict().items()})
    sd["pose"], sd["transl"] = m.pose.weight.detach().cpu().clone(), m.transl.weight.detach().cpu().clone()
    sd["geo"] = m.geo_feature.detach().cpu().clone()
    sd["bn_running"] = m.net.bn_running.detach().cpu().clone()
    sd["counts"] = torch.tensor([int(st.num_batches_tracked) for st in m.net._states.values()])
    return sd


def _same_state(a, b):
    return a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)


def _error(pose, transl, true_pose, true_transl):
    return float(torch.cat([pose - true_pose, transl - true_transl], 1).norm())


@pytest.mark.parametrize("stage", [1, 2])
@pytest.mark.parametrize("body", ["smpl", "smplx"])
def test_recovers_known_poses(body, stage):
    """The error is measured over what was displaced: the perturbed pose components and transl.  The other components start at the
    known pose and are free too; those with little effect on a 128^2 render of the synthetic body (hands, feet, face) are barely
    observable and drift by up to a few tenths of a radian, most in stage 2, where every joint also moves the input map."""
    m, mapper, frames, tp, tt = _problem(body, stage)
    before = _model_state(m)
    fitter = PoseFitter(m, iters=150, pose_mapper=mapper)
    pose, transl, report = fitter.fit(frames)
    assert _same_state(before, _model_state(m))
    assert all(p.grad is None for p in m.net.parameters())
    init_p = torch.stack([f["pose_data"] for f in frames])
    init_t = torch.stack([f["transl_data"] for f in frames])
    P = PERTURBED
    e0, e1 = _error(init_p[:, P], init_t, tp[:, P], tt), _error(pose[:, P], transl, tp[:, P], tt)
    assert e1 <= 0.5 * e0, (e0, e1)
    for r in report:
        assert r["fitted_loss"] <= r["initial_loss"] and 0 <= r["best_iter"] <= 150
    assert sum(r["fitted_loss"] for r in report) < 0.1 * sum(r["initial_loss"] for r in report)


def test_stage1_chunk_independence():
    """A frame's fit does not depend on its chunk.  The rasterizer's backward adds gradients with floating-point atomics, so two fits
    of the same frame differ in the last bits of each gradient; Adam's normalised steps can carry such a difference into a component
    whose gradient is near zero by up to a step of lr per iteration.  Tolerance: 1e-2 (rad / m) per component, and the fitted
    losses within 1e-2 relative (1.4e-3 was seen on an H100)."""
    m, _, frames, _, _ = _problem("smpl", 1, n=8, seed=1)
    p8, t8, r8 = PoseFitter(m, iters=40, chunk=8).fit(frames)
    p3, t3, r3 = PoseFitter(m, iters=40, chunk=3).fit(frames)
    assert (p8 - p3).abs().max() < 1e-2 and (t8 - t3).abs().max() < 1e-2
    for a, b in zip(r8, r3):
        assert a["initial_loss"] == b["initial_loss"]                  # the forward is deterministic
        assert abs(a["fitted_loss"] - b["fitted_loss"]) <= 1e-2 * a["fitted_loss"]


def test_iters_zero_returns_the_input_poses():
    m, _, frames, _, _ = _problem("smplx", 1, n=3)
    pose, transl, report = PoseFitter(m, iters=0).fit(frames)
    assert torch.equal(pose, torch.stack([f["pose_data"] for f in frames]))
    assert torch.equal(transl, torch.stack([f["transl_data"] for f in frames]))
    assert all(r["best_iter"] == 0 and r["fitted_loss"] == r["initial_loss"] for r in report)


@pytest.mark.parametrize("stage", [1, 2])
def test_forced_overflow_gives_the_same_fit(stage):
    """The same tolerances as the chunk test; in stage 2 the forward differs in the last bits too (the decoder's BatchNorm sums use
    atomics), so the initial losses agree to 1e-5 relative there."""
    m, mapper, frames, _, _ = _problem("smpl", stage, n=3)
    ref = PoseFitter(m, iters=20, pose_mapper=mapper).fit(frames)
    f = PoseFitter(m, iters=20, pose_mapper=mapper, capacity=64)
    got = f.fit(frames)
    assert f.overflows >= 1
    assert (got[0] - ref[0]).abs().max() < 1e-2 and (got[1] - ref[1]).abs().max() < 1e-2
    for a, b in zip(got[2], ref[2]):
        assert abs(a["initial_loss"] - b["initial_loss"]) <= (0.0 if stage == 1 else 1e-5 * b["initial_loss"])
        assert abs(a["fitted_loss"] - b["fitted_loss"]) <= 1e-2 * b["fitted_loss"]


@pytest.mark.parametrize("body", ["smpl", "smplx"])
def test_stage2_map_gradient_is_live(body):
    """The pose gradient of the stage-2 loss with the map built from the pose differs from the one with the map held constant."""
    from gaussianavatar_b200.losses import image_loss
    from gaussianavatar_b200.avatar_model import kept_state
    m, mapper, frames, _, _ = _problem(body, 2, n=1)
    it = frames[0]
    cams = m._batch_cameras({k: [it[k]] for k in ("FovX", "FovY", "world_view_transform", "full_proj_transform")}, 1, DEV)
    rest = it["rest_pose"][None].to(DEV) if body == "smplx" else None
    grads = []
    with kept_state(m):
        for detach in (False, True):
            p = it["pose_data"][None].to(DEV).requires_grad_(True)
            t = it["transl_data"][None].to(DEV).requires_grad_(True)
            pm, tm = (p.detach(), t.detach()) if detach else (p, t)
            inp = mapper(pm, rest, tm) if rest is not None else mapper(pm, tm)
            batch = {"inp_pos_map": inp, "rest_pose": rest, "_cams": cams, "height": [SIDE], "width": [SIDE]}
            means, scales, colors, _, _ = m._stage2_gaussians(batch, pose=p, transl=t)
            img = m._render_frames(batch, means, scales, colors)
            loss = image_loss(img, it["original_image"][None].to(DEV), 0.2)
            grads.append(torch.cat(torch.autograd.grad(loss, (p, t)), 1))
    live, const = grads
    assert torch.isfinite(live).all() and const.norm() > 0
    assert _rel(live, const) > 1e-3


def test_tool_end_to_end(tmp_path):
    from gaussianavatar_b200.config import OptimizationParams
    from gaussianavatar_b200.dataset import MonoDataset_test
    from gaussianavatar_b200.metrics import PeakSignalNoiseRatio
    from PIL import Image
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from dataset_fixture import write_synthetic_dataset
    mp = write_synthetic_dataset(str(tmp_path), N=1000, S=32, num_frames=4, side=96, seed=0)
    torch.manual_seed(0)
    m = AvatarModel(mp, NetworkParams(nf=8), OptimizationParams(), train=True)
    m.training_setup()
    with torch.no_grad():
        sd = m.net.state_dict()
        sd["decoder.conv8N.bias"] = torch.tensor([-5.3])
        m.net.load_state_dict(sd, strict=False)
    m.save(7)
    mp2 = type(mp)(**{**vars(mp), "batch_size": 1})
    model = AvatarModel(mp2, NetworkParams(nf=8), OptimizationParams(), train=False)
    model.load(7)
    test_dir = os.path.join(mp.source_path, "test")
    parms = torch.load(os.path.join(test_dir, "smpl_parms.pth"), weights_only=False)
    true_pose, true_transl = parms["body_pose"].float(), parms["trans"].float()
    ds = MonoDataset_test(mp2)

    def render(pose, transl):
        out = []
        with torch.no_grad():
            for i in range(len(ds)):
                it = ds[i]
                batch = {k: [it[k]] for k in ("FovX", "FovY", "world_view_transform", "full_proj_transform", "height", "width")}
                batch.update(pose_data=pose[i:i + 1].to(DEV), transl_data=transl[i:i + 1].to(DEV))
                out.append(model.render_free_stage1(batch, 59400)[0])
        return torch.stack(out)

    # the split's images are renders at the true poses; its pose file holds perturbed ones
    imgs = render(true_pose, true_transl)
    for i, name in enumerate(sorted(os.listdir(os.path.join(test_dir, "images")))):
        u8 = (imgs[i].clamp(0, 1) * 255 + 0.5).byte().permute(1, 2, 0).cpu().numpy()
        Image.fromarray(u8, "RGB").save(os.path.join(test_dir, "images", name))
        Image.fromarray(np.full(u8.shape[:2], 255, np.uint8), "L").save(os.path.join(test_dir, "masks", name))
    g = torch.Generator().manual_seed(3)
    bad_pose = true_pose.clone()
    bad_pose[:, PERTURBED] += torch.randn(bad_pose.shape[0], len(PERTURBED), generator=g) * 0.08
    bad_transl = true_transl + torch.randn(true_transl.shape, generator=g) * 0.03
    torch.save(dict(parms, body_pose=bad_pose, trans=bad_transl), os.path.join(test_dir, "smpl_parms.pth"))
    cmd = [sys.executable, os.path.join(ROOT, "tools", "fit_poses.py"), "-s", mp.source_path, "-m", mp.model_path, "--project_path",
           mp.project_path, "--smpl_model", os.path.join(mp.smpl_model_path, "SMPL_NEUTRAL.pkl"), "--query_posmap_size",
           str(mp.query_posmap_size), "--inp_posmap_size", str(mp.inp_posmap_size), "--epoch", "7", "--stage", "1", "--body", "smpl",
           "--iters", "60"]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    fit = torch.load(os.path.join(test_dir, "smpl_parms_fit.pth"), weights_only=False)
    assert set(fit) == set(parms) and torch.equal(fit["beta"], parms["beta"])
    assert torch.equal(torch.load(os.path.join(test_dir, "smpl_parms.pth"), weights_only=False)["body_pose"], bad_pose)
    import json
    with open(os.path.join(test_dir, "smpl_parms_fit.json")) as fh:
        rep = json.load(fh)
    assert len(rep["frames"]) == len(ds)
    gt = torch.stack([ds[i]["original_image"] for i in range(len(ds))]).to(DEV)
    psnr = PeakSignalNoiseRatio(data_range=1.0).to(DEV)
    before = float(psnr(render(bad_pose, bad_transl), gt))
    psnr.reset()
    after = float(psnr(render(fit["body_pose"].float(), fit["trans"].float()), gt))
    assert after > before + 1.0, (before, after)
