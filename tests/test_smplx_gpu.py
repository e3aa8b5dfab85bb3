"""GPU: the SMPL-X (55-joint) path — joint transforms against the reference's `smplx.SMPLX` (tests/golden/smplx_A.npz) and fp64
autograd of the oracle, 55-joint LBS against the fp64 oracle, and whole stage-1 / stage-2 steps through
`AvatarModel(..., smpl_type='smplx')` on a synthetic folder against the oracle chain."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import avatar_oracle as ao
from oracle import avatar_oracle_smplx as aox

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEV = "cuda:0"


def _rel(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30)


def _oracle_C(J, pose66, rest99, transl, inv_cano):
    return ao.cano2live(aox.smplx_joint_transforms(J, pose66, rest99, transl), inv_cano[None])


# ------------------------------------------------------------------------------------------------------ joint transforms
def test_cano2live_smplx_matches_reference_fixture_and_autograd():
    from gaussianavatar_b200 import synthetic as syn
    from gaussianavatar_b200.body import SMPLX
    from gaussianavatar_b200.ops import Cano2Live
    d = np.load(os.path.join(GOLD, "smplx_A.npz"))
    a = syn.make_avatar_assets(100, 16, seed=0, body="smplx")
    J = torch.tensor(d["rest_joints"])
    inv_cano = torch.linalg.inv(a.cano_joint_mats)
    pose = torch.tensor(d["pose66"], device=DEV, requires_grad=True)
    rest = torch.tensor(d["rest99"], device=DEV)
    transl = torch.tensor(d["transl"], device=DEV, requires_grad=True)
    C = Cano2Live.apply(SMPLX, pose, rest, transl, J.to(DEV), inv_cano.to(DEV).contiguous())
    assert C.shape == (pose.shape[0], 55, 12)
    ref = torch.matmul(torch.tensor(d["A"]), inv_cano[None])[:, :, :3, :].reshape(-1, 55, 12)
    assert (C.detach().cpu() - ref).abs().max() < 5e-6
    g = torch.randn(C.shape, generator=torch.Generator().manual_seed(0))
    (C * g.to(DEV)).sum().backward()
    p64 = torch.tensor(d["pose66"]).double().requires_grad_(True)
    t64 = torch.tensor(d["transl"]).double().requires_grad_(True)
    C64 = _oracle_C(J.double(), p64, torch.tensor(d["rest99"]).double(), t64, inv_cano.double())[:, :, :3, :].reshape(-1, 55, 12)
    (C64 * g.double()).sum().backward()
    assert pose.grad.shape == (pose.shape[0], 66)
    assert _rel(pose.grad.cpu(), p64.grad) < 1e-4
    assert _rel(transl.grad.cpu(), t64.grad) < 1e-5


def test_cano2live_rejects_bad_smplx_shapes():
    from gaussianavatar_b200.body import SMPLX
    from gaussianavatar_b200.ops import Cano2Live
    z = lambda *s: torch.zeros(*s, device=DEV)
    with pytest.raises(ValueError, match="rest_pose"):
        Cano2Live.apply(SMPLX, z(2, 66), z(2, 6), z(2, 3), z(55, 3), z(55, 4, 4))
    with pytest.raises(ValueError, match="pose"):
        Cano2Live.apply(SMPLX, z(2, 72), z(2, 99), z(2, 3), z(55, 3), z(55, 4, 4))


# ------------------------------------------------------------------------------------------------------------------ LBS
@pytest.mark.parametrize("per_frame", [False, True], ids=["shared", "per_frame"])
@pytest.mark.parametrize("B", [1, 3, 8])
@pytest.mark.parametrize("N", [1, 255, 257, 777, 1000])
def test_lbs_55_joints_forward_backward(N, B, per_frame):
    from gaussianavatar_b200 import synthetic as syn
    from gaussianavatar_b200.ops import LbsAssemble
    S = int(math.ceil(math.sqrt(N))) + 2
    a = syn.make_avatar_assets(N, S, seed=2, body="smplx")
    g = torch.Generator().manual_seed(4 + N + B)
    frames = B if per_frame else 1
    dec = torch.randn(frames * S * S, 8, generator=g)
    dec[:, 3:7] = torch.rand(frames * S * S, 4, generator=g)
    pose, rest, transl = syn.synthetic_smplx_poses(B, seed=1)
    C = _oracle_C(a.rest_joints, pose, rest, transl, torch.linalg.inv(a.cano_joint_mats))                    # [B,55,4,4]
    vidx = torch.nonzero(a.valid_idx).reshape(-1).to(torch.int32)
    w56 = F.pad(a.query_lbs, (0, 1)).contiguous()
    dec_d = dec.to(DEV).requires_grad_(True)
    C_d = C[:, :, :3, :].reshape(B, 55, 12).contiguous().to(DEV).requires_grad_(True)
    it = 300 if N % 2 else 5000
    mul = 1e-3 * it if it < 1000 else 1.0
    means, scales, colors = LbsAssemble.apply(dec_d, C_d, vidx.to(DEV), a.query_points.to(DEV), w56.to(DEV), mul, per_frame)
    dec64 = dec.double().requires_grad_(True)
    C64 = C.double().requires_grad_(True)
    d3 = dec64.reshape(frames, S * S, 8).transpose(1, 2).expand(B, -1, -1)
    o = ao.assemble_and_skin(d3[:, :3], d3[:, 3:4], d3[:, 4:7], a.valid_idx, a.query_points.double()[None].expand(B, -1, -1),
                             a.query_lbs.double()[None].expand(B, -1, -1), C64, it)
    assert (means.detach().cpu() - o["means3D"].detach()).abs().max() < 2e-6
    assert (scales.detach().cpu() - o["scales"].detach()).abs().max() < 1e-6
    assert (colors.detach().cpu() - o["colors"].detach()).abs().max() < 1e-6
    gm, gs, gc = (torch.randn(B, N, 3, generator=g) for _ in range(3))
    ((means * gm.to(DEV)).sum() + (scales * gs.to(DEV)).sum() + (colors * gc.to(DEV)).sum()).backward()
    ((o["means3D"] * gm.double()).sum() + (o["scales"] * gs.double()).sum() + (o["colors"] * gc.double()).sum()).backward()
    assert _rel(dec_d.grad.cpu()[:, :7], dec64.grad[:, :7]) < 1e-5
    assert (dec_d.grad.cpu()[:, 7] == 0).all()
    assert _rel(C_d.grad.cpu().reshape(B, 55, 3, 4), C64.grad[:, :, :3, :]) < 1e-5


# -------------------------------------------------------------------------------------------------------- end to end
def _folder_model(tmp_path, N, S, F_, side, inp, stage2=False, nf=None):
    from dataset_fixture_smplx import write_synthetic_smplx_dataset
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams, OptimizationParams
    mp = write_synthetic_smplx_dataset(str(tmp_path), N=N, S=S, num_frames=F_, side=side, inp=inp, stage2=stage2)
    torch.manual_seed(0)
    m = AvatarModel(mp, NetworkParams(nf=nf) if nf else NetworkParams(), OptimizationParams(), train=True)
    with torch.no_grad():
        sd = m.net.state_dict(); sd["decoder.conv8N.bias"] = torch.tensor([-3.6]); m.net.load_state_dict(sd, strict=False)
    return mp, m


def _collate(items):
    from gaussianavatar_b200.workload import to_cuda
    batch = {k: (torch.stack([torch.as_tensor(it[k]) for it in items]) if not isinstance(items[0][k], (int, float)) else [it[k] for it in items])
             for k in items[0]}
    batch["pose_idx"] = torch.tensor([it["pose_idx"] for it in items])
    return to_cuda(batch, DEV)[0]


def _oracle_images(o, cam, N, side, B):
    from oracle import raster_oracle as ro
    rots = np.zeros((N, 4), np.float32); rots[:, 0] = 1
    rs = []
    for b in range(B):
        rs.append(ro.forward(o["means3D"][b].detach().numpy(), o["colors"][b].detach().numpy(), np.ones(N, np.float32),
                             o["scales"][b].detach().numpy(), rots, np.ones(3, np.float32), cam["world_view_transform"].numpy(),
                             cam["full_proj_transform"].numpy(), math.tan(cam["FovX"] / 2), math.tan(cam["FovY"] / 2), side, side))
    return rs


def test_train_stage1_smplx_end_to_end_vs_oracle_chain(tmp_path):
    """AvatarModel(smpl_type='smplx') built from the reference's folder layout: a stage-1 step (rest_pose from the batch) against the
    oracle chain; then the reference-layout checkpoint round-trips through save / load."""
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams, OptimizationParams
    N, S, F_, side, B = 3000, 64, 5, 128, 2
    mp, m = _folder_model(tmp_path, N, S, F_, side, 16)
    assert m.pose.weight.shape == (F_, 66) and m._query_lbs.shape == (N, 56) and (m._query_lbs[:, 55] == 0).all()
    assert m.query_lbs.shape == (B, N, 55) and m._inv_cano.shape == (55, 4, 4)
    m.training_setup()
    ds = m.train_dataset
    items = [ds[1], ds[3]]
    batch = _collate(items)
    assert batch["rest_pose"].shape == (B, 99)
    images, full_pred, offset_loss, geo_loss, scale_loss = m.train_stage1(batch, 5000)
    p = {k: v.cpu() for k, v in m.net.state_dict().items() if "running" not in k and "num_batches" not in k}
    geo = m.geo_feature.detach().cpu()
    res, sc, shs = ao.pop_forward(p, geo, S, B=B)
    ids = batch["pose_idx"].cpu()
    C = _oracle_C(m._rest_joints.cpu(), m.pose.weight.detach().cpu()[ids], batch["rest_pose"].cpu().float(),
                  m.transl.weight.detach().cpu()[ids], m._inv_cano.cpu())
    q, w = m._query_points.cpu(), m._query_lbs.cpu()[:, :55]
    o = ao.assemble_and_skin(res, sc, shs, m.valid_idx.cpu(), q[None].expand(B, -1, -1), w[None].expand(B, -1, -1), C, 5000, geo_feature=geo)
    assert (full_pred.detach().cpu() - o["means3D"]).abs().max() < 5e-5
    assert abs(offset_loss.item() - o["offset_loss"].item()) < 1e-6 * max(1, abs(o["offset_loss"].item()))
    assert abs(scale_loss.item() - o["scale_loss"].item()) < 1e-6
    for b, r in enumerate(_oracle_images(o, items[0], N, side, B)):
        err = np.abs(images[b].detach().cpu().numpy() - r.image).mean()
        assert err <= 1e-4, err
        assert (r.image < 0.99).mean() > 0.02      # the body is actually on screen
    (images.mean() + offset_loss + geo_loss + scale_loss).backward()
    assert torch.isfinite(m.net.flat.grad).all() and m.net.flat.grad.abs().sum() > 0
    gp = m.pose.weight.grad.coalesce()
    assert gp.values().shape == (B, 66) and torch.isfinite(gp.values()).all() and gp.values().abs().sum() > 0
    # a rest_pose of the wrong width (the SMPL test poses leave 6 columns past 66) is refused before any launch
    bad = dict(batch, rest_pose=torch.zeros(B, 6, device=DEV))
    with pytest.raises(ValueError, match="rest_pose"):
        m.train_stage1(bad, 5000)
    with pytest.raises(ValueError, match="rest_pose"):
        m.train_stage1({k: v for k, v in batch.items() if k != "rest_pose"}, 5000)
    # checkpoint round-trip (model/avatar_model.py:163-202 layout)
    m.step(1)
    m.save(3)
    torch.manual_seed(1)
    m2 = AvatarModel(mp, NetworkParams(), OptimizationParams(), train=True)
    m2.training_setup()
    m2.load(3)
    assert torch.equal(m2.pose.weight, m.pose.weight) and m2.pose.weight.shape == (F_, 66)
    assert torch.equal(m2.transl.weight, m.transl.weight) and torch.equal(m2.geo_feature, m.geo_feature)
    assert torch.equal(m2.net.flat, m.net.flat)
    with torch.no_grad():
        a1 = m.train_stage1(batch, 5000)[1]
        a2 = m2.train_stage1(batch, 5000)[1]
    assert torch.allclose(a1, a2, rtol=0, atol=1e-6)


def test_render_free_stage1_smplx_on_test_items(tmp_path):
    """render_free_stage1 on the test dataset's items (pose_data [66] + rest_pose [99]) equals the oracle chain; the hand / face pose
    of the item is what moves the hands."""
    N, S, F_, side = 2000, 48, 4, 64
    mp, m = _folder_model(tmp_path, N, S, F_, side, 16)
    te = m.getTestDataset()
    item = te[2]
    assert item["pose_data"].shape == (66,) and item["rest_pose"].shape == (99,)
    tb = _collate([item])
    with torch.no_grad():
        img = m.render_free_stage1(tb, 59400)
        p = {k: v.cpu() for k, v in m.net.state_dict().items() if "running" not in k and "num_batches" not in k}
    assert img.shape == (1, 3, side, side) and torch.isfinite(img).all()
    res, sc, shs = ao.pop_forward(p, m.geo_feature.detach().cpu(), S, B=1)
    C = _oracle_C(m._rest_joints.cpu(), item["pose_data"][None].float(), item["rest_pose"][None].float(), item["transl_data"][None].float(),
                  m._inv_cano.cpu())
    o = ao.assemble_and_skin(res, sc, shs, m.valid_idx.cpu(), m._query_points.cpu()[None], m._query_lbs.cpu()[None, :, :55], C, 59400)
    r = _oracle_images(o, item, N, side, 1)[0]
    assert np.abs(img[0].cpu().numpy() - r.image).mean() <= 1e-4
    tb2 = dict(tb, rest_pose=tb["rest_pose"] + 0.8)
    with torch.no_grad():
        img2 = m.render_free_stage1(tb2, 59400)
    assert (img2 - img).abs().max().item() > 1e-2


def test_train_stage2_smplx_step_vs_oracle_chain(tmp_path):
    """A stage-2 step (pose encoder -> per-frame decoder -> 55-joint LBS -> rasterizer) against the oracle chain's forward; the backward
    reaches the pose encoder and the 66-wide pose table."""
    from gaussianavatar_b200.trainer import AvatarTrainer
    N, S, F_, side, inp, B = 700, 48, 4, 64, 32, 2
    mp, m = _folder_model(tmp_path, N, S, F_, side, inp, stage2=True, nf=8)
    tr = AvatarTrainer(m, use_graph=False)
    items = [m.train_dataset[0], m.train_dataset[2]]
    batch = _collate(items)
    with torch.backends.cudnn.flags(allow_tf32=False):
        loss, image = tr.loss(batch, 3000, epoch=1)
        m.zero_grad(1)
        loss.backward()
        p = {k: v.cpu() for k, v in m.net.state_dict().items() if "running" not in k and "num_batches" not in k}
        pe = {k: v.detach().cpu() for k, v in m.pose_encoder.named_parameters()}
        pf = ao.unet5ds_forward(pe, batch["inp_pos_map"].cpu().float())
    res, sc, shs = ao.pop_forward(p, m.geo_feature.detach().cpu(), S, B=B, pose_featmap=pf)
    ids = batch["pose_idx"].cpu()
    C = _oracle_C(m._rest_joints.cpu(), m.pose.weight.detach().cpu()[ids], batch["rest_pose"].cpu().float(),
                  m.transl.weight.detach().cpu()[ids], m._inv_cano.cpu())
    o = ao.assemble_and_skin(res, sc, shs, m.valid_idx.cpu(), m._query_points.cpu()[None].expand(B, -1, -1),
                             m._query_lbs.cpu()[None, :, :55].expand(B, -1, -1), C, 3000, ramp=False)
    rs = _oracle_images(o, items[0], N, side, B)
    img = torch.stack([torch.tensor(r.image, dtype=torch.float32) for r in rs])
    gt = batch["original_image"].cpu().float()
    ref_loss = (0.8 * ao.l1_loss_w(img, gt) + 0.2 * (1 - ao.ssim(img, gt))).item() + 10.0 * o["offset_loss"].item() + 10.0 * torch.mean(pf ** 2).item()
    assert abs(loss.item() - ref_loss) < 1e-4 * max(1.0, abs(ref_loss)), (loss.item(), ref_loss)
    assert np.abs(image.detach().cpu().numpy() - img.numpy()).mean() < 1e-4
    assert all(torch.isfinite(v.grad).all() and v.grad.abs().sum() > 0 for v in m.pose_encoder.parameters() if v.grad is not None)
    gp = m.pose.weight.grad.coalesce()
    assert gp.values().shape[1] == 66 and torch.isfinite(gp.values()).all()


@pytest.mark.tf32
def test_graphed_step_follows_rest_pose_changes():
    """The whole-step CUDA graph reads each step's rest_pose: with the learning rates at zero (the parameters stay put), the graphed
    steps' losses equal the eager steps' while only the hand / face pose changes from step to step."""
    from gaussianavatar_b200.trainer import Stage1Trainer
    from gaussianavatar_b200.workload import Stage1Workload

    def run(use_graph):
        wl = Stage1Workload(3, 2, device=DEV, N=4000, S=64, side=128, inp_posmap_size=32, body="smplx")
        with torch.no_grad():
            sd = wl.model.net.state_dict(); sd["decoder.conv8N.bias"] = torch.tensor([-3.6]); wl.model.net.load_state_dict(sd, strict=False)
        wl.make_ground_truth()
        wl.model.opt_parms.lr_net = 0.0
        wl.model.opt_parms.lr_geomfeat = 0.0
        tr = Stage1Trainer(wl.model, use_graph=use_graph)
        g = torch.Generator().manual_seed(5)
        out = []
        for i in range(4):
            batch = wl.device_batch([0, 1])
            batch["rest_pose"] = (torch.randn(2, 99, generator=g) * 1.2).to(DEV)
            out.append(float(tr.step(batch, 5000 + i, epoch=1)))
        tr.finish()
        assert bool(tr._graphs) == use_graph
        return out

    eager = run(False)
    graph = run(True)
    assert max(eager) - min(eager) > 1e-4, eager              # the hand / face pose does change the loss
    for i, (le, lg) in enumerate(zip(eager, graph)):
        assert abs(le - lg) < 1e-5 * max(1.0, abs(le)), (eager, graph)
        # and each replay is its own step's loss, not the captured step's or another one's
        assert abs(le - lg) < 0.1 * min(abs(lg - eager[j]) for j in range(len(eager)) if j != i), (eager, graph)
