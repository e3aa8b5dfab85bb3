"""GPU parity of the non-rasterizer stages (through the C ABI) against the oracle and against fixtures generated from
the reference's own modules (tests/golden, oracle/gen_golden.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import avatar_oracle as ao

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEV = "cuda:0"


def _rel(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30)


# ---------------------------------------------------------------------------------------------------------------- SMPL
def test_cano2live_smpl_matches_reference_fixture_and_autograd():
    from gaussianavatar_b200 import synthetic as syn
    from gaussianavatar_b200.body import SMPL
    from gaussianavatar_b200.ops import Cano2Live
    d = np.load(os.path.join(GOLD, "smpl_A.npz"))
    a = syn.make_avatar_assets(100, 16, seed=0)
    J = torch.tensor(d["rest_joints"])
    inv_cano = torch.linalg.inv(a.cano_joint_mats)
    pose = torch.tensor(d["pose"], device=DEV, requires_grad=True)
    transl = torch.tensor(d["transl"], device=DEV, requires_grad=True)
    C = Cano2Live.apply(SMPL, pose, None, transl, J.to(DEV), inv_cano.to(DEV).contiguous())
    # fixture: A straight from the reference's lbs(); cano2live = A @ inv(A_cano)  (avatar_model.py:296)
    ref = torch.matmul(torch.tensor(d["A"]), inv_cano[None])[:, :, :3, :].reshape(-1, 24, 12)
    assert (C.detach().cpu() - ref).abs().max() < 5e-6
    g = torch.randn(C.shape, generator=torch.Generator().manual_seed(0))
    (C * g.to(DEV)).sum().backward()
    p64 = torch.tensor(d["pose"]).double().requires_grad_(True)
    t64 = torch.tensor(d["transl"]).double().requires_grad_(True)
    C64 = ao.cano2live(ao.smpl_joint_transforms(J.double(), p64, t64), inv_cano.double()[None])[:, :, :3, :].reshape(-1, 24, 12)
    (C64 * g.double()).sum().backward()
    assert _rel(pose.grad.cpu(), p64.grad) < 1e-4
    assert _rel(transl.grad.cpu(), t64.grad) < 1e-5


# ----------------------------------------------------------------------------------------------------------------- LBS
@pytest.mark.parametrize("N,S,B,it", [(1000, 40, 2, 5000), (777, 32, 3, 300), (300, 20, 1, 999)])
def test_lbs_assemble_forward_backward(N, S, B, it):
    from gaussianavatar_b200 import synthetic as syn
    from gaussianavatar_b200.ops import LbsAssemble
    a = syn.make_avatar_assets(N, S, seed=2)
    g = torch.Generator().manual_seed(4)
    dec = torch.randn(S * S, 8, generator=g)
    dec[:, 3:7] = torch.rand(S * S, 4, generator=g)
    pose, transl = syn.synthetic_poses(B, seed=1)
    C = ao.cano2live(ao.smpl_joint_transforms(a.rest_joints, pose, transl), torch.linalg.inv(a.cano_joint_mats)[None])   # [B,24,4,4]
    vidx = torch.nonzero(a.valid_idx).reshape(-1).to(torch.int32)
    dec_d = dec.to(DEV).requires_grad_(True)
    C_d = C[:, :, :3, :].reshape(B, 24, 12).contiguous().to(DEV).requires_grad_(True)
    mul = 1e-3 * it if it < 1000 else 1.0
    means, scales, colors = LbsAssemble.apply(dec_d, C_d, vidx.to(DEV), a.query_points.to(DEV), a.query_lbs.to(DEV), mul)
    dec64 = dec.double().requires_grad_(True)
    C64 = C.double().requires_grad_(True)
    o = ao.assemble_and_skin(dec64[:, :3].t()[None].expand(B, -1, -1), dec64[:, 3:4].t()[None].expand(B, -1, -1),
                             dec64[:, 4:7].t()[None].expand(B, -1, -1), a.valid_idx, a.query_points.double()[None].expand(B, -1, -1),
                             a.query_lbs.double()[None].expand(B, -1, -1), C64, it)
    assert (means.detach().cpu() - o["means3D"].detach()).abs().max() < 2e-6
    assert (scales.detach().cpu() - o["scales"].detach()).abs().max() < 1e-6
    assert (colors.detach().cpu() - o["colors"].detach()).abs().max() < 1e-6
    gm, gs, gc = (torch.randn(B, N, 3, generator=g) for _ in range(3))
    ((means * gm.to(DEV)).sum() + (scales * gs.to(DEV)).sum() + (colors * gc.to(DEV)).sum()).backward()
    ((o["means3D"] * gm.double()).sum() + (o["scales"] * gs.double()).sum() + (o["colors"] * gc.double()).sum()).backward()
    assert _rel(dec_d.grad.cpu()[:, :7], dec64.grad[:, :7]) < 1e-5
    assert _rel(C_d.grad.cpu().reshape(B, 24, 3, 4), C64.grad[:, :, :3, :]) < 1e-5


# ------------------------------------------------------------------------------------------------------------- decoder
@pytest.mark.parametrize("name", ["pop_s32_in16.npz", "pop_s32_in32.npz", "pop_s48_in128.npz"])
def test_decoder_matches_reference_fixture(name):
    """Forward outputs, BatchNorm running statistics, weight / geo_feature gradients of the reference's POP_no_unet."""
    from gaussianavatar_b200.network import POP_no_unet
    d = np.load(os.path.join(GOLD, name))
    inp, S, B, seed = int(d["inp"]), int(d["S"]), int(d["B"]), int(d["seed"])
    net = POP_no_unet(c_geom=64, hsize=128).to(DEV)
    net.load_state_dict(ao.seeded_pop_params(seed), strict=False)
    g = torch.Generator().manual_seed(seed + 1)
    geo = (torch.randn(1, 64, inp, inp, generator=g) * 0.01).to(DEV).requires_grad_(True)
    uv = torch.tensor(d["uv"], device=DEV)
    res, sc, shs = net(None, geo.expand(B, -1, -1, -1).contiguous(), uv[None].expand(B, -1, -1).contiguous())
    assert res.shape == (B, 3, S * S) and sc.shape == (B, 1, S * S) and shs.shape == (B, 3, S * S)
    # strict-FP32 CUDA-core path vs the reference on CPU fp32
    for got, key, tol in ((res, "res", 2e-4), (sc, "scales", 5e-5), (shs, "shs", 5e-5)):
        err = np.abs(got.detach().cpu().numpy() - d[key]).max()
        assert err < tol, (key, err)
    gr, gs, gc = (torch.randn(res.shape, generator=g), torch.randn(sc.shape, generator=g), torch.randn(shs.shape, generator=g))
    ((res * gr.to(DEV)).sum() + (sc * gs.to(DEV)).sum() + (shs * gc.to(DEV)).sum()).backward()
    grads = {k: v.cpu().numpy() for k, v in net.reference_grads().items()}
    names = [str(n) for n in d["grad_names"]]
    norms = np.array([np.linalg.norm(grads[n]) for n in names])
    bias_before_bn = [i for i, n in enumerate(names) if n.endswith(".bias") and "conv8" not in n and ".bn" not in n]
    keep = [i for i in range(len(names)) if i not in bias_before_bn]
    assert np.abs(norms[keep] - d["grad_norms"][keep]).max() / d["grad_norms"].max() < 2e-3
    for k in d.files:
        if k.startswith("grad:"):
            n = k[5:]
            if n in ("decoder.conv1.bias", "decoder.conv6N.bias"):
                assert np.abs(grads[n]).max() < 5e-3      # exactly-zero gradient (bias in front of BatchNorm)
                continue
            got = grads[n][:8, :8] if n.startswith("geom_proc") else grads[n]
            assert _rel(got, d[k]) < 3e-3, (n, _rel(got, d[k]))
    gg = geo.grad.cpu().numpy()
    assert abs(np.linalg.norm(gg) - float(d["geo_grad_norm"])) / float(d["geo_grad_norm"]) < 2e-3
    assert _rel(gg[:, ::4, ::max(1, inp // 8), ::max(1, inp // 8)], d["geo_grad_sub"]) < 3e-3
    sd = net.state_dict()
    assert np.abs(sd["decoder.bn1.running_mean"].cpu().numpy() - d["bn1_running_mean"]).max() < 1e-5
    assert np.abs(sd["decoder.bn1.running_var"].cpu().numpy() - d["bn1_running_var"]).max() < 1e-5


def test_decoder_state_dict_roundtrip_reference_names():
    from gaussianavatar_b200.network import POP_no_unet
    net = POP_no_unet(c_geom=64, hsize=128).to(DEV)
    p = ao.seeded_pop_params(11)
    net.load_state_dict(p, strict=False)
    sd = net.state_dict()
    for k, v in p.items():
        assert torch.equal(sd[k].cpu(), v), k
    assert "decoder.bn7SH.running_var" in sd and "decoder.bn1.num_batches_tracked" in sd
    assert sum(v.numel() for k, v in sd.items() if "running" not in k and "num_batches" not in k) == 493063   # SURVEY B.1


# -------------------------------------------------------------------------------------------------------- end to end
def _make_model(N, S, side, B, seed=0, inp=32):
    from gaussianavatar_b200 import synthetic as syn
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, TEST_POSE_K, make_camera, scaled_intrinsics
    assets = syn.make_avatar_assets(N, S, seed=seed)
    tp = np.load(os.path.join(GOLD, "test_pose_subset.npz"))
    pose, transl = torch.tensor(tp["body_pose"]), torch.tensor(tp["trans"])
    cam = make_camera(scaled_intrinsics(TEST_POSE_K, side), TEST_POSE_EXTRINSIC, side, side)
    frames = [dict(pose_idx=i, FovX=cam.FovX, FovY=cam.FovY, height=side, width=side, world_view_transform=cam.world_view_transform,
                   full_proj_transform=cam.full_proj_transform, camera_center=cam.camera_center) for i in range(pose.shape[0])]
    torch.manual_seed(seed)
    model = AvatarModel.from_assets(assets, frames, pose, transl, batch_size=B, device=DEV)
    model.model_parms.inp_posmap_size = inp
    model.net_set(1)
    return model, assets, cam, pose, transl


def test_train_stage1_end_to_end_vs_oracle_chain():
    """Whole frame: SMPL -> net -> LBS -> rasterizer vs the chain of oracles (image mean-L1 <= 1e-4, SURVEY App. C)."""
    from oracle import raster_oracle as ro
    import math
    N, S, side, B = 3000, 64, 128, 2
    model, assets, cam, pose, transl = _make_model(N, S, side, B)
    with torch.no_grad():
        # make the Gaussians visible: scale head bias -> sigmoid ~ 0.02 m
        sd = model.net.state_dict()
        sd["decoder.conv8N.bias"] = torch.tensor([-3.9])
        model.net.load_state_dict(sd, strict=False)
    idx = torch.tensor([3, 17], device=DEV)
    batch = dict(pose_idx=idx, FovX=[cam.FovX] * B, FovY=[cam.FovY] * B, height=[side] * B, width=[side] * B,
                 world_view_transform=[cam.world_view_transform.to(DEV)] * B, full_proj_transform=[cam.full_proj_transform.to(DEV)] * B,
                 camera_center=[cam.camera_center.to(DEV)] * B)
    images, full_pred, offset_loss, geo_loss, scale_loss = model.train_stage1(batch, 5000)
    assert images.shape == (B, 3, side, side) and full_pred.shape == (B, N, 3)
    # oracle chain on CPU
    p = {k: v.cpu() for k, v in model.net.state_dict().items() if "running" not in k and "num_batches" not in k}
    geo = model.geo_feature.detach().cpu()
    res, sc, shs = ao.pop_forward(p, geo, S, B=B)
    A = ao.smpl_joint_transforms(assets.rest_joints, pose[idx.cpu()], transl[idx.cpu()])
    C = ao.cano2live(A, torch.linalg.inv(assets.cano_joint_mats)[None])
    o = ao.assemble_and_skin(res, sc, shs, assets.valid_idx, assets.query_points[None].expand(B, -1, -1),
                             assets.query_lbs[None].expand(B, -1, -1), C, 5000, geo_feature=geo)
    assert (full_pred.detach().cpu() - o["means3D"]).abs().max() < 5e-5
    assert abs(offset_loss.item() - o["offset_loss"].item()) < 1e-6 * max(1, abs(o["offset_loss"].item()))
    assert abs(scale_loss.item() - o["scale_loss"].item()) < 1e-6
    assert abs(geo_loss.item() - o["geo_loss"].item()) < 1e-9
    rots = np.zeros((N, 4), np.float32); rots[:, 0] = 1
    for b in range(B):
        ref = ro.forward(o["means3D"][b].numpy(), o["colors"][b].numpy(), np.ones(N, np.float32), o["scales"][b].numpy(), rots,
                         np.ones(3, np.float32), cam.world_view_transform.numpy(), cam.full_proj_transform.numpy(),
                         math.tan(cam.FovX / 2), math.tan(cam.FovY / 2), side, side)
        err = np.abs(images[b].detach().cpu().numpy() - ref.image).mean()
        assert err <= 1e-4, err
        assert (ref.image < 0.99).mean() > 0.02      # the body is actually on screen
    # and the whole thing back-propagates into every trainable tensor
    loss = images.mean() + offset_loss + geo_loss + scale_loss
    loss.backward()
    assert model.net.flat.grad is not None and torch.isfinite(model.net.flat.grad).all() and model.net.flat.grad.abs().sum() > 0
    assert model.geo_feature.grad is not None and torch.isfinite(model.geo_feature.grad).all()
    assert model.pose.weight.grad is not None


def test_reference_signature_constructor_reads_the_dataset_folder(tmp_path):
    """AvatarModel(model_parms, net_parms, opt_parms) (model/avatar_model.py:20-121) on a synthetic folder in the reference's layout:
    the staged tensors equal the in-memory construction from the same assets, the DataLoader yields reference-shaped batches and a
    stage-1 step, the test / novel-pose datasets render."""
    from dataset_fixture import write_synthetic_dataset
    from gaussianavatar_b200 import synthetic as syn
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams, OptimizationParams
    from gaussianavatar_b200.losses import image_loss
    from gaussianavatar_b200.workload import to_cuda
    N, S, F = 600, 32, 5
    mp = write_synthetic_dataset(str(tmp_path), N=N, S=S, num_frames=F, side=64, inp=16)
    torch.manual_seed(0)
    m = AvatarModel(mp, NetworkParams(), OptimizationParams(), train=True)
    a = syn.make_avatar_assets(N, S, seed=0)
    pose, transl = syn.synthetic_poses(F, seed=0)
    ref = AvatarModel.from_assets(a, [], pose, transl, batch_size=2)
    assert torch.equal(m.valid_idx, ref.valid_idx) and torch.equal(m.valid_index, ref.valid_index)
    for name in ("_query_points", "_query_lbs", "_inv_cano"):
        assert torch.allclose(getattr(m, name), getattr(ref, name), atol=1e-6), name
    assert torch.allclose(m._rest_joints, ref._rest_joints, atol=1e-5)
    assert torch.equal(m.pose.weight, ref.pose.weight) and torch.equal(m.transl.weight, ref.transl.weight)
    assert m.geo_feature.shape == (1, 64, 16, 16)

    m.training_setup()
    batch = next(iter(m.getTrainDataloader()))
    assert batch["original_image"].shape == (2, 3, 64, 64) and batch["world_view_transform"].shape == (2, 4, 4)
    batch, _ = to_cuda(batch, DEV)
    image, points, offset_loss, geo_loss, scale_loss = m.train_stage1(batch, 2000)
    loss = image_loss(image, batch["original_image"].float(), 0.2) + 10.0 * offset_loss + geo_loss + 3e-2 * scale_loss
    m.zero_grad(1); loss.backward(); m.step(1)
    assert torch.isfinite(loss) and image.shape == (2, 3, 64, 64) and (image < 0.999).any()

    te = m.getTestDataset()
    item = te[0]
    tb, _ = to_cuda({k: (v[None] if torch.is_tensor(v) else [v]) for k, v in item.items()}, DEV)
    tb["pose_idx"] = torch.tensor([item["pose_idx"]], device=DEV)
    with torch.no_grad():
        img = m.render_free_stage1(tb, 59400)
    assert img.shape == (1, 3, 64, 64)
    nv = m.getNovelposeDataset()
    assert len(nv) == 4 and nv[0]["height"] == 1024


def test_inference_model_caches_the_frame_invariant_decoder_output():
    """render_novel_pose.py path (avatar_model.py:467-554): an inference model evaluates the stage-1 net once; the frames rendered from
    the cached output are the frames a model that re-evaluates it every time renders (SURVEY.md §8e)."""
    from gaussianavatar_b200 import synthetic as syn
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.workload import Stage1Workload
    wl = Stage1Workload(3, 1, device=DEV, N=4000, S=64, side=128, inp_posmap_size=32)
    m = wl.model
    pose, transl = syn.synthetic_poses(3, seed=4)
    batches = [dict(pose_idx=torch.tensor([0], device=DEV), pose_data=pose[i:i + 1].to(DEV), transl_data=transl[i:i + 1].to(DEV),
                    **wl.camera_fields(1)) for i in range(3)]
    with torch.no_grad():
        m.cache_decoder = False
        ref = [m.render_free_stage1(b, 59400).clone() for b in batches]
        m.cache_decoder = True
        m.invalidate_decoder_cache()
        n0 = list(m.net._states.values())[0].num_batches_tracked
        got = [m.render_free_stage1(b, 59400).clone() for b in batches]
        n1 = list(m.net._states.values())[0].num_batches_tracked
        assert n1 == n0 + 1, (n0, n1)          # evaluated once for the three frames
    for a, b in zip(got, ref):          # the re-evaluated net differs by the summation order of its BatchNorm statistics (double atomics):
        d = (a - b).abs()               # round-off everywhere, except where that round-off flips a rasterizer threshold (alpha < 1/255, the
        # 3-sigma tile rectangle, T < 1e-4): a flipped Gaussian changes a handful of pixels by at most its own cut-off contribution (~1e-2).
        # The order of the atomics differs from run to run, so the bounds must hold for a few flips, not for none.
        assert torch.quantile(d.flatten(), 0.999).item() < 1e-4, torch.quantile(d.flatten(), 0.999).item()
        assert d.max().item() < 5e-2, d.max().item()
        assert d.mean().item() < 2e-5, d.mean().item()
    assert (got[0] - got[1]).abs().mean().item() > 1e-4, (got[0] - got[1]).abs().mean().item()


# ------------------------------------------------------------------------------------------------------------- stage 2
@pytest.mark.parametrize("mode", ["fp32", pytest.param("tf32", marks=pytest.mark.tf32)])
def test_stage2_decoder_with_pose_featmap_matches_reference_fixture(mode):
    """POP_no_unet.forward(pose_featmap=[B,64,h,h], ...) (model/network.py:55-58): per-frame decoder rows, BatchNorm statistics over
    both frames — outputs, parameter / geo_feature / pose_featmap gradients of the reference module."""
    from gaussianavatar_b200.network import POP_no_unet
    d = np.load(os.path.join(GOLD, "pop_s32_in16_pose.npz"))
    inp, S, B, seed = int(d["inp"]), int(d["S"]), int(d["B"]), int(d["seed"])
    otol, gtol = (2e-4, 3e-3) if mode == "fp32" else (5e-3, 3e-2)
    net = POP_no_unet(c_geom=64, hsize=128).to(DEV)
    assert net.tensor_cores == (mode == "tf32")
    net.load_state_dict(ao.seeded_pop_params(seed), strict=False)
    g = torch.Generator().manual_seed(seed + 1)
    geo = (torch.randn(1, 64, inp, inp, generator=g) * 0.01).to(DEV).requires_grad_(True)
    pf = torch.tensor(d["pose_featmap"], device=DEV).requires_grad_(True)
    _ = torch.randn(B, 64, inp, inp, generator=g)                      # keeps the generator in step with the fixture's draws
    uv = torch.tensor(d["uv"], device=DEV)
    res, sc, shs = net(pf, geo.expand(B, -1, -1, -1).contiguous(), uv[None].expand(B, -1, -1).contiguous())
    assert res.shape == (B, 3, S * S) and sc.shape == (B, 1, S * S) and shs.shape == (B, 3, S * S)
    for got, key in ((res, "res"), (sc, "scales"), (shs, "shs")):
        ref = d[key]
        assert np.abs(got.detach().cpu().numpy() - ref).max() < otol * max(1.0, np.abs(ref).max()), key
    gr, gs, gc = (torch.randn(res.shape, generator=g), torch.randn(sc.shape, generator=g), torch.randn(shs.shape, generator=g))
    ((res * gr.to(DEV)).sum() + (sc * gs.to(DEV)).sum() + (shs * gc.to(DEV)).sum()).backward()
    grads = {k: v.cpu().numpy() for k, v in net.reference_grads().items()}
    for k in d.files:
        if k.startswith("grad:"):
            n = k[5:]
            if n in ("decoder.conv1.bias", "decoder.conv6N.bias"):
                continue
            got = grads[n][:8, :8] if n.startswith("geom_proc") else grads[n]
            assert _rel(got, d[k]) < gtol, (n, _rel(got, d[k]))
    assert _rel(pf.grad.cpu().numpy(), d["pose_grad"]) < gtol
    assert abs(np.linalg.norm(geo.grad.cpu().numpy()) - float(d["geo_grad_norm"])) / float(d["geo_grad_norm"]) < gtol


def test_lbs_assemble_per_frame_decoder_output():
    """Stage 2: every frame has its own decoder rows; forward and backward against the stage-1 kernel run frame by frame."""
    from gaussianavatar_b200 import synthetic as syn
    from gaussianavatar_b200.ops import LbsAssemble
    N, S, B = 900, 40, 3
    a = syn.make_avatar_assets(N, S, seed=2)
    g = torch.Generator().manual_seed(0)
    dec = torch.randn(B * S * S, 8, generator=g).to(DEV).requires_grad_(True)
    C = (torch.eye(4)[:3].reshape(1, 1, 12) + 0.05 * torch.randn(B, 24, 12, generator=g)).to(DEV).requires_grad_(True)
    vi = torch.nonzero(a.valid_idx).reshape(-1).to(torch.int32).to(DEV)
    q, w = a.query_points.to(DEV), a.query_lbs.to(DEV)
    gm, gs, gc = (torch.randn(B, N, 3, generator=g).to(DEV) for _ in range(3))
    m, s, c = LbsAssemble.apply(dec, C, vi, q, w, 0.7, True)
    ((m * gm).sum() + (s * gs).sum() + (c * gc).sum()).backward()
    for b in range(B):
        db = dec.detach()[b * S * S:(b + 1) * S * S].clone().requires_grad_(True)
        Cb = C.detach()[b:b + 1].clone().requires_grad_(True)
        mb, sb, cb = LbsAssemble.apply(db, Cb, vi, q, w, 0.7)
        assert torch.equal(mb[0], m[b]) and torch.equal(sb[0], s[b]) and torch.equal(cb[0], c[b])
        ((mb * gm[b:b + 1]).sum() + (sb * gs[b:b + 1]).sum() + (cb * gc[b:b + 1]).sum()).backward()
        assert torch.allclose(dec.grad[b * S * S:(b + 1) * S * S], db.grad, atol=1e-6)
        assert torch.allclose(C.grad[b], Cb.grad[0], rtol=1e-4, atol=1e-5)


def test_train_stage2_end_to_end_vs_oracle_chain(tmp_path):
    """One whole stage-2 step (model/avatar_model.py:369-463, train.py:79-97) on a synthetic dataset folder: pose encoder -> per-frame
    decoder -> LBS -> rasterizer -> loss -> backward, against the CPU oracle chain (reference-pinned pose encoder / POP / SMPL / losses
    restatements + the C rasterizer oracle); then save / stage2_load round-trips the reference's `pose_encoder.pth` layout."""
    import math
    from dataset_fixture import write_synthetic_dataset
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams, OptimizationParams
    from gaussianavatar_b200.trainer import AvatarTrainer
    from gaussianavatar_b200.workload import to_cuda
    from oracle import raster_oracle as ro
    N, S, F, side, inp = 700, 48, 4, 64, 32          # five stride-2 steps need a >= 32 input map (UnetNoCond5DS: "for posmap size=32")
    mp = write_synthetic_dataset(str(tmp_path), N=N, S=S, num_frames=F, side=side, inp=inp, stage2=True)
    torch.manual_seed(0)
    m = AvatarModel(mp, NetworkParams(nf=8), OptimizationParams(), train=True)
    with torch.no_grad():
        sd = m.net.state_dict(); sd["decoder.conv8N.bias"] = torch.tensor([-3.5]); m.net.load_state_dict(sd, strict=False)
    tr = AvatarTrainer(m, use_graph=False)
    ds = m.train_dataset
    items = [ds[1], ds[2]]
    batch = {k: (torch.stack([torch.as_tensor(it[k]) for it in items]) if not isinstance(items[0][k], (int, float)) else [it[k] for it in items])
             for k in items[0]}
    batch["pose_idx"] = torch.tensor([it["pose_idx"] for it in items])
    batch, _ = to_cuda(batch, DEV)
    B = 2
    with torch.backends.cudnn.flags(allow_tf32=False):       # strict-FP32 comparison: the pose encoder's cuDNN convs in fp32 like the decoder path under test
        loss, image = tr.loss(batch, 3000, epoch=1)
        m.zero_grad(1)
        loss.backward()
    # ---- oracle chain ----
    p = {k: v.cpu().clone().requires_grad_(True) for k, v in m.net.state_dict().items() if "running" not in k and "num_batches" not in k}
    pe = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in m.pose_encoder.named_parameters()}
    geo = m.geo_feature.detach().cpu().clone().requires_grad_(True)
    ids = batch["pose_idx"].cpu()
    pose = m.pose.weight.detach().cpu()[ids].clone(); transl = m.transl.weight.detach().cpu()[ids].clone()
    pf = ao.unet5ds_forward(pe, batch["inp_pos_map"].cpu().float())
    res, sc, shs = ao.pop_forward(p, geo, S, B=B, pose_featmap=pf)
    A = ao.smpl_joint_transforms(m._rest_joints.cpu(), pose, transl)
    C = torch.matmul(A, m._inv_cano.cpu()[None])
    q, w = m._query_points.cpu(), m._query_lbs.cpu()
    o = ao.assemble_and_skin(res, sc, shs, m.valid_idx.cpu(), q[None].expand(B, -1, -1), w[None].expand(B, -1, -1), C, 3000, ramp=False)
    cam = items[0]
    rots = np.zeros((N, 4), np.float32); rots[:, 0] = 1
    rs, imgs = [], []
    for b in range(B):
        r = ro.forward(o["means3D"][b].detach().numpy(), o["colors"][b].detach().numpy(), np.ones(N, np.float32), o["scales"][b].detach().numpy(),
                       rots, np.ones(3, np.float32), cam["world_view_transform"].numpy(), cam["full_proj_transform"].numpy(),
                       math.tan(cam["FovX"] / 2), math.tan(cam["FovY"] / 2), side, side)
        rs.append(r); imgs.append(torch.tensor(r.image, dtype=torch.float32))
    img = torch.stack(imgs).requires_grad_(True)
    gt = batch["original_image"].cpu().float()
    li = 0.8 * ao.l1_loss_w(img, gt) + 0.2 * (1 - ao.ssim(img, gt))
    li.backward()
    gm, gc, gs = [], [], []
    for b in range(B):
        gb = rs[b].backward(img.grad[b].numpy())
        gm.append(torch.tensor(gb["d_means3D"], dtype=torch.float32)); gc.append(torch.tensor(gb["d_colors"], dtype=torch.float32))
        gs.append(torch.tensor(gb["d_scales"], dtype=torch.float32))
    reg = 10.0 * o["offset_loss"] + 10.0 * torch.mean(pf ** 2)
    ref_loss = li.item() + reg.item()
    torch.autograd.backward([o["means3D"], o["colors"], o["scales"], reg], [torch.stack(gm), torch.stack(gc), torch.stack(gs), torch.ones(())])
    assert abs(loss.item() - ref_loss) < 1e-4 * max(1.0, abs(ref_loss)), (loss.item(), ref_loss)
    assert np.abs(image.detach().cpu().numpy() - img.detach().numpy()).mean() < 1e-4
    got = {k: v.cpu() for k, v in m.net.reference_grads().items()}
    worst = 0.0
    for k, v in p.items():
        if k.endswith(".bias") and ".bn" not in k and "conv8" not in k:
            continue
        worst = max(worst, _rel(got[k].numpy(), v.grad.numpy()))
    assert worst < 1e-2, worst
    for k, v in m.pose_encoder.named_parameters():
        assert _rel(v.grad.cpu().numpy(), pe[k].grad.numpy()) < 2e-2, k
    # one optimizer step, then the reference's stage-2 checkpoint layout round-trips
    m.step(1)
    m.save(7)
    ck = torch.load(os.path.join(m.model_path, "net/iteration_7", "pose_encoder.pth"), weights_only=False)
    assert set(ck) == {"pose_encoder", "geo_feature", "pose", "transl", "net", "optimizer", "scheduler"}
    assert "conv3.conv.weight" in ck["pose_encoder"] and "upconv5.up.bias" in ck["pose_encoder"]
    before = m.pose_encoder.conv3.conv.weight.detach().clone()
    with torch.no_grad():
        m.pose_encoder.conv3.conv.weight.zero_()
    mp2 = mp
    m.model_parms.project_path = ""
    m.stage2_load(7)
    assert torch.equal(m.pose_encoder.conv3.conv.weight, before)
    with torch.no_grad():
        out = m.render_free_stage2(batch, 3000)
    assert out.shape == (B, 3, side, side) and torch.isfinite(out).all()


def test_decoder_backward_after_a_newer_forward_fails_loudly():
    """ADVICE r1: the decoder's activations live in one workspace per state; a stale backward must raise, not silently use them."""
    from gaussianavatar_b200.network import POP_no_unet
    net = POP_no_unet(c_geom=64, hsize=128).to(DEV)
    geo = (torch.randn(1, 64, 16, 16) * 0.01).to(DEV).requires_grad_(True)
    d1 = net.forward_packed(geo, 32, 1)
    d2 = net.forward_packed(geo, 32, 1)
    with pytest.raises(RuntimeError, match="overwritten"):
        d1.sum().backward()
    d2.sum().backward()
    assert torch.isfinite(net.flat.grad).all()
