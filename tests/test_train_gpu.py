"""GPU parity of the fused loss, the fused Adam and one whole stage-1 training step against the oracle chain."""
import math
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


def test_losses_match_reference_fixture():
    from gaussianavatar_b200.losses import image_loss, l1_loss_w, ssim
    d = np.load(os.path.join(GOLD, "losses.npz"))
    a = torch.tensor(d["img"], device=DEV, requires_grad=True)
    b = torch.tensor(d["gt"], device=DEV)
    assert abs(l1_loss_w(a, b).item() - float(d["l1"])) < 1e-6
    assert abs(ssim(a, b).item() - float(d["ssim"])) < 2e-6
    loss = image_loss(a, b, 0.2)
    assert abs(loss.item() - (0.8 * float(d["l1"]) + 0.2 * (1 - float(d["ssim"])))) < 2e-6
    loss.backward()
    assert _rel(a.grad.cpu().numpy(), d["grad"]) < 2e-4


@pytest.mark.parametrize("shape", [(1, 3, 37, 53), (2, 3, 64, 96), (1, 3, 16, 200)])
def test_losses_vs_oracle_odd_sizes(shape):
    from gaussianavatar_b200.losses import image_loss
    g = torch.Generator().manual_seed(shape[2])
    a, b = torch.rand(shape, generator=g), torch.rand(shape, generator=g)
    a64 = a.double().requires_grad_(True)
    ref = 0.8 * ao.l1_loss_w(a64, b.double()) + 0.2 * (1 - ao.ssim(a64, b.double()))
    ref.backward()
    ad = a.to(DEV).requires_grad_(True)
    up = torch.tensor(1.7, device=DEV)
    (image_loss(ad, b.to(DEV), 0.2) * up).backward()
    assert abs(image_loss(ad, b.to(DEV), 0.2).item() - ref.item()) < 2e-6
    assert _rel(ad.grad.cpu().numpy() / 1.7, a64.grad.numpy()) < 2e-4


def test_losses_with_uniform_background_tiles_vs_oracle():
    """Frames whose background equals the target exactly (GaussianAvatar's white background): the kernels skip the blurs for tiles whose
    whole window support is identical; loss and gradient still match the fp64 oracle."""
    from gaussianavatar_b200.losses import image_loss
    g = torch.Generator().manual_seed(5)
    H, W = 160, 224
    gt = torch.ones(2, 3, H, W)
    gt[:, :, 40:120, 60:150] = torch.rand(2, 3, 80, 90, generator=g)
    img = gt.clone()
    img[:, :, 50:130, 70:170] = torch.rand(2, 3, 80, 100, generator=g)          # differs from gt inside and partly outside the figure
    a64 = img.double().requires_grad_(True)
    ref = 0.8 * ao.l1_loss_w(a64, gt.double()) + 0.2 * (1 - ao.ssim(a64, gt.double()))
    ref.backward()
    ad = img.to(DEV).requires_grad_(True)
    loss = image_loss(ad, gt.to(DEV), 0.2)
    loss.backward()
    assert abs(loss.item() - ref.item()) < 2e-6
    assert _rel(ad.grad.cpu().numpy(), a64.grad.numpy()) < 2e-4
    assert (ad.grad[:, :, :20, :20] == 0).all()                                  # far background: exactly nothing


def test_fused_adam_matches_torch_adam():
    from gaussianavatar_b200.optim import FusedAdam
    g = torch.Generator().manual_seed(0)
    p0 = torch.randn(10007, generator=g)
    pa = torch.nn.Parameter(p0.clone().to(DEV)); pb = torch.nn.Parameter(p0.clone().to(DEV))
    oa = FusedAdam([{"params": [pa], "lr": 3e-3}])
    ob = torch.optim.Adam([{"params": [pb], "lr": 3e-3}])
    for s in range(5):
        gr = torch.randn(10007, generator=g).to(DEV) * (10.0 ** (s - 2))
        pa.grad = gr.clone(); pb.grad = gr.clone()
        oa.step(); ob.step()
    assert (pa - pb).abs().max().item() < 1e-6
    assert oa.state_dict()["state"][0]["exp_avg"].shape == ob.state_dict()["state"][0]["exp_avg"].shape


@pytest.mark.parametrize("mode", ["fp32", pytest.param("tf32", marks=pytest.mark.tf32)])
def test_train_step_gradients_vs_oracle_chain(mode):
    """d loss / d (net params, geo_feature, pose, transl) of one stage-1 step: CUDA chain vs the CPU oracle chain
    (torch autograd for the net / SMPL / LBS / losses + the C oracle's rasterizer backward).  Runs on the strict-FP32 decoder
    path (tight tolerance) and on the production tensor-core TF32 path (the tolerance SURVEY.md App. C assigns to TF32)."""
    tol = 5e-3 if mode == "fp32" else 3e-2
    from gaussianavatar_b200.trainer import Stage1Trainer
    from gaussianavatar_b200.workload import Stage1Workload
    from oracle import raster_oracle as ro
    N, S, side, B = 4000, 64, 128, 2
    wl = Stage1Workload(3, B, device=DEV, N=N, S=S, side=side, inp_posmap_size=32)
    with torch.no_grad():
        sd = wl.model.net.state_dict(); sd["decoder.conv8N.bias"] = torch.tensor([-3.9]); wl.model.net.load_state_dict(sd, strict=False)
    wl.make_ground_truth()
    assert wl.model.net.tensor_cores == (mode == "tf32")
    tr = Stage1Trainer(wl.model)
    ids = [4, 5]
    batch = wl.device_batch(ids)
    loss, image = tr.loss(batch, 5000, epoch=1)
    wl.model.zero_grad(1)
    loss.backward()
    m = wl.model
    # ---- oracle chain ----
    p = {k: v.cpu().clone().requires_grad_(True) for k, v in m.net.state_dict().items() if "running" not in k and "num_batches" not in k}
    geo = m.geo_feature.detach().cpu().clone().requires_grad_(True)
    pose = m.pose.weight.detach().cpu()[ids].clone().requires_grad_(True)
    transl = m.transl.weight.detach().cpu()[ids].clone().requires_grad_(True)
    a = dict(valid=m.valid_idx.cpu(), q=m._query_points.cpu(), w=m._query_lbs.cpu(), J=m._rest_joints.cpu(), ic=m._inv_cano.cpu())
    res, sc, shs = ao.pop_forward(p, geo, S, B=B)
    A = ao.smpl_joint_transforms(a["J"], pose, transl)
    C = torch.matmul(A, a["ic"][None])
    o = ao.assemble_and_skin(res, sc, shs, a["valid"], a["q"][None].expand(B, -1, -1), a["w"][None].expand(B, -1, -1), C, 5000, geo_feature=geo)
    cam = wl.cam
    rots = np.zeros((N, 4), np.float32); rots[:, 0] = 1
    rs, imgs = [], []
    for b in range(B):
        r = ro.forward(o["means3D"][b].detach().numpy(), o["colors"][b].detach().numpy(), np.ones(N, np.float32), o["scales"][b].detach().numpy(),
                       rots, np.ones(3, np.float32), cam.world_view_transform.numpy(), cam.full_proj_transform.numpy(),
                       math.tan(cam.FovX / 2), math.tan(cam.FovY / 2), side, side)
        rs.append(r); imgs.append(torch.tensor(r.image, dtype=torch.float32))
    img = torch.stack(imgs).requires_grad_(True)
    gt = wl.gt_dev[ids].cpu()
    li = 0.8 * ao.l1_loss_w(img, gt) + 0.2 * (1 - ao.ssim(img, gt))
    li.backward()
    gm, gc, gs = [], [], []
    for b in range(B):
        gb = rs[b].backward(img.grad[b].numpy())
        gm.append(torch.tensor(gb["d_means3D"], dtype=torch.float32)); gc.append(torch.tensor(gb["d_colors"], dtype=torch.float32))
        gs.append(torch.tensor(gb["d_scales"], dtype=torch.float32))
    reg = 3e-2 * o["scale_loss"] + 10.0 * o["offset_loss"] + o["geo_loss"]
    ref_loss = li.item() + reg.item()
    torch.autograd.backward([o["means3D"], o["colors"], o["scales"], reg], [torch.stack(gm), torch.stack(gc), torch.stack(gs), torch.ones(())])
    assert abs(loss.item() - ref_loss) < (2e-5 if mode == "fp32" else 2e-3) * max(1.0, abs(ref_loss))
    got = {k: v.cpu() for k, v in m.net.reference_grads().items()}
    worst = 0.0
    for k, v in p.items():
        if k.endswith(".bias") and ".bn" not in k and "conv8" not in k:
            continue                                     # exactly-zero gradients (bias in front of BatchNorm)
        worst = max(worst, _rel(got[k].numpy(), v.grad.numpy()))
    assert worst < tol, worst
    assert _rel(m.geo_feature.grad.cpu().numpy(), geo.grad.numpy()) < tol
    pg = m.pose.weight.grad.coalesce()
    dense = torch.zeros_like(m.pose.weight).index_add_(0, pg.indices()[0], pg.values()).cpu()
    assert _rel(dense[ids].numpy(), pose.grad.numpy()) < tol
    tg = m.transl.weight.grad.coalesce()
    dense_t = torch.zeros_like(m.transl.weight).index_add_(0, tg.indices()[0], tg.values()).cpu()
    assert _rel(dense_t[ids].numpy(), transl.grad.numpy()) < tol
    # and an optimizer step moves the parameters by Adam's first-step rule: |delta| == lr (sign of the gradient)
    before = m.net.flat.detach().clone()
    tr.sync_gradients(); m.optimizer.grad_scale = 1.0; m.step(1)
    delta = (m.net.flat.detach() - before)
    nz = m.net.flat.grad.abs() > 1e-4      # well above Adam's eps = 1e-8
    assert torch.allclose(delta[nz].abs(), torch.full_like(delta[nz], 3e-3), rtol=2e-3)
    assert torch.equal(torch.sign(delta[nz]), -torch.sign(m.net.flat.grad[nz]))


@pytest.mark.tf32
def test_graphed_step_matches_eager_step():
    """The whole-step CUDA graph (forward + loss + backward in one launch, static inputs) computes what the eager step computes:
    same loss, same gradients (up to float-atomics noise), over several steps with changing batches."""
    from gaussianavatar_b200.trainer import Stage1Trainer
    from gaussianavatar_b200.workload import Stage1Workload

    def run(use_graph):
        wl = Stage1Workload(3, 2, device=DEV, N=4000, S=64, side=128, inp_posmap_size=32)
        with torch.no_grad():
            sd = wl.model.net.state_dict(); sd["decoder.conv8N.bias"] = torch.tensor([-3.9]); wl.model.net.load_state_dict(sd, strict=False)
        wl.make_ground_truth()
        tr = Stage1Trainer(wl.model, use_graph=use_graph)
        out = []
        for i in range(4):
            loss = tr.step(wl.device_batch(wl.frame_ids(i)), 5000 + i, epoch=1)
            out.append((float(loss), wl.model.net.flat.grad.detach().clone(), wl.model.geo_feature.grad.detach().clone()))
        tr.finish()
        assert bool(tr._graphs) == use_graph
        return out, wl.model.net.flat.detach().clone(), wl.model.net.state_dict()["decoder.bn3.num_batches_tracked"]

    eager, flat_e, nbt_e = run(False)
    graph, flat_g, nbt_g = run(True)
    assert int(nbt_e) == int(nbt_g)
    # step 1 starts from identical parameters: gradients agree to atomics noise
    assert abs(eager[0][0] - graph[0][0]) < 1e-5 * max(1.0, abs(eager[0][0]))
    assert _rel(graph[0][1].cpu().numpy(), eager[0][1].cpu().numpy()) < 1e-3
    assert _rel(graph[0][2].cpu().numpy(), eager[0][2].cpu().numpy()) < 1e-3
    # later steps: Adam turns round-off level gradient differences into +-lr flips of a few parameters; the losses stay together
    for (le, _, _), (lg, _, _) in zip(eager, graph):
        assert abs(le - lg) < 2e-3 * max(1.0, abs(le))
    assert (flat_e - flat_g).abs().max().item() <= 4 * 2 * 3e-3 + 1e-6
