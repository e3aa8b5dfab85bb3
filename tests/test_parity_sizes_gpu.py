"""GPU parity of the PRODUCTION path at BASELINE.json sizes (VERDICT r1 "next round" item 1).

Production path = what bench.py times: decoder MLP on the TF32 tensor-core kernels, frames of a batch rendered on the
two alternating streams, sub-tile culling in the compositing kernels.  Every test here is marked `tf32`, which makes
tests/conftest.py leave GA_DECODER_FP32 unset.

  config 2 (50k Gaussians, UV 256^2, 512^2)   one WHOLE stage-1 train step vs the oracle chain
  config 3 (200k Gaussians, UV 512^2, 1024^2) one frame, rasterizer forward + backward vs the C oracle

Stage-wise bars (SURVEY.md App. C): rasterizer integer stages bit-exact, image mean-L1 <= 1e-4, rasterizer gradients rel-L2
<= 5e-4 (the oracle rasterizer is fed the Gaussians the CUDA chain produced, so these bars do not absorb TF32 noise of the
feature net); net / geo_feature / pose gradients of the whole chain within the TF32 tolerance (3e-2) of the fp32 oracle chain.
"""
import math

import numpy as np
import pytest
import torch

from oracle import avatar_oracle as ao

pytestmark = [pytest.mark.gpu, pytest.mark.tf32]
DEV = "cuda:0"


def _rel(a, b):
    a = np.asarray(a, dtype=np.float64).reshape(np.asarray(b).shape); b = np.asarray(b, dtype=np.float64)
    return np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30)


def _oracle_frame(means, colors, scales, cam, side):
    from oracle import raster_oracle as ro
    N = means.shape[0]
    rots = np.zeros((N, 4), np.float32); rots[:, 0] = 1
    return ro.forward(means, colors, np.ones(N, np.float32), scales, rots, np.ones(3, np.float32), cam.world_view_transform.numpy(),
                      cam.full_proj_transform.numpy(), math.tan(cam.FovX / 2), math.tan(cam.FovY / 2), side, side)


def _check_raster_state(v, o, H, W):
    """Per-stage parity of one frame: CUDA views `v` vs oracle forward `o`."""
    assert v["num_rendered"] == o.num_rendered
    np.testing.assert_array_equal(v["radii"].numpy(), o.get("radii"))
    np.testing.assert_array_equal(v["tiles_touched"].numpy(), o.get("tiles"))
    vis = o.get("radii") > 0
    np.testing.assert_array_equal(v["rect"].numpy().astype(np.int32)[vis], o.get("rect")[vis])
    np.testing.assert_array_equal(v["depth"].numpy().view(np.uint32)[vis], o.get("depth").astype(np.float32).view(np.uint32)[vis])
    np.testing.assert_array_equal(v["keys_sorted"].numpy().view(np.uint64), o.get("keys"))
    np.testing.assert_array_equal(v["vals_sorted"].numpy().view(np.uint32), o.get("vals"))
    np.testing.assert_array_equal(v["ranges"].numpy().view(np.uint32), o.get("ranges"))
    nc_mismatch = int((v["n_contrib"].numpy().view(np.uint32) != o.get("n_contrib")).sum())
    assert nc_mismatch <= max(2, H * W // 2000), nc_mismatch
    assert np.abs(v["final_T"].numpy() - o.get("final_T")).mean() <= 1e-4


def test_config3_frame_raster_forward_backward_vs_oracle():
    """200k Gaussians / 1024^2: the Gaussians the production chain (TF32 decoder + LBS) produces for one pose, rasterized
    by the CUDA path and by the C oracle; backward with a random image gradient."""
    from gaussianavatar_b200.rasterizer import GaussianRasterizationSettings, rasterize_backward, rasterize_forward
    from gaussianavatar_b200.workload import Stage1Workload
    wl = Stage1Workload(3, 1, device=DEV)
    assert wl.model.net.tensor_cores
    m, c = wl.model, wl._cam_dev
    with torch.no_grad():
        means, scales, colors, _ = m._posed_gaussians(torch.tensor([3], device=DEV), 5000)
    rs = GaussianRasterizationSettings(c.height, c.width, math.tan(c.FovX / 2), math.tan(c.FovY / 2), m.background, 1.0,
                                       c.world_view_transform, c.full_proj_transform, 0, c.camera_center, False, False)
    color, radii, ctx = rasterize_forward(means[0], colors[0], m.fix_opacity, scales[0], m.fix_rotation, rs)
    o = _oracle_frame(means[0].cpu().numpy(), colors[0].cpu().numpy(), scales[0].cpu().numpy(), wl.cam, wl.side)
    assert o.num_rendered > 500_000           # the config-3 regime: >256-entry tile lists, 6 sort passes
    _check_raster_state(ctx.views(), o, wl.side, wl.side)
    img = color.cpu().numpy().astype(np.float64)
    assert np.abs(img - o.image).mean() <= 1e-4
    gw = torch.randn(3, wl.side, wl.side, generator=torch.Generator().manual_seed(5))
    d_means3D, _, d_colors, _, d_scales, _ = rasterize_backward(ctx, means[0], colors[0], scales[0], m.fix_rotation, rs, gw.to(DEV),
                                                                want_opacity=False, want_rotations=False, want_means2D=False)
    gb = o.backward(gw.numpy())
    assert _rel(d_colors.cpu().numpy(), gb["d_colors"]) < 2e-4
    assert _rel(d_means3D.cpu().numpy(), gb["d_means3D"]) < 5e-4
    assert _rel(d_scales.cpu().numpy(), gb["d_scales"]) < 5e-4


def test_config2_whole_train_step_production_path_vs_oracle_chain():
    """50k Gaussians / 512^2, B = 2 frames: loss, images, rasterizer stages and every gradient of one stage-1 step."""
    from gaussianavatar_b200.trainer import Stage1Trainer
    from gaussianavatar_b200.workload import Stage1Workload
    B = 2
    wl = Stage1Workload(2, B, device=DEV)
    N, S, side = wl.N, wl.S, wl.side
    assert (N, side) == (50_000, 512) and wl.model.net.tensor_cores
    wl.make_ground_truth()
    tr = Stage1Trainer(wl.model)
    m = wl.model
    ids = [6, 7]
    batch = wl.device_batch(ids)
    loss, image = tr.loss(batch, 5000, epoch=1)
    g_means, g_scales, g_colors = m._last_gaussians
    for t in (g_means, g_scales, g_colors):
        t.retain_grad()
    image.retain_grad()
    m.zero_grad(1)
    loss.backward()
    torch.cuda.synchronize()

    # ---- stage-wise: the oracle rasterizer on the Gaussians the CUDA chain produced ----
    gt = wl.gt_dev[ids].cpu()
    img_c = image.detach().cpu()
    ref_img = img_c.clone().requires_grad_(True)
    li = 0.8 * ao.l1_loss_w(ref_img, gt) + 0.2 * (1 - ao.ssim(ref_img, gt))
    li.backward()
    assert _rel(image.grad.cpu().numpy(), ref_img.grad.numpy()) < 2e-4            # fused L1+SSIM backward at 512^2
    for b in range(B):
        o = _oracle_frame(g_means[b].detach().cpu().numpy(), g_colors[b].detach().cpu().numpy(), g_scales[b].detach().cpu().numpy(), wl.cam, side)
        assert np.abs(img_c[b].numpy().astype(np.float64) - o.image).mean() <= 1e-4
        gb = o.backward(image.grad[b].cpu().numpy())
        assert _rel(g_colors.grad[b].cpu().numpy(), gb["d_colors"]) < 5e-4
        assert _rel(g_means.grad[b].cpu().numpy(), gb["d_means3D"]) < 5e-4
        # d_scales of the chain additionally carries d(scale_loss): compare after removing that constant
        ds = g_scales.grad[b].cpu().numpy() - 3e-2 / (B * N * 3)
        assert _rel(ds, gb["d_scales"]) < 1e-3
        o.close()

    # ---- end to end: fp32 oracle chain (torch CPU + C rasterizer) vs the TF32 production chain ----
    from oracle import raster_oracle as ro
    p = {k: v.cpu().clone().requires_grad_(True) for k, v in m.net.state_dict().items() if "running" not in k and "num_batches" not in k}
    geo = m.geo_feature.detach().cpu().clone().requires_grad_(True)
    pose = m.pose.weight.detach().cpu()[ids].clone().requires_grad_(True)
    transl = m.transl.weight.detach().cpu()[ids].clone().requires_grad_(True)
    res, sc, shs = ao.pop_forward(p, geo, S, B=B)
    A = ao.smpl_joint_transforms(m._rest_joints.cpu(), pose, transl)
    C = torch.matmul(A, m._inv_cano.cpu()[None])
    q, w = m._query_points.cpu(), m._query_lbs.cpu()
    oo = ao.assemble_and_skin(res, sc, shs, m.valid_idx.cpu(), q[None].expand(B, -1, -1), w[None].expand(B, -1, -1), C, 5000, geo_feature=geo)
    rs, imgs = [], []
    for b in range(B):
        r = _oracle_frame(oo["means3D"][b].detach().numpy(), oo["colors"][b].detach().numpy(), oo["scales"][b].detach().numpy(), wl.cam, side)
        rs.append(r); imgs.append(torch.tensor(r.image, dtype=torch.float32))
    img = torch.stack(imgs).requires_grad_(True)
    li = 0.8 * ao.l1_loss_w(img, gt) + 0.2 * (1 - ao.ssim(img, gt))
    li.backward()
    gm, gc, gs = [], [], []
    for b in range(B):
        gb = rs[b].backward(img.grad[b].numpy())
        gm.append(torch.tensor(gb["d_means3D"], dtype=torch.float32)); gc.append(torch.tensor(gb["d_colors"], dtype=torch.float32))
        gs.append(torch.tensor(gb["d_scales"], dtype=torch.float32))
    reg = 3e-2 * oo["scale_loss"] + 10.0 * oo["offset_loss"] + oo["geo_loss"]
    ref_loss = li.item() + reg.item()
    torch.autograd.backward([oo["means3D"], oo["colors"], oo["scales"], reg], [torch.stack(gm), torch.stack(gc), torch.stack(gs), torch.ones(())])
    assert abs(loss.item() - ref_loss) < 2e-3 * max(1.0, abs(ref_loss))
    assert np.abs(img_c.numpy() - img.detach().numpy()).mean() < 2e-3             # TF32 colours / offsets vs fp32: context, not the 1e-4 bar
    got = {k: v.cpu() for k, v in m.net.reference_grads().items()}
    worst = 0.0
    for k, v in p.items():
        if k.endswith(".bias") and ".bn" not in k and "conv8" not in k:
            continue                                     # exactly-zero gradients (bias in front of BatchNorm)
        worst = max(worst, _rel(got[k].numpy(), v.grad.numpy()))
    assert worst < 3e-2, worst
    assert _rel(m.geo_feature.grad.cpu().numpy(), geo.grad.numpy()) < 3e-2
    pg = m.pose.weight.grad.coalesce()
    dense = torch.zeros_like(m.pose.weight).index_add_(0, pg.indices()[0], pg.values()).cpu()
    assert _rel(dense[ids].numpy(), pose.grad.numpy()) < 3e-2
