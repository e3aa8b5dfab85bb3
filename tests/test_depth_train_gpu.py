"""GPU: training an avatar against depth maps end to end.

  * The target depth is plane 0 of one synthetic avatar's `rasterize_batch_depth`; for a second avatar the depth term's gradient in
    means3D (through `rasterize_batch_with_depth` and `depth_loss`) is a descent direction.
  * `rasterize_batch_with_depth` returns `rasterize_batch_depth`'s images and depth bit for bit, and with no depth gradient its
    gradients are `rasterize_batch`'s.
  * Stage 1 with the term: graphed and eager steps give the same loss and gradients (the graph tests' tolerances); a short run with
    the term lowers the mean |m - d*| on counted pixels more than the same run without it.
  * Stage 2 runs a step with the term, from a dataset folder with depths/.
"""
import os

import numpy as np
import pytest
import torch

from gaussianavatar_b200.losses import depth_loss
from gaussianavatar_b200.rasterizer import RasterBatchPlan, rasterize_batch, rasterize_batch_depth, rasterize_batch_with_depth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _rel(a, b):
    return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30))


def _workload(seed=0):
    from gaussianavatar_b200.workload import Stage1Workload
    wl = Stage1Workload(3, 2, device=DEV, seed=seed, N=4000, S=64, side=128, inp_posmap_size=32)
    with torch.no_grad():
        sd = wl.model.net.state_dict(); sd["decoder.conv8N.bias"] = torch.tensor([-3.9]); wl.model.net.load_state_dict(sd, strict=False)
    wl.make_ground_truth()
    return wl


def _target_depth(wl_target, frames):
    """Plane 0 of the target avatar's depth pass for each frame [F,H,W] (rasterize_batch_depth, forward only)."""
    m = wl_target.model
    out = []
    with torch.no_grad():
        for f0 in range(0, frames, 2):
            ids = [f0, f0 + 1]
            batch = wl_target.device_batch(ids)
            means, scales, colors, _ = m._posed_gaussians(batch["pose_idx"], 5000)
            cams = m._batch_cameras(batch, 2, m.device)
            plan = RasterBatchPlan(2, means.shape[1], wl_target.side, wl_target.side, m.device)
            _, depth = rasterize_batch_depth(means, colors, scales, m.fix_rotation, m.fix_opacity, cams, m.background, plan)
            assert plan.check(wait=True)
            out.append(depth[:, 0].clone())
    return torch.cat(out)


@pytest.fixture(scope="module")
def target():
    wl = _workload(seed=1)
    d = _target_depth(wl, 8)
    assert float((d > 0).float().mean()) > 0.1
    return d


def _with_depth(wl, ids, target):
    b = wl.device_batch(ids)
    b["depth"] = target[torch.tensor(ids, device=DEV)].contiguous()
    return b


def test_forward_equals_depth_pass_and_plain_gradients():
    wl = _workload()
    m = wl.model
    batch = wl.device_batch([0, 1])
    with torch.no_grad():
        means, scales, colors, _ = m._posed_gaussians(batch["pose_idx"], 5000)
    cams = m._batch_cameras(batch, 2, m.device)
    P = means.shape[1]
    args = lambda t: (t[0], t[1], t[2], m.fix_rotation, m.fix_opacity, cams, m.background)
    with torch.no_grad():
        plan_r = RasterBatchPlan(2, P, wl.side, wl.side, m.device)
        img_r, depth_r = rasterize_batch_depth(*args((means, colors, scales)), plan_r)
    leaf = [t.clone().requires_grad_(True) for t in (means, colors, scales)]
    plan = RasterBatchPlan(2, P, wl.side, wl.side, m.device)
    img, depth = rasterize_batch_with_depth(*args(leaf), plan)
    assert plan.check(wait=True) and plan_r.check(wait=True)
    assert torch.equal(img, img_r) and torch.equal(depth, depth_r)
    gw = torch.randn_like(img)
    (img * gw).sum().backward()                             # no depth gradient: ga_rasterb_backward's gradients
    leaf2 = [t.clone().requires_grad_(True) for t in (means, colors, scales)]
    plan2 = RasterBatchPlan(2, P, wl.side, wl.side, m.device)
    (rasterize_batch(*args(leaf2), plan2) * gw).sum().backward()
    for a, b in zip(leaf, leaf2):
        assert _rel(a.grad.cpu().numpy(), b.grad.cpu().numpy()) < 1e-5


def test_depth_gradient_is_a_descent_direction(target):
    wl = _workload()
    m = wl.model
    batch = _with_depth(wl, [2, 3], target)
    with torch.no_grad():
        means, scales, colors, _ = m._posed_gaussians(batch["pose_idx"], 5000)
    cams = m._batch_cameras(batch, 2, m.device)
    plan = RasterBatchPlan(2, means.shape[1], wl.side, wl.side, m.device)

    def loss_at(x, grad=False):
        x = x.clone().requires_grad_(grad)
        _, depth = rasterize_batch_with_depth(x, colors, scales, m.fix_rotation, m.fix_opacity, cams, m.background, plan)
        loss, n = depth_loss(depth, batch["depth"], 1.0, return_count=True)
        assert plan.check(wait=True)
        if grad:
            loss.backward()
        return float(loss), int(n), x.grad

    l0, n0, g = loss_at(means, True)
    assert n0 > 500 and l0 > 0 and float(g.abs().max()) > 0
    step = -g / g.abs().max()
    predicted = float((g * step).sum())
    for t in (1e-4, 3e-5):
        l1, _, _ = loss_at(means + t * step)
        print(f"\ndepth train: step {t:g}: loss {l0:.6g} -> {l1:.6g} (first order {t * predicted:.3g})")
        assert l1 < l0


def _train(wl, target, steps, use_graph, with_depth, lam=1.0, it0=5000):
    from gaussianavatar_b200.trainer import Stage1Trainer
    wl.model.opt_parms.lambda_depth = lam
    tr = Stage1Trainer(wl.model, use_graph=use_graph)
    out = []
    for i in range(steps):
        ids = wl.frame_ids(i % 4)
        batch = _with_depth(wl, ids, target) if with_depth else wl.device_batch(ids)
        loss = tr.step(batch, it0 + i, epoch=1)
        out.append((float(loss), wl.model.net.flat.grad.detach().clone(), wl.model.geo_feature.grad.detach().clone()))
    tr.finish()
    return tr, out


@pytest.mark.tf32
def test_graphed_step_with_depth_matches_eager_step(target):
    """test_train_gpu's graphed-versus-eager comparison and tolerances with the depth term.  lambda_depth = 0.1 keeps the total loss
    at that test's scale (its later-step tolerance is absolute: Adam turns round-off level gradient differences into +-lr flips)."""
    wl_e, wl_g = _workload(), _workload()
    tr_e, eager = _train(wl_e, target, 4, False, True, lam=0.1)
    tr_g, graph = _train(wl_g, target, 4, True, True, lam=0.1)
    assert bool(tr_g._graphs) and not tr_e._graphs
    assert all(k[3] and not k[-1] for k in tr_g._graphs)           # the key carries the depth flag; the last word is LPIPS's
    assert abs(eager[0][0] - graph[0][0]) < 1e-5 * max(1.0, abs(eager[0][0]))
    assert _rel(graph[0][1].cpu().numpy(), eager[0][1].cpu().numpy()) < 1e-3
    assert _rel(graph[0][2].cpu().numpy(), eager[0][2].cpu().numpy()) < 1e-3
    for (le, _, _), (lg, _, _) in zip(eager, graph):
        assert abs(le - lg) < 2e-3 * max(1.0, abs(le))
    assert (wl_e.model.net.flat - wl_g.model.net.flat).abs().max().item() <= 4 * 2 * 3e-3 + 1e-6
    # the graphed loss carries the depth term: without it the first step's loss is lower by lambda * depth_loss
    _, plain = _train(_workload(), target, 1, False, False)
    assert eager[0][0] > plain[0][0] + 1e-4


def _mean_abs_error(wl, target, frames=8):
    m = wl.model
    err, n = 0.0, 0
    with torch.no_grad():
        for f0 in range(0, frames, 2):
            ids = [f0, f0 + 1]
            batch = wl.device_batch(ids)
            means, scales, colors, _ = m._posed_gaussians(batch["pose_idx"], 5000)
            cams = m._batch_cameras(batch, 2, m.device)
            plan = RasterBatchPlan(2, means.shape[1], wl.side, wl.side, m.device)
            _, depth = rasterize_batch_depth(means, colors, scales, m.fix_rotation, m.fix_opacity, cams, m.background, plan)
            assert plan.check(wait=True)
            t = target[f0:f0 + 2]
            c = (t > 0) & (depth[:, 1] != 0)
            err += float((depth[:, 0] - t).abs()[c].sum())
            n += int(c.sum())
    return err / max(n, 1)


# H100 80GB HBM3 (700 W), two runs: mean |m - d*| 0.0456 before; after 60 colour-only steps 0.203 / 0.172, after 60 steps with the
# term 0.0202 / 0.0240 (the decoder's float atomics make runs differ in the last bits, and training amplifies that)
STEPS, MARGIN = 60, 0.5


def test_short_run_with_depth_lowers_depth_error(target):
    wl0 = _workload()
    before = _mean_abs_error(wl0, target)
    _train(wl0, target, STEPS, True, False)
    without = _mean_abs_error(wl0, target)
    wl1 = _workload()
    _train(wl1, target, STEPS, True, True)
    with_depth = _mean_abs_error(wl1, target)
    print(f"\ndepth train: mean |m - d*| before {before:.5g}, after {STEPS} steps without the term {without:.5g}, with it {with_depth:.5g}")
    assert with_depth < MARGIN * without and with_depth < before


def test_stage2_step_with_depth(tmp_path):
    from dataset_fixture import write_synthetic_dataset
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams, OptimizationParams
    from gaussianavatar_b200.trainer import AvatarTrainer
    from gaussianavatar_b200.workload import to_cuda
    mp = write_synthetic_dataset(str(tmp_path), N=700, S=48, num_frames=4, side=64, inp=32, stage2=True)
    mp.depth_maps = True
    folder = os.path.join(mp.source_path, "train")
    os.makedirs(os.path.join(folder, "depths"))
    for n in os.listdir(os.path.join(folder, "images")):
        np.save(os.path.join(folder, "depths", n.split(".")[0] + ".npy"), np.full((64, 64), 2.0, np.float32))
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
    assert batch["depth"].shape == (2, 64, 64)
    loss, _ = tr.loss(batch, 3000, epoch=1)
    plain = dict(batch)
    del plain["depth"]
    loss_plain, _ = tr.loss(plain, 3000, epoch=1)
    dl = depth_loss(m.last_depth.detach(), batch["depth"], 1.0)
    assert float(dl) > 0 and abs(float(loss) - float(loss_plain) - float(dl)) <= 1e-4 * max(1.0, float(loss))
    before = [p.detach().clone() for p in m.pose_encoder.parameters()]
    loss = tr.step(batch, 3000, epoch=1)
    tr.finish()
    assert np.isfinite(float(loss))
    assert any(not torch.equal(a, b.detach()) for a, b in zip(before, m.pose_encoder.parameters()))
