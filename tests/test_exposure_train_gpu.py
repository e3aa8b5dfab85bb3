"""GPU: the per-frame exposure table through AvatarModel, the trainer, the pose fitter and data parallelism.

Identity rows render the exposure-off images bit for bit.  A known-answer capture (a fixed avatar rendered under known per-frame
transforms, frame 0 at identity) is recovered by training and by PoseFitter(exposure=True).  Graphed and eager steps agree, a skipped
(overflowed) step leaves the table and its moments alone, a stage-2 step trains the table, and two NCCL ranks keep equal tables.
"""
import os
import tempfile

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from gaussianavatar_b200.avatar_model import identity_exposure

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SMALL = dict(N=4000, S=64, side=128, inp_posmap_size=32)


def _workload(seed=0, frames=8, exposure=True, B=2):
    from gaussianavatar_b200.workload import Stage1Workload
    wl = Stage1Workload(3, B, device=DEV, seed=seed, num_frames=frames, **SMALL)
    with torch.no_grad():
        sd = wl.model.net.state_dict(); sd["decoder.conv8N.bias"] = torch.tensor([-3.9]); wl.model.net.load_state_dict(sd, strict=False)
    if exposure:
        m = wl.model
        m.model_parms.train_exposure = True
        m.exposure = torch.nn.Parameter(identity_exposure(wl.num_frames, DEV))
    return wl


def _true_table(frames, seed=5, a=0.1, t=0.04):
    g = torch.Generator().manual_seed(seed)
    E = identity_exposure(frames, "cpu")
    E[1:, :, :3] += a * torch.randn(frames - 1, 3, 3, generator=g)
    E[1:, :, 3] += t * torch.randn(frames - 1, 3, generator=g)
    return E.to(DEV)


def _fix_avatar(wl, seed=3):
    """A fixed avatar: the decoder's output frozen, its colours spread over [0.15, 0.85] so that A and t are told apart."""
    m = wl.model
    with torch.no_grad():
        dec = m.net.forward_packed(m.geo_feature, int(m.model_parms.query_posmap_size), wl.B).detach().clone()
        g = torch.Generator(device=DEV).manual_seed(seed)
        dec[:, 4:7] = 0.15 + 0.7 * torch.rand(dec.shape[0], 3, device=DEV, generator=g)
    m.net.forward_packed = lambda geo, S, batch: dec
    return dec


def _capture(wl, E):
    """Ground truth: every frame rendered with its row of E (a batch's `exposure`)."""
    m = wl.model
    imgs = []
    with torch.no_grad():
        for f0 in range(0, wl.num_frames, wl.B):
            idx = torch.arange(f0, f0 + wl.B, device=DEV)
            batch = dict(pose_idx=idx, exposure=E[idx], **wl.camera_fields(wl.B))
            imgs.append(m.render_free_stage1(batch, 5000).clone())
    wl.gt_dev = torch.cat(imgs).contiguous()


def _train(wl, steps, use_graph=False, it0=5000, record=None):
    """record: a list that receives (exposure gradient, table) after each step."""
    from gaussianavatar_b200.trainer import Stage1Trainer
    tr = Stage1Trainer(wl.model, use_graph=use_graph)
    losses = []
    for i in range(steps):
        losses.append(float(tr.step(wl.device_batch(wl.frame_ids(i % (wl.num_frames // wl.B))), it0 + i, epoch=1)))
        if record is not None:
            m = wl.model
            record.append((m.exposure.grad.detach().clone(), m.exposure.detach().clone()))
    tr.finish()
    return tr, losses


def _image_loss(wl):
    from gaussianavatar_b200.losses import image_loss
    m = wl.model
    out = []
    with torch.no_grad():
        for f0 in range(0, wl.num_frames, wl.B):
            b = wl.device_batch(list(range(f0, f0 + wl.B)))
            img = m.train_stage1(b, 5000)[0]
            out.append(float(image_loss(img, b["original_image"], m.opt_parms.lambda_dssim)))
    return float(np.mean(out))


def test_identity_rows_render_the_exposure_off_images():
    wl = _workload()
    m = wl.model
    batch = dict(pose_idx=torch.tensor([0, 3], device=DEV), **wl.camera_fields(2))
    with torch.no_grad():
        dec = m._stage1_decoder(2)
        images = []
        for table in (m.exposure, None):
            means, scales, colors = m._assemble(dec, m.pose(batch["pose_idx"]), m.transl(batch["pose_idx"]), exposure=table,
                                                exposure_idx=None if table is None else batch["pose_idx"])
            images.append(m._render_frames(batch, means, scales, colors))
    assert torch.equal(images[0], images[1])


def test_training_recovers_known_exposures():
    """Fixed avatar, 8 frames under known [A | t] (frame 0 identity), 400 steps of B = 2: each entry within 0.05 of the truth (A and t),
    row 0 exactly identity, and a lower image loss than the same steps without the table."""
    wl = _workload(frames=8)
    m = wl.model
    m.opt_parms.epochs = 100                      # 100 epochs x 4 batches: the rate falls from 1e-2 to 1e-3 over the 400 steps
    _fix_avatar(wl)
    E = _true_table(8)
    _capture(wl, E)
    loss0 = _image_loss(wl)
    _train(wl, 400)
    got = m.exposure.detach()
    err = (got - E).abs()
    print(f"\nexposure: max |A - A*| {float(err[..., :3].max()):.4g}, max |t - t*| {float(err[..., 3].max()):.4g}, "
          f"loss {loss0:.5g} -> {_image_loss(wl):.5g}")
    assert torch.equal(got[0], torch.eye(3, 4, device=DEV))
    assert float(err.max()) < 0.05
    with_table = _image_loss(wl)

    wl2 = _workload(frames=8, exposure=False)
    _fix_avatar(wl2)
    wl2.gt_dev = wl.gt_dev
    _train(wl2, 400)
    without = _image_loss(wl2)
    print(f"exposure: image loss after 400 steps with the table {with_table:.5g}, without {without:.5g}")
    assert with_table < 0.7 * without


def test_posefitter_recovers_a_test_frames_exposure():
    from gaussianavatar_b200.posefit import PoseFitter
    wl = _workload(frames=4)
    m = wl.model
    _fix_avatar(wl)
    E = _true_table(4, seed=9)
    _capture(wl, E)
    cam = wl.camera_fields(1)
    items = []
    for f in (1, 2, 3):
        items.append(dict(original_image=wl.gt_dev[f], FovX=cam["FovX"][0], FovY=cam["FovY"][0], height=cam["height"][0],
                          width=cam["width"][0], world_view_transform=cam["world_view_transform"][0],
                          full_proj_transform=cam["full_proj_transform"][0], pose_data=m.pose.weight[f].detach().cpu(),
                          transl_data=m.transl.weight[f].detach().cpu()))
    pose, transl, report, table = PoseFitter(m, iters=400, exposure=True).fit(items)
    err = (table.to(DEV) - E[1:]).abs()
    ratio = float(err.square().mean().sqrt() / (E[1:] - identity_exposure(3, DEV)).square().mean().sqrt())
    print(f"\nposefit exposure: max |A - A*| {float(err[..., :3].max()):.4g}, max |t - t*| {float(err[..., 3].max()):.4g}, "
          f"rms error / rms distance from identity {ratio:.3g}, losses {[(r['initial_loss'], r['fitted_loss']) for r in report]}")
    assert float(err.max()) < 0.05 and ratio < 0.5
    assert all(r["fitted_loss"] < 0.5 * r["initial_loss"] for r in report)
    # without the flag: the three-value result of before
    assert len(PoseFitter(m, iters=2).fit(items[:1])) == 3


@pytest.mark.tf32
def test_graphed_step_matches_eager_step():
    def run(use_graph, record):
        wl = _workload()
        wl.make_ground_truth()
        tr, losses = _train(wl, 4, use_graph, record=record)
        return wl, tr, losses
    rec_e, rec_g = [], []
    wl_e, tr_e, eager = run(False, rec_e)
    wl_g, tr_g, graph = run(True, rec_g)
    assert tr_g._graphs and all(k[-2] and not k[-1] for k in tr_g._graphs)    # the exposure flag goes before LPIPS's
    for le, lg in zip(eager, graph):
        assert abs(le - lg) < 2e-3 * max(1.0, abs(le))
    te, tg = wl_e.model.exposure.detach(), wl_g.model.exposure.detach()
    assert torch.equal(te[0], torch.eye(3, 4, device=DEV)) and torch.equal(tg[0], torch.eye(3, 4, device=DEV))
    moved = (tg - identity_exposure(tg.shape[0], DEV)).abs().amax((1, 2))
    assert float(moved[1:8].min()) > 0                           # frames 1..7 were stepped
    # the gradient each path hands to Adam, step by step: the same up to the decoder's float-atomic noise (the tolerance of the
    # loss and net-gradient comparisons of test_depth_train_gpu), and nonzero in exactly the rows of the step's frames
    def rel(a, b):
        return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))
    for i, ((ge, _), (gg, _)) in enumerate(zip(rec_e, rec_g)):
        rows = set(range(2 * i, 2 * i + 2)) - {0}
        assert {int(r) for r in torch.nonzero(gg.abs().amax((1, 2))).flatten()} == rows
        assert rel(gg, ge) < 1e-3, (i, rel(gg, ge))
    # Adam's first step moves each entry by ~lr against the sign of its gradient: both tables move that way wherever the gradient
    # is not round-off level against the largest
    ge = rec_e[0][0]
    strong = ge.abs() > 1e-2 * ge.abs().max()
    d_e = rec_e[0][1] - identity_exposure(te.shape[0], DEV)
    d_g = rec_g[0][1] - identity_exposure(te.shape[0], DEV)
    assert int(strong.sum()) >= 6
    assert torch.equal(d_e[strong].sign(), -ge[strong].sign()) and torch.equal(d_g[strong].sign(), -ge[strong].sign())
    assert wl_g.model.exposure_optimizer.step_count == wl_e.model.exposure_optimizer.step_count == 4


def test_skipped_step_leaves_table_and_moments():
    wl = _workload()
    wl.make_ground_truth()
    tr, _ = _train(wl, 2)
    m = wl.model
    opt = m.exposure_optimizer
    before = [t.detach().clone() for t in (m.exposure, opt.exp_avg, opt.exp_avg_sq)]
    n = opt.step_count
    g = torch.randn_like(m.exposure)
    g[0] = 0.0                                                              # the anchor row's gradient, as the kernel writes it
    m.exposure.grad = g
    opt.skip_flag = torch.ones(1, dtype=torch.int32, device=DEV)            # the rasterizer's overflow word, set
    opt.step()
    torch.cuda.synchronize()
    for a, b in zip(before, (m.exposure, opt.exp_avg, opt.exp_avg_sq)):
        assert torch.equal(a, b.detach())
    tr._undo_host_step(1)                                                    # the host side of the skipped step
    assert opt.step_count == n
    opt.skip_flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    opt.step()
    torch.cuda.synchronize()
    assert not torch.equal(before[0], m.exposure.detach()) and torch.equal(before[0][0], m.exposure.detach()[0])


def test_stage2_step_trains_the_table(tmp_path):
    from dataset_fixture import write_synthetic_dataset
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams, OptimizationParams
    from gaussianavatar_b200.trainer import AvatarTrainer
    from gaussianavatar_b200.workload import to_cuda
    mp_ = write_synthetic_dataset(str(tmp_path), N=700, S=48, num_frames=4, side=64, inp=32, stage2=True)
    mp_.train_exposure = True
    torch.manual_seed(0)
    m = AvatarModel(mp_, NetworkParams(nf=8), OptimizationParams(), train=True)
    assert m.exposure is not None and tuple(m.exposure.shape) == (4, 3, 4)
    tr = AvatarTrainer(m, use_graph=False)
    items = [m.train_dataset[0], m.train_dataset[2]]
    batch = {k: (torch.stack([torch.as_tensor(it[k]) for it in items]) if not isinstance(items[0][k], (int, float)) else [it[k] for it in items])
             for k in items[0]}
    batch["pose_idx"] = torch.tensor([it["pose_idx"] for it in items])
    batch, _ = to_cuda(batch, DEV)
    loss = tr.step(batch, 3000, epoch=1)
    tr.finish()
    assert np.isfinite(float(loss))
    E = m.exposure.detach()
    eye = torch.eye(3, 4, device=DEV)
    assert torch.equal(E[0], eye) and torch.equal(E[1], eye) and torch.equal(E[3], eye)
    assert not torch.equal(E[2], eye)
    # the checkpoint carries the table into a stage-2 save and back
    m.model_path = str(tmp_path / "out")
    m.save(7)
    saved = torch.load(os.path.join(m.model_path, "net/iteration_7/pose_encoder.pth"), weights_only=False)
    assert torch.equal(saved["exposure"].to(DEV), E) and saved["exposure_optimizer"]["step"] == 1


def _dp_worker(rank, world, port, path):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import torch.distributed as dist
    from gaussianavatar_b200.trainer import Stage1Trainer
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    global DEV
    DEV = f"cuda:{rank}"
    wl = _workload()
    wl.make_ground_truth()
    tr = Stage1Trainer(wl.model)
    for i in range(3):
        tr.step(wl.device_batch(wl.frame_ids(i, rank, world)), 5000 + i, epoch=1)
    tr.finish()
    torch.cuda.synchronize()
    torch.save(wl.model.exposure.detach().cpu(), f"{path}.{rank}")
    dist.barrier(device_ids=[rank])
    dist.destroy_process_group()


def test_two_nccl_ranks_keep_equal_tables():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ctx = mp.get_context("spawn")
    port = 29900 + (os.getpid() % 300)
    path = os.path.join(tempfile.mkdtemp(), "exp")
    procs = [ctx.Process(target=_dp_worker, args=(r, 2, port, path)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(600)
        assert p.exitcode == 0
    tables = [torch.load(f"{path}.{r}") for r in range(2)]
    assert torch.equal(tables[0], tables[1])
    assert not torch.equal(tables[0], identity_exposure(tables[0].shape[0], "cpu"))
