"""CPU: the exposure table's C ABI argument checks, its checkpoint entries (round trip, checkpoints without them, the stage 1 ->
stage 2 carry-over), option namespaces without the new fields, the learning-rate schedule and the gloo all-reduce bucket with the
table's gradient appended."""
import os
import types

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from gaussianavatar_b200 import _lib
from gaussianavatar_b200.avatar_model import AvatarModel, identity_exposure
from gaussianavatar_b200.optim import ExposureAdam, log_linear_lr

FAKE = 256     # a non-NULL address: every refusal below happens before anything is read or launched


def _refused(rc, text):
    assert rc != 0
    assert text in _lib.lib().ga_last_error().decode()


def test_abi_refuses_bad_arguments():
    L = _lib.lib()
    fwd = lambda F, E=FAKE, idx=FAKE, N=10, B=1: L.ga_lbs_forward_exposure(N, B, 24, 24, 1.0, 0, FAKE, FAKE, FAKE, FAKE, FAKE, F, E, idx,
                                                                             FAKE, FAKE, FAKE, None)
    _refused(fwd(0), "num_exposures 0")
    _refused(fwd(2, E=None), "NULL pointer")
    _refused(fwd(2, idx=None), "NULL pointer")
    _refused(fwd(2, B=9), "bad LBS dims")
    assert L.ga_lbs_exposure_workspace_bytes(10, 24) == 4 * 12 * 8
    assert L.ga_lbs_exposure_workspace_bytes(300 * 256, 24) == 4 * 12 * 8 * 264       # two CTAs per SM on 132 SMs
    assert L.ga_lbs_exposure_workspace_bytes(300 * 256, 55) == 4 * 12 * 8 * 132
    assert L.ga_lbs_exposure_workspace_bytes(0, 24) == 0

    def bwd(F=2, dE=FAKE, ws=FAKE, nbytes=384, J=24, ld=24):
        return L.ga_lbs_backward_exposure(10, 1, J, ld, 16, 1.0, 0, FAKE, FAKE, FAKE, FAKE, FAKE, F, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE,
                                          FAKE, dE, ws, nbytes, None)
    _refused(bwd(F=0), "num_exposures 0")
    _refused(bwd(dE=None), "NULL pointer")
    _refused(bwd(nbytes=380), "exposure workspace of 380 bytes")
    _refused(bwd(ws=None), "exposure workspace")
    _refused(bwd(J=55, ld=24), "lbs_ld 24")


def _stub(frames, tmp=None):
    """The parts of an AvatarModel the checkpoint code touches, on the CPU."""
    m = types.SimpleNamespace(device=torch.device("cpu"), exposure=torch.nn.Parameter(identity_exposure(frames, "cpu")),
                              exposure_optimizer=None, _dec_cache=None, net=torch.nn.Linear(2, 2), pose=torch.nn.Embedding(frames, 3),
                              transl=torch.nn.Embedding(frames, 3), geo_feature=torch.nn.Parameter(torch.zeros(1, 2)))
    for name in ("_exposure_state", "_load_exposure", "stage_load"):
        setattr(m, name, types.MethodType(getattr(AvatarModel, name), m))
    return m


class _StubAdam:
    def __init__(self):
        self.sd = None

    def state_dict(self):
        return {"step": 7, "exp_avg": torch.full((3, 3, 4), 0.5), "exp_avg_sq": torch.full((3, 3, 4), 0.25)}

    def load_state_dict(self, sd):
        self.sd = sd


def test_checkpoint_round_trip_and_missing_key(tmp_path):
    a = _stub(3)
    with torch.no_grad():
        a.exposure[1] += 0.25
        a.exposure[2, :, 3] = torch.tensor([0.1, -0.2, 0.3])
    a.exposure_optimizer = _StubAdam()
    path = os.path.join(tmp_path, "net.pth")
    torch.save({"net": a.net.state_dict(), **a._exposure_state()}, path)
    saved = torch.load(path, weights_only=False)
    assert tuple(saved["exposure"].shape) == (3, 3, 4) and saved["exposure_optimizer"]["step"] == 7
    b = _stub(3)
    b.exposure_optimizer = _StubAdam()
    b._load_exposure(saved)
    assert torch.equal(b.exposure.detach(), a.exposure.detach())
    assert b.exposure_optimizer.sd["step"] == 7
    # a checkpoint without the key (the reference's, or one written without the table) loads identity
    with torch.no_grad():
        b.exposure.mul_(3.0)
    b._load_exposure({"net": {}})
    assert torch.equal(b.exposure.detach(), identity_exposure(3, "cpu"))
    with pytest.raises(ValueError, match="checkpoint exposure"):
        b._load_exposure({"exposure": torch.zeros(4, 3, 4)})
    # a model without the table writes no entry and ignores one
    c = _stub(3)
    c.exposure = None
    assert c._exposure_state() == {}
    c._load_exposure(saved)


def test_stage1_table_carries_into_stage2(tmp_path):
    s1 = _stub(4)
    with torch.no_grad():
        s1.exposure[3, 0, 0] = 1.5
    torch.save({"net": s1.net.state_dict(), "pose": s1.pose.state_dict(), "transl": s1.transl.state_dict(), "geo_feature": s1.geo_feature,
                **s1._exposure_state()}, os.path.join(tmp_path, "net.pth"))
    s2 = _stub(4)
    s2.exposure_optimizer = _StubAdam()
    s2.stage_load(str(tmp_path))
    assert torch.equal(s2.exposure.detach(), s1.exposure.detach())
    assert s2.exposure_optimizer.sd is None            # the table carries over; its Adam state starts afresh in stage 2


def test_namespaces_without_the_new_fields():
    """The reference's option namespaces have no train_exposure / exposure_lr_*: the table is off and the rates default."""
    from gaussianavatar_b200.config import ModelParams, OptimizationParams
    assert ModelParams().train_exposure is False
    op = OptimizationParams()
    assert (op.exposure_lr_init, op.exposure_lr_final) == (0.01, 0.001)
    m = types.SimpleNamespace(exposure=torch.nn.Parameter(identity_exposure(5, "cpu")), opt_parms=types.SimpleNamespace(epochs=3),
                              train_dataset=list(range(10)), batch_size=2)
    m.exposure_schedule_steps = types.MethodType(AvatarModel.exposure_schedule_steps, m)
    AvatarModel.exposure_setup(m)
    opt = m.exposure_optimizer
    assert (opt.total_steps, opt.lr_init, opt.lr_final) == (15, 0.01, 0.001)
    assert getattr(types.SimpleNamespace(), "train_exposure", False) is False


def test_learning_rate_falls_log_linearly():
    assert log_linear_lr(0, 100, 0.01, 0.001) == pytest.approx(0.01, rel=1e-12)
    assert log_linear_lr(50, 100, 0.01, 0.001) == pytest.approx(0.01 * 0.1 ** 0.5, rel=1e-12)
    assert log_linear_lr(100, 100, 0.01, 0.001) == pytest.approx(0.001, rel=1e-12)
    assert log_linear_lr(1000, 100, 0.01, 0.001) == pytest.approx(0.001, rel=1e-12)
    opt = ExposureAdam(torch.nn.Parameter(identity_exposure(2, "cpu")), 10)
    rows = opt._hyper_rows(25)
    assert rows.shape[0] >= 25
    assert float(rows[0, 0]) == pytest.approx(0.01, rel=1e-6) and float(rows[24, 0]) == pytest.approx(0.001, rel=1e-6)
    assert float(rows[4, 4]) == pytest.approx(1 - 0.9 ** 5, rel=1e-6)
    assert float(rows[4, 5]) == pytest.approx((1 - 0.999 ** 5) ** 0.5, rel=1e-6)


def _bucket_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from gaussianavatar_b200.trainer import Stage1Trainer
    g = torch.Generator().manual_seed(300 + rank)
    flat, geo, exp = torch.nn.Parameter(torch.zeros(50)), torch.nn.Parameter(torch.zeros(1, 2, 3, 3)), torch.nn.Parameter(torch.zeros(4, 3, 4))
    for t in (flat, geo, exp):
        t.grad = torch.randn(t.shape, generator=g)
    local = torch.cat([flat.grad.reshape(-1), geo.grad.reshape(-1), exp.grad.reshape(-1)])
    tr = Stage1Trainer.__new__(Stage1Trainer)
    tr.world, tr.group = world, None
    tr.model = types.SimpleNamespace(net=types.SimpleNamespace(flat=flat), geo_feature=geo, exposure=exp,
                                     model_parms=types.SimpleNamespace(train_stage=1))
    tr.sync_gradients()
    gathered = [torch.zeros_like(local) for _ in range(world)]
    dist.all_gather(gathered, local)
    expect = torch.stack(gathered).sum(0)
    bk = tr._bucket
    ok = (bk.numel() == 50 + 18 + 48 + 1 and torch.allclose(bk[:-1], expect, atol=1e-6) and float(bk[-1]) == 0.0
          and exp.grad.data_ptr() == bk[68:116].data_ptr() and tuple(exp.grad.shape) == (4, 3, 4))
    if rank == 0:
        out.put(bool(ok))
    dist.barrier()
    dist.destroy_process_group()


def test_gloo_bucket_carries_the_exposure_gradient():
    """[net.flat.grad | geo_feature.grad | exposure.grad | overflow flag], one all-reduce; the table's gradient becomes a bucket view."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 30100 + (os.getpid() % 400)
    procs = [ctx.Process(target=_bucket_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    assert q.get(timeout=10) is True


def test_fit_file_gains_the_exposure_key(tmp_path):
    """tools/fit_poses.py --exposure: the fitted rows under `exposure` [F,3,4] (identity past the fitted frames), other keys unchanged."""
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import fit_poses
    g = torch.Generator().manual_seed(0)
    d = dict(beta=torch.randn(1, 10, generator=g), body_pose=torch.randn(6, 72, generator=g), trans=torch.randn(6, 3, generator=g))
    src, dst = str(tmp_path / "smpl_parms.pth"), str(tmp_path / fit_poses.OUT_NAME)
    torch.save(d, src)
    pose, transl = torch.randn(4, 72, generator=g), torch.randn(4, 3, generator=g)
    E = torch.eye(3, 4).repeat(4, 1, 1) + 0.1 * torch.randn(4, 3, 4, generator=g)
    fit_poses.write_fit(src, dst, pose, transl, E)
    out = torch.load(dst, weights_only=False)
    assert set(out) == {"beta", "body_pose", "trans", "exposure"}
    assert torch.equal(out["exposure"][:4], E) and torch.equal(out["exposure"][4:], torch.eye(3, 4).repeat(2, 1, 1))
    assert torch.equal(out["body_pose"][:4], pose) and torch.equal(out["beta"], d["beta"])


@pytest.mark.parametrize("fused", [True, False], ids=["fused_adam", "torch_adam"])
@pytest.mark.parametrize("exposure", [False, True], ids=["no_exposure", "exposure"])
@pytest.mark.parametrize("world", [1, 2])
def test_each_gradient_is_divided_by_world_once(fused, exposure, world):
    """The trainer's per-step optimiser set-up: with FusedAdam the 1/world factor goes into the kernels (grad_scale) and the
    gradients stay as summed; with another optimiser the gradients are divided once; the exposure table's Adam takes 1/world in its
    rows whatever the main optimiser is, and the same skip flag."""
    from gaussianavatar_b200.optim import FusedAdam
    from gaussianavatar_b200.trainer import Stage1Trainer
    flat, geo = torch.nn.Parameter(torch.zeros(10)), torch.nn.Parameter(torch.zeros(2, 3))
    grads = [torch.full((10,), 4.0), torch.full((2, 3), 6.0)]
    flat.grad, geo.grad = grads[0].clone(), grads[1].clone()
    groups = [{"params": [flat], "lr": 1e-3}, {"params": [geo], "lr": 1e-3}]
    opt = FusedAdam(groups) if fused else torch.optim.Adam(groups)
    table = torch.nn.Parameter(identity_exposure(3, "cpu")) if exposure else None
    m = types.SimpleNamespace(optimizer=opt, exposure=table, exposure_optimizer=ExposureAdam(table, 10) if exposure else None)
    tr = Stage1Trainer.__new__(Stage1Trainer)
    tr.model, tr.world = m, world
    tr._skip = torch.ones(1, dtype=torch.int32)
    tr._prepare_updates()
    scale = 1.0 / world
    if fused:
        assert opt.grad_scale == scale and torch.equal(flat.grad, grads[0]) and torch.equal(geo.grad, grads[1])
        assert opt.skip_flag is (tr._skip if world > 1 else None)
    else:
        assert torch.equal(flat.grad, grads[0] * scale) and torch.equal(geo.grad, grads[1] * scale)
    if exposure:
        eo = m.exposure_optimizer
        assert eo.grad_scale == scale and eo.skip_flag is (tr._skip if world > 1 else None)
        assert float(eo._hyper_rows(1)[0, 6]) == scale


def test_schedule_spans_this_ranks_steps_and_undo_follows_launches():
    m = types.SimpleNamespace(exposure=torch.nn.Parameter(identity_exposure(5, "cpu")), opt_parms=types.SimpleNamespace(epochs=3),
                              train_dataset=list(range(16)), batch_size=2)
    m.exposure_schedule_steps = types.MethodType(AvatarModel.exposure_schedule_steps, m)
    assert AvatarModel.exposure_schedule_steps(m) == 24 and AvatarModel.exposure_schedule_steps(m, 2) == 12
    AvatarModel.exposure_setup(m, 2)
    opt = m.exposure_optimizer
    assert opt.total_steps == 12
    first = opt._hyper_rows(1).clone()
    opt.total_steps = 24                                   # the rows follow a new schedule length
    assert float(opt._hyper_rows(1)[6, 0]) > float(first[6, 0])
    opt.step_count = 5
    opt.step()                                             # no gradient: nothing launched, nothing to take back
    assert opt.step_count == 5 and not opt.launched
    opt.undo()
    assert opt.step_count == 5
    opt.launched = True                                    # as after a launched step
    opt.undo()
    assert opt.step_count == 4 and not opt.launched
