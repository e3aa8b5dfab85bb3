"""NCCL correctness of the data-parallel path (needs >= 2 GPUs; skipped otherwise): two ranks x 2 frames produce the same
averaged gradients and the same updated parameters as one rank x 4 frames (SURVEY.md §8e, App. C "DP" row).  Runs the
production configuration (TF32 decoder, frame streams).  Needs two GPUs: `python -m pytest tests/test_dist_gpu.py -m gpu`."""
import os
import tempfile

import pytest
import torch
import torch.multiprocessing as mp

pytestmark = [pytest.mark.gpu, pytest.mark.tf32]
SMALL = dict(N=4000, S=64, side=128, inp_posmap_size=32)


def _one_step(device, B, rank, world):
    from gaussianavatar_b200.trainer import Stage1Trainer
    from gaussianavatar_b200.workload import Stage1Workload
    wl = Stage1Workload(3, B, device=device, **SMALL)
    with torch.no_grad():
        sd = wl.model.net.state_dict(); sd["decoder.conv8N.bias"] = torch.tensor([-3.9]); wl.model.net.load_state_dict(sd, strict=False)
    wl.make_ground_truth()
    tr = Stage1Trainer(wl.model)
    batch = wl.device_batch(wl.frame_ids(0, rank, world))
    tr.step(batch, 5000, epoch=1)
    torch.cuda.synchronize()
    m = wl.model
    return dict(flat=m.net.flat.detach().cpu(), geo=m.geo_feature.detach().cpu(), g_flat=m.net.flat.grad.cpu() / world,
                g_geo=m.geo_feature.grad.cpu() / world)


def _worker(rank, world, port, path):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    os.environ.pop("GA_DECODER_FP32", None)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    out = _one_step(f"cuda:{rank}", 2, rank, world)
    torch.save(out, f"{path}.{rank}")
    dist.barrier(device_ids=[rank])
    dist.destroy_process_group()


def test_two_ranks_x2_frames_equal_one_rank_x4_frames():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ctx = mp.get_context("spawn")
    port = 29600 + (os.getpid() % 300)
    path = os.path.join(tempfile.mkdtemp(), "dp")
    procs = [ctx.Process(target=_worker, args=(r, 2, port, path)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(600)
        assert p.exitcode == 0
    ranks = [torch.load(f"{path}.{r}") for r in range(2)]
    one = _one_step("cuda:0", 4, 0, 1)

    def rel(a, b):
        return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()

    # both ranks hold the same all-reduced gradient and the same updated parameters
    assert torch.equal(ranks[0]["g_flat"], ranks[1]["g_flat"]) and torch.equal(ranks[0]["flat"], ranks[1]["flat"])
    assert torch.equal(ranks[0]["geo"], ranks[1]["geo"])
    # ... equal to the single-process B = 4 step up to float-atomics / summation-order noise
    assert rel(ranks[0]["g_flat"], one["g_flat"]) < 1e-3
    assert rel(ranks[0]["g_geo"], one["g_geo"]) < 1e-3
    # Adam's first step moves every parameter by ~lr * sign(g): identical except where the gradient is at round-off level
    for k, lr in (("flat", 3e-3), ("geo", 5e-4)):
        d = (ranks[0][k] - one[k]).abs()
        assert d.max().item() <= 2.001 * lr
        assert (d > 1e-2 * lr).float().mean().item() < 0.01
