#!/usr/bin/env python
"""Headline benchmark: stage-1 train-step FPS at 200k Gaussians / 1024^2 (BASELINE.json configs[2]; configs[3] semantics
for N > 1: every rank renders its own frames, one all-reduce of the shared feature-net gradients).

    python bench.py --gpus 1 --steps 20 --warmup 3
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P bench.py --gpus N ...
    python bench.py --impl reference ...      # the CPU arm: the reference's algorithm (oracle port) on the host cores
    python bench.py ... --dump-outputs DIR    # also write what the last timed step computed, as DIR/<name>.npy

One "step" = SMPL pose -> feature net -> LBS -> rasterize B frames -> L1+SSIM loss -> backward -> Adam (train.py:66-97).
Rank 0 prints ONE JSON line.  Timing: CUDA events on the launching stream, barrier + synchronize on both sides, max over
ranks.  `value` has inputs resident in HBM; `e2e` goes through the public API with HOST (pinned) batches, the H2D copy
and the loss read-back inside the timed region.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

METRIC = "train_step_fps_200k_gaussians_1024sq"
UNIT = "frames/s"


# ---------------------------------------------------------------------------------------------------------------------
class ClockSampler:
    """SM clock / throttle reasons sampled DURING the timed region, in-process through NVML (`pynvml`, three cheap queries every
    50 ms from a daemon thread).  An external `nvidia-smi -lms 100` loop can stall kernel launches while it runs; it is only the
    fallback when pynvml is unavailable."""
    REASONS = (("hw_slowdown", 0x8), ("hw_thermal_slowdown", 0x40), ("sw_thermal_slowdown", 0x20), ("sw_power_cap", 0x4))

    def __init__(self, gpu_index: int):
        self.gpu, self.rows, self._p, self._stop, self._thr, self._h = gpu_index, [], None, False, None, None

    def start(self):
        try:
            import pynvml
            pynvml.nvmlInit()
            vis = os.environ.get("CUDA_VISIBLE_DEVICES")
            phys = int(vis.split(",")[self.gpu]) if vis and all(v.strip().isdigit() for v in vis.split(",")) else self.gpu
            self._h = pynvml.nvmlDeviceGetHandleByIndex(phys)
            self._nv = pynvml
            self._max_sm = pynvml.nvmlDeviceGetMaxClockInfo(self._h, pynvml.NVML_CLOCK_SM)      # static, and slow to query (4 ms avg, 25 ms max under load)

            def loop():
                nv, h = self._nv, self._h
                while not self._stop:
                    try:
                        sm = nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM)
                        mx = self._max_sm
                        rs = nv.nvmlDeviceGetCurrentClocksEventReasons(h) if hasattr(nv, "nvmlDeviceGetCurrentClocksEventReasons") \
                            else nv.nvmlDeviceGetCurrentClocksThrottleReasons(h)
                        self.rows.append((float(sm), float(mx), int(rs)))
                    except Exception:
                        pass
                    time.sleep(0.05)
            self._thr = threading.Thread(target=loop, daemon=True)
            self._thr.start()
            return
        except Exception:
            self._h = None
        try:
            q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
                 "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
            self._p = subprocess.Popen(["nvidia-smi", f"--id={self.gpu}", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-lms", "250"],
                                       stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self._p = None

    def _read(self):
        for line in self._p.stdout:
            c = [x.strip() for x in line.split(",")]
            try:
                bits = sum(bit for (name, bit), v in zip(self.REASONS, c[2:6]) if v.lower().startswith("active"))
                self.rows.append((float(c[0]), float(c[1]), bits))
            except (ValueError, IndexError):
                continue

    def stop(self) -> dict:
        self._stop = True
        if self._thr is not None:
            self._thr.join(timeout=1.0)
        if self._p is not None:
            time.sleep(0.3)
            self._p.terminate()
        if self._thr is None and self._p is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["clock sampling unavailable"]}
        sm = [r[0] for r in self.rows]
        mx = [r[1] for r in self.rows]
        reasons = sorted({name for r in self.rows for name, bit in self.REASONS if r[2] & bit})
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None, "reasons": reasons,
                "samples": len(sm), "how": "pynvml thread, 50 ms" if self._thr is not None else "nvidia-smi -lms 250"}


def measured_peaks() -> dict:
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        d["_source"] = "measured (MEASURED_PEAKS.json)"
        return d
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "bf16_tflops_sustained": 989.0, "_source": "H100 SXM data sheet (700 W), not measured"}


# ---------------------------------------------------------------------------------------------------------------------
# CPU arm: the reference's algorithm for the same step, restated in oracle/ (the reference itself cannot travel to the GPU
# box: it needs /root/reference plus CUDA-only / un-installed dependencies, SURVEY.md §0).  One step = ONE frame at full size.
# ---------------------------------------------------------------------------------------------------------------------
def cpu_reference_step_factory(config: int):
    import math
    import numpy as np
    import torch
    from gaussianavatar_b200 import synthetic as syn
    from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, TEST_POSE_K, make_camera, scaled_intrinsics
    from gaussianavatar_b200.workload import load_poses
    from oracle import avatar_oracle as ao
    from oracle import raster_oracle as ro

    torch.set_num_threads(os.cpu_count() or 1)
    N, S, side = syn.CONFIGS[config]
    a = syn.make_avatar_assets(N, S, seed=0)
    pose, transl, _ = load_poses(32)
    cam = make_camera(scaled_intrinsics(TEST_POSE_K, side), TEST_POSE_EXTRINSIC, side, side)
    p = {k: v.clone().requires_grad_(True) for k, v in ao.seeded_pop_params(0).items()}
    with torch.no_grad():
        p["decoder.conv8N.bias"].fill_(-5.3)
        for k in p:
            if ".bn" in k:
                p[k].copy_(torch.ones_like(p[k]) if k.endswith("weight") else torch.zeros_like(p[k]))
    geo = (torch.randn(1, 64, 128, 128, generator=torch.Generator().manual_seed(0)) * 0.01).requires_grad_(True)
    opt = torch.optim.Adam([{"params": list(p.values()), "lr": 3e-3}, {"params": [geo], "lr": 5e-4}])
    inv_cano = torch.linalg.inv(a.cano_joint_mats)[None]
    rots = np.zeros((N, 4), np.float32); rots[:, 0] = 1
    gt = torch.rand(1, 3, side, side, generator=torch.Generator().manual_seed(2))
    tanx, tany = math.tan(cam.FovX / 2), math.tan(cam.FovY / 2)

    def step(i: int):
        f = i % pose.shape[0]
        ps = pose[f:f + 1].clone().requires_grad_(True)
        tr = transl[f:f + 1].clone().requires_grad_(True)
        res, sc, shs = ao.pop_forward(p, geo, S, B=1)
        C = ao.cano2live(ao.smpl_joint_transforms(a.rest_joints, ps, tr), inv_cano)
        o = ao.assemble_and_skin(res, sc, shs, a.valid_idx, a.query_points[None], a.query_lbs[None], C, 5000, geo_feature=geo)
        means, colors, scales = o["means3D"][0], o["colors"][0], o["scales"][0]
        r = ro.forward(means.detach().numpy(), colors.detach().numpy(), np.ones(N, np.float32), scales.detach().numpy(), rots,
                       np.ones(3, np.float32), cam.world_view_transform.numpy(), cam.full_proj_transform.numpy(), tanx, tany, side, side)
        img = torch.tensor(r.image, dtype=torch.float32)[None].requires_grad_(True)
        loss_img = 0.8 * ao.l1_loss_w(img, gt) + 0.2 * (1.0 - ao.ssim(img, gt))
        loss_img.backward()
        gb = r.backward(img.grad[0].numpy())
        opt.zero_grad()
        reg = 3e-2 * o["scale_loss"] + 10.0 * o["offset_loss"] + o["geo_loss"]
        torch.autograd.backward([means, colors, scales, reg],
                                [torch.tensor(gb["d_means3D"], dtype=torch.float32), torch.tensor(gb["d_colors"], dtype=torch.float32),
                                 torch.tensor(gb["d_scales"], dtype=torch.float32), torch.ones(())])
        opt.step()
        r.close()
        return float(loss_img.detach())

    return step, dict(N=N, S=S, side=side)


def run_reference_arm(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return 0
    import torch
    step, dims = cpu_reference_step_factory(args.config)
    cores = os.cpu_count() or 1
    t0 = time.perf_counter(); step(0); t_first = time.perf_counter() - t0      # first call also warms the allocator
    budget_s = 200.0
    warm = max(0, min(args.warmup, int(0.25 * budget_s / max(t_first, 1e-3)) - 1))
    for i in range(warm):
        step(1 + i)
    steps = max(1, min(args.steps, int(0.75 * budget_s / max(t_first, 1e-3))))
    t0 = time.perf_counter()
    for i in range(steps):
        step(1 + warm + i)
    dt = time.perf_counter() - t0
    fps = steps / dt
    sample = (f"{steps} of the requested {args.steps} steps executed (bounded to ~{budget_s:.0f}s of CPU work); one step = ONE "
              f"{dims['N']}-Gaussian / {dims['side']}^2 frame: feature net + SMPL + LBS (torch CPU, {torch.get_num_threads()} threads) + C/OpenMP "
              f"rasterizer fwd+bwd + L1/SSIM + Adam")
    line = {"impl": "reference", "metric": METRIC, "value": fps, "unit": UNIT, "n_gpus": args.gpus, "steps": steps, "warmup": warm,
            "ms_per_step": 1e3 * dt / steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
            "data": "synthetic", "config": {"workload": f"config{args.config}: {dims['N']} Gaussians, {dims['side']}x{dims['side']}, stage-1 train step, 1 frame/step on host cores"},
            "cpu_baseline": {"value": fps, "unit": UNIT, "cores": cores, "kind": "port", "sample": sample},
            "e2e": {"value": fps, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}, "gpu_launches": 0}
    print(json.dumps(line), flush=True)
    return 0


# ---------------------------------------------------------------------------------------------------------------------
def dump_outputs(out_dir: str, trainer, loss, batch, iteration: int, start_params) -> None:
    """What the last timed step computed from the seeded parameters: its loss (float64, [1]), the gradients it left on the feature
    net (`net_grad`, the flat buffer) and on geo_feature (`geo_feature_grad`), and the frames it rendered (`images`, [B,3,H,W]; the
    step keeps no copy of them, so the same forward runs again, untimed, on the step's inputs).  Gradients carry the run-to-run
    scatter of float-atomic reduction order: compare them with a tolerance."""
    import numpy as np
    import torch
    m = trainer.model
    os.makedirs(out_dir, exist_ok=True)
    torch.cuda.synchronize()
    np.save(os.path.join(out_dir, "loss.npy"), loss.detach().double().reshape(1).cpu().numpy())
    np.save(os.path.join(out_dir, "net_grad.npy"), m.net.flat.grad.detach().float().cpu().numpy())
    np.save(os.path.join(out_dir, "geo_feature_grad.npy"), m.geo_feature.grad.detach().float().cpu().numpy())
    with torch.no_grad():
        m.net.flat.copy_(start_params[0])
        m.geo_feature.copy_(start_params[1])
        _, image = trainer.loss(batch, iteration, epoch=1)
    np.save(os.path.join(out_dir, "images.npy"), image.detach().float().cpu().numpy())


def algorithmic_cost(N, S, side, R, B):
    """Per-launch algorithmic bytes / flops of the kernels we report rooflines for (DESIGN.md §6; SURVEY.md §8d)."""
    M = S * S
    T = ((side + 15) // 16) ** 2
    bits = 32 + max(1, (T - 1).bit_length())
    passes = (bits + 7) // 8
    raster_fwd_bytes = N * (56 + 40 + 8) + R * (12 + 8 + passes * 24 + 8 + 40) + side * side * 20 + T * 8
    return dict(
        raster_fwd_bytes=raster_fwd_bytes,
        mlp_layer_fwd_flops=2.0 * M * 128 * 128, mlp_layer_fwd_bytes=2.0 * M * 128 * 4,
        mlp_fwd_flops=363264.0 * M, mlp_fwdbwd_flops=3 * 363264.0 * M,
        lbs_bytes=N * (96 + 12 + 32 + 4) + B * N * 36)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--config", type=int, default=3, help="BASELINE.md §4 config number (3 = 200k / 1024^2 stage-1 loop)")
    ap.add_argument("--frames-per-gpu", type=int, default=2, help="frames per step and GPU (reference batch_size=2)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-extra", action="store_true", help="skip the config-4 (1 frame/GPU) and config-5 (novel-pose) side measurements")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last one computed (loss, gradients, rendered frames) as DIR/<name>.npy; "
                         "that step starts from the seeded initial parameters, so its inputs are the same on every run")
    args = ap.parse_args()
    args.warmup = max(3, args.warmup) if args.impl == "ours" else args.warmup
    if args.impl == "reference":
        return run_reference_arm(args)

    # stdout carries exactly ONE JSON line: anything else a library prints there (NCCL's version banner, ...) goes to stderr
    real_stdout = os.dup(1)
    os.dup2(2, 1)

    import torch
    import torch.distributed as dist
    from gaussianavatar_b200 import _lib
    from gaussianavatar_b200.trainer import Stage1Trainer
    from gaussianavatar_b200.workload import Stage1Workload, to_cuda

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device (there is no CPU fallback for the product path)")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    B = args.frames_per_gpu
    torch.cuda.set_stream(torch.cuda.Stream(device=dev))      # everything below runs on one non-default stream (graph capture needs that)

    wl = Stage1Workload(args.config, B, device=dev)
    wl.make_ground_truth()
    trainer = Stage1Trainer(wl.model, fused_adam=True)
    # The backward accumulates per-Gaussian and per-weight gradients with float atomics whose order varies from run to run, and Adam
    # carries that into the parameters of every later step.  With --dump-outputs the last timed step therefore starts from the seeded
    # initial parameters (two small device copies inside the timed region), so that its inputs are identical on every run.
    start_params = (wl.model.net.flat.detach().clone(), wl.model.geo_feature.detach().clone()) if args.dump_outputs else None
    iteration0 = 5000      # >= 1000: no scale ramp (SURVEY.md §8d)

    def barrier():
        if world > 1:
            dist.barrier(device_ids=[local])
        torch.cuda.synchronize()

    # every distinct batch of the frame pool is built on the device once, before anything is timed: "inputs already resident in HBM"
    dev_batches = {}
    for i in range(wl.num_frames):
        ids = tuple(wl.frame_ids(i, rank, world))
        if ids not in dev_batches:
            dev_batches[ids] = wl.device_batch(list(ids))
    torch.cuda.synchronize()

    _sleep_ms = float(os.environ.get("GA_VALUE_SLEEP_MS", "0"))       # experiment hook (never set by the driver)
    if os.environ.get("GA_VALUE_CLONE") == "1":
        for b in dev_batches.values():
            b["original_image"] = b["original_image"].clone()

    def run_value(n, start, restore_last=False):
        loss = None
        t0 = time.perf_counter()
        trainer.host_wait_s = trainer.host_enqueue_s = 0.0
        diag_ev = [] if (os.environ.get("GA_BENCH_DIAG") == "1" and rank == 0 and n > 2) else None
        for i in range(n):
            batch = dev_batches[tuple(wl.frame_ids(start + i, rank, world))]
            if _sleep_ms:
                time.sleep(_sleep_ms * 1e-3)
            if restore_last and i == n - 1:
                with torch.no_grad():
                    wl.model.net.flat.copy_(start_params[0])
                    wl.model.geo_feature.copy_(start_params[1])
            loss = trainer.step(batch, iteration0 + start + i, epoch=1)
            if diag_ev is not None:
                e = torch.cuda.Event(enable_timing=True); e.record(); diag_ev.append(e)
        if os.environ.get("GA_BENCH_DIAG") == "1" and rank == 0 and n > 2:
            print(f"value diag: host wait-for-status {1e3 * trainer.host_wait_s / n:.2f} ms/step, enqueue {1e3 * trainer.host_enqueue_s / n:.2f} ms/step", file=sys.stderr, flush=True)
        trainer.host_wait_s = trainer.host_enqueue_s = 0.0
        if diag_ev:
            torch.cuda.synchronize()
            print("value diag per-step ms:", " ".join(f"{a.elapsed_time(b):.2f}" for a, b in zip(diag_ev[:-1], diag_ev[1:])), file=sys.stderr, flush=True)
        if os.environ.get("GA_BENCH_DIAG") == "1" and rank == 0 and n > 2:
            print(f"value diag (rank 0): host enqueue loop {1e3 * (time.perf_counter() - t0) / n:.2f} ms per step", file=sys.stderr, flush=True)
        return loss

    h2d_bytes = [0]
    copy_stream = torch.cuda.Stream(device=dev)
    loss_host = [torch.zeros((), dtype=torch.float32).pin_memory() for _ in range(4)]

    def run_e2e(n, start):
        """Public-API loop with HOST batches: the next batch's H2D copy (pinned -> device, side stream) is prefetched while
        the current step computes, as a DataLoader with pin_memory would; every step's loss is copied back to pinned host
        memory and read two steps later (so the read-back never stalls the enqueue).  All of it is inside the timed region."""
        last = 0.0
        lag = int(os.environ.get("GA_E2E_LAG", "2"))           # the loss of step i is read when step i + lag has been enqueued
        diag = os.environ.get("GA_BENCH_DIAG") == "1" and rank == 0
        t_fetch = t_step = t_wait = 0.0
        pending = []

        def fetch(i):
            hb = wl.host_batch(wl.frame_ids(start + i, rank, world))
            with torch.cuda.stream(copy_stream):
                b, nb = to_cuda(hb, dev)
                ev = torch.cuda.Event(); ev.record(copy_stream)
            h2d_bytes[0] = nb
            return b, ev

        nxt = fetch(0)
        for i in range(n):
            t0 = time.perf_counter()
            batch, ev = nxt
            torch.cuda.current_stream().wait_event(ev)
            for t in batch.values():
                if torch.is_tensor(t):
                    t.record_stream(torch.cuda.current_stream())
            if i + 1 < n:
                nxt = fetch(i + 1)
            t1 = time.perf_counter()
            loss = trainer.step(batch, iteration0 + start + i, epoch=1)
            buf = loss_host[i % len(loss_host)]
            buf.copy_(loss.detach(), non_blocking=True)        # device -> host read of the step's result (train.py:101)
            done = torch.cuda.Event(); done.record()
            t2 = time.perf_counter()
            pending.append((buf, done))
            if len(pending) > lag:
                b0, d0 = pending.pop(0)
                d0.synchronize(); last = float(b0)
            t3 = time.perf_counter()
            t_fetch += t1 - t0; t_step += t2 - t1; t_wait += t3 - t2
        for b0, d0 in pending:
            d0.synchronize(); last = float(b0)
        if diag and n > 2:
            print(f"e2e diag (rank 0, per step): fetch {1e3 * t_fetch / n:.2f} ms, enqueue {1e3 * t_step / n:.2f} ms, wait {1e3 * t_wait / n:.2f} ms", file=sys.stderr, flush=True)
        return last

    last_out = [None]

    def timed(fn, n, start):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        last_out[0] = fn(n, start)
        e1.record()
        barrier()
        ms = e0.elapsed_time(e1)
        if world > 1:
            t = torch.tensor([ms], device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms = float(t.item())
        return ms

    # ---- launch-mode calibration (untimed, part of the warm-up) ----------------------------------------------------------
    # The step runs either as ~120 eager launches or as ONE replayed CUDA graph (+ the optimizer launches).  Which is faster depends
    # on the machine: a replayed graph can cost the device more per step than back-to-back stream launches, but a slow host cannot
    # keep 120 launches per step ahead of the GPU.  Both compute the same thing (tests/test_train_gpu.py::test_graphed_step_matches_eager_step),
    # so measure and pick.
    calib = None
    if os.environ.get("GA_STEP_GRAPH") is None and world == 1:
        def ms_per_step(n, start):
            torch.cuda.synchronize(); t = time.perf_counter()
            run_value(n, start)
            trainer.finish(); torch.cuda.synchronize()
            return 1e3 * (time.perf_counter() - t) / n
        trainer.use_graph = False
        run_value(3, 0)
        eager_ms = ms_per_step(10, 3)
        trainer.use_graph = True
        run_value(3, 13)                      # captures the graph
        graph_ms = ms_per_step(10, 16)
        trainer.use_graph = graph_ms < eager_ms
        calib = {"eager_ms_per_step": round(eager_ms, 3), "graph_ms_per_step": round(graph_ms, 3), "chosen": "graph" if trainer.use_graph else "eager"}

    # ---- warm-up, then the timed region (inputs resident in HBM) -------------------------------------------------------
    clocks = ClockSampler(local)
    if rank == 0:
        clocks.start()                     # nvidia-smi needs ~1 s to start sampling: begin before the warm-up steps
    run_value(args.warmup, 0)
    clocks.rows.clear()                    # keep only samples taken during the timed region
    l0 = _lib.launch_count() + trainer.replayed_launches
    ms_value = timed(lambda n, start: run_value(n, start, restore_last=start_params is not None), args.steps, args.warmup)
    launches = _lib.launch_count() + trainer.replayed_launches - l0      # eager launches + the kernels inside the replayed step graphs
    clk = clocks.stop() if rank == 0 else {}
    fps = world * B * args.steps / (ms_value * 1e-3)
    if args.dump_outputs:
        trainer.finish()                   # settle the last step: it is run again if its binning buffer overflowed
        if rank == 0:
            last = args.warmup + args.steps - 1
            dump_outputs(args.dump_outputs, trainer, last_out[0], dev_batches[tuple(wl.frame_ids(last, rank, world))], iteration0 + last,
                         start_params)

    # ---- end to end through the public API with host batches ----------------------------------------------------------
    e2e = None
    if not args.no_e2e:
        run_e2e(2, args.warmup + args.steps)
        ms_e2e = timed(run_e2e, args.steps, args.warmup + args.steps + 2)
        e2e = {"value": world * B * args.steps / (ms_e2e * 1e-3), "unit": UNIT, "h2d_bytes_per_step": int(h2d_bytes[0]),
               "d2h_bytes_per_step": 4, "ms_per_step": ms_e2e / args.steps}

    # ---- per-kernel CUDA-event pass (same steps again, rank-local) -> roofline ---------------------------------------
    trainer.finish()
    graph_mode, trainer.use_graph = trainer.use_graph, False      # per-kernel events need eager launches (a replayed graph carries none)
    _lib.profile(True)
    _lib.profile_report()
    nprof = min(args.steps, 5)
    run_value(nprof, 2 * args.warmup + 2 * args.steps + 4)
    trainer.finish()
    prof = _lib.profile_report()
    _lib.profile(False)
    trainer.use_graph = graph_mode
    per_step = {k: (n / nprof, ms / nprof) for k, (n, ms) in prof.items()}
    total_kernel_ms = sum(ms for _, ms in per_step.values())

    peaks = measured_peaks()
    # the rasterizer's instance count for the cost model (one forward outside the timed region)
    with torch.no_grad():
        from gaussianavatar_b200.rasterizer import GaussianRasterizationSettings, rasterize_forward
        import math
        bt = wl.device_batch(wl.frame_ids(0, rank, world))
        means, scales, colors, _ = wl.model._posed_gaussians(bt["pose_idx"], iteration0)
        c = wl._cam_dev
        rs = GaussianRasterizationSettings(c.height, c.width, math.tan(c.FovX / 2), math.tan(c.FovY / 2), wl.model.background, 1.0,
                                           c.world_view_transform, c.full_proj_transform, 0, c.camera_center, False, False)
        _, _, rctx = rasterize_forward(means[0], colors[0], wl.model.fix_opacity, scales[0], wl.model.fix_rotation, rs)
        R = rctx.num_rendered
    cost = algorithmic_cost(wl.N, wl.S, wl.side, R, B)

    def kms(*names):
        return sum(per_step[n][1] for n in names if n in per_step)

    M = wl.S * wl.S
    plane = 4.0 * M * 128                      # bytes of one [M,128] fp32 activation / gradient plane
    feat = 4.0 * M * 72
    # algorithmic HBM bytes of ALL launches of a kernel in one step (DESIGN.md §4): what must cross HBM at least once
    tc_bwd_bytes = 10 * (4 * plane) + (2 * plane + 2 * feat) + (2 * plane + 3 * feat)     # 10 full layers + the two 72-wide input layers
    tc_fwd_bytes = 10 * (2 * plane) + (feat + plane) + (feat + plane) + (3 * plane - 2 * plane)   # 9 full + L1 + L5a + L5b (accumulating: +1 plane read)
    tc_flops = 3 * 363264.0 * M
    mlp_ms = kms("mlp_tc_fwd", "mlp_tc_bwd") + sum(v[1] for k, v in per_step.items() if k.startswith("mlp_") and not k.startswith("mlp_tc"))
    dominant = max(per_step.items(), key=lambda kv: kv[1][1])[0] if per_step else None

    def hbm_roof(name, nbytes, label):
        ms = kms(name)
        n = per_step[name][0] if name in per_step else 0
        gbs = nbytes / (ms * 1e-3) / 1e9 if ms > 0 else None
        return {"kernel": label, "bound": "hbm", "achieved": gbs, "peak": peaks["hbm_gbs"], "unit": "GB/s",
                "frac": gbs / peaks["hbm_gbs"] if gbs else None, "traffic": None,
                "launches_per_step": n, "ms_per_step": ms,
                "avg_launch_ms": ms / n if n else None, "algorithmic_bytes_per_step": nbytes,
                "share_of_kernel_time": ms / total_kernel_ms if total_kernel_ms else None, "peak_source": peaks["_source"]}

    if dominant in ("mlp_tc_bwd", "mlp_tc_fwd"):
        roofline = hbm_roof("mlp_tc_bwd", tc_bwd_bytes, "tc_bwd_kernel (fused dgrad+wgrad of one decoder layer, TF32 tensor cores): all launches of one step")
        roofline["tensor_tflops_all_mlp"] = tc_flops / (mlp_ms * 1e-3) / 1e12 if mlp_ms > 0 else None
    else:
        mlp_tflops = tc_flops / (mlp_ms * 1e-3) / 1e12 if mlp_ms > 0 else None
        tf32_peak = peaks["bf16_tflops_sustained"] / 2.0
        roofline = {"kernel": "decoder MLP GEMMs (strict-FP32 CUDA-core path)", "bound": "tensor", "achieved": mlp_tflops, "peak": tf32_peak,
                    "unit": "TFLOP/s", "frac": (mlp_tflops / tf32_peak) if mlp_tflops else None, "traffic": None,
                    "peak_source": peaks["_source"] + "; tf32 dense = 1/2 x bf16 sustained", "ms_per_step": mlp_ms,
                    "share_of_kernel_time": mlp_ms / total_kernel_ms if total_kernel_ms else None}
    fwd_roofline = hbm_roof("mlp_tc_fwd", tc_fwd_bytes, "tc_fwd_kernel (one decoder layer forward, TF32 tensor cores): all launches of one step")
    raster_fwd_names = ["preprocess_fwd_kernel", "tile_scan_kernel", "bucket_scatter_kernel", "tile_sort_kernel", "render_fwd_kernel"]
    raster_fwd_ms = kms(*raster_fwd_names) / B          # per frame
    raster_bwd_ms = kms("render_bwd_kernel", "preprocess_bwd_kernel") / B
    raster_gbs = cost["raster_fwd_bytes"] / (raster_fwd_ms * 1e-3) / 1e9 if raster_fwd_ms > 0 else None
    raster_roofline = {"kernel": "rasterizer forward K1-K6, per frame (bytes: SURVEY.md §8d model of upstream's pipeline)", "bound": "hbm", "achieved": raster_gbs,
                       "peak": peaks["hbm_gbs"], "unit": "GB/s", "frac": raster_gbs / peaks["hbm_gbs"] if raster_gbs else None, "traffic": None,
                       "algorithmic_bytes": cost["raster_fwd_bytes"], "ms_per_frame": raster_fwd_ms, "num_rendered": R,
                       "bwd_ms_per_frame": raster_bwd_ms, "peak_source": peaks["_source"]}
    # per stage (SURVEY.md §8d): the streaming stages against HBM with THIS pipeline's algorithmic bytes per frame (DESIGN.md §4 table),
    # the compositing kernels as (pixel x list-entry) interactions per second — they are instruction / latency bound, not HBM bound
    T_tiles = ((wl.side + 15) // 16) ** 2
    stage_bytes = {"preprocess_fwd_kernel": wl.N * 100 + R * 4, "tile_scan_kernel": T_tiles * 28, "bucket_scatter_kernel": wl.N * 12 + R * 8,
                   "tile_sort_kernel": R * 100, "preprocess_bwd_kernel": wl.N * 150}
    raster_stages = {}
    for k, nbytes in stage_bytes.items():
        ms = kms(k) / B
        gbs = nbytes / (ms * 1e-3) / 1e9 if ms > 0 else None
        raster_stages[k] = {"bound": "hbm", "ms_per_frame": ms, "algorithmic_bytes": nbytes, "achieved_gbs": gbs,
                            "frac": gbs / peaks["hbm_gbs"] if gbs else None}
    try:
        pv = plan_views = wl.model._last_plan.views() if getattr(wl.model, "_last_plan", None) is not None else None
        inter = float(sum(int(v["n_contrib"].to(torch.int64).sum()) for v in pv)) / max(1, len(pv)) if pv else None
    except Exception:
        inter = None
    for k in ("render_fwd_kernel", "render_bwd_kernel"):
        ms = kms(k) / B
        raster_stages[k] = {"bound": "instruction issue / latency", "ms_per_frame": ms, "pixel_entry_interactions": inter,
                            "ginteractions_per_s": inter / (ms * 1e-3) / 1e9 if (inter and ms > 0) else None}
    raster_roofline["stages"] = raster_stages

    # ---- BASELINE configs 4 and 5 next to the headline (VERDICT r1 item 6) ---------------------------------------------------
    extra = {}
    step_graph_used = bool(trainer.use_graph and trainer._graphs)
    if not args.no_extra:
        trainer.finish()
        del trainer
        wl.model._raster_plans = {}
        torch.cuda.empty_cache()

        def timed_loop(fn, n):
            barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); fn(n); e1.record()
            barrier()
            ms = e0.elapsed_time(e1)
            if world > 1:
                t = torch.tensor([ms], device=dev)
                dist.all_reduce(t, op=dist.ReduceOp.MAX)
                ms = float(t.item())
            return ms

        # config 4 literally: ONE pose per GPU per step (8 poses / step over 8 GPUs), the decoder no longer amortised over 2 frames
        wl4 = Stage1Workload(4, 1, device=dev)
        wl4.make_ground_truth()
        tr4 = Stage1Trainer(wl4.model, fused_adam=True)

        batches4 = {}
        for i in range(wl4.num_frames):
            ids = tuple(wl4.frame_ids(i, rank, world))
            if ids not in batches4:
                batches4[ids] = wl4.device_batch(list(ids))
        torch.cuda.synchronize()

        def run4(n, start=[0]):
            for i in range(n):
                tr4.step(batches4[tuple(wl4.frame_ids(start[0] + i, rank, world))], iteration0 + start[0] + i, epoch=1)
            start[0] += n
        run4(max(3, args.warmup))
        ms4 = timed_loop(run4, args.steps)
        tr4.finish()
        extra["config4_one_pose_per_gpu"] = {"value": world * args.steps / (ms4 * 1e-3), "unit": UNIT, "ms_per_step": ms4 / args.steps,
                                             "global_batch": world, "workload": "config4: 200000 Gaussians, 1024x1024, stage-1 train step, 1 frame/GPU/step"}
        del tr4, wl4
        torch.cuda.empty_cache()

        # config 5: novel-pose rendering (render_novel_pose.py:12-33 -> AvatarModel.render_free_stage1), forward only, 500k Gaussians / 2048^2;
        # an inference model evaluates the frame-invariant stage-1 net once (cached), per frame: SMPL -> LBS -> rasterizer
        from gaussianavatar_b200.workload import load_poses
        wl5 = Stage1Workload(5, 1, device=dev)
        m5 = wl5.model
        m5.cache_decoder = True
        poses5, transl5, _ = load_poses(32)
        pin = lambda t: t.contiguous().pin_memory()
        host_frames = [(pin(poses5[i:i + 1]), pin(transl5[i:i + 1])) for i in range(poses5.shape[0])]
        dev_frames = [(p.to(dev), t.to(dev)) for p, t in host_frames]
        cam5 = wl5.camera_fields(1)
        idx0 = torch.zeros(1, dtype=torch.long, device=dev)
        out_host = torch.empty(1, 3, wl5.side, wl5.side).pin_memory()
        m5.defer_raster_check = True

        def run5(n, start=[0], e2e=False):
            with torch.no_grad():
                for i in range(n):
                    f = (start[0] + i * world + rank) % len(dev_frames)
                    if e2e:
                        p, t = host_frames[f][0].to(dev, non_blocking=True), host_frames[f][1].to(dev, non_blocking=True)
                    else:
                        p, t = dev_frames[f]
                    img = m5.render_free_stage1(dict(pose_idx=idx0, pose_data=p, transl_data=t, **cam5), 59400)
                    if e2e:
                        out_host.copy_(img, non_blocking=True)       # the frame goes back to the host (render_novel_pose.py:32 saves it)
            start[0] += n * world
            return m5.raster_ok(wait=True)               # False: the binning buffer overflowed (and has been grown)
        run5(4); run5(4)
        assert run5(4), "binning buffer still overflowing after two warm-up rounds"
        n5 = max(args.steps, 20)
        ok5 = []
        ms5 = timed_loop(lambda n: ok5.append(run5(n)), n5)
        ms5e = timed_loop(lambda n: ok5.append(run5(n, e2e=True)), n5)
        assert all(ok5), "binning buffer overflow during the timed novel-pose loop"
        plan5 = m5._last_plan
        extra["config5_novel_pose"] = {"value": world * n5 / (ms5 * 1e-3), "unit": UNIT, "ms_per_frame": ms5 / n5,
                                       "e2e": {"value": world * n5 / (ms5e * 1e-3), "unit": UNIT, "ms_per_frame": ms5e / n5,
                                               "h2d_bytes_per_frame": 300, "d2h_bytes_per_frame": int(out_host.numel() * 4)},
                                       "num_rendered": int(plan5.status_host[0]), "frames": n5,
                                       "workload": f"config5: {wl5.N} Gaussians, UV {wl5.S}^2, {wl5.side}x{wl5.side}, novel-pose forward "
                                                   "(decoder output cached across frames), 1 frame per GPU at a time"}
        # per-stage kernel times of one novel-pose frame
        _lib.profile(True); _lib.profile_report()
        run5(5)
        torch.cuda.synchronize()
        p5 = _lib.profile_report(); _lib.profile(False)
        extra["config5_novel_pose"]["kernel_ms_per_frame"] = {k: round(ms / 5, 4) for k, (n, ms) in sorted(p5.items(), key=lambda kv: -kv[1][1])}
        T5 = ((wl5.side + 15) // 16) ** 2
        R5 = int(plan5.status_host[0])
        # algorithmic HBM bytes of the streaming stages of ONE frame (DESIGN.md §4): K1 reads 56 B / writes 44 B per Gaussian (+4 B per
        # instance of tile-count atomics), K3 reads 12 B per Gaussian and writes 8 B per instance, K4 reads 8 B, gathers 40 B and writes
        # 52 B per instance, K6 streams 48 B per instance per sub-tile pass (L1/L2 resident) and writes 36 B per pixel
        stage_bytes = {"preprocess_fwd_kernel": wl5.N * 100 + R5 * 4, "bucket_scatter_kernel": wl5.N * 12 + R5 * 8,
                       "tile_sort_kernel": R5 * 100, "tile_scan_kernel": T5 * 28}
        extra["config5_novel_pose"]["stage_rooflines"] = {
            k: {"algorithmic_bytes": b, "achieved_gbs": (b / (p5[k][1] / 5 * 1e-3) / 1e9) if k in p5 and p5[k][1] > 0 else None,
                "frac_of_hbm": (b / (p5[k][1] / 5 * 1e-3) / 1e9 / peaks["hbm_gbs"]) if k in p5 and p5[k][1] > 0 else None}
            for k, b in stage_bytes.items()}
        del wl5, m5
        torch.cuda.empty_cache()

    cpu_baseline = None
    if rank == 0 and not args.no_cpu_baseline:
        torch.cuda.synchronize()
        warm, _ = cpu_reference_step_factory(1)            # small config: warms torch's CPU kernels / thread pool only
        warm(0)
        step, dims = cpu_reference_step_factory(args.config)
        t0 = time.perf_counter()
        step(0)
        dt = time.perf_counter() - t0
        cpu_baseline = {"value": 1.0 / dt, "unit": UNIT, "cores": os.cpu_count(), "kind": "port",
                        "sample": f"1 full-size single-frame train step of the oracle port (torch CPU all cores + C/OpenMP rasterizer, fwd+bwd+Adam), {dt:.1f}s"}

    if rank == 0:
        line = {"metric": METRIC, "value": fps, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
                "ms_per_step": ms_value / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
                "dtype": "tf32" if wl.model.net.tensor_cores else "f32", "data": "synthetic",
                "config": {"workload": f"config{args.config}: {wl.N} Gaussians, UV {wl.S}^2, {wl.side}x{wl.side}, stage-1 train step (feature net + "
                                       f"L1/SSIM), {B} frames/GPU/step, global batch {B * world}", "poses": wl.pose_source,
                           "l2_policy": "inputs and activations (>1.5 GB/step) exceed the 50 MB L2; no explicit flush",
                           "parallelism": f"dp{world} (frames sharded, 1 all-reduce of 1.56M fp32 grads)",
                           "step_graph": step_graph_used, "step_mode_calibration": calib},
                "clocks": clk, "e2e": e2e, "gpu_launches": int(launches), "roofline": roofline, "mlp_fwd_roofline": fwd_roofline, "raster_roofline": raster_roofline,
                "cpu_baseline": cpu_baseline, **extra,
                "kernel_ms_per_step": {k: round(v[1], 4) for k, v in sorted(per_step.items(), key=lambda kv: -kv[1][1])},
                "dominant_kernel": dominant}
        sys.stdout.flush()
        os.write(real_stdout, (json.dumps(line) + "\n").encode())
    if world > 1:
        dist.barrier(device_ids=[local])
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
