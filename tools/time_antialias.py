"""Preprocess kernel times and stage-1 step time with the antialiasing setting on and off, alternated in one run.  Run on the GPU box:
    python tools/time_antialias.py --config 3 --steps 40 > antialias_c3.json
Two identical workloads (config 3: 200k Gaussians, 1024^2, B = 2 by default) train side by side with the whole-step CUDA graph, one
with `antialiasing` set on its model; each step is timed with CUDA events around the trainer's step, the two alternating.  Then the
library's per-kernel CUDA-event profile gives K1 (preprocess_fwd_kernel) and the fused K8/K9 (preprocess_bwd_kernel) of the batched
forward / backward on the same Gaussians in each mode.  The card name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gaussianavatar_b200 import _lib  # noqa: E402
from gaussianavatar_b200.rasterizer import RasterBatchPlan, rasterize_batch  # noqa: E402
from gaussianavatar_b200.trainer import Stage1Trainer  # noqa: E402
from gaussianavatar_b200.workload import Stage1Workload  # noqa: E402
from time_raster import card  # noqa: E402


def kernel_times(wl, iters):
    """Mean per-call times (us) of K1 and K8/K9 over `iters` batched forward + backward calls, filter off then on."""
    m = wl.model
    batch = wl.device_batch(wl.frame_ids(0))
    with torch.no_grad():
        means, scales, colors, _ = m._posed_gaussians(batch["pose_idx"], 5000)
    cams = m._batch_cameras(batch, wl.B, m.device)
    out = {}
    for on in (False, True):
        plan = RasterBatchPlan(wl.B, means.shape[1], wl.side, wl.side, m.device, antialiasing=on)
        args = [t.detach().clone().requires_grad_(True) for t in (means, colors, scales)]
        gw = torch.randn(wl.B, 3, wl.side, wl.side, device=m.device)

        def one():
            img = rasterize_batch(args[0], args[1], args[2], m.fix_rotation, m.fix_opacity, cams, m.background, plan)
            (img * gw).sum().backward()
        for _ in range(3):
            one()
            plan.check(wait=True)
        torch.cuda.synchronize()
        _lib.profile_report()
        _lib.profile(True)
        for _ in range(iters):
            one()
        rep = _lib.profile_report()
        _lib.profile(False)
        for name in ("preprocess_fwd_kernel", "preprocess_bwd_kernel"):
            n, ms = rep[name]
            out[f"{'aa' if on else 'plain'}_{name}_us"] = round(1e3 * ms / n, 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=3)
    ap.add_argument("--frames", type=int, default=2, help="frames per step (B)")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--kernel_iters", type=int, default=50)
    args = ap.parse_args()
    dev = "cuda:0"
    wls = {"plain": Stage1Workload(args.config, args.frames, device=dev), "aa": Stage1Workload(args.config, args.frames, device=dev)}
    wls["aa"].model.antialiasing = True
    for wl in wls.values():
        wl.make_ground_truth()
    trainers = {k: Stage1Trainer(wl.model) for k, wl in wls.items()}
    times = {k: [] for k in wls}
    losses = {k: 0.0 for k in wls}
    for i in range(args.warmup + args.steps):
        for k, wl in wls.items():                  # alternate the two step by step
            batch = wl.device_batch(wl.frame_ids(i))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            loss = trainers[k].step(batch, 5000 + i, epoch=1)
            e1.record()
            torch.cuda.synchronize()
            if i >= args.warmup:
                times[k].append(e0.elapsed_time(e1))
            losses[k] = float(loss)
    for tr in trainers.values():
        tr.finish()
    out = dict(config=args.config, B=args.frames, side=wls["plain"].side, P=wls["plain"].N, steps=args.steps,
               graphed={k: bool(tr._graphs) for k, tr in trainers.items()})
    for k, t in times.items():
        t = sorted(t)
        out[f"{k}_step_ms_median"] = round(t[len(t) // 2], 3)
        out[f"{k}_step_ms_min"] = round(t[0], 3)
        out[f"{k}_last_loss"] = losses[k]
    out["aa_overhead_ms_median"] = round(out["aa_step_ms_median"] - out["plain_step_ms_median"], 3)
    out.update(kernel_times(wls["plain"], args.kernel_iters))
    out.update(card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
