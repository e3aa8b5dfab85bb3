"""Stage-1 step time with and without the depth term, alternated step by step in one run.  Run on the GPU box:
    python tools/time_depth_train.py --config 3 --steps 40 > depth_train_c3.json
Two identical workloads (config 3: 200k Gaussians, 1024^2, B = 2 by default) train side by side with the whole-step CUDA graph; one
gets batches that carry a target depth (its own initial mean depth, scaled by 1.02, so the term has a gradient everywhere it
counts) and lambda_depth, the other the plain batches.  Each step is timed with CUDA events around the trainer's step (the graph
replay and Adam), the two trainers alternating.  The card name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gaussianavatar_b200.rasterizer import RasterBatchPlan, rasterize_batch_depth  # noqa: E402
from gaussianavatar_b200.trainer import Stage1Trainer  # noqa: E402
from gaussianavatar_b200.workload import Stage1Workload  # noqa: E402
from time_raster import card  # noqa: E402


def target_depth(wl):
    m = wl.model
    out = []
    with torch.no_grad():
        for f0 in range(0, wl.num_frames, wl.B):
            ids = [(f0 + j) % wl.num_frames for j in range(wl.B)]
            batch = wl.device_batch(ids)
            means, scales, colors, _ = m._posed_gaussians(batch["pose_idx"], 5000)
            cams = m._batch_cameras(batch, wl.B, m.device)
            plan = RasterBatchPlan(wl.B, means.shape[1], wl.side, wl.side, m.device)
            _, depth = rasterize_batch_depth(means, colors, scales, m.fix_rotation, m.fix_opacity, cams, m.background, plan)
            assert plan.check(wait=True)
            out.append(depth[:, 0] * 1.02)
    return torch.cat(out)[:wl.num_frames].contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=3)
    ap.add_argument("--frames", type=int, default=2, help="frames per step (B)")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--lambda_depth", type=float, default=1.0)
    args = ap.parse_args()
    dev = "cuda:0"
    wls = {"plain": Stage1Workload(args.config, args.frames, device=dev), "depth": Stage1Workload(args.config, args.frames, device=dev)}
    for wl in wls.values():
        wl.make_ground_truth()
    target = target_depth(wls["depth"])
    wls["depth"].model.opt_parms.lambda_depth = args.lambda_depth
    trainers = {k: Stage1Trainer(wl.model) for k, wl in wls.items()}
    times = {k: [] for k in wls}
    losses = {k: 0.0 for k in wls}
    for i in range(args.warmup + args.steps):
        for k, wl in wls.items():                  # alternate the two step by step
            ids = wl.frame_ids(i)
            batch = wl.device_batch(ids)
            if k == "depth":
                batch["depth"] = target[torch.tensor(ids, device=dev)]
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
               lambda_depth=args.lambda_depth, graphed={k: bool(tr._graphs) for k, tr in trainers.items()})
    for k, t in times.items():
        t = sorted(t)
        out[f"{k}_step_ms_median"] = round(t[len(t) // 2], 3)
        out[f"{k}_step_ms_min"] = round(t[0], 3)
        out[f"{k}_last_loss"] = losses[k]
    out["depth_overhead_ms_median"] = round(out["depth_step_ms_median"] - out["plain_step_ms_median"], 3)
    out.update(card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
