"""Stage-1 step time with the per-frame exposure table on and off, alternated in one run, and the skinning kernels behind it.  Run on
the GPU box:
    python tools/time_exposure.py --config 3 --steps 40 > exposure_c3.json
Two identical workloads (config 3: 200k Gaussians, 1024^2, B = 2 by default) train side by side with the whole-step CUDA graph, one
with an exposure table on its model (ModelParams.train_exposure); each step is timed with CUDA events around the trainer's step, the
two alternating.  Then the library's per-kernel CUDA-event profile gives the skinning forward / backward of both variants and the
exposure gradient's reduction on the same inputs.  The card name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gaussianavatar_b200 import _lib  # noqa: E402
from gaussianavatar_b200.avatar_model import identity_exposure  # noqa: E402
from gaussianavatar_b200.trainer import Stage1Trainer  # noqa: E402
from gaussianavatar_b200.workload import Stage1Workload  # noqa: E402
from time_raster import card  # noqa: E402


def kernel_times(wl, iters):
    """Mean per-call times (us) of the LBS launches with the table and without it."""
    m = wl.model
    batch = wl.device_batch(wl.frame_ids(0))
    idx = batch["pose_idx"]
    with torch.no_grad():
        dec = m._stage1_decoder(wl.B)
    out = {}
    for table in (None, m.exposure.detach()):
        pose, transl = m.pose.weight.detach()[idx].clone().requires_grad_(True), m.transl.weight.detach()[idx]
        for _ in range(3):
            means, scales, colors = m._assemble(dec, pose, transl, exposure=table, exposure_idx=None if table is None else idx)
            torch.autograd.backward([means, colors], [torch.ones_like(means), torch.ones_like(colors)])
        torch.cuda.synchronize()
        _lib.profile_report()
        _lib.profile(True)
        for _ in range(iters):
            means, scales, colors = m._assemble(dec, pose, transl, exposure=table, exposure_idx=None if table is None else idx)
            torch.autograd.backward([means, colors], [torch.ones_like(means), torch.ones_like(colors)])
        rep = _lib.profile_report()
        _lib.profile(False)
        for name, (n, ms) in rep.items():
            if name.startswith("lbs"):
                out[f"{name}_us"] = round(1e3 * ms / n, 2)
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
    wls = {"plain": Stage1Workload(args.config, args.frames, device=dev), "exposure": Stage1Workload(args.config, args.frames, device=dev)}
    m = wls["exposure"].model
    m.model_parms.train_exposure = True
    m.exposure = torch.nn.Parameter(identity_exposure(wls["exposure"].num_frames, dev))
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
    out["exposure_overhead_ms_median"] = round(out["exposure_step_ms_median"] - out["plain_step_ms_median"], 3)
    out.update(kernel_times(wls["exposure"], args.kernel_iters))
    out.update(card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
