"""SMPL vs SMPL-X cost of the config-3 stage-1 training step.  Run on the GPU box:
    python tools/time_lbs_smplx.py --steps 30 --rounds 3 > smplx_c3.json
Builds the config-3 workload (N = 200,000 Gaussians, 512^2 UV map, 1024^2 frames, two frames per step) once on the synthetic SMPL body
and once on the synthetic SMPL-X body (55 joints, a hand / face pose per frame), then
  1. times whole steps (whole-step CUDA graph, the default trainer) with CUDA events, alternating SMPL and SMPL-X round by round;
  2. in a separate eager pass with the library profiler on, reports the joint-transform and `lbs_kernel` instantiations per step with
     their bandwidth on algorithmic bytes (weights, query points, decoder rows and valid index read once per step; per-frame outputs
     / gradients).
The card name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gaussianavatar_b200 import _lib  # noqa: E402
from gaussianavatar_b200.trainer import Stage1Trainer  # noqa: E402
from gaussianavatar_b200.workload import Stage1Workload  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


def card():
    """Name, power limit and max SM clock of cuda:0, read with a query (nothing is changed)."""
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return dict(gpu=torch.cuda.get_device_name(0), nvidia_smi=q)


def lbs_bytes(N, B, ld, backward):
    """Algorithmic bytes of one stage-1 LBS launch: the weight row (ld floats), valid index, query point and decoder row once per
    Gaussian; means / scales / colours out (forward) or their gradients in and the decoder-row gradient out (backward) per frame."""
    per_gaussian = 4 * ld + 4 + 12 + 32 + (32 if backward else 0)
    return N * per_gaussian + B * N * 36


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=3)
    ap.add_argument("--frames", type=int, default=2)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_lbs_smplx.py needs a CUDA device")
    dev = "cuda:0"
    runs = {}
    for body in ("smpl", "smplx"):
        wl = Stage1Workload(args.config, args.frames, device=dev, body=body)
        wl.make_ground_truth()
        runs[body] = dict(wl=wl, tr=Stage1Trainer(wl.model), it=0)

    def steps(body, n, trainer=None):
        r = runs[body]
        tr = trainer or r["tr"]
        for _ in range(n):
            i = r["it"]
            tr.step(r["wl"].device_batch(r["wl"].frame_ids(i)), 5000 + i, epoch=1)
            r["it"] += 1
        tr.finish()

    for body in runs:                           # warm-up: allocator, graph capture, module loads
        steps(body, 3)
    torch.cuda.synchronize()
    ms = {b: [] for b in runs}
    for _ in range(args.rounds):
        for body in runs:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            steps(body, args.steps)
            e1.record()
            e1.synchronize()
            ms[body].append(e0.elapsed_time(e1) / args.steps)

    # profiler pass: eager steps (graph replays bypass the library's per-launch events)
    kern = {}
    for body in runs:
        eager = Stage1Trainer(runs[body]["wl"].model, use_graph=False)
        steps(body, 2, eager)
        _lib.profile(True)
        _lib.profile_report()
        steps(body, args.steps, eager)
        rep = _lib.profile_report()
        _lib.profile(False)
        wl = runs[body]["wl"]
        ld = 56 if body == "smplx" else 24
        out = {}
        for name, (n, tot) in rep.items():
            if name.startswith("lbs_kernel") or name.startswith("smpl"):
                per_step = tot / args.steps
                d = dict(launches_per_step=n / args.steps, ms_per_step=round(per_step, 4))
                if name.startswith("lbs_kernel"):
                    nb = lbs_bytes(wl.N, wl.B, ld, "bwd" in name)
                    d.update(algorithmic_bytes=nb, tb_per_s=round(nb / (per_step * 1e-3 / (n / args.steps)) / 1e12, 3),
                             share_of_datasheet_hbm=round(nb / (per_step * 1e-3 / (n / args.steps)) / HBM_BYTES_PER_S, 3))
                out[name] = d
        kern[body] = out

    res = dict(tool="time_lbs_smplx", config=args.config, N=runs["smpl"]["wl"].N, frames_per_step=args.frames, steps=args.steps,
               rounds=args.rounds, card=card(),
               step_ms={b: [round(x, 4) for x in v] for b, v in ms.items()},
               step_ms_median={b: round(statistics.median(v), 4) for b, v in ms.items()},
               kernels=kern)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
