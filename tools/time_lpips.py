"""LPIPS timing on the GPU box:
    python tools/time_lpips.py --iters 50 --rounds 3 > lpips.json
(a) LPIPS forward + backward at 1024^2, B = 2 (4 images through the network, 2 backward), the library against the oracle's network
    in fp32 on cuDNN (torch defaults: TF32 convolutions), alternating call by call in one process; medians over --iters calls per
    round, --rounds rounds for the spread.  A separate pass with the library's event profiler gives per-kernel times and TFLOP/s
    on FLOPs computed from shapes.
(b) The graphed stage-1 config-3 step with the LPIPS term active (epoch > lpips_start_iter) against the same trainer before it,
    alternating blocks of steps.
The card name, power limit and max SM clock are read in the same run.  Seeded random weights: the time does not depend on them.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from gaussianavatar_b200 import _lib  # noqa: E402
from gaussianavatar_b200.lpips import LPIPS  # noqa: E402
from oracle import lpips_oracle as lo  # noqa: E402
from time_raster import card  # noqa: E402

DATASHEET_TF32_TFLOPS = 495.0      # H100 SXM, dense


def kernel_flops(B, H, W):
    """Algorithmic FLOPs (2 per multiply-add) of each named convolution launch of one forward (2B images) + backward (B images)."""
    ms = lo.map_shapes(H, W)
    out = {}
    for k in range(5):
        h, w = ms[k]
        K = lo.KERNELS[k] ** 2 * lo.IN_CHANNELS[k]
        out[f"lpips_conv{k + 1}"] = 2.0 * 2 * B * h * w * lo.CHANNELS[k] * K
        if k > 0:
            out[f"lpips_dgrad{k + 1}"] = 2.0 * B * h * w * lo.CHANNELS[k] * K
    h, w = ms[0]
    out["lpips_img_grad"] = 2.0 * B * h * w * 64 * 363
    return out


def time_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0)


def part_a(args, dev):
    B, H, W = 2, 1024, 1024
    sd = lo.random_state_dict(0)
    lib_net = LPIPS(sd, device=dev)
    ref_net = lo.LpipsOracle(sd).to(dev)             # fp32, cuDNN
    g = torch.Generator(device=dev).manual_seed(1)
    x0 = torch.rand(B, 3, H, W, generator=g, device=dev)
    x1 = torch.rand(B, 3, H, W, generator=g, device=dev)
    a = x0.clone().requires_grad_(True)

    def run(net):
        a.grad = None
        net(a, x1, normalize=True).sum().backward()

    lib_call, ref_call = (lambda: run(lib_net)), (lambda: run(ref_net))
    for _ in range(5):
        lib_call(); ref_call()
    # the two agree (a sanity check on what is being timed, not the parity test)
    run(lib_net); gl = a.grad.clone(); vl = lib_net(x0, x1, normalize=True)
    run(ref_net); gr = a.grad.clone(); vr = ref_net(x0, x1, normalize=True)
    agree = dict(value_rel=float(((vl - vr).abs() / vr.abs()).max()), grad_rel_l2=float((gl - gr).norm() / gr.norm()))
    rounds = []
    for _ in range(args.rounds):
        tl, tr = [], []
        for _ in range(args.iters):
            tl.append(time_ms(lib_call))
            tr.append(time_ms(ref_call))
        rounds.append(dict(library_ms=statistics.median(tl), cudnn_ms=statistics.median(tr)))
    # per-kernel pass (profiler on: its events slow the host, so it is not part of the numbers above)
    _lib.profile(True)
    _lib.profile_report()
    n = 20
    for _ in range(n):
        lib_call()
    rep = _lib.profile_report()
    _lib.profile(False)
    flops = kernel_flops(B, H, W)
    kernels = {}
    for name, (cnt, ms) in sorted(rep.items()):
        if not name.startswith("lpips_"):
            continue
        per = ms / n
        row = dict(ms=round(per, 4), launches=cnt // n)
        if name in flops:
            row["tflops"] = round(flops[name] / (per * 1e-3) / 1e12, 1)
            row["share_of_tf32_datasheet"] = round(row["tflops"] / DATASHEET_TF32_TFLOPS, 3)
        kernels[name] = row
    total_flops = sum(flops.values())
    med_lib = statistics.median(r["library_ms"] for r in rounds)
    return dict(shape=[B, 3, H, W], iters=args.iters, rounds=rounds, agree=agree, kernels=kernels,
                kernel_sum_ms=round(sum(k["ms"] for k in kernels.values()), 4), conv_gflop=round(total_flops / 1e9, 1),
                library_tflops_end_to_end=round(total_flops / (med_lib * 1e-3) / 1e12, 1))


def part_b(args, dev):
    from gaussianavatar_b200.trainer import Stage1Trainer
    from gaussianavatar_b200.workload import Stage1Workload
    B = 2
    wl = Stage1Workload(3, B, device=dev)
    wl.make_ground_truth()
    tr = Stage1Trainer(wl.model, perceptual_loss=LPIPS(lo.random_state_dict(0), device=dev))
    batches = [wl.device_batch(wl.frame_ids(i)) for i in range(4)]
    it = [5000]
    start = tr.opt.lpips_start_iter

    def steps(epoch, n):
        for i in range(n):
            tr.step(batches[i % len(batches)], it[0], epoch=epoch)
            it[0] += 1

    for e in (start, start + 1):
        steps(e, 3)
    tr.finish()
    res = {"inactive": [], "active": []}
    for _ in range(args.step_rounds):
        for key, e in (("inactive", start), ("active", start + 1)):
            ms = time_ms(lambda: steps(e, args.step_block))
            res[key].append(B * args.step_block / (ms * 1e-3))
    tr.finish()
    graphs = [list(k) for k in tr._graphs]
    return dict(config=3, frames_per_step=B, steps_per_block=args.step_block, graphs=graphs,
                fps_inactive=[round(x, 1) for x in res["inactive"]], fps_active=[round(x, 1) for x in res["active"]],
                fps_inactive_median=round(statistics.median(res["inactive"]), 1),
                fps_active_median=round(statistics.median(res["active"]), 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--step-block", type=int, default=20)
    ap.add_argument("--step-rounds", type=int, default=5)
    ap.add_argument("--skip-step", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_lpips.py needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_stream(torch.cuda.Stream(device=dev))      # graph capture in part (b) needs a non-default stream
    out = dict(card=card(), lpips=part_a(args, dev))
    if not args.skip_step:
        out["step"] = part_b(args, dev)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
