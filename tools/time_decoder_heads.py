"""Time the decoder's layer-6 launches (tensor-core path), alternated in one process at config-3 size (M = 512^2 x 1 UV pixels;
--M to change), and print each form's algorithmic HBM bytes and the rate they imply.

  layer-6 forward   3 x ga_tc_linear_forward (one per head)  vs  ga_tc_linear_forward_heads(heads = 3), which the decoder uses
  layer-6 backward  the mode 1 -> 2 -> 3 chain the decoder uses, and a timing probe of it with layer 5's output read from HBM once

Chain bytes: dZ6 / Y6 of each head, Y5 three times, dZ5 stored, reduce-added (read + write of lines that are not resident) and
re-read + stored: 14 planes.  A one-launch form (three-CTA clusters summing dX over distributed shared memory) would move 8.

Bytes count every operand once (an ideal cache): a [M,128] fp32 plane per activation read or written.  The per-head layer-6
forward reads its input once per head; the one-launch form reads it once.

    python tools/time_decoder_heads.py [--M 262144] [--reps 5] [--iters 20]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gaussianavatar_b200 import _lib as L  # noqa: E402

DEV = "cuda:0"


def p(t):
    return None if t is None else t.data_ptr()


def timed(fn, iters):
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--M", type=int, default=512 * 512)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    M = args.M
    g = torch.Generator(device=DEV).manual_seed(0)
    st = torch.cuda.current_stream().cuda_stream
    lib = L.lib()

    def rn(*s, scale=1.0):
        return torch.randn(*s, device=DEV, generator=g) * scale

    def pos(*s):
        return torch.rand(*s, device=DEV, generator=g) + 0.5

    Y5, a5, b5 = rn(M, 128), pos(128), rn(128, scale=0.5)
    W6, bias6 = rn(384, 128, scale=1 / 11.3), rn(384)
    Y6 = torch.empty(M, 384, device=DEV)
    stat = torch.zeros(2, 384, dtype=torch.float64, device=DEV)

    def fwd_old():
        for h in range(3):
            L.check(lib.ga_tc_linear_forward(M, 128, p(Y5), 128, p(a5), p(b5), p(W6[h * 128:]), 128, p(bias6[h * 128:]), p(Y6[:, h * 128:]),
                                             384, 0, p(stat[0, h * 128:]), p(stat[1, h * 128:]), st))

    def fwd_new():
        L.check(lib.ga_tc_linear_forward_heads(M, 3, 128, p(Y5), 128, p(a5), p(b5), p(W6), 128, 128 * 128, p(bias6), p(Y6), 384, 128, 0,
                                               p(stat[0]), p(stat[1]), 128, st))

    # layer-6 backward as the decoder runs it: three launches, modes 1 (store raw dX), 2 (reduce-add in L2), 3 (add, activation
    # backward, store), each reading layer 5's output Y5.  The probe form points heads 1 and 2 at a single Y5 row (ldp = 0), which
    # stays in L2: its results are meaningless, its time is that of the chain with Y5 read from HBM once.
    W6b, dW6 = rn(384, 128, scale=1 / 11.3), torch.zeros(384, 128, device=DEV)
    dZ6b = rn(M, 384, scale=0.01)
    bc6 = [torch.stack([pos(128), rn(128, scale=0.01), rn(128, scale=0.01), rn(128, scale=0.1), pos(128)]).contiguous() for _ in range(3)]
    pc5 = torch.stack([pos(128), rn(128, scale=0.5), rn(128, scale=0.1), pos(128)]).contiguous()
    dZ5 = torch.empty(M, 128, device=DEV)
    s5 = torch.zeros(2, 128, dtype=torch.float64, device=DEV)

    def l6_chain(y5_once):
        for h in range(3):
            c = h * 128
            ldp = 0 if (y5_once and h > 0) else 128
            L.check(lib.ga_tc_linear_backward_ex(M, p(dZ6b[:, c:]), p(Y6[:, c:]), 384, p(bc6[h]), p(Y5), ldp, p(pc5), p(W6b[c:]), 128,
                                                 p(dW6[c:]), 128, p(dZ5), 128, h + 1, p(s5[0]), p(s5[1]), 128, 0, st))

    plane = M * 128 * 4
    forms = {
        "l6_fwd_per_head": (fwd_old, 6 * plane),
        "l6_fwd_heads": (fwd_new, 4 * plane),
        "l6_bwd_chain": (lambda: l6_chain(False), 14 * plane),
        "l6_bwd_chain_y5_once_probe": (lambda: l6_chain(True), 12 * plane),
    }
    times = {k: [] for k in forms}
    for _ in range(args.reps):
        for k, (fn, _) in forms.items():
            times[k].append(timed(fn, args.iters))
    out = {"device": torch.cuda.get_device_name(0), "M": M}
    for k, (fn, nbytes) in forms.items():
        ms = min(times[k])
        out[k] = {"ms_min": round(ms, 4), "ms_all": [round(t, 4) for t in times[k]], "GB": round(nbytes / 1e9, 3),
                  "TB_per_s": round(nbytes / ms / 1e9, 3)}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
