"""Rasterizer micro-benchmark on the synthetic avatar scene (SURVEY.md §8d "Raster micro-bench").  Run on the GPU box:
    python tools/time_raster.py --config 3 --iters 50 > raster_c3.json
"""
import argparse
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gaussianavatar_b200 import synthetic as syn  # noqa: E402
from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, TEST_POSE_K, make_camera, scaled_intrinsics  # noqa: E402
from gaussianavatar_b200.rasterizer import GaussianRasterizationSettings, rasterize_backward, rasterize_forward  # noqa: E402


def make_scene(config, dev):
    N, S, side = syn.CONFIGS[config]
    a = syn.make_avatar_assets(N, S)
    g = torch.Generator().manual_seed(0)
    means = a.query_points + torch.tensor([0.0, -0.13, 0.0])      # undo most of the canonical lift: body centred in view
    scales = (0.005 * torch.exp(0.35 * torch.randn(N, 1, generator=g))).repeat(1, 3)
    colors = torch.rand(N, 3, generator=g)
    rots = torch.zeros(N, 4); rots[:, 0] = 1
    opac = torch.ones(N, 1)
    cam = make_camera(scaled_intrinsics(TEST_POSE_K, side), TEST_POSE_EXTRINSIC, side, side).to(dev)
    rs = GaussianRasterizationSettings(side, side, math.tan(cam.FovX / 2), math.tan(cam.FovY / 2), torch.ones(3, device=dev), 1.0,
                                       cam.world_view_transform, cam.full_proj_transform, 0, cam.camera_center, False, False)
    t = [x.to(dev).contiguous() for x in (means, colors, opac, scales, rots)]
    return t, rs, side


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    (means, colors, opac, scales, rots), rs, side = make_scene(args.config, dev)
    gw = torch.randn(3, side, side, device=dev)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    fw, bw = [], []
    R = 0
    for it in range(args.iters + 5):
        e0, e1, e2 = ev(), ev(), ev()
        e0.record()
        color, radii, ctx = rasterize_forward(means, colors, opac, scales, rots, rs)
        e1.record()
        rasterize_backward(ctx, means, colors, scales, rots, rs, gw, want_opacity=False, want_rotations=False, want_means2D=False)
        e2.record()
        torch.cuda.synchronize()
        if it >= 5:
            fw.append(e0.elapsed_time(e1)); bw.append(e1.elapsed_time(e2))
        R = ctx.num_rendered
    fw.sort(); bw.sort()
    out = dict(config=args.config, P=int(means.shape[0]), side=side, num_rendered=R, visible=int((radii > 0).sum()),
               covered=float((color.mean(0) < 0.999).float().mean()),
               fwd_ms_median=fw[len(fw) // 2], bwd_ms_median=bw[len(bw) // 2], fwd_ms_min=fw[0], bwd_ms_min=bw[0])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
