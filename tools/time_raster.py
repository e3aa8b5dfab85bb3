"""Rasterizer micro-benchmark on the synthetic avatar scene (SURVEY.md §8d "Raster micro-bench").  Run on the GPU box:
    python tools/time_raster.py --config 3 --iters 50 > raster_c3.json
With --sh-degree D and / or --cov3d-precomp the per-frame forward + backward is also timed with SH colours (16 coefficients per
Gaussian, degree D) and / or precomputed 3D covariances, alternating iteration by iteration with the precomputed-colour,
scale / rotation baseline, and a second pass with the library profiler reports K1 and the fused K8/K9 per mode with their
bandwidth on algorithmic bytes.  The card name and power limit are read in the same run.
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gaussianavatar_b200 import synthetic as syn  # noqa: E402
from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, TEST_POSE_K, make_camera, scaled_intrinsics  # noqa: E402
from gaussianavatar_b200 import _lib  # noqa: E402
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


def card():
    """Name, power limit and max SM clock of cuda:0, read with a query (nothing is changed)."""
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return dict(gpu=torch.cuda.get_device_name(0), nvidia_smi=q)


def k1_bytes(P, vis, M_read, cov, sh):
    """Algorithmic bytes of K1: means + opacity + (Sigma | scale + rotation) in, per-Gaussian state out (depth, xy, conic,
    cov3D, tiles, rect, radii); with SH the coefficients of the visible Gaussians in and rgb + clamp bits out."""
    b = P * (12 + 4 + (24 if cov else 28)) + P * (4 + 8 + 16 + 24 + 4 + 8 + 4)
    return b + (vis * 12 * M_read + P * 13 if sh else 0)


def k89_bytes(P, vis, M, M_read, cov, sh):
    """Algorithmic bytes of the fused K8/K9 as time_raster calls it (no opacity / rotation / means2D gradients): means, radii,
    cov3D, dL/dmean2D, dL/dconic in; d_means3D and d_scales (or d_cov3D) out; scales + rotations in without cov3D; with SH
    dL/drgb + clamp bits in for all, the active coefficients of the visible Gaussians in and the whole d_sh out."""
    b = P * (12 + 4 + 24 + 8 + 16) + P * (12 + (24 if cov else 12)) + (0 if cov else P * 28)
    return b + (P * 13 + vis * 12 * M_read + P * 12 * M if sh else 0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--sh-degree", type=int, default=None, help="also time SH colours of this degree (16 coefficients per Gaussian)")
    ap.add_argument("--cov3d-precomp", action="store_true", help="also time precomputed 3D covariances")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    (means, colors, opac, scales, rots), rs, side = make_scene(args.config, dev)
    gw = torch.randn(3, side, side, device=dev)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    N = int(means.shape[0])

    sh = args.sh_degree is not None
    cov = args.cov3d_precomp
    modes = {"base": {}}
    if sh or cov:
        kw = {}
        if sh:
            g = torch.Generator().manual_seed(1)
            shs = 0.1 * torch.randn(N, 16, 3, generator=g)
            shs[:, 0] = (colors.cpu() - 0.5) / 0.28209479177387814
            kw["shs"] = shs.to(dev).contiguous()
            rs = rs._replace(sh_degree=args.sh_degree)
        if cov:      # the Sigma K1 builds from the scene's scales / rotations: the same image, the same lists
            kw["cov3D_precomp"] = rasterize_forward(means, colors, opac, scales, rots, rs)[2].views()["cov3d"].to(dev).contiguous()
        modes["ext"] = kw

    def step(kw):
        color, radii, ctx = rasterize_forward(means, None if "shs" in kw else colors, opac, None if "cov3D_precomp" in kw else scales,
                                              None if "cov3D_precomp" in kw else rots, rs, **kw)
        mark = ev()
        mark.record()
        rasterize_backward(ctx, means, None if "shs" in kw else colors, None if "cov3D_precomp" in kw else scales,
                           None if "cov3D_precomp" in kw else rots, rs, gw, want_opacity=False, want_rotations=False, want_means2D=False,
                           **({"return_sh_cov3D": True} if kw else {}))
        return color, radii, ctx, mark

    times = {m: ([], []) for m in modes}
    res = {}
    for it in range(args.iters + 5):
        for m, kw in modes.items():          # alternate the modes iteration by iteration
            e0, e2 = ev(), ev()
            e0.record()
            color, radii, ctx, e1 = step(kw)
            e2.record()
            torch.cuda.synchronize()
            if it >= 5:
                times[m][0].append(e0.elapsed_time(e1)); times[m][1].append(e1.elapsed_time(e2))
            res[m] = (color, radii, ctx)
    color, radii, ctx = res["base"]
    fw, bw = (sorted(x) for x in times["base"])
    out = dict(config=args.config, P=N, side=side, num_rendered=ctx.num_rendered, visible=int((radii > 0).sum()),
               covered=float((color.mean(0) < 0.999).float().mean()),
               fwd_ms_median=fw[len(fw) // 2], bwd_ms_median=bw[len(bw) // 2], fwd_ms_min=fw[0], bwd_ms_min=bw[0])
    if len(modes) > 1:
        vis = out["visible"]
        M_read = (args.sh_degree + 1) ** 2 if sh else 0
        fe, be = (sorted(x) for x in times["ext"])
        out.update(mode=("sh%d" % args.sh_degree if sh else "") + ("+cov3d" if cov else ""), ext_fwd_ms_median=fe[len(fe) // 2],
                   ext_bwd_ms_median=be[len(be) // 2], ext_fwd_ms_min=fe[0], ext_bwd_ms_min=be[0],
                   image_max_abs_diff_vs_base=float((res["ext"][0] - color).abs().max()))
        # second pass, profiler on: per-kernel times of K1 and the fused K8/K9 in each mode
        for m, kw in modes.items():
            for _ in range(3):
                step(kw)
            torch.cuda.synchronize()
            _lib.profile_report()
            _lib.profile(True)
            for _ in range(args.iters):
                step(kw)
            rep = _lib.profile_report()
            _lib.profile(False)
            e_sh, e_cov = m == "ext" and sh, m == "ext" and cov
            for name, nbytes in (("preprocess_fwd_kernel", k1_bytes(N, vis, M_read, e_cov, e_sh)),
                                 ("preprocess_bwd_kernel", k89_bytes(N, vis, 16, M_read, e_cov, e_sh))):
                n, ms = rep[name]
                us = 1e3 * ms / n
                out[f"{m}_{name}_us"] = round(us, 2)
                out[f"{m}_{name}_MB"] = round(nbytes / 1e6, 2)
                out[f"{m}_{name}_GBps"] = round(nbytes / (us * 1e-6) / 1e9, 1)
    out.update(card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
