"""Cost of rendering the animated avatar inside a 3D Gaussian Splatting scene (animate.Animator with scene=...): the synthetic
avatar at 200k Gaussians (S = 512) in synthetic scenes of 1M and 3M Gaussians at SH degree 3, 1920 x 1080 frames, the shipped
test-pose camera.  Run on the GPU box:
    python tools/time_scene.py > scene.json
For each scene and chunk = 1, 2, 4, 8, stage 1 (graph replays, RGB):
  device_ms_per_frame         CUDA events around back-to-back replays of the chunk's graph, the scene player and the avatar-only
                              player alternated round by round in this process (avatar_ms_per_frame)
  k1_ms / k1_floor_ms         the composite K1 (preprocess_fwd_kernel, library event profiler, eager launches) per call, and the
                              least time its bytes take at 3.35 TB/s: the scene read once, Ps (12 + 12 + 16 + 4 + 4 * 3 M) bytes,
                              plus the dynamic inputs and the per-frame state written, B (P + Ps) 80 bytes (K1 reads the scene
                              once per frame, so B > 1 cannot reach this floor)
  instances_per_frame         status word 0 / B (the binning capacity a chunk needs), binning_bytes_per_frame the buffer that
                              holds them, default_capacity_fits whether 6 B (P + Ps) held them
The card's name, power limit and clocks are read in the same run.
"""
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from gaussianavatar_b200 import _lib  # noqa: E402
from gaussianavatar_b200 import animate as an  # noqa: E402
from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, TEST_POSE_K, scaled_intrinsics  # noqa: E402
from gaussianavatar_b200.dataset import camera_item  # noqa: E402
from gaussianavatar_b200.scene import GaussianScene  # noqa: E402
from time_animate import clip, events_ms, model  # noqa: E402
from time_posmap import card  # noqa: E402

W, H, DEGREE = 1920, 1080, 3
SCENES = (1_000_000, 3_000_000)
HBM_BYTES_PER_S = 3.35e12


def synthetic_scene(Ps, seed=0):
    """A room-sized cloud around the avatar (the camera sits at z ~ 2.4 looking down -z): anisotropic Gaussians of 1-4 cm, opacities
    0.1..0.99, SH degree 3 with a mid-grey DC term."""
    g = torch.Generator().manual_seed(seed)
    M = (DEGREE + 1) ** 2
    means = (torch.rand(Ps, 3, generator=g) - 0.5) * torch.tensor([6.0, 4.0, 6.0]) + torch.tensor([0.0, 0.0, -1.5])
    scales = 0.02 * torch.exp(0.5 * torch.randn(Ps, 3, generator=g))
    rots = torch.randn(Ps, 4, generator=g)
    rots = rots / rots.norm(dim=1, keepdim=True)
    opac = 0.1 + 0.89 * torch.rand(Ps, generator=g)
    shs = 0.2 * torch.randn(Ps, M, 3, generator=g)
    shs[:, 0] += 0.3
    return GaussianScene(means, scales, rots, opac, shs, DEGREE)


def main():
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    res = card()
    res["config"] = dict(avatar_gaussians=200_000, S=512, width=W, height=H, sh_degree=DEGREE, channels=3)
    K = scaled_intrinsics(TEST_POSE_K, W)
    K[0, 2], K[1, 2] = W / 2.0, H / 2.0
    cam = camera_item(K, TEST_POSE_EXTRINSIC, H, W)
    m, _ = model(1)
    P = int(m._query_points.shape[0])
    c = clip(17)
    for Ps in SCENES:
        scene = synthetic_scene(Ps).to(m.device)
        M = (DEGREE + 1) ** 2
        for b in (1, 2, 4, 8):
            try:
                res[f"scene{Ps}_chunk{b}"] = one_chunk(m, cam, c, scene, P, Ps, M, b)
            except torch.OutOfMemoryError as e:
                res[f"scene{Ps}_chunk{b}"] = dict(out_of_memory=str(e).split(".")[0])
            print(json.dumps({f"scene{Ps}_chunk{b}": res[f"scene{Ps}_chunk{b}"]}), file=sys.stderr, flush=True)
            torch.cuda.empty_cache()
        res[f"scene{Ps}_peak_memory_gb"] = torch.cuda.max_memory_allocated() / 1e9
        del scene
        torch.cuda.empty_cache()
    res["card_after"] = card()["nvidia_smi"]
    print(json.dumps(res, indent=1))


def one_chunk(m, cam, c, scene, P, Ps, M, b):
    """One chunk size: the scene and avatar-only players' graph replays alternated, then the composite K1 from the profiler."""
    players = {}
    for key, sc in (("scene", scene), ("avatar", None)):
        anim = an.Animator(m, cam, H, W, chunk=b, scene=sc)
        for _ in anim.frames(c, 30.0):              # warm-up: graphs captured, binning grown to what the chunks need
            pass
        sched = anim.schedule(c, 30.0)
        with torch.no_grad():
            render = anim._stage1_setup(sched.times[None], [sched.align], sched.cams)
            render(0, b, 0)
        players[key] = (anim, render)
    rounds = {"scene": [], "avatar": []}
    with torch.no_grad():
        for _ in range(5):
            for key, (anim, render) in players.items():
                rounds[key].append(events_ms(lambda: render(0, b, 0), 10, rounds=1)[0] / b)
    anim = players["scene"][0]
    plan = anim._plans[b]
    torch.cuda.synchronize()
    plan.check(wait=True)
    inst, capacity, overflows = int(plan.status_host[0]), plan.capacity, anim.overflows
    del players, anim, plan
    torch.cuda.empty_cache()
    eager = an.Animator(m, cam, H, W, chunk=b, scene=scene, graphs=False, capacity=capacity)
    for _ in eager.frames(c, 30.0):
        pass
    torch.cuda.synchronize()
    _lib.profile(True)
    for _ in eager.frames(c, 30.0):
        pass
    rep = _lib.profile_report()
    _lib.profile(False)
    del eager
    n_calls, k1_total = rep.get("preprocess_fwd_kernel", (0, 0.0))
    floor_bytes = Ps * (12 + 12 + 16 + 4 + 4 * 3 * M) + b * P * (12 + 12) + b * (P + Ps) * 80
    return dict(device_ms_per_frame=statistics.median(rounds["scene"]), device_rounds_ms=rounds["scene"],
                avatar_ms_per_frame=statistics.median(rounds["avatar"]), avatar_rounds_ms=rounds["avatar"],
                k1_ms=k1_total / max(n_calls, 1), k1_floor_ms=1e3 * floor_bytes / HBM_BYTES_PER_S,
                instances_per_frame=inst / b, binning_bytes_per_frame=_lib.lib().ga_rasterb_binning_bytes(b, H, W, inst) / b,
                default_capacity=6 * b * (P + Ps), default_capacity_fits=inst <= 6 * b * (P + Ps), overflows_while_warming=overflows,
                kernels_ms_per_frame={k: ms / len(sched.times) for k, (_, ms) in rep.items()})


if __name__ == "__main__":
    main()
