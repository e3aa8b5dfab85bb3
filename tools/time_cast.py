"""Cost of rendering several avatars together (animate.Ensemble), of their visibility mattes and of the depth pass: 1, 2 and 4
actors of the synthetic avatar at 200k Gaussians (S = 512, the same model on its own clip per actor, placed side by side),
1920 x 1080 frames, the shipped test-pose camera, with no scene and with the 1M-Gaussian synthetic scene of tools/time_scene.py.
Run on the GPU box:
    python tools/time_cast.py [--actors 1 2] > cast.json
For each scene, actor count and chunk = 2, 8, stage 1 (graph replays, RGB):
  device_ms_per_frame         CUDA events around back-to-back replays of the chunk's graph, mattes and depth off
  mattes_ms_per_frame         the same with mattes on
  depth_ms_per_frame          the same with depth on (mattes off); the three players alternate round by round in this process
  render_fwd_ms / render_fwd_mattes_ms / render_fwd_depth_ms   the compositing kernel alone per frame, plain, with mattes and with
                              depth (library event profiler, eager launches)
The card's name, power limit and clocks are read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from gaussianavatar_b200 import _lib  # noqa: E402
from gaussianavatar_b200 import animate as an  # noqa: E402
from gaussianavatar_b200 import synthetic as syn  # noqa: E402
from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, TEST_POSE_K, scaled_intrinsics  # noqa: E402
from gaussianavatar_b200.dataset import camera_item  # noqa: E402
from gaussianavatar_b200.scene import Placement  # noqa: E402
from time_animate import events_ms, model  # noqa: E402
from time_posmap import card  # noqa: E402
from time_scene import synthetic_scene  # noqa: E402

W, H = 1920, 1080
ACTORS = (1, 2, 4)
CHUNKS = (2, 8)
KEYS = 17


def actors(m, n):
    """n actors of model m, each on its own synthetic clip, side by side 0.7 apart around actor 0."""
    out = []
    for k in range(n):
        pose, transl = syn.synthetic_poses(KEYS, seed=1 + k)
        place = None if k == 0 else Placement.from_axis_angle(1.0, [0.0, 0.0, 0.0], [0.7 * ((k + 1) // 2) * (-1) ** k, 0.0, -0.3 * k])
        out.append(an.Actor(m, an.MotionClip(pose, transl, 30.0, "smpl"), place))
    return out


VARIANTS = {"plain": {}, "mattes": dict(mattes=True), "depth": dict(depth=True)}
KERNELS = {"plain": "render_fwd_kernel", "mattes": "render_fwd_mattes_kernel", "depth": "render_fwd_depth_kernel"}


def player(cast, cam, b, scene, variant, capacity=None):
    ens = an.Ensemble(cast, cam, H, W, chunk=b, scene=scene, capacity=capacity, **VARIANTS[variant])
    for _ in ens.frames(30.0):                        # warm-up: graphs captured, binning grown to what the chunks need
        pass
    times, aligns, cams = ens._playback(30.0)
    with torch.no_grad():
        render = ens._stage1_setup(times, aligns, cams)
        render(0, b, 0)
    return ens, render


def one(cast, cam, b, scene):
    players = {key: player(cast, cam, b, scene, key) for key in VARIANTS}
    rounds = {key: [] for key in VARIANTS}
    with torch.no_grad():
        for _ in range(5):
            for key, (_, render) in players.items():
                rounds[key].append(events_ms(lambda: render(0, b, 0), 10, rounds=1)[0] / b)
    capacity = players["plain"][0]._plans[b].capacity
    overflows = {k: p[0].overflows for k, p in players.items()}
    del players
    torch.cuda.empty_cache()
    kernels = {}
    for key in VARIANTS:
        ens = an.Ensemble(cast, cam, H, W, chunk=b, scene=scene, graphs=False, capacity=capacity, **VARIANTS[key])
        for _ in ens.frames(30.0):
            pass
        torch.cuda.synchronize()
        _lib.profile(True)
        n = 0
        for _, f, *_ in ens.frames(30.0):
            n += f.shape[0]
        rep = _lib.profile_report()
        _lib.profile(False)
        kernels[key] = rep.get(KERNELS[key], (0, 0.0))[1] / n
        del ens
        torch.cuda.empty_cache()
    return dict(device_ms_per_frame=statistics.median(rounds["plain"]), device_rounds_ms=rounds["plain"],
                mattes_ms_per_frame=statistics.median(rounds["mattes"]), mattes_rounds_ms=rounds["mattes"],
                depth_ms_per_frame=statistics.median(rounds["depth"]), depth_rounds_ms=rounds["depth"],
                render_fwd_ms=kernels["plain"], render_fwd_mattes_ms=kernels["mattes"], render_fwd_depth_ms=kernels["depth"],
                overflows_while_warming=overflows)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--actors", type=int, nargs="+", default=list(ACTORS), help="actor counts to time (default 1 2 4)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    res = card()
    res["config"] = dict(avatar_gaussians=200_000, S=512, width=W, height=H, scene_gaussians=1_000_000, channels=3, clip_keys=KEYS)
    K = scaled_intrinsics(TEST_POSE_K, W)
    K[0, 2], K[1, 2] = W / 2.0, H / 2.0
    cam = camera_item(K, TEST_POSE_EXTRINSIC, H, W)
    m, _ = model(1)
    for Ps in (0, 1_000_000):
        scene = synthetic_scene(Ps).to(m.device) if Ps else None
        for n in args.actors:
            cast = actors(m, n)
            for b in CHUNKS:
                key = f"scene{Ps}_actors{n}_chunk{b}"
                try:
                    res[key] = one(cast, cam, b, scene)
                except torch.OutOfMemoryError as e:
                    res[key] = dict(out_of_memory=str(e).split(".")[0])
                print(json.dumps({key: res[key]}), file=sys.stderr, flush=True)
                torch.cuda.empty_cache()
        del scene
        torch.cuda.empty_cache()
    res["peak_memory_gb"] = torch.cuda.max_memory_allocated() / 1e9
    res["mattes_over_plain"] = {k: v["mattes_ms_per_frame"] / v["device_ms_per_frame"] for k, v in res.items()
                                if isinstance(v, dict) and "mattes_ms_per_frame" in v}
    res["depth_over_plain"] = {k: v["depth_ms_per_frame"] / v["device_ms_per_frame"] for k, v in res.items()
                               if isinstance(v, dict) and "depth_ms_per_frame" in v}
    res["depth_kernel_over_plain"] = {k: v["render_fwd_depth_ms"] / v["render_fwd_ms"] for k, v in res.items()
                                      if isinstance(v, dict) and v.get("render_fwd_ms")}
    res["card_after"] = card()["nvidia_smi"]
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
