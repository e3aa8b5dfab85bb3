"""Cost of rendering several avatars together (animate.Ensemble) and of their visibility mattes: 1, 2 and 4 actors of the synthetic
avatar at 200k Gaussians (S = 512, the same model on its own clip per actor, placed side by side), 1920 x 1080 frames, the shipped
test-pose camera, with no scene and with the 1M-Gaussian synthetic scene of tools/time_scene.py.  Run on the GPU box:
    python tools/time_cast.py > cast.json
For each scene, actor count and chunk = 2, 8, stage 1 (graph replays, RGB):
  device_ms_per_frame         CUDA events around back-to-back replays of the chunk's graph, mattes off
  mattes_ms_per_frame         the same with mattes on; the two players alternate round by round in this process
  render_fwd_ms / render_fwd_mattes_ms   the compositing kernel alone per frame, without and with mattes (library event profiler,
                              eager launches)
The card's name, power limit and clocks are read in the same run.
"""
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


def player(cast, cam, b, scene, mattes, capacity=None):
    ens = an.Ensemble(cast, cam, H, W, chunk=b, mattes=mattes, scene=scene, capacity=capacity)
    for _ in ens.frames(30.0):                        # warm-up: graphs captured, binning grown to what the chunks need
        pass
    times, aligns, cams = ens._playback(30.0)
    with torch.no_grad():
        render = ens._stage1_setup(times, aligns, cams)
        render(0, b, 0)
    return ens, render


def one(cast, cam, b, scene):
    players = {key: player(cast, cam, b, scene, key == "mattes") for key in ("plain", "mattes")}
    rounds = {"plain": [], "mattes": []}
    with torch.no_grad():
        for _ in range(5):
            for key, (_, render) in players.items():
                rounds[key].append(events_ms(lambda: render(0, b, 0), 10, rounds=1)[0] / b)
    capacity = players["plain"][0]._plans[b].capacity
    overflows = {k: p[0].overflows for k, p in players.items()}
    del players
    torch.cuda.empty_cache()
    kernels = {}
    for key in ("plain", "mattes"):
        ens = an.Ensemble(cast, cam, H, W, chunk=b, mattes=key == "mattes", scene=scene, graphs=False, capacity=capacity)
        for _ in ens.frames(30.0):
            pass
        torch.cuda.synchronize()
        _lib.profile(True)
        n = 0
        for _, f, _ in ens.frames(30.0):
            n += f.shape[0]
        rep = _lib.profile_report()
        _lib.profile(False)
        name = "render_fwd_mattes_kernel" if key == "mattes" else "render_fwd_kernel"
        kernels[key] = rep.get(name, (0, 0.0))[1] / n
        del ens
        torch.cuda.empty_cache()
    return dict(device_ms_per_frame=statistics.median(rounds["plain"]), device_rounds_ms=rounds["plain"],
                mattes_ms_per_frame=statistics.median(rounds["mattes"]), mattes_rounds_ms=rounds["mattes"],
                render_fwd_ms=kernels["plain"], render_fwd_mattes_ms=kernels["mattes"], overflows_while_warming=overflows)


def main():
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
        for n in ACTORS:
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
    res["card_after"] = card()["nvidia_smi"]
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
