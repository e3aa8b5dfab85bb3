"""Cost of the animation player (gaussianavatar_b200.animate) on the synthetic avatar at 200k Gaussians (S = 512), 1024^2 frames,
the shipped test-pose camera.  Run on the GPU box:
    python tools/time_animate.py > animate.json
Stage 1, chunk = 1, 2, 4, 8 (RGB):
  device_ms_per_frame   CUDA events around back-to-back replays of the chunk's graph (sample -> cano2live -> LBS -> raster -> pack)
  latency_ms            from the chunk's start on the compute stream to its bytes in pinned memory (events on both streams)
  sustained_fps         wall-clock frames per second of `Animator.frames` over a 300-frame playback, copy-out included
Stage 2 (S = 512, 128^2 input maps, pose encoder nf = 32): sustained frames per second, one frame per forward.
kernels_ms_per_frame: per-kernel split of stage 1 at chunk 8 from the library's event profiler (eager launches, graphs off).
The card's name, power limit and clocks are read in the same run.
"""
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from gaussianavatar_b200 import _lib, synthetic as syn  # noqa: E402
from gaussianavatar_b200 import animate as an  # noqa: E402
from gaussianavatar_b200.avatar_model import AvatarModel  # noqa: E402
from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, TEST_POSE_K  # noqa: E402
from gaussianavatar_b200.config import NetworkParams  # noqa: E402
from gaussianavatar_b200.dataset import camera_item  # noqa: E402
from time_posmap import card  # noqa: E402

N, S, SIDE, INP = 200_000, 512, 1024, 128


def model(stage):
    a = syn.make_avatar_assets(N, S, seed=0)
    pose, transl = syn.synthetic_poses(8, seed=0)
    fields = dict(train_stage=2, inp_posmap_size=INP) if stage == 2 else {}
    torch.manual_seed(0)
    m = AvatarModel.from_assets(a, [], pose, transl, batch_size=1, train=False, net_parms=NetworkParams(), **fields)
    with torch.no_grad():
        sd = m.net.state_dict()
        sd["decoder.conv8N.bias"] = torch.tensor([-5.3])
        m.net.load_state_dict(sd, strict=False)
    mapper = None
    if stage == 2:
        from gaussianavatar_b200.posmap import PoseMapper
        t = syn.make_uv_template(0)
        mapper = PoseMapper(syn.smpl_mesh_model(a.body, t), a.body.betas[0], t, INP)
    return m, mapper


def clip(T):
    pose, transl = syn.synthetic_poses(T, seed=1)
    return an.MotionClip(pose, transl, 30.0, "smpl")


def events_ms(fn, iters, rounds=5, stream_end=None):
    out = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record(stream_end) if stream_end is not None else b.record()
        b.synchronize()
        out.append(a.elapsed_time(b) / iters)
    return statistics.median(out), out


def sustained(anim, c):
    for _ in anim.frames(c, 30.0):        # warm-up: graphs captured, buffers sized
        pass
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = 0
    for _, f in anim.frames(c, 30.0):
        n += f.shape[0]
    return n / (time.perf_counter() - t0), n


def main():
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    res = card()
    res["config"] = dict(gaussians=N, S=S, side=SIDE, channels=3)
    cam = camera_item(TEST_POSE_K, TEST_POSE_EXTRINSIC, SIDE, SIDE)
    m, _ = model(1)
    long_clip = clip(301)
    for b in (1, 2, 4, 8):
        anim = an.Animator(m, cam, SIDE, SIDE, chunk=b)
        fps, n = sustained(anim, long_clip)
        sched = anim.schedule(long_clip, 30.0)
        with torch.no_grad():
            render = anim._stage1_setup(sched.times[None], [sched.align], sched.cams)
            render(0, b, 0)
            dev_ms, dev_rounds = events_ms(lambda: render(0, b, 0), 20)
        lat = []
        for _ in range(10):
            a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a0.record()
            anim._enqueue(render, 0, b, 0)
            a1.record(anim._copy_stream)
            a1.synchronize()
            lat.append(a0.elapsed_time(a1))
        res[f"stage1_chunk{b}"] = dict(device_ms_per_frame=dev_ms / b, device_rounds_ms=dev_rounds, latency_ms=statistics.median(lat),
                                       sustained_fps=fps, frames=n, captures=anim.captures, overflows=anim.overflows)
    anim = an.Animator(m, cam, SIDE, SIDE, chunk=8, graphs=False)
    c16 = clip(16)
    for _ in anim.frames(c16, 30.0):
        pass
    torch.cuda.synchronize()
    _lib.profile(True)
    for _ in anim.frames(c16, 30.0):
        pass
    rep = _lib.profile_report()
    _lib.profile(False)
    res["kernels_ms_per_frame"] = {k: ms / 16 for k, (cnt, ms) in sorted(rep.items(), key=lambda kv: -kv[1][1])}
    del anim, m
    torch.cuda.empty_cache()

    m2, mapper = model(2)
    anim = an.Animator(m2, cam, SIDE, SIDE, chunk=4, pose_mapper=mapper)
    fps, n = sustained(anim, clip(17))
    res["stage2"] = dict(S=S, inp_posmap_size=INP, sustained_fps=fps, ms_per_frame=1e3 / fps, frames=n)
    res["card_after"] = card()["nvidia_smi"]
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
