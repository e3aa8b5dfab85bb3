"""Cost of test-time pose fitting (gaussianavatar_b200.posefit) on the synthetic avatar at 200k Gaussians (S = 512), 1024^2 frames,
the shipped test-pose camera.  Run on the GPU box:
    python tools/time_posefit.py > posefit.json
  stage1_chunk{8,1}     device time per frame-iteration (CUDA events around `PoseFitter.fit` of 8 frames, divided by frames x
                        (iters + 1) forwards; iters backwards), chunk 8 and chunk 1
  stage2                the same for stage 2 (S = 512, 128^2 input maps, pose encoder nf = 32), one frame per forward
  kernels               ga_smpl_vertices_backward (B = 8), ga_smplx_vertices_backward (B = 8) and ga_posmap_fill_backward (S = 512,
                        B = 1 and 8): mean kernel time from the library's event profiler over 50 calls (both kernels of the vertex
                        backward), against the byte floor at the data sheet's 3.35 TB/s (posedirs once; the fill's d_out, bary, CSR
                        and d_verts)
  kernels_ms_per_frame_iteration   stage 1 at chunk 8, split per library kernel by the library's event profiler
The card's name, power limit and clocks are read in the same run.
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from gaussianavatar_b200 import _lib, synthetic as syn  # noqa: E402
from gaussianavatar_b200.posefit import PoseFitter  # noqa: E402
from gaussianavatar_b200.posmap import PoseMapper, SmplxPoseMapper, vertices_backward  # noqa: E402
from time_animate import model, N, SIDE, INP  # noqa: E402
from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, TEST_POSE_K  # noqa: E402
from gaussianavatar_b200.dataset import camera_item  # noqa: E402
from time_posmap import card  # noqa: E402

HBM = 3.35e12      # bytes / s, H100 SXM data sheet
FRAMES, ITERS = 8, 10


def frames(m, n):
    cam = camera_item(TEST_POSE_K, TEST_POSE_EXTRINSIC, SIDE, SIDE)
    pose, transl = syn.synthetic_poses(n, seed=2)
    gt = torch.ones(3, SIDE, SIDE)
    return [dict(cam, original_image=gt, pose_data=pose[i], transl_data=transl[i]) for i in range(n)]


def fit_ms(fitter, items):
    fitter.fit(items)                         # warm-up: plans sized, modules loaded
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fitter.fit(items)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / (len(items) * (fitter.iters + 1))


def kernel_ms(fn, n=50):
    """{kernel name: mean ms per call} of the library's launches in fn, timed by its event profiler."""
    fn()
    torch.cuda.synchronize()
    _lib.profile(True)
    for _ in range(n):
        fn()
    rep = _lib.profile_report()
    _lib.profile(False)
    return {k: ms / n for k, (cnt, ms) in rep.items()}


def kernels():
    out = {}
    for body, B in (("smpl", 8), ("smplx", 8)):
        if body == "smpl":
            bd, t = syn.make_body(0), syn.make_uv_template(0)
            mp = PoseMapper(syn.smpl_mesh_model(bd, t), bd.betas[0], t, 512)
            p, tr = syn.synthetic_poses(B)
            r = None
        else:
            bd, t = syn.make_smplx_body(0), syn.make_smplx_uv_template(0)
            mp = SmplxPoseMapper(syn.smplx_mesh_model(bd, t, syn.smplx_posedirs(0)), bd.betas[0], t, 512)
            p, r, tr = syn.synthetic_smplx_poses(B)
            r = r.cuda()
        p = p.cuda()
        g = torch.randn(B, mp.V, 3, device="cuda")
        split = kernel_ms(lambda: vertices_backward(mp, p, r, g))
        ms = sum(split.values())
        floor = mp.posedirs.numel() * 4 / HBM * 1e3
        out[f"{body}_vertices_backward_B{B}"] = dict(ms=ms, split_ms=split, floor_ms=floor, share_of_floor=floor / ms)
        offsets, entries = mp.vertex_csr()
        nnz = int(offsets[-1])
        for Bf in (1, 8):
            d = torch.randn(Bf, 3, 512, 512, device="cuda")
            ms = sum(kernel_ms(lambda: mp.fill_backward(d)).values())
            nbytes = Bf * 3 * 512 * 512 * 4 + nnz * 4 * 2 + (mp.V + 1) * 4 + Bf * mp.V * 3 * 4
            floor = nbytes / HBM * 1e3
            out[f"{body}_fill_backward_S512_B{Bf}"] = dict(ms=ms, bytes=nbytes, floor_ms=floor, share_of_floor=floor / ms)
    return out


def main():
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    res = card()
    res["config"] = dict(gaussians=N, S=512, side=SIDE, frames=FRAMES, iters=ITERS)
    res["kernels"] = kernels()
    m, _ = model(1)
    items = frames(m, FRAMES)
    for chunk in (8, 1):
        f = PoseFitter(m, iters=ITERS, chunk=chunk)
        res[f"stage1_chunk{chunk}"] = dict(device_ms_per_frame_iteration=fit_ms(f, items), overflows=f.overflows)
    f = PoseFitter(m, iters=ITERS, chunk=8)
    f.fit(items)
    torch.cuda.synchronize()
    _lib.profile(True)
    f.fit(items)
    rep = _lib.profile_report()
    _lib.profile(False)
    res["kernels_ms_per_frame_iteration"] = {k: ms / (FRAMES * (ITERS + 1)) for k, (cnt, ms) in sorted(rep.items(), key=lambda kv: -kv[1][1])}
    del m, f
    torch.cuda.empty_cache()
    m2, mapper = model(2)
    f = PoseFitter(m2, iters=ITERS, pose_mapper=mapper)
    res["stage2"] = dict(S=512, inp_posmap_size=INP, device_ms_per_frame_iteration=fit_ms(f, frames(m2, 2)), overflows=f.overflows)
    res["card_after"] = card()["nvidia_smi"]
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
