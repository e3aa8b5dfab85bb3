"""Cost of the soft silhouette (csrc/silhouette.cu) and of one pose-refinement iteration.  Run on the GPU box:
    python tools/time_silhouette.py > silhouette.json
The synthetic SMPL body, B = 8 frames per call at 540^2 and 1080^2: `ga_silhouette_forward` and `ga_silhouette_backward` times
(CUDA events over back-to-back calls, workspace preallocated) beside their byte floor at 3.35 TB/s (inputs read once, outputs
written once: verts, faces, CSR, cameras, masks, sil / d_verts), and one `PoseRefiner` iteration over 100 frames (the difference of
10 and 0 iterations, divided by 10).  The card's name and power limit are read in the same run.
"""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from gaussianavatar_b200 import _lib, synthetic as syn  # noqa: E402
from gaussianavatar_b200._lib import ptr  # noqa: E402
from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, make_camera  # noqa: E402
from gaussianavatar_b200.mesh_render import cameras  # noqa: E402
from gaussianavatar_b200.posmap import BodyPoser  # noqa: E402
from gaussianavatar_b200.silhouette import PoseRefiner, SilhouetteRenderer  # noqa: E402
from time_posmap import card, time_us  # noqa: E402

HBM = 3.35e12


def _K(side):
    s = side / 1024.0
    return np.array([[1100.0 * s, 0, side / 2], [0, 1100.0 * s, side / 2], [0, 0, 1]], np.float32)


def main():
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    res = card()
    s = torch.cuda.current_stream().cuda_stream
    L = _lib.lib()
    body, t = syn.make_body(0), syn.make_uv_template(0)
    poser = BodyPoser(syn.smpl_mesh_model(body, t), body.betas[0])
    B = 8
    for side in (540, 1080):
        pose, transl = syn.synthetic_poses(B, seed=1)
        verts = poser.vertices(pose, transl)
        r = SilhouetteRenderer(poser.faces, poser.V)
        cams = cameras([make_camera(_K(side), TEST_POSE_EXTRINSIC, side, side)] * B).cuda()
        sil = torch.empty(B, side, side, device="cuda")
        masks = (r.render(verts, cams, side, side) > 0.5).to(torch.uint8) * 255
        loss = torch.empty(B, device="cuda")
        d = torch.empty(B, r.V, 3, device="cuda")
        w = torch.ones(B, device="cuda")
        ws = torch.empty(L.ga_silhouette_workspace_bytes(B, r.V, r.F, side, side), dtype=torch.uint8, device="cuda")
        fwd, _ = time_us(lambda: _lib.check(L.ga_silhouette_forward(B, r.V, r.F, side, side, 1.0, ptr(verts), ptr(r.faces), ptr(cams), ptr(masks),
                                                                    ptr(ws), ptr(sil), ptr(loss), s)), 50)
        bwd, _ = time_us(lambda: _lib.check(L.ga_silhouette_backward(B, r.V, r.F, side, side, 1.0, ptr(verts), ptr(r.faces), ptr(r.adj_offsets),
                                                                     ptr(r.adj_faces), ptr(cams), ptr(masks), ptr(w), ptr(ws), ptr(d), s)), 50)
        px = B * side * side
        common = B * r.V * 12 + r.F * 12 + B * 160 + px
        floor_f = (common + px * 4 + B * 4) / HBM * 1e6
        floor_b = (common + (r.V + 1) * 4 + 3 * r.F * 4 + B * r.V * 12) / HBM * 1e6
        res[f"smpl_B{B}_{side}"] = dict(forward_us=fwd, backward_us=bwd, forward_floor_us=floor_f, backward_floor_us=floor_b,
                                        covered_fraction=float((masks > 0).float().mean()))
        # one refinement iteration over 100 frames at this size
        n = 100
        pose, transl = syn.synthetic_poses(n, seed=2)
        cam = cameras([make_camera(_K(side), TEST_POSE_EXTRINSIC, side, side)])[0].cuda()
        mk = torch.cat([(r.render(poser.vertices(pose[i:i + 8], transl[i:i + 8]), cam[None].expand(len(pose[i:i + 8]), -1).contiguous(),
                                  side, side) > 0.5).to(torch.uint8) * 255 for i in range(0, n, 8)])
        times = {}
        for iters in (0, 10, 0, 10):
            ref = PoseRefiner(poser, r, iters=iters)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ref.refine(pose + 0.05, transl, cam, mk)
            torch.cuda.synchronize()
            times[iters] = time.perf_counter() - t0
        res[f"refine_iteration_100_frames_{side}_ms"] = (times[10] - times[0]) / 10 * 1e3
    res["card_after"] = card()["nvidia_smi"]
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
