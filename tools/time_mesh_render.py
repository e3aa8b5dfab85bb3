"""Cost of the mesh overlay render (csrc/mesh_render.cu, `ga_mesh_render`) at 1024^2.  Run on the GPU box:
    python tools/time_mesh_render.py > mesh_render.json
For B = 1, 2 and 8 frames per call: the synthetic SMPL (6890 vertices, 13416 faces) and SMPL-X (10475 vertices, 20384 faces) bodies
posed by `ga_smpl_vertices` / `ga_smplx_vertices` in front of the shipped test-pose camera, and a close-up of three faces that each
cover most of the frame (the tile pass).  Times are CUDA events around many back-to-back calls (workspace preallocated), reported
per call and per frame; the card's name, power limit and max SM clock are read in the same run.
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from gaussianavatar_b200 import _lib, synthetic as syn  # noqa: E402
from gaussianavatar_b200._lib import ptr  # noqa: E402
from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, TEST_POSE_K, make_camera  # noqa: E402
from gaussianavatar_b200.mesh_render import MeshRenderer, cameras  # noqa: E402
from gaussianavatar_b200.posmap import BodyPoser, SmplxBodyPoser  # noqa: E402
from time_posmap import card, time_us  # noqa: E402

SIDE = 1024


def meshes(B):
    bs, ts = syn.make_body(0), syn.make_uv_template(0)
    pose, transl = syn.synthetic_poses(B, seed=1)
    yield "smpl", BodyPoser(syn.smpl_mesh_model(bs, ts), bs.betas[0]).vertices(pose, transl), ts[1], TEST_POSE_EXTRINSIC
    bx, tx = syn.make_smplx_body(0), syn.make_smplx_uv_template(0)
    pose, rest, transl = syn.synthetic_smplx_poses(B, seed=1)
    yield "smplx", SmplxBodyPoser(syn.smplx_mesh_model(bx, tx, syn.smplx_posedirs(0)), bx.betas[0]).vertices(pose, rest, transl), tx[1], \
        TEST_POSE_EXTRINSIC
    X = torch.tensor([[-50, -50, 4.0], [50, -50, 6.0], [50, 50, 6.0], [-50, 50, 4.0], [-40, -40, 3.0], [40, -30, 3.5], [0, 40, 3.2]])
    yield "closeup", X[None].expand(B, -1, -1).contiguous().cuda(), np.array([[0, 1, 2], [0, 2, 3], [4, 5, 6]]), np.eye(4)


def main():
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    res = card()
    s = torch.cuda.current_stream().cuda_stream
    L = _lib.lib()
    for B in (1, 2, 8):
        for name, verts, faces, extr in meshes(B):
            r = MeshRenderer(faces, verts.shape[1])
            cams = cameras([make_camera(TEST_POSE_K, extr, SIDE, SIDE)] * B).cuda()
            rgb = torch.empty(B, 3, SIDE, SIDE, device="cuda")
            fid = torch.empty(B, SIDE, SIDE, dtype=torch.int32, device="cuda")
            depth = torch.empty(B, SIDE, SIDE, device="cuda")
            ws = torch.empty(L.ga_mesh_render_workspace_bytes(B, r.V, r.F, SIDE, SIDE), dtype=torch.uint8, device="cuda")
            med, rounds = time_us(lambda: _lib.check(L.ga_mesh_render(B, r.V, r.F, SIDE, SIDE, ptr(verts), ptr(r.faces), ptr(r.adj_offsets),
                                                                      ptr(r.adj_faces), ptr(cams), *r.color, None, ptr(ws), ptr(fid),
                                                                      ptr(depth), ptr(rgb), s)), 100)
            res[f"{name}_B{B}"] = dict(us_per_call=med, us_per_frame=med / B, rounds_us=rounds, faces=r.F,
                                       drawn_fraction=float((fid >= 0).float().mean()))
    res["card_after"] = card()["nvidia_smi"]
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
