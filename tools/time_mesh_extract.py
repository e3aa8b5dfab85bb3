"""Cost of mesh extraction (gaussianavatar_b200.mesh_extract) on the synthetic avatar at 200k Gaussians (S = 512), SMPL and SMPL-X,
res = 256, 64 views of 512^2.  Run on the GPU box:
    python tools/time_mesh_extract.py > mesh_extract.json
Per body, from the library's event profiler over whole extractions (after a warm-up one):
  integrate_ms      the 8 integration launches (64 views), and their byte floor: 28 B read + 28 B written per sample and launch
  count_ms, scan_ms, emit_ms   the three mesher passes, each with its byte floor (state read once, counts / offsets / mesh written)
  extract_ms        one whole extract_mesh (posing, 64 renders, fusion, meshing, the totals read-back), CUDA events
The card's name and power limit are read in the same run.  Floors use 3.35 TB/s (H100 SXM data sheet).
"""
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from gaussianavatar_b200 import _lib, synthetic as syn  # noqa: E402
from gaussianavatar_b200.avatar_model import AvatarModel  # noqa: E402
from gaussianavatar_b200.config import NetworkParams  # noqa: E402
from gaussianavatar_b200.mesh_extract import extract_mesh, fusion_grid, posed_gaussians  # noqa: E402
from time_posmap import card  # noqa: E402

N, S, RES, VIEWS, SIZE = 200_000, 512, 256, 64, 512
BW = 3.35e12


def model(body):
    a = syn.make_avatar_assets(N, S, seed=0, body=body)
    pose, transl = syn.synthetic_poses(2, seed=0)
    if body == "smplx":
        pose = pose[:, :66].contiguous()
    torch.manual_seed(0)
    m = AvatarModel.from_assets(a, [], pose, transl, batch_size=1, train=False, net_parms=NetworkParams())
    with torch.no_grad():
        sd = m.net.state_dict()
        sd["decoder.conv8N.bias"] = torch.tensor([-5.3])
        m.net.load_state_dict(sd, strict=False)
    rest = syn.synthetic_smplx_poses(1, seed=0)[1].cuda() if body == "smplx" else None
    return m, pose[:1].cuda(), transl[:1].cuda(), rest


def floor_ms(nbytes):
    return nbytes / BW * 1e3


def main():
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    res = card()
    res["config"] = dict(gaussians=N, S=S, res=RES, views=VIEWS, size=SIZE)
    for body in ("smpl", "smplx"):
        m, pose, transl, rest = model(body)
        run = lambda: extract_mesh(m, pose, transl, rest, res=RES, views=VIEWS, size=SIZE)
        verts, faces, _ = run()                                     # warm-up
        torch.cuda.synchronize()
        with torch.no_grad():
            means, scales, _ = posed_gaussians(m, pose, transl, rest)
        _, _, dims, _ = fusion_grid(means, scales, RES, 4)
        n = dims[0] * dims[1] * dims[2]
        V, F = int(verts.shape[0]), int(faces.shape[0])
        reps = 5
        _lib.profile(True)
        for _ in range(reps):
            run()
        rep = _lib.profile_report()
        _lib.profile(False)
        k = {name: ms / reps for name, (cnt, ms) in rep.items()}
        wall = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            run()
            b.record()
            b.synchronize()
            wall.append(a.elapsed_time(b))
        launches = (VIEWS + 7) // 8
        res[body] = dict(
            grid=dims, samples=n, vertices=V, faces=F,
            integrate_ms=k.get("tsdf_integrate_kernel"), integrate_floor_ms=floor_ms(launches * 56 * n),
            count_ms=k.get("tsdf_count_kernel"), count_floor_ms=floor_ms(12 * n + 9 * n),
            scan_ms=k.get("tsdf_scan"), scan_floor_ms=floor_ms(2 * 2 * 4 * n),
            emit_ms=k.get("tsdf_emit_kernel"), emit_floor_ms=floor_ms(12 * n + 9 * n + 24 * V + 12 * F),
            extract_ms=statistics.median(wall), extract_rounds_ms=wall,
            kernels_ms=dict(sorted(k.items(), key=lambda kv: -kv[1])))
        del m
        torch.cuda.empty_cache()
    res["card_after"] = card()["nvidia_smi"]
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
