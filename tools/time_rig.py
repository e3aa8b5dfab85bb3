"""Cost of the rigged-mesh export (gaussianavatar_b200.rig) on the synthetic avatar at 200k Gaussians (S = 512), SMPL and SMPL-X,
res = 256, 64 views of 512^2, k = 8 neighbours, 4 influences.  Run on the GPU box:
    python tools/time_rig.py > rig.json
Per body:
  skin_weights_ms   ga_skin_weights alone on the canonical mesh's vertices and the canonical Gaussians, CUDA events, median of 10
  distance_evals    vertices x Gaussians, and the rate they were evaluated at
  rig_ms            one whole extract_rigged_mesh (canonical Gaussians, 64 renders, fusion, meshing, skin weights), CUDA events
The card's name and power limit are read in the same run.
"""
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from gaussianavatar_b200 import rig as rg  # noqa: E402
from gaussianavatar_b200.avatar_model import kept_state  # noqa: E402
from time_mesh_extract import RES, SIZE, VIEWS, model  # noqa: E402
from time_posmap import card  # noqa: E402

K_NEAR, INFLUENCES = 8, 4


def events(fn, reps):
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return out


def main():
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    res = card()
    res["config"] = dict(gaussians=200_000, S=512, res=RES, views=VIEWS, size=SIZE, k=K_NEAR, influences=INFLUENCES)
    for body in ("smpl", "smplx"):
        m, _, _, _ = model(body)
        run = lambda: rg.extract_rigged_mesh(m, res=RES, views=VIEWS, size=SIZE, k=K_NEAR, influences=INFLUENCES)
        rig = run()                                                 # warm-up
        torch.cuda.synchronize()
        with torch.no_grad(), kept_state(m):
            means = rg.canonical_gaussians(m)[0][0].contiguous()
        V, N = int(rig.verts.shape[0]), int(means.shape[0])
        skin = lambda: rg.skin_weights(rig.verts, means, m._query_lbs, m.body.joints, K_NEAR, INFLUENCES)
        skin()
        sw = events(skin, 10)
        whole = events(run, 5)
        ms = statistics.median(sw)
        res[body] = dict(vertices=V, faces=int(rig.faces.shape[0]), gaussians=N, distance_evals=V * N,
                         skin_weights_ms=ms, skin_weights_rounds_ms=sw, distance_evals_per_s=V * N / (ms * 1e-3),
                         rig_ms=statistics.median(whole), rig_rounds_ms=whole)
        del m, rig
        torch.cuda.empty_cache()
    res["card_after"] = card()["nvidia_smi"]
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
