"""Cost of the body-topology rig export (gaussianavatar_b200.rig.extract_body_rig) on the tube-bodied synthetic SMPL avatar of
tests/body_rig_fixture.py at S = 512 (about 230k Gaussians), for L = 0, 1, 2 midpoint subdivisions.  Run on the GPU box:
    python tools/time_body_rig.py > body_rig.json
Per L:
  vertices, faces      the rig's mesh
  fit_ms               fit_body_mesh alone (FIT_ITERATIONS preconditioned CG steps), CUDA events, median of 5
  cg_relative_residual its final |b - A d| / |b|
  pushpull_ms          ga_texture_pushpull of the 512^2 colour map, median of 20
  resolve_ms           ga_mesh_shade_unlit (texture) of 8 frames of 1024^2 after one ga_mesh_render, median of 20
  export_ms            one whole extract_body_rig (canonical Gaussians, topology, layout, fit, texture, weights), median of 3
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
from gaussianavatar_b200 import _lib  # noqa: E402
from gaussianavatar_b200 import mesh_extract as me  # noqa: E402
from gaussianavatar_b200 import rig as rg  # noqa: E402
from gaussianavatar_b200._lib import ptr  # noqa: E402
from gaussianavatar_b200.mesh_render import MeshRenderer  # noqa: E402
from gaussianavatar_b200.posmap import CANO_TRANSL, canonical_pose  # noqa: E402
from body_rig_fixture import tube_avatar  # noqa: E402
from time_posmap import card  # noqa: E402

S, FRAMES, SIDE = 512, 8, 1024


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
    m, mapper, template, _, _, _ = tube_avatar("smpl", 1, S=S)
    dev = m.device
    res["config"] = dict(gaussians=int(m.valid_index.numel()), S=S, lam=rg.FIT_LAMBDA, iterations=rg.FIT_ITERATIONS, frames=FRAMES,
                         side=SIDE)
    for L in (0, 1, 2):
        rig = rg.extract_body_rig(m, template, subdiv=L, pose_mapper=mapper)
        topo = rg.body_topology(template, mapper.weights, L)
        pose, rest = m.body.split(canonical_pose("smpl").to(dev))
        x0 = rg.subdivide_points(mapper.posed(pose, rest, torch.tensor([CANO_TRANSL], device=dev))[0], topo)
        layout = rg.UVLayout(topo.faces, topo.uvs, topo.uv_faces, topo.V, S, dev)
        M = (layout.face_id >= 0).float()
        target = layout.fill(x0) + 0.003 * torch.randn(3, S, S, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
        fit = events(lambda: rg.fit_body_mesh(layout, topo, x0, target, M), 5)
        _, rel = rg.fit_body_mesh(layout, topo, x0, target, M)
        img = torch.rand(3, S, S, device=dev)
        mask = torch.rand(S, S, device=dev) < 0.5
        pp = events(lambda: rg.texture_pushpull(img, mask), 20)
        vid, tex, faces = rg.seam_split(rig)
        X = rig.verts[torch.from_numpy(vid).to(dev)][None].expand(FRAMES, -1, -1).contiguous()
        cams = me.fusion_cameras(rig.verts.mean(0).cpu().numpy(), 1.0, FRAMES, SIDE).to(dev)
        mr = MeshRenderer(faces, X.shape[1], device=dev)
        _, fid, _ = mr.render(X, cams, SIDE, SIDE)
        uvs, texture = torch.from_numpy(tex).to(dev), rig.texture.float().div(255.0).contiguous()
        rgb = torch.empty(FRAMES, 3, SIDE, SIDE, device=dev)
        resolve = lambda: _lib.check(_lib.lib().ga_mesh_shade_unlit(FRAMES, X.shape[1], len(faces), SIDE, SIDE, ptr(X), ptr(mr.faces), ptr(cams),
                                                                      ptr(fid), None, ptr(uvs), ptr(texture), S, S, None, ptr(rgb),
                                                                      torch.cuda.current_stream().cuda_stream), "ga_mesh_shade_unlit")
        resolve()
        rs = events(resolve, 20)
        whole = events(lambda: rg.extract_body_rig(m, template, subdiv=L, pose_mapper=mapper), 3)
        res[f"L{L}"] = dict(vertices=topo.V, faces=len(topo.faces), fit_ms=statistics.median(fit), fit_rounds_ms=fit,
                            cg_relative_residual=float(rel), pushpull_ms=statistics.median(pp), resolve_ms=statistics.median(rs),
                            export_ms=statistics.median(whole), export_rounds_ms=whole, avatar_fit=rig.fit)
    res["card_after"] = card()["nvidia_smi"]
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
