"""ORACLE — TEST INFRASTRUCTURE ONLY.  Generates the position-map fixtures by importing the UNMODIFIED reference modules from
/root/reference (read-only, never copied).  Run in the build container only (the GPU box has no /root/reference):

    python oracle/gen_golden_posmap.py                        # both fixtures
    python oracle/gen_golden_posmap.py gen_posmap_vertices    # only the named generators

  posmap_vertices.npz   the reference's `submodules.smplx.lbs.lbs` (fp64) on the synthetic body (synthetic.make_body, non-zero
                        posedirs) for the T-pose and the first poses of test_pose_subset.npz with their translations, plus
                        body_models.py:382's `vertices += transl`.  All 6890 vertices would be 0.7 MB: the fixture keeps 512 fixed
                        vertices per pose and each pose's vertex mean and mean square over all of them.
  posmap_obj_parser.npz the reference's `load_obj_mesh(..., with_texture=True)` (scripts/posmap_generator/lib/renderer/mesh.py) on
                        posmap_obj_parser.obj, a small OBJ with triangles, quads, `v/vt`, `v/vt/vn` and texture indices that differ
                        from the vertex indices (a seam), also written here.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(REF, "scripts"))
OUT = os.path.join(ROOT, "tests", "golden")

from gaussianavatar_b200 import synthetic as syn          # noqa: E402

N_KEEP = 512
N_POSES = 8


def gen_posmap_vertices():
    from submodules.smplx.lbs import lbs
    body = syn.make_body(0)
    sub = np.load(os.path.join(OUT, "test_pose_subset.npz"))
    pose = np.concatenate([np.zeros((1, 72), np.float32), sub["body_pose"][:N_POSES]]).astype(np.float32)
    transl = np.concatenate([np.zeros((1, 3), np.float32), sub["trans"][:N_POSES]]).astype(np.float32)
    B = pose.shape[0]
    d = torch.float64
    with torch.no_grad():
        verts, _ = lbs(body.betas.to(d).expand(B, -1), torch.from_numpy(pose).to(d), body.v_template.to(d)[None], body.shapedirs.to(d),
                       body.posedirs.to(d), body.J_regressor.to(d), body.parents, body.lbs_weights.to(d))
        verts = verts + torch.from_numpy(transl).to(d)[:, None]
    v = verts.numpy()
    keep = np.sort(np.random.default_rng(5).choice(v.shape[1], N_KEEP, replace=False))
    np.savez_compressed(os.path.join(OUT, "posmap_vertices.npz"), pose=pose, transl=transl, betas=body.betas[0].numpy(), body_seed=0,
                        keep=keep, verts=v[:, keep].astype(np.float64), mean=v.mean(1), mean_sq=(v ** 2).mean(1))


OBJ_TEXT = """# parser case: triangles, quads, v/vt and v/vt/vn, vt indices that differ from v indices
v 0.0 0.0 0.0
v 1.0 0.0 0.0
v 1.0 1.0 0.0
v 0.0 1.0 0.0
v 2.0 0.0 0.5
v 2.0 1.0 0.5
vt 0.10 0.10
vt 0.40 0.10
vt 0.40 0.40
vt 0.10 0.40
vt 0.60 0.10
vt 0.90 0.10
vt 0.90 0.40
vt 0.60 0.40
vn 0.0 0.0 1.0
vn 0.0 1.0 0.0
f 1/1 2/2 3/3
f 1/1/1 3/3/1 4/4/2
f 2/5 5/6 6/7 3/8
f 2/5/1 5/6/1 6/7/2 3/8/2

f 4/4 3/3 6/7
"""


def gen_posmap_obj_parser():
    from posmap_generator.lib.renderer.mesh import load_obj_mesh
    path = os.path.join(OUT, "posmap_obj_parser.obj")
    with open(path, "w") as fh:
        fh.write(OBJ_TEXT)
    verts, faces, uvs, faces_uv = load_obj_mesh(path, with_texture=True)
    np.savez_compressed(os.path.join(OUT, "posmap_obj_parser.npz"), verts=verts, faces=faces, uvs=uvs, faces_uv=faces_uv)


GENERATORS = (gen_posmap_vertices, gen_posmap_obj_parser)

if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    names = sys.argv[1:] or [g.__name__ for g in GENERATORS]
    for name in names:
        globals()[name]()
    for f in ("posmap_vertices.npz", "posmap_obj_parser.npz", "posmap_obj_parser.obj"):
        print(f, os.path.getsize(os.path.join(OUT, f)))
