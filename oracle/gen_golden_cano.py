"""ORACLE — TEST INFRASTRUCTURE ONLY.  Generates the canonical-asset fixtures by importing the UNMODIFIED reference modules from
/root/reference (read-only, never copied).  Run in the build container only (the GPU box has no /root/reference):

    python oracle/gen_golden_cano.py                         # every fixture
    python oracle/gen_golden_cano.py gen_cano_smplx          # only the named generators

  cano_smplx_vertices.npz  the reference's own `smplx.SMPLX(use_pca=False, flat_hand_mean=True)` (fp64) on a synthetic
                           SMPLX_NEUTRAL.npz with non-zero posedirs (synthetic.smplx_posedirs) and the faces of
                           synthetic.make_smplx_uv_template: the canonical pose of arguments/__init__.py (smplx_cpose_param, transl
                           (0, 0.30, 0)), the T-pose, random poses and large finger angles.  `.vertices` (transl added,
                           body_models.py:1273-1275) as 512 fixed vertices per pose plus each pose's vertex mean and mean square, and
                           `.A`.
  cano_smpl.npz            the reference's own `smplx.SMPL` (fp64) on the synthetic SMPL_NEUTRAL.pkl (synthetic.smpl_mesh_model) at
                           the canonical pose and translation of scripts/gen_pose_map_cano_smpl.py:60-70 (smpl_cpose_param): the
                           same vertex summary and `.A`, the matrices that script saves as smpl_cano_joint_mat.pth.
  cano_lbs_weights.npz     the reference's `gen_lbs_weight_from_ori` (utils/general_utils.py:245-259) on the synthetic skinning
                           weights of both bodies, with the face ids and barycentric weights of the library's layout of the synthetic
                           UV templates at S = 16 (the texel faces as `get_face_per_pixel` forms them: background reads face 0).

The reference's `arguments` module imports pytorch3d.transforms for a constant the canonical pose does not use; a stub stands in.
"""
import os
import pickle
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)
OUT = os.path.join(ROOT, "tests", "golden")

from gaussianavatar_b200 import synthetic as syn          # noqa: E402
from oracle import posmap_oracle as po                    # noqa: E402

N_KEEP = 512
W_SIZE = 16


def _cpose():
    """smpl_cpose_param, smplx_cpose_param of the reference's own arguments module."""
    stub = types.ModuleType("pytorch3d")
    stub.transforms = types.SimpleNamespace(euler_angles_to_matrix=lambda x, order: x, matrix_to_axis_angle=lambda x: x)
    sys.modules.setdefault("pytorch3d", stub)
    sys.modules.setdefault("pytorch3d.transforms", stub.transforms)
    import arguments
    return arguments.smpl_cpose_param.clone(), arguments.smplx_cpose_param.clone()


def _summary(v, seed):
    keep = np.sort(np.random.default_rng(seed).choice(v.shape[1], N_KEEP, replace=False))
    return dict(keep=keep, verts=v[:, keep], mean=v.mean(1), mean_sq=(v ** 2).mean(1))


def gen_cano_smplx():
    from submodules import smplx as ref_smplx
    _, cpose = _cpose()
    body = syn.make_smplx_body(0)
    template = syn.make_smplx_uv_template(0)
    g = torch.Generator().manual_seed(31)
    B = 8
    pose = torch.zeros(B, 66, dtype=torch.float64); rest = torch.zeros(B, 99, dtype=torch.float64)
    transl = torch.zeros(B, 3, dtype=torch.float64)
    pose[0] = cpose[0, :66].double(); rest[0] = cpose[0, 66:].double(); transl[0] = torch.tensor([0.0, 0.30, 0.0])   # canonical
    # 1: T-pose; 2..5: random; 6, 7: large finger angles (up to 2.5 rad)
    pose[2:6] = torch.randn(4, 66, generator=g, dtype=torch.float64) * 0.3
    rest[2:6] = torch.randn(4, 99, generator=g, dtype=torch.float64) * 0.3
    transl[2:6] = torch.randn(4, 3, generator=g, dtype=torch.float64) * 0.2
    pose[6:] = torch.randn(2, 66, generator=g, dtype=torch.float64) * 0.2
    rest[6:, :9] = torch.randn(2, 9, generator=g, dtype=torch.float64) * 0.2
    rest[6:, 9:] = (torch.rand(2, 90, generator=g, dtype=torch.float64) * 2 - 1) * 2.5
    pose, rest, transl = pose.float().double(), rest.float().double(), transl.float().double()     # exact in fp32 too
    betas = body.betas.double().expand(B, -1).contiguous()
    with tempfile.TemporaryDirectory() as tmp:
        syn.write_smplx_model_npz(os.path.join(tmp, "SMPLX_NEUTRAL.npz"), body, seed=0, posedirs=syn.smplx_posedirs(0), faces=template[1])
        m = ref_smplx.SMPLX(model_path=tmp, gender="neutral", use_pca=False, num_pca_comps=45, flat_hand_mean=True, batch_size=B,
                            dtype=torch.float64).eval()
        assert float(m.pose_mean.abs().sum()) == 0.0 and float(m.posedirs.abs().sum()) > 0
        with torch.no_grad():
            out = m.forward(betas=betas, global_orient=pose[:, :3], transl=transl, body_pose=pose[:, 3:66], jaw_pose=rest[:, :3],
                            leye_pose=rest[:, 3:6], reye_pose=rest[:, 6:9], left_hand_pose=rest[:, 9:54], right_hand_pose=rest[:, 54:])
    v = out.vertices.numpy()
    np.savez_compressed(os.path.join(OUT, "cano_smplx_vertices.npz"), betas=body.betas[0].numpy(), pose66=pose.float().numpy(),
                        rest99=rest.float().numpy(), transl=transl.float().numpy(), A=out.A.numpy(), body_seed=0, **_summary(v, 6))


def gen_cano_smpl():
    from submodules import smplx as ref_smplx
    cpose, _ = _cpose()
    body = syn.make_body(0)
    with tempfile.TemporaryDirectory() as tmp:
        with open(os.path.join(tmp, "SMPL_NEUTRAL.pkl"), "wb") as fh:
            pickle.dump(syn.smpl_mesh_model(body, syn.make_uv_template(0)), fh)
        m = ref_smplx.SMPL(model_path=tmp, gender="neutral", batch_size=1, dtype=torch.float64).eval()
        with torch.no_grad():       # scripts/gen_pose_map_cano_smpl.py:60-66
            out = m.forward(betas=body.betas.double(), global_orient=cpose[:, :3].double(), transl=torch.tensor([[0, 0.30, 0]]).double(),
                            body_pose=cpose[:, 3:].double())
    v = out.vertices.numpy()
    np.savez_compressed(os.path.join(OUT, "cano_smpl.npz"), betas=body.betas[0].numpy(), pose=cpose.numpy(), transl=np.array([[0, 0.30, 0]], np.float32),
                        A=out.A.numpy(), body_seed=0, **_summary(v, 7))


def gen_cano_lbs_weights():
    from utils.general_utils import gen_lbs_weight_from_ori, get_face_per_pixel
    res = {}
    for name, body, template in (("smpl", syn.make_body(0), syn.make_uv_template(0)),
                                 ("smplx", syn.make_smplx_body(0), syn.make_smplx_uv_template(0))):
        face_id, bary = po.layout(template[2].astype(np.float32)[template[3]], W_SIZE)
        faces_px = get_face_per_pixel(torch.from_numpy(face_id).long(), torch.from_numpy(template[1]).long())
        w = gen_lbs_weight_from_ori(body.lbs_weights.float(), torch.from_numpy(bary), faces_px)
        res.update({f"{name}/face_id": face_id, f"{name}/bary": bary, f"{name}/lbs_map": w.numpy()})
    np.savez_compressed(os.path.join(OUT, "cano_lbs_weights.npz"), S=W_SIZE, **res)


GENERATORS = (gen_cano_smplx, gen_cano_smpl, gen_cano_lbs_weights)
FILES = ("cano_smplx_vertices.npz", "cano_smpl.npz", "cano_lbs_weights.npz")

if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    names = sys.argv[1:] or [g.__name__ for g in GENERATORS]
    for name in names:
        globals()[name]()
    for f in FILES:
        print(f, os.path.getsize(os.path.join(OUT, f)))
