"""ORACLE — TEST INFRASTRUCTURE ONLY.  Generates the SMPL-X fixtures tests/golden/smplx_A.npz and tests/golden/dataset_items_smplx.npz
by importing the UNMODIFIED reference modules from /root/reference (read-only, never copied).  Run in the build container only (the
GPU box has no /root/reference):

    python oracle/gen_golden_smplx.py                      # both fixtures
    python oracle/gen_golden_smplx.py gen_smplx_A          # only the named generators

The model file the reference loads is the synthetic SMPLX_NEUTRAL.npz of gaussianavatar_b200.synthetic (no licensed asset needed).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)
OUT = os.path.join(ROOT, "tests", "golden")

from gaussianavatar_b200 import synthetic as syn          # noqa: E402


def gen_smplx_A():
    """The reference's own `smplx.SMPLX` (use_pca=False, flat_hand_mean=True, as model/avatar_model.py:46 builds it) on the synthetic
    SMPLX_NEUTRAL.npz, called with the argument split of model/avatar_model.py:281-289: T-pose, star pose, random poses and large
    finger angles.  Stores the inputs, the reference's rest joints J_regressor (v_template + shapedirs beta) and A."""
    import tempfile
    from submodules import smplx as ref_smplx
    from submodules.smplx.lbs import blend_shapes, vertices2joints
    body = syn.make_smplx_body(0)
    g = torch.Generator().manual_seed(21)
    pose = torch.zeros(10, 66); rest = torch.zeros(10, 99); transl = torch.zeros(10, 3)
    pose[1] = torch.tensor(syn.star_pose()[:66]).float()                                  # star pose
    pose[2:8] = torch.randn(6, 66, generator=g) * 0.3                                     # random
    rest[2:8] = torch.randn(6, 99, generator=g) * 0.3
    transl[1:8] = torch.randn(7, 3, generator=g) * 0.2
    pose[8:] = torch.randn(2, 66, generator=g) * 0.2                                      # large finger angles (up to ~2.5 rad)
    rest[8:, :9] = torch.randn(2, 9, generator=g) * 0.2
    rest[8:, 9:] = (torch.rand(2, 90, generator=g) * 2 - 1) * 2.5
    B = pose.shape[0]
    betas = body.betas.expand(B, -1).contiguous()
    with tempfile.TemporaryDirectory() as tmp:
        syn.write_smplx_model_npz(os.path.join(tmp, "SMPLX_NEUTRAL.npz"), body, seed=0)
        m = ref_smplx.SMPLX(model_path=tmp, gender="neutral", use_pca=False, num_pca_comps=45, flat_hand_mean=True, batch_size=B).eval()
        assert float(m.pose_mean.abs().sum()) == 0.0
        with torch.no_grad():
            out = m.forward(betas=betas, global_orient=pose[:, :3], transl=transl, body_pose=pose[:, 3:66], jaw_pose=rest[:, :3],
                            leye_pose=rest[:, 3:6], reye_pose=rest[:, 6:9], left_hand_pose=rest[:, 9:54], right_hand_pose=rest[:, 54:])
            J = vertices2joints(m.J_regressor, m.v_template[None] + blend_shapes(betas[:1], m.shapedirs))[0]
        parents = m.parents.numpy()
    np.savez_compressed(os.path.join(OUT, "smplx_A.npz"), betas=body.betas[0].numpy(), pose66=pose.numpy(), rest99=rest.numpy(),
                        transl=transl.numpy(), rest_joints=J.numpy(), A=out.A.numpy(), parents=parents, body_seed=0)


def gen_dataset_items_smplx():
    """Items of the reference's own dataset classes (scene/dataset_mono.py) on the synthetic SMPL-X folder tests/dataset_fixture_smplx.py
    writes: every item of the training, test and novel-pose sets, including `rest_pose`."""
    import tempfile
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from dataset_fixture_smplx import write_synthetic_smplx_dataset
    from scene import dataset_mono as ref
    _orig = ref.getProjectionMatrix
    ref.getProjectionMatrix = lambda **kw: _orig(**{**kw, "K": np.asarray(kw["K"]).astype(np.float64)})
    fields = ("original_image", "world_view_transform", "projection_matrix", "full_proj_transform", "camera_center")
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        mp = write_synthetic_smplx_dataset(tmp)
        mp.no_mask = 1      # as gen_dataset_items: the reference's masked branch does not run under this image's Pillow
        sets = dict(train=ref.MonoDataset_train(mp, device="cpu"), test=ref.MonoDataset_test(mp, device="cpu"),
                    novel_pose=ref.MonoDataset_novel_pose(mp, device="cpu"))
        for name, dset in sets.items():
            out[f"{name}/len"] = np.array(len(dset))
            for i in range(len(dset)):
                item = dset[i]
                for k in fields + ("pose_data", "transl_data", "rest_pose"):
                    if k in item:
                        out[f"{name}/{i}/{k}"] = np.asarray(item[k], dtype=np.float64)
                if "original_image" in item:
                    img = np.asarray(item["original_image"], dtype=np.float32).reshape(-1)
                    out[f"{name}/{i}/original_image"] = img[np.random.default_rng(i).choice(img.size, 64, replace=False)]
                out[f"{name}/{i}/scalars"] = np.array([item["FovX"], item["FovY"], item["width"], item["height"], item["pose_idx"]], dtype=np.float64)
    np.savez_compressed(os.path.join(OUT, "dataset_items_smplx.npz"), **out)


GENERATORS = (gen_smplx_A, gen_dataset_items_smplx)

if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    names = sys.argv[1:] or [g.__name__ for g in GENERATORS]
    for name in names:
        globals()[name]()
    for f in ("smplx_A.npz", "dataset_items_smplx.npz"):
        print(f, os.path.getsize(os.path.join(OUT, f)))
