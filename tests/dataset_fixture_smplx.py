"""Writes a small synthetic SMPL-X dataset folder in the reference's layout (scene/dataset_mono.py:83-96 + the SMPL-X assets
model/avatar_model.py:45-53 reads): `smpl_parms.pth` with a [F,165] body_pose (pose 66 | rest_pose 99), the `_smplx` UV mask,
canonical position map, LBS map [S,S,55], canonical joint matrices [55,4,4] and a synthetic SMPLX_NEUTRAL.npz.  Deterministic from a
seed.  Test helper, not product."""
import os
from os.path import join

import numpy as np
import torch
from PIL import Image

from gaussianavatar_b200 import synthetic as syn
from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, TEST_POSE_K, scaled_intrinsics
from gaussianavatar_b200.config import ModelParams


def smplx_body_pose(num_frames, seed):
    pose, rest, transl = syn.synthetic_smplx_poses(num_frames, seed=seed)
    return torch.cat([pose, rest], 1), transl


def write_synthetic_smplx_dataset(root, N=600, S=32, num_frames=5, side=64, inp=16, seed=0, stage2=False) -> ModelParams:
    g = np.random.default_rng(seed)
    a = syn.make_avatar_assets(N, S, seed=seed, body="smplx")
    body_pose, transl = smplx_body_pose(num_frames, seed)
    K = scaled_intrinsics(TEST_POSE_K, side)
    project, source, testf, smplx_dir = join(root, "project"), join(root, "data"), join(root, "novel"), join(root, "smplx_models")
    for split in ("train", "test"):
        d = join(source, split)
        os.makedirs(join(d, "images"), exist_ok=True); os.makedirs(join(d, "masks"), exist_ok=True)
        for f in range(num_frames):
            img = g.integers(0, 256, size=(side, side, 3), dtype=np.uint8)
            yy, xx = np.mgrid[0:side, 0:side]
            mask = (((yy - side / 2) ** 2 + (xx - side / 2 - f) ** 2) < (side / 3) ** 2).astype(np.uint8) * 255
            Image.fromarray(img, "RGB").save(join(d, "images", f"{f:05d}.png"))
            Image.fromarray(mask, "L").save(join(d, "masks", f"{f:05d}.png"))
        np.savez(join(d, "cam_parms.npz"), intrinsic=K, extrinsic=TEST_POSE_EXTRINSIC)
        smpl = dict(beta=a.body.betas.clone(), body_pose=body_pose.clone(), trans=transl.clone())
        torch.save(smpl, join(d, "smpl_parms.pth")); torch.save(smpl, join(d, "smpl_parms_pred.pth"))
        posmap = np.zeros((S * S, 3), np.float32); posmap[a.valid_idx.numpy()] = a.query_points.numpy()
        np.savez(join(d, f"query_posemap_{S}_cano_smplx.npz"), **{f"posmap{S}": posmap.reshape(S, S, 3)})
        torch.save(a.cano_joint_mats.clone(), join(d, "smplx_cano_joint_mat.pth"))
        if stage2:
            os.makedirs(join(d, "inp_map"), exist_ok=True)
            for f in range(num_frames):
                pm = g.normal(0, 0.3, size=(inp, inp, 3)).astype(np.float32)
                np.savez(join(d, "inp_map", "inp_posemap_%s_%s.npz" % (str(inp), str(f).zfill(8))), **{f"posmap{inp}": pm})
    os.makedirs(testf, exist_ok=True)
    np.savez(join(testf, "cam_parms.npz"), intrinsic=TEST_POSE_K, extrinsic=TEST_POSE_EXTRINSIC)
    npose, ntransl = smplx_body_pose(4, seed + 1)
    torch.save(dict(beta=a.body.betas.clone(), body_pose=npose, trans=ntransl), join(testf, "smpl_parms.pth"))
    os.makedirs(join(project, "assets", "uv_masks"), exist_ok=True)
    uv = np.full(S * S, -1, np.int32); uv[a.valid_idx.numpy()] = np.arange(N) % 20908     # face ids; -1 = not on the body
    np.save(join(project, "assets", "uv_masks", f"uv_mask{S}_with_faceid_smplx.npy"), uv.reshape(S, S))
    lbs = np.zeros((S * S, 55), np.float32); lbs[a.valid_idx.numpy()] = a.query_lbs.numpy()
    np.save(join(project, "assets", f"lbs_map_smplx_{S}.npy"), lbs.reshape(S, S, 55))
    os.makedirs(smplx_dir, exist_ok=True)
    syn.write_smplx_model_npz(join(smplx_dir, "SMPLX_NEUTRAL.npz"), a.body, seed=seed)
    return ModelParams(source_path=source, model_path=join(root, "out"), project_path=project, smplx_model_path=smplx_dir, test_folder=testf,
                       smpl_type="smplx", train_stage=2 if stage2 else 1, query_posmap_size=S, inp_posmap_size=inp, batch_size=2)
