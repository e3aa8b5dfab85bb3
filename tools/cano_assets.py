"""A subject's canonical assets for SMPL or SMPL-X, built on the GPU in the reference's file formats (no OpenGL).

    python tools/cano_assets.py FOLDER --body smpl  --model SMPL_NEUTRAL.pkl  --uv_template template_mesh_smpl_uv.obj  --size 512
    python tools/cano_assets.py FOLDER --body smplx --model SMPLX_NEUTRAL.npz --uv_template template_mesh_smplx_uv.obj --size 512
    python tools/cano_assets.py FOLDER ... --check

Reads `beta` from FOLDER/smpl_parms.pth, builds everything with gaussianavatar_b200.posmap.canonical_assets and writes

  FOLDER/query_posemap_{S}_cano_{body}.npz           key posmap{S}, [S,S,3] float32 (scripts/gen_pose_map_cano_smpl.py renders it)
  FOLDER/{body}_cano_joint_mat.pth                   [1,J,4,4] float32, the canonical pose's A (the same script's torch.save)
  ASSETS/uv_masks/uv_mask{S}_with_faceid_{body}.npy  [S,S] int32 face ids, -1 for background
  ASSETS/lbs_map_{body}_{S}.npy                      [S,S,J] float32 texel skinning weights
  ASSETS/bary_coords_uv_map/bary_coords_{body}_uv{S}.npy  [S,S,3] float32 barycentric weights

ASSETS is --assets, by default ./assets (the reference reads its assets under the working directory).  FOLDER is the split folder
AvatarModel reads (e.g. data/subject/train).  The coverage of the face-id mask follows the library's rules, not GL's (DESIGN.md,
PARITY UNPINNED).

--check writes nothing: it compares with the files already present and prints one JSON line with the largest absolute difference
of each file, the largest of them, the number of texels whose face id differs and the files that are missing.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gaussianavatar_b200.body import load_model  # noqa: E402
from gaussianavatar_b200.posmap import canonical_assets  # noqa: E402


def output_paths(folder, assets, body, S):
    return dict(posmap=os.path.join(folder, f"query_posemap_{S}_cano_{body}.npz"),
                joint_mats=os.path.join(folder, f"{body}_cano_joint_mat.pth"),
                face_id=os.path.join(assets, "uv_masks", f"uv_mask{S}_with_faceid_{body}.npy"),
                lbs_map=os.path.join(assets, f"lbs_map_{body}_{S}.npy"),
                bary=os.path.join(assets, "bary_coords_uv_map", f"bary_coords_{body}_uv{S}.npy"))


def _load(key, path, S):
    if key == "posmap":
        return np.load(path)[f"posmap{S}"]
    if key == "joint_mats":
        return torch.as_tensor(torch.load(path, weights_only=False)).numpy()
    return np.load(path)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("folder")
    ap.add_argument("--body", choices=("smpl", "smplx"), default="smpl")
    ap.add_argument("--model", required=True, help="SMPL_{GENDER}.pkl or SMPLX_{GENDER}.npz")
    ap.add_argument("--uv_template", required=True, help="the body's UV template OBJ")
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--assets", default=os.path.join(os.getcwd(), "assets"), help="assets directory (default: ./assets)")
    ap.add_argument("--check", action="store_true", help="compare with the existing files instead of writing")
    a = ap.parse_args(argv)
    S = a.size
    for path in (os.path.join(a.folder, "smpl_parms.pth"), a.model, a.uv_template):
        if not os.path.exists(path):
            ap.error(f"{path} not found")
    beta = torch.as_tensor(torch.load(os.path.join(a.folder, "smpl_parms.pth"), weights_only=False)["beta"]).float().reshape(-1, 10)[0]
    res = canonical_assets(load_model(a.model), beta, a.uv_template, S, body=a.body)
    got = dict(posmap=res.posmap.cpu().numpy(), joint_mats=res.joint_mats[None].cpu().numpy(), face_id=res.face_id.cpu().numpy(),
               lbs_map=res.lbs_map.cpu().numpy(), bary=res.bary.cpu().numpy())
    paths = output_paths(a.folder, a.assets, a.body, S)
    if a.check:
        out = dict(body=a.body, size=S, missing_files=[], max_abs_error={})
        for key, path in paths.items():
            if not os.path.exists(path):
                out["missing_files"].append(path)
                continue
            ref = _load(key, path, S)
            if key == "face_id":
                out["face_id_mismatches"] = int((ref.reshape(S, S) != got[key]).sum())
            else:
                out["max_abs_error"][key] = float(np.abs(ref.astype(np.float64).reshape(got[key].shape) - got[key]).max())
        out["max_abs_error_all"] = max(out["max_abs_error"].values(), default=0.0)
        print(json.dumps(out))
        return 0
    for path in paths.values():
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    np.savez(paths["posmap"], **{f"posmap{S}": got["posmap"]})
    torch.save(torch.from_numpy(got["joint_mats"]), paths["joint_mats"])
    np.save(paths["face_id"], got["face_id"])
    np.save(paths["lbs_map"], got["lbs_map"])
    np.save(paths["bary"], got["bary"])
    print(json.dumps(dict(body=a.body, size=S, covered_texels=int((got["face_id"] >= 0).sum()), written=list(paths.values()))))
    return 0


if __name__ == "__main__":
    sys.exit(main())
