"""Stage-2 input position maps of a data folder, written on the GPU in the reference's file format.

    python tools/pose_maps.py FOLDER --smpl_model SMPL_NEUTRAL.pkl --uv_template template_mesh_smpl_uv.obj --size 128
    python tools/pose_maps.py FOLDER ... --check [--uv_mask uv_mask128_with_faceid_smpl.npy]

Reads the SMPL parameters of FOLDER (smpl_parms_pred.pth if it exists, which is what the stage-2 datasets read, else
smpl_parms.pth; or --params), builds every frame's map with gaussianavatar_b200.posmap.PoseMapper and writes
FOLDER/inp_map/inp_posemap_{S}_{idx:08d}.npz with the key posmap{S}, [S,S,3] float32: the files the reference's
scripts/gen_pose_map_our_smpl.py renders with OpenGL.

--check writes nothing: it compares the maps with the files already in FOLDER/inp_map (and the face ids with --uv_mask, the
reference's uv_mask{S}_with_faceid_smpl.npy) and prints one JSON line with the largest absolute map difference and the number of
texels whose face id differs.
"""
import argparse
import json
import os
import pickle
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gaussianavatar_b200.posmap import PoseMapper  # noqa: E402

CHUNK = 64      # frames per device call


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("folder")
    ap.add_argument("--smpl_model", required=True, help="SMPL_{GENDER}.pkl")
    ap.add_argument("--uv_template", required=True, help="template_mesh_smpl_uv.obj")
    ap.add_argument("--size", type=int, default=128)
    ap.add_argument("--params", default=None, help="SMPL parameter file in FOLDER (default: smpl_parms_pred.pth, else smpl_parms.pth)")
    ap.add_argument("--check", action="store_true", help="compare with the existing files instead of writing")
    ap.add_argument("--uv_mask", default=None, help="with --check: uv_mask{S}_with_faceid_smpl.npy to compare the face ids with")
    a = ap.parse_args(argv)
    S = a.size
    params = a.params or ("smpl_parms_pred.pth" if os.path.exists(os.path.join(a.folder, "smpl_parms_pred.pth")) else "smpl_parms.pth")
    smpl_data = torch.load(os.path.join(a.folder, params), weights_only=False)
    pose = torch.as_tensor(smpl_data["body_pose"]).float()
    transl = torch.as_tensor(smpl_data["trans"]).float()
    beta = torch.as_tensor(smpl_data["beta"]).float().reshape(-1, 10)[0]
    with open(a.smpl_model, "rb") as fh:
        sm = pickle.load(fh, encoding="latin1")
    mapper = PoseMapper(sm, beta, a.uv_template, S)
    out_dir = os.path.join(a.folder, "inp_map")
    if not a.check:
        os.makedirs(out_dir, exist_ok=True)
    max_err, n_missing = 0.0, 0
    for s in range(0, pose.shape[0], CHUNK):
        maps = mapper(pose[s:s + CHUNK], transl[s:s + CHUNK]).permute(0, 2, 3, 1).cpu().numpy()      # [b,S,S,3]
        for i, m in enumerate(maps):
            fn = os.path.join(out_dir, "inp_posemap_%s_%s.npz" % (S, str(s + i).zfill(8)))
            if a.check:
                if not os.path.exists(fn):
                    n_missing += 1
                    continue
                ref = np.load(fn)[f"posmap{S}"]
                max_err = max(max_err, float(np.abs(ref.astype(np.float64) - m).max()))
            else:
                np.savez(fn, **{f"posmap{S}": np.ascontiguousarray(m, np.float32)})
    if not a.check:
        print(json.dumps(dict(written=int(pose.shape[0]), folder=out_dir, size=S)))
        return 0
    res = dict(frames=int(pose.shape[0]), missing_files=n_missing, max_abs_map_error=max_err, size=S)
    if a.uv_mask:
        ref_id = np.load(a.uv_mask).reshape(S, S)
        res["face_id_mismatches"] = int((ref_id != mapper.face_id.cpu().numpy()).sum())
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
