"""Write the stage-1-refined SMPL / SMPL-X poses of a checkpoint into a data folder (the reference's
scripts/export_stage_1_smpl.py).

    python tools/export_stage1_poses.py OUT/net/iteration_200 DATA/train
    python tools/export_stage1_poses.py OUT/net/iteration_200 DATA/train --body smplx

Reads CKPT_DIR/net.pth["pose"] / ["transl"] (the `pose` / `transl` embedding state dicts that AvatarModel.save and the reference's
save write) and FOLDER/smpl_parms.pth, and writes FOLDER/smpl_parms_pred.pth: the same dict with the first F rows of body_pose and
trans replaced by the F refined rows, everything else kept.  SMPL trains all 72 pose columns; SMPL-X trains the global and body
pose (66 columns), so only body_pose[:F, :66] is replaced and the jaw, eye and hand pose [66:] is kept.  Plain torch, no GPU.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gaussianavatar_b200.body import body_of  # noqa: E402


def export(ckpt_dir, folder, body="smpl"):
    saved = torch.load(os.path.join(ckpt_dir, "net.pth"), map_location="cpu", weights_only=False)
    pose = torch.as_tensor(saved["pose"]["weight"]).detach().float()
    transl = torch.as_tensor(saved["transl"]["weight"]).detach().float()
    smpl = torch.load(os.path.join(folder, "smpl_parms.pth"), map_location="cpu", weights_only=False)
    bp = torch.as_tensor(smpl["body_pose"]).clone()
    tr = torch.as_tensor(smpl["trans"]).clone()
    width = body_of(body).pose_width
    F = pose.shape[0]
    if pose.dim() != 2 or pose.shape[1] != width or tuple(transl.shape) != (F, 3):
        raise ValueError(f"checkpoint pose {tuple(pose.shape)} / transl {tuple(transl.shape)}: expected [F,{width}] / [F,3] for {body}")
    if bp.dim() != 2 or bp.shape[1] < width or bp.shape[0] < F or tr.shape[0] < F:
        raise ValueError(f"smpl_parms.pth body_pose {tuple(bp.shape)} / trans {tuple(tr.shape)} cannot take {F} rows of {width} columns")
    bp[:F, :width] = pose.to(bp.dtype)
    tr[:F] = transl.to(tr.dtype)
    smpl["body_pose"], smpl["trans"] = bp, tr
    out = os.path.join(folder, "smpl_parms_pred.pth")
    torch.save(smpl, out)
    return out, F


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("ckpt_dir", help="directory holding net.pth")
    ap.add_argument("folder", help="data folder holding smpl_parms.pth")
    ap.add_argument("--body", choices=("smpl", "smplx"), default="smpl")
    a = ap.parse_args(argv)
    out, F = export(a.ckpt_dir, a.folder, a.body)
    print(json.dumps(dict(written=out, frames=F, body=a.body)))
    return 0


if __name__ == "__main__":
    sys.exit(main())
