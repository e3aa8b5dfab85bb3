"""Fit the SMPL / SMPL-X poses of a split's frames to its images through a trained avatar, before eval.py renders them.

    python tools/fit_poses.py -s DATA -m MODEL --epoch N --stage 1 --body smpl
    python tools/fit_poses.py -s DATA -m MODEL --epoch N --stage 2 --body smplx --smpl_model SMPLX_NEUTRAL.npz \
        --uv_template template_mesh_smplx_uv.obj --iters 100

DATA / MODEL are the reference's -s / -m folders; stage 1 loads net/iteration_N/net.pth (`load`), stage 2 pose_encoder.pth
(`stage2_load`).  The split's poses come from the file its stage's dataset reads (stage 1: smpl_parms.pth, stage 2:
smpl_parms_pred.pth); stage 2 builds its input maps from the pose being fitted and never reads inp_map/.  Writes
DATA/<split>/smpl_parms_fit.pth in the input file's format ({beta, body_pose, trans}; SMPL-X's rest columns copied unchanged) and
DATA/<split>/smpl_parms_fit.json (per-frame initial and fitted loss, best iteration).  --exposure also fits each frame's colour
transform [A | t] and adds it to the pose file as `exposure` [F,3,4]; the test dataset's items then carry it and render_free_stage1 /
render_free_stage2 apply it.  The input file is never overwritten.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

OUT_NAME = "smpl_parms_fit.pth"
REPORT_NAME = "smpl_parms_fit.json"


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("-s", "--source_path", required=True)
    ap.add_argument("-m", "--model_path", required=True)
    ap.add_argument("--project_path", default=os.getcwd(), help="folder holding assets/ (UV masks, LBS maps)")
    ap.add_argument("--epoch", type=int, required=True)
    ap.add_argument("--stage", type=int, choices=(1, 2), default=1)
    ap.add_argument("--body", choices=("smpl", "smplx"), default="smpl")
    ap.add_argument("--split", default="test", help="the folder under DATA whose frames are fitted")
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--lr", type=float, default=5e-3)
    ap.add_argument("--smpl_model", default=None, help="SMPL_{GENDER}.pkl / SMPLX_{GENDER}.npz (its folder is the model path)")
    ap.add_argument("--smpl_gender", default="neutral")
    ap.add_argument("--uv_template", default=None, help="stage 2: the body's UV template OBJ")
    ap.add_argument("--query_posmap_size", type=int, default=512)
    ap.add_argument("--inp_posmap_size", type=int, default=128)
    ap.add_argument("--nf", type=int, default=32, help="stage 2: the pose encoder's base width")
    ap.add_argument("--white_background", type=int, choices=(0, 1), default=1)
    ap.add_argument("--antialiasing", action="store_true", help="render with 3DGS's antialiasing setting (for an avatar trained with it)")
    ap.add_argument("--exposure", action="store_true", help="also fit each frame's exposure and white balance [A | t]")
    a = ap.parse_args(argv)
    if a.iters < 0:
        ap.error(f"--iters {a.iters} is negative")
    if not a.lr > 0:
        ap.error(f"--lr {a.lr} is not positive")
    if a.stage == 2 and not (a.smpl_model and a.uv_template):
        ap.error("--stage 2 needs --smpl_model and --uv_template for the input position maps")
    if not os.path.isdir(os.path.join(a.source_path, a.split)):
        ap.error(f"no split folder {os.path.join(a.source_path, a.split)}")
    if not os.path.exists(input_path(a)):
        ap.error(f"no pose file {input_path(a)}")
    return a


def input_path(a):
    return os.path.join(a.source_path, a.split, "smpl_parms.pth" if a.stage == 1 else "smpl_parms_pred.pth")


def write_fit(src, dst, pose, transl, exposure=None):
    """Copy of the pose file `src` with body_pose[:n, :pose width] and trans[:n] replaced by the fitted rows; every other entry and
    column (beta, SMPL-X's rest columns, frames past n) unchanged.  exposure [n,3,4]: stored as `exposure` [F,3,4], identity past n."""
    if os.path.abspath(src) == os.path.abspath(dst):
        raise ValueError(f"{dst}: the fit must not overwrite its input")
    d = dict(torch.load(src, map_location="cpu", weights_only=False))
    body = torch.as_tensor(d["body_pose"]).clone()
    trans = torch.as_tensor(d["trans"]).clone()
    n, w = pose.shape
    body[:n, :w] = pose.to(body.dtype)
    trans[:n] = transl.to(trans.dtype)
    d["body_pose"], d["trans"] = body, trans
    if exposure is not None:
        table = torch.eye(3, 4).repeat(body.shape[0], 1, 1)
        table[:n] = exposure.float()
        d["exposure"] = table
    torch.save(d, dst)


def main(argv=None):
    a = parse_args(argv)
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import ModelParams, NetworkParams, OptimizationParams
    from gaussianavatar_b200.dataset import MonoDataset_test
    from gaussianavatar_b200.posefit import PoseFitter

    model_dir = os.path.dirname(os.path.abspath(a.smpl_model)) if a.smpl_model else ""
    mp = ModelParams(source_path=a.source_path, model_path=a.model_path, project_path=a.project_path, smpl_model_path=model_dir,
                     smplx_model_path=model_dir, smpl_gender=a.smpl_gender, smpl_type=a.body, train_stage=a.stage,
                     query_posmap_size=a.query_posmap_size, inp_posmap_size=a.inp_posmap_size, batch_size=1,
                     white_background=bool(a.white_background), antialiasing=bool(a.antialiasing))
    model = AvatarModel(mp, NetworkParams(nf=a.nf), OptimizationParams(), train=False)
    pose_mapper = None
    if a.stage == 1:
        model.load(a.epoch)
    else:
        model.stage2_load(a.epoch)
        from gaussianavatar_b200.body import load_model
        from gaussianavatar_b200.posmap import PoseMapper
        pose_mapper = PoseMapper(load_model(a.smpl_model), model.betas[0], a.uv_template, a.inp_posmap_size, device=model.device,
                                 body=model.body)

    # the maps come from the pose being fitted: the dataset need not read inp_map/
    dmp = ModelParams(**{**vars(mp), "inp_posmap_from_pose": True})
    dataset = type("SplitDataset", (MonoDataset_test,), {"split": a.split})(dmp)
    frames = [dataset[i] for i in range(len(dataset))]
    fitter = PoseFitter(model, iters=a.iters, lr=a.lr, pose_mapper=pose_mapper, exposure=a.exposure)
    pose, transl, report, *exposure = fitter.fit(frames)

    split_dir = os.path.join(a.source_path, a.split)
    write_fit(input_path(a), os.path.join(split_dir, OUT_NAME), pose, transl, exposure[0] if exposure else None)
    with open(os.path.join(split_dir, REPORT_NAME), "w") as fh:
        json.dump(dict(stage=a.stage, body=a.body, iters=a.iters, lr=a.lr, exposure=a.exposure, frames=report), fh, indent=1)
    init = sum(r["initial_loss"] for r in report) / max(1, len(report))
    fit = sum(r["fitted_loss"] for r in report) / max(1, len(report))
    print(json.dumps(dict(frames=len(report), mean_initial_loss=round(init, 6), mean_fitted_loss=round(fit, 6),
                          out=os.path.join(split_dir, OUT_NAME))))
    return 0


if __name__ == "__main__":
    sys.exit(main())
