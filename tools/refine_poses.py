"""Turn a monocular capture with raw SMPL estimates into a training folder: refine every frame's pose against its mask with the
library's soft silhouette (`silhouette.PoseRefiner`), then split the frames and write them in the reference's data layout.  Stands in
for InstantAvatar's pose preprocessing plus the reference's scripts/sample_romp2gsavatar.py (without pytorch3d, OpenGL or that
script's hard-coded paths).

    python tools/refine_poses.py CAPTURE --smpl_model SMPL_NEUTRAL.pkl --out DATA [--iters 100 --sigma 1 --lambda_smooth 0 --lambda_prior 0]

CAPTURE holds images/, masks/ (same file names as the images; >= 128 is the subject), cameras.npz (intrinsic, extrinsic) and the
poses (--poses, default poses.npz): betas (10 values), transl, and global_orient + body_pose or thetas [N,72].  Frames are taken in
sorted image-name order.  Writes CAPTURE/poses_optimized.npz (the input's keys, refined values), then DATA/train and DATA/test, each
with images/, masks/, cam_parms.npz and smpl_parms.pth (beta [1,10], body_pose [F,72], trans [F,3]).  The split is InstantAvatar's:
N // 5 validation frames every `length` frames from offset length // 2; the first half of them is the test split, the rest is
dropped, and every other frame is a training frame.  --iters 0 refines nothing (the conversion alone, no GPU needed).  Prints one
JSON line: frame counts, the objective and the mean hard IoU (ga_mesh_render coverage against the masks) before and after.
"""
import argparse
import json
import os
import shutil
import sys

import numpy as np
import torch
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def split(n: int):
    """(train indices, test indices) of an n-frame capture."""
    num_val = n // 5
    if num_val == 0:
        raise ValueError(f"{n} frames: the split needs at least 5")
    length = int(1 / num_val * n)
    val = list(range(n))[length // 2::length]
    held = set(val)
    train = [i for i in range(n) if i not in held]
    return train, val[:len(val) // 2]


def thetas(poses: dict) -> np.ndarray:
    """[N,72] float32: global_orient | body_pose, or thetas."""
    if "thetas" in poses:
        return np.asarray(poses["thetas"], np.float32).reshape(-1, 72)
    return np.concatenate([np.asarray(poses["global_orient"], np.float32).reshape(-1, 3),
                           np.asarray(poses["body_pose"], np.float32).reshape(-1, 69)], 1)


def smpl_parms(poses: dict, theta: np.ndarray, idx) -> dict:
    return dict(beta=torch.from_numpy(np.asarray(poses["betas"], np.float32).reshape(1, 10).copy()),
                body_pose=torch.from_numpy(theta[idx].copy()).reshape(len(idx), 72),
                trans=torch.from_numpy(np.asarray(poses["transl"], np.float32).reshape(-1, 3)[idx].copy()).reshape(len(idx), 3))


def read_mask(path) -> np.ndarray:
    m = np.array(Image.open(path))
    return (m if m.ndim == 2 else m[..., 0]).astype(np.uint8)


def refine(a, names, poses, theta):
    """Refined theta [N,72] and transl [N,3] and the report of `PoseRefiner`."""
    from gaussianavatar_b200.camera import make_camera
    from gaussianavatar_b200.mesh_render import cameras
    from gaussianavatar_b200.body import load_model
    from gaussianavatar_b200.posmap import BodyPoser
    from gaussianavatar_b200.silhouette import PoseRefiner, SilhouetteRenderer
    cam = np.load(os.path.join(a.capture, "cameras.npz"))
    masks = np.stack([read_mask(os.path.join(a.capture, "masks", n)) for n in names])
    H, W = masks.shape[1:]
    poser = BodyPoser(load_model(a.smpl_model), torch.from_numpy(np.asarray(poses["betas"], np.float32).reshape(-1)[:10].copy()))
    renderer = SilhouetteRenderer(poser.faces, poser.V, sigma=a.sigma, device=poser.device)
    refiner = PoseRefiner(poser, renderer, iters=a.iters, lr=a.lr, lambda_smooth=a.lambda_smooth, lambda_prior=a.lambda_prior)
    K, extr = np.asarray(cam["intrinsic"]).reshape(3, 3), np.asarray(cam["extrinsic"])
    cams = cameras([make_camera(K, extr, H, W)])[0]
    transl = np.asarray(poses["transl"], np.float32).reshape(-1, 3)[:len(names)]
    pose, tr, report = refiner.refine(torch.from_numpy(theta[:len(names)].copy()), torch.from_numpy(transl.copy()), cams,
                                      torch.from_numpy(masks))
    return pose.numpy(), tr.numpy(), report


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("capture")
    ap.add_argument("--smpl_model", default=None, help="SMPL_{GENDER}.pkl (needed when --iters > 0)")
    ap.add_argument("--out", required=True)
    ap.add_argument("--poses", default="poses.npz", help="pose file in CAPTURE")
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--lr", type=float, default=1e-2)
    ap.add_argument("--sigma", type=float, default=1.0, help="silhouette softness, pixels^2")
    ap.add_argument("--lambda_smooth", type=float, default=0.0)
    ap.add_argument("--lambda_prior", type=float, default=0.0)
    a = ap.parse_args(argv)
    if a.iters < 0:
        ap.error("--iters must be >= 0")
    if a.iters > 0 and not a.smpl_model:
        ap.error("--smpl_model is needed to refine (--iters > 0)")
    names = sorted(os.listdir(os.path.join(a.capture, "images")))
    n = len(names)
    missing = [x for x in names if not os.path.exists(os.path.join(a.capture, "masks", x))]
    if missing:
        raise FileNotFoundError(f"masks/ has no {missing[0]} (masks must have the images' file names)")
    with np.load(os.path.join(a.capture, a.poses)) as z:
        poses = {k: z[k] for k in z.files}
    theta = thetas(poses)
    if theta.shape[0] < n:
        raise ValueError(f"{n} images but {theta.shape[0]} poses in {a.poses}")
    train, test = split(n)
    result = dict(frames=n, train=len(train), test=len(test), iters=a.iters)
    if a.iters > 0:
        pose, transl, rep = refine(a, names, poses, theta)
        theta = theta.copy()
        theta[:n] = pose
        poses = dict(poses)
        t = np.asarray(poses["transl"], np.float32).copy()
        t.reshape(-1, 3)[:n] = transl
        poses["transl"] = t
        if "thetas" in poses:
            poses["thetas"] = theta.reshape(np.shape(poses["thetas"]))
        else:
            poses["global_orient"] = theta[:, :3].reshape(np.shape(poses["global_orient"])).copy()
            poses["body_pose"] = theta[:, 3:].reshape(np.shape(poses["body_pose"])).copy()
        result.update(objective_before=rep["objective_before"], objective_after=rep["objective_after"],
                      mean_iou_before=rep["mean_iou_before"], mean_iou_after=rep["mean_iou_after"])
    np.savez(os.path.join(a.capture, "poses_optimized.npz"), **poses)
    cam = np.load(os.path.join(a.capture, "cameras.npz"))
    for part, idx in (("train", train), ("test", test)):
        d = os.path.join(a.out, part)
        for sub in ("images", "masks"):
            os.makedirs(os.path.join(d, sub), exist_ok=True)
        np.savez(os.path.join(d, "cam_parms.npz"), intrinsic=np.array(cam["intrinsic"]), extrinsic=np.array(cam["extrinsic"]))
        torch.save(smpl_parms(poses, theta, idx), os.path.join(d, "smpl_parms.pth"))
        for i in idx:
            for sub in ("images", "masks"):
                shutil.copy(os.path.join(a.capture, sub, names[i]), os.path.join(d, sub, names[i]))
    print(json.dumps(result))
    return 0


if __name__ == "__main__":
    sys.exit(main())
