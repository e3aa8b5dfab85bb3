"""Animate a trained avatar along a motion clip on the GPU, streaming the frames out as they render.

    python tools/animate.py -s DATA -m MODEL --epoch N --stage 1 --motion walk.npz --body smpl --fps 30 --align_to 0 --png OUT
    python tools/animate.py -s DATA -m MODEL --epoch N --stage 1 --motion clip.pth --clip_fps 30 --body smpl --fps 60 --rgba --raw - \
        | ffmpeg -f rawvideo -pix_fmt rgba -s 1024x1024 -r 60 -i - out.mov
    python tools/animate.py -s DATA -m MODEL --epoch N --stage 2 --motion walk.npz --body smpl --smpl_model SMPL_NEUTRAL.pkl \
        --uv_template template_mesh_smpl_uv.obj --fps 30 --align_to 0 --raw frames.rgb

DATA / MODEL are the reference's -s / -m folders; stage 1 loads net/iteration_N/net.pth (`load`), stage 2 pose_encoder.pth
(`stage2_load`).  --motion: an AMASS SMPL+H / SMPL-X .npz, or a smpl_parms.pth (its rate from --clip_fps).  Cameras: DATA/train's
cam_parms.npz (--camera dataset) or its orbit around the clip's first pelvis (--camera orbit); --size W H scales the intrinsics.
--png DIR writes DIR/{:05d}.png; --raw FILE (or - for stdout) writes the frames back to back as H x W x 3 (--rgba: 4) bytes.

--scene PLY renders the avatar inside a 3D Gaussian Splatting scene (3DGS's point_cloud.ply), both splatted in one sort so that
each occludes the other; --place S RX RY RZ TX TY TZ puts the avatar's world into the scene's (x_scene = S R x + T, R an
axis-angle).  Dataset and orbit cameras are carried along with the avatar; --camera scene:K takes camera K of the cameras.json of
the 3DGS model folder holding point_cloud/iteration_*/point_cloud.ply (or of --scene_cameras), at its own size unless --size.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gaussianavatar_b200.animate import Animator, MotionClip, OrbitCamera  # noqa: E402
from gaussianavatar_b200.avatar_model import AvatarModel  # noqa: E402
from gaussianavatar_b200.config import ModelParams, NetworkParams, OptimizationParams  # noqa: E402
from gaussianavatar_b200.dataset import camera_item  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("-s", "--source_path", required=True)
    ap.add_argument("-m", "--model_path", required=True)
    ap.add_argument("--project_path", default=os.getcwd(), help="folder holding assets/ (UV masks, LBS maps)")
    ap.add_argument("--epoch", type=int, required=True)
    ap.add_argument("--stage", type=int, choices=(1, 2), default=1)
    ap.add_argument("--motion", required=True)
    ap.add_argument("--clip_fps", type=float, default=None, help="the clip's frame rate (required for a .pth; overrides an .npz's)")
    ap.add_argument("--body", choices=("smpl", "smplx"), default="smpl")
    ap.add_argument("--smpl_model", default=None, help="SMPL_{GENDER}.pkl / SMPLX_{GENDER}.npz (its folder is the model path)")
    ap.add_argument("--smpl_gender", default="neutral")
    ap.add_argument("--uv_template", default=None, help="stage 2: the body's UV template OBJ")
    ap.add_argument("--query_posmap_size", type=int, default=512)
    ap.add_argument("--inp_posmap_size", type=int, default=128)
    ap.add_argument("--nf", type=int, default=32, help="stage 2: the pose encoder's base width")
    ap.add_argument("--fps", type=float, default=30.0, help="output frame rate")
    ap.add_argument("--speed", type=float, default=1.0)
    ap.add_argument("--align_to", type=int, default=None, help="map clip frame 0 onto this training frame")
    ap.add_argument("--camera", default="dataset", help="dataset | orbit | scene:K (camera K of the scene's cameras.json)")
    ap.add_argument("--scene", default=None, help="a 3DGS point_cloud.ply to render the avatar in")
    ap.add_argument("--place", type=float, nargs=7, metavar=("S", "RX", "RY", "RZ", "TX", "TY", "TZ"), default=None,
                    help="the avatar in the scene: x_scene = S R x + T, R from the axis-angle (RX, RY, RZ)")
    ap.add_argument("--scene_cameras", default=None, help="cameras.json for --camera scene:K (default: the 3DGS model folder's)")
    ap.add_argument("--size", type=int, nargs=2, metavar=("W", "H"), default=None)
    ap.add_argument("--chunk", type=int, default=None, help="frames per rasterizer call (default 8, with --scene 2)")
    ap.add_argument("--rgba", action="store_true")
    ap.add_argument("--png", default=None)
    ap.add_argument("--raw", default=None)
    a = ap.parse_args(argv)
    if a.png is None and a.raw is None:
        ap.error("nothing to write: give --png DIR and / or --raw FILE")
    scene_cam = None
    if a.camera.startswith("scene:"):
        if a.scene is None:
            ap.error("--camera scene:K needs --scene")
        try:
            scene_cam = int(a.camera[len("scene:"):])
        except ValueError:
            ap.error(f"--camera {a.camera}: K must be an integer")
    elif a.camera not in ("dataset", "orbit"):
        ap.error(f"--camera {a.camera}: dataset, orbit or scene:K")
    if a.place is not None and a.scene is None:
        ap.error("--place needs --scene")

    model_dir = os.path.dirname(os.path.abspath(a.smpl_model)) if a.smpl_model else ""
    mp = ModelParams(source_path=a.source_path, model_path=a.model_path, project_path=a.project_path, smpl_model_path=model_dir,
                     smplx_model_path=model_dir, smpl_gender=a.smpl_gender, smpl_type=a.body, train_stage=a.stage,
                     query_posmap_size=a.query_posmap_size, inp_posmap_size=a.inp_posmap_size, batch_size=1)
    model = AvatarModel(mp, NetworkParams(nf=a.nf), OptimizationParams(), train=False)
    pose_mapper = None
    if a.stage == 1:
        model.load(a.epoch)
    else:
        model.stage2_load(a.epoch)
        if not (a.smpl_model and a.uv_template):
            ap.error("--stage 2 needs --smpl_model and --uv_template for the input position maps")
        from gaussianavatar_b200.body import load_model
        from gaussianavatar_b200.posmap import PoseMapper
        pose_mapper = PoseMapper(load_model(a.smpl_model), model.betas[0], a.uv_template, a.inp_posmap_size, device=model.device,
                                 body=model.body)

    cam = np.load(os.path.join(a.source_path, "train", "cam_parms.npz"))
    K, E = np.array(cam["intrinsic"], np.float32).reshape(3, 3), np.asarray(cam["extrinsic"], np.float64)
    from PIL import Image
    img_dir = os.path.join(a.source_path, "train", "images")
    W0, H0 = Image.open(os.path.join(img_dir, sorted(os.listdir(img_dir))[0])).size
    W, H = a.size if a.size else (W0, H0)
    K[0, :] *= W / W0
    K[1, :] *= H / H0
    cameras = camera_item(K, E, H, W) if a.camera == "dataset" else OrbitCamera(K, E)

    scene = placement = None
    if a.scene is not None:
        from gaussianavatar_b200.scene import GaussianScene, Placement, load_scene_cameras, scene_cameras_path
        scene = GaussianScene.load_ply(a.scene)
        if a.place is not None:
            placement = Placement.from_axis_angle(a.place[0], a.place[1:4], a.place[4:7])
        if scene_cam is not None:
            cams = load_scene_cameras(a.scene_cameras or scene_cameras_path(a.scene))
            if not 0 <= scene_cam < len(cams):
                ap.error(f"--camera scene:{scene_cam}: the scene has cameras 0..{len(cams) - 1}")
            cameras = cams[scene_cam]
            if not a.size:
                W, H = cameras.width, cameras.height

    clip = MotionClip.load(a.motion, a.body, fps=a.clip_fps)
    anim = Animator(model, cameras, H, W, chunk=a.chunk if a.stage == 1 else 1, channels=4 if a.rgba else 3, pose_mapper=pose_mapper,
                    scene=scene, placement=placement)
    if a.png:
        os.makedirs(a.png, exist_ok=True)
    raw = None if a.raw is None else (sys.stdout.buffer if a.raw == "-" else open(a.raw, "wb"))
    mode = "RGBA" if a.rgba else "RGB"
    n = 0
    t0 = time.perf_counter()
    try:
        for first, frames in anim.frames(clip, a.fps, a.speed, a.align_to):
            arr = frames.numpy()
            if raw is not None:
                raw.write(arr.tobytes())
            if a.png:
                for k in range(arr.shape[0]):
                    Image.fromarray(arr[k], mode).save(os.path.join(a.png, "{:05d}.png".format(first + k)))
            n += arr.shape[0]
    finally:
        if raw is not None and raw is not sys.stdout.buffer:
            raw.close()
    dt = time.perf_counter() - t0
    print(json.dumps(dict(frames=n, width=W, height=H, channels=4 if a.rgba else 3, seconds=round(dt, 4),
                          fps=round(n / dt, 2) if dt > 0 else None)), file=sys.stderr if a.raw == "-" else sys.stdout)
    return 0


if __name__ == "__main__":
    sys.exit(main())
