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

--cast CAST.json renders several avatars together (at most 8), each on its own clip, in one sort per tile so that each hides the
others.  It replaces -s / -m / --motion / --body / --stage: the file is a list of actors, each an object with the single-avatar
fields
    source_path, model_path, epoch, motion                                  (required)
    stage (1), body ("smpl"), clip_fps, speed (1), align_to, place [S RX RY RZ TX TY TZ], smpl_model, smpl_gender ("neutral"),
    uv_template, query_posmap_size (512), inp_posmap_size (128), nf (32), white_background (true), antialiasing (false)
The first actor's dataset gives the cameras; each actor's `place` puts its world into the scene's (without a scene, into the
first actor's placed world).  The output, camera and scene flags are shared; the playback lasts as long as the longest clip, a
shorter one holding its last pose.
--antialiasing renders the avatar with 3DGS's `antialiasing` setting (Mip-Splatting's screen-space filter); give it for an avatar
trained with ModelParams.antialiasing, so that it looks right at any --size or camera distance.  A cast entry's `antialiasing`
does the same, and the actors of one cast must share it.  --scene_antialiasing does it for a --scene trained with the setting
(the PLY does not record it); the avatar's and the scene's modes are independent.
--mattes DIR writes DIR/{:05d}_{k}.png, actor k's visible matte (8-bit greyscale: the weight its Gaussians add to each pixel),
with --cast or for the single avatar (its visible mask inside a scene).
--depth DIR writes DIR/{:05d}.npy, float32 [2,H,W]: plane 0 the mean, plane 1 the median view depth of the composited frame (the
shared world's units, 0 where there is no surface), from the same compositing pass as the frame; with --cast, --scene, --mattes
or for the single avatar.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gaussianavatar_b200.animate import Actor, Animator, Ensemble, MotionClip, OrbitCamera  # noqa: E402
from gaussianavatar_b200.avatar_model import AvatarModel  # noqa: E402
from gaussianavatar_b200.config import ModelParams, NetworkParams, OptimizationParams  # noqa: E402
from gaussianavatar_b200.dataset import camera_item  # noqa: E402


CAST_REQUIRED = ("source_path", "model_path", "epoch", "motion")
CAST_DEFAULTS = dict(stage=1, body="smpl", clip_fps=None, speed=1.0, align_to=None, place=None, smpl_model=None, smpl_gender="neutral",
                     uv_template=None, query_posmap_size=512, inp_posmap_size=128, nf=32, white_background=True, antialiasing=False)


def read_cast(path):
    """The actors of a --cast file, each a dict of every field (defaults filled in) with its clip loaded as "clip".  Raises
    ValueError naming the entry: a missing or unknown field, a bad value, a clip that is not of the entry's body, or backgrounds
    or antialiasing modes that differ from the first actor's."""
    with open(path) as f:
        try:
            raw = json.load(f)
        except json.JSONDecodeError as e:
            raise ValueError(f"{path}: not JSON ({e})") from None
    if not isinstance(raw, list) or not 1 <= len(raw) <= 8:
        raise ValueError(f"{path}: a list of 1..8 actors")
    out = []
    for k, e in enumerate(raw):
        where = f"{path}: actor {k}"
        if not isinstance(e, dict):
            raise ValueError(f"{where}: an object with the actor's fields")
        missing = [f for f in CAST_REQUIRED if f not in e]
        if missing:
            raise ValueError(f"{where}: missing {', '.join(missing)}")
        unknown = sorted(set(e) - set(CAST_REQUIRED) - set(CAST_DEFAULTS))
        if unknown:
            raise ValueError(f"{where}: unknown field {', '.join(unknown)}")
        d = {**CAST_DEFAULTS, **e}
        if d["stage"] not in (1, 2) or d["body"] not in ("smpl", "smplx"):
            raise ValueError(f"{where}: stage {d['stage']!r} (1 or 2), body {d['body']!r} (smpl or smplx)")
        if d["place"] is not None and len(d["place"]) != 7:
            raise ValueError(f"{where}: place has {len(d['place'])} values (S RX RY RZ TX TY TZ)")
        if d["stage"] == 2 and not (d["smpl_model"] and d["uv_template"]):
            raise ValueError(f"{where}: stage 2 needs smpl_model and uv_template for the input position maps")
        if bool(d["white_background"]) != bool(out[0]["white_background"] if out else d["white_background"]):
            raise ValueError(f"{where}: white_background {d['white_background']}, actor 0 renders on "
                             f"{'white' if out[0]['white_background'] else 'black'}: the actors must share one background")
        if out and bool(d["antialiasing"]) != bool(out[0]["antialiasing"]):
            raise ValueError(f"{where}: antialiasing {bool(d['antialiasing'])}, actor 0 renders with antialiasing "
                             f"{bool(out[0]['antialiasing'])}: the actors must share one mode")
        try:
            d["clip"] = MotionClip.load(d["motion"], d["body"], fps=d["clip_fps"])
        except ValueError as err:
            raise ValueError(f"{where}: {err}") from None
        out.append(d)
    return out


def load_actor(d, project_path, placement):
    """An `Actor` for one actor's fields (the single avatar's flags or a --cast entry)."""
    model_dir = os.path.dirname(os.path.abspath(d["smpl_model"])) if d["smpl_model"] else ""
    mp = ModelParams(source_path=d["source_path"], model_path=d["model_path"], project_path=project_path, smpl_model_path=model_dir,
                     smplx_model_path=model_dir, smpl_gender=d["smpl_gender"], smpl_type=d["body"], train_stage=d["stage"],
                     query_posmap_size=d["query_posmap_size"], inp_posmap_size=d["inp_posmap_size"], batch_size=1,
                     white_background=bool(d["white_background"]), antialiasing=bool(d["antialiasing"]))
    model = AvatarModel(mp, NetworkParams(nf=d["nf"]), OptimizationParams(), train=False)
    pose_mapper = None
    if d["stage"] == 1:
        model.load(d["epoch"])
    else:
        model.stage2_load(d["epoch"])
        from gaussianavatar_b200.body import load_model
        from gaussianavatar_b200.posmap import PoseMapper
        pose_mapper = PoseMapper(load_model(d["smpl_model"]), model.betas[0], d["uv_template"], d["inp_posmap_size"], device=model.device,
                                 body=model.body)
    return Actor(model, d["clip"], placement, d["align_to"], d["speed"], pose_mapper)


def main(argv=None):
    pre = argparse.ArgumentParser(add_help=False)
    pre.add_argument("--cast", default=None)
    cast_given = pre.parse_known_args(argv)[0].cast is not None
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("-s", "--source_path", required=not cast_given)
    ap.add_argument("-m", "--model_path", required=not cast_given)
    ap.add_argument("--project_path", default=os.getcwd(), help="folder holding assets/ (UV masks, LBS maps)")
    ap.add_argument("--epoch", type=int, required=not cast_given)
    ap.add_argument("--stage", type=int, choices=(1, 2), default=None, help="1 (default) or 2")
    ap.add_argument("--motion", required=not cast_given)
    ap.add_argument("--clip_fps", type=float, default=None, help="the clip's frame rate (required for a .pth; overrides an .npz's)")
    ap.add_argument("--body", choices=("smpl", "smplx"), default=None, help="smpl (default) or smplx")
    ap.add_argument("--cast", default=None, help="a JSON list of actors rendered together (replaces -s, -m, --motion, --body, --stage)")
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
    ap.add_argument("--antialiasing", action="store_true",
                    help="render the avatar with 3DGS's antialiasing setting (for an avatar trained with it)")
    ap.add_argument("--scene_antialiasing", action="store_true", help="render --scene with 3DGS's antialiasing setting (for a scene "
                    "trained with it)")
    ap.add_argument("--scene_cameras", default=None, help="cameras.json for --camera scene:K (default: the 3DGS model folder's)")
    ap.add_argument("--size", type=int, nargs=2, metavar=("W", "H"), default=None)
    ap.add_argument("--chunk", type=int, default=None, help="frames per rasterizer call (default 8, with --scene 2)")
    ap.add_argument("--rgba", action="store_true")
    ap.add_argument("--png", default=None)
    ap.add_argument("--raw", default=None)
    ap.add_argument("--mattes", default=None, help="DIR: each avatar's visible matte as DIR/{:05d}_{k}.png")
    ap.add_argument("--depth", default=None, help="DIR: each frame's mean and median depth as DIR/{:05d}.npy, float32 [2,H,W]")
    a = ap.parse_args(argv)
    if a.png is None and a.raw is None and a.mattes is None and a.depth is None:
        ap.error("nothing to write: give --png DIR, --raw FILE, --mattes DIR and / or --depth DIR")
    if a.cast is not None:
        given = [f for f, v in (("-s", a.source_path), ("-m", a.model_path), ("--epoch", a.epoch), ("--motion", a.motion), ("--body", a.body),
                                ("--stage", a.stage), ("--antialiasing", a.antialiasing or None)) if v is not None]
        if given:
            ap.error(f"--cast replaces {', '.join(given)}: give each actor's in the cast file")
        try:
            specs = read_cast(a.cast)
        except (OSError, ValueError) as e:
            ap.error(str(e))
    else:
        a.body, a.stage = a.body or "smpl", a.stage or 1
        specs = [dict(source_path=a.source_path, model_path=a.model_path, epoch=a.epoch, stage=a.stage, body=a.body, motion=a.motion,
                      clip_fps=a.clip_fps, speed=a.speed, align_to=a.align_to, place=a.place, smpl_model=a.smpl_model,
                      smpl_gender=a.smpl_gender, uv_template=a.uv_template, query_posmap_size=a.query_posmap_size,
                      inp_posmap_size=a.inp_posmap_size, nf=a.nf, white_background=True, antialiasing=a.antialiasing)]
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
    if a.scene_antialiasing and a.scene is None:
        ap.error("--scene_antialiasing needs --scene")
    if a.place is not None and (a.scene is None or a.cast is not None):
        ap.error("--place needs --scene" if a.cast is None else "--place: give each actor's place in the cast file")
    if a.cast is None and a.stage == 2 and not (a.smpl_model and a.uv_template):
        ap.error("--stage 2 needs --smpl_model and --uv_template for the input position maps")
    if a.cast is None:
        specs[0]["clip"] = None          # loaded after the model, as before

    from gaussianavatar_b200.scene import Placement
    place = lambda d: None if d["place"] is None else Placement.from_axis_angle(d["place"][0], d["place"][1:4], d["place"][4:7])
    actors = [load_actor(d, a.project_path, place(d)) for d in specs]

    src = specs[0]["source_path"]
    cam = np.load(os.path.join(src, "train", "cam_parms.npz"))
    K, E = np.array(cam["intrinsic"], np.float32).reshape(3, 3), np.asarray(cam["extrinsic"], np.float64)
    from PIL import Image
    img_dir = os.path.join(src, "train", "images")
    W0, H0 = Image.open(os.path.join(img_dir, sorted(os.listdir(img_dir))[0])).size
    W, H = a.size if a.size else (W0, H0)
    K[0, :] *= W / W0
    K[1, :] *= H / H0
    cameras = camera_item(K, E, H, W) if a.camera == "dataset" else OrbitCamera(K, E)

    scene = None
    if a.scene is not None:
        from gaussianavatar_b200.scene import GaussianScene, load_scene_cameras, scene_cameras_path
        scene = GaussianScene.load_ply(a.scene, antialiasing=a.scene_antialiasing)
        if scene_cam is not None:
            cams = load_scene_cameras(a.scene_cameras or scene_cameras_path(a.scene))
            if not 0 <= scene_cam < len(cams):
                ap.error(f"--camera scene:{scene_cam}: the scene has cameras 0..{len(cams) - 1}")
            cameras = cams[scene_cam]
            if not a.size:
                W, H = cameras.width, cameras.height

    if a.cast is None:
        actors[0].clip = MotionClip.load(a.motion, a.body, fps=a.clip_fps)
    chunk = a.chunk if all(d["stage"] == 1 for d in specs) else 1
    channels = 4 if a.rgba else 3
    if a.cast is None and a.mattes is None:
        x = actors[0]
        anim = Animator(x.model, cameras, H, W, chunk=chunk, channels=channels, pose_mapper=x.pose_mapper, scene=scene,
                        placement=x.placement, depth=a.depth is not None)
        playback = ((first, frames, None, *depth) for first, frames, *depth in anim.frames(x.clip, a.fps, x.speed, x.align_to))
    else:
        try:
            ens = Ensemble(actors, cameras, H, W, chunk=chunk, channels=channels, mattes=a.mattes is not None, scene=scene,
                           depth=a.depth is not None)
        except ValueError as e:
            ap.error(str(e))
        playback = ens.frames(a.fps)
    for d in (a.png, a.mattes, a.depth):
        if d:
            os.makedirs(d, exist_ok=True)
    raw = None if a.raw is None else (sys.stdout.buffer if a.raw == "-" else open(a.raw, "wb"))
    mode = "RGBA" if a.rgba else "RGB"
    n = 0
    t0 = time.perf_counter()
    try:
        for first, frames, mattes, *depth in playback:
            arr = frames.numpy()
            if raw is not None:
                raw.write(arr.tobytes())
            if a.png:
                for k in range(arr.shape[0]):
                    Image.fromarray(arr[k], mode).save(os.path.join(a.png, "{:05d}.png".format(first + k)))
            if mattes is not None:
                mt = mattes.numpy()
                for k in range(mt.shape[0]):
                    for j in range(mt.shape[1]):
                        Image.fromarray(mt[k, j], "L").save(os.path.join(a.mattes, "{:05d}_{}.png".format(first + k, j)))
            if depth:
                dp = depth[0].numpy()
                for k in range(dp.shape[0]):
                    np.save(os.path.join(a.depth, "{:05d}.npy".format(first + k)), dp[k])
            n += arr.shape[0]
    finally:
        if raw is not None and raw is not sys.stdout.buffer:
            raw.close()
    dt = time.perf_counter() - t0
    print(json.dumps(dict(frames=n, width=W, height=H, channels=channels, seconds=round(dt, 4),
                          fps=round(n / dt, 2) if dt > 0 else None)), file=sys.stderr if a.raw == "-" else sys.stdout)
    return 0


if __name__ == "__main__":
    sys.exit(main())
