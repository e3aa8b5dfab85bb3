"""Extract a coloured, watertight mesh of a trained avatar in a training frame's pose or along a motion clip, on the GPU.

    python tools/extract_mesh.py -s DATA -m MODEL --epoch N --frame 0 --frame 12 --out meshes
    python tools/extract_mesh.py -s DATA -m MODEL --epoch N --motion walk.npz --fps 10 --align_to 0 --format obj --out meshes

DATA / MODEL / --epoch / --stage / --body and the stage-2 flags are tools/animate.py's.  --frame K (repeatable) poses the avatar with
training frame K's pose and writes OUT/frame_{K:05d}.{ply,obj}; --motion CLIP samples the clip at --fps (as the animation player
does, --align_to mapping its first frame onto a training frame) and writes OUT/{:05d}.{ply,obj}, one mesh per output frame.
--res samples along the grid's longest side, --views fusion views of --size x --size pixels, --trunc the truncation in voxels,
--min_carve the views that must see through a sample to carve it.  --iou prints each mesh's silhouette IoU against the avatar's own
(median depth > 0) from the dataset camera.  --antialiasing renders the fusion views and every reference render with 3DGS's
`antialiasing` setting, for an avatar trained with ModelParams.antialiasing.  One JSON line per mesh goes to stdout.

    python tools/extract_mesh.py -s DATA -m MODEL --epoch N --format glb --motion walk.npz --fps 30 --out rig

--format glb writes one rigged mesh, OUT/avatar.glb (gaussianavatar_b200.rig): the canonical mesh, the body skeleton and
--influences (4 or 8) skin weights per vertex, with --motion CLIP baked in as an animation at --fps (--up: the clip world's up
axis, by default -y for a smpl_parms.pth or with --align_to, else z).  --iou poses the rig at every baked frame, or at each --frame K
without a clip, and prints its silhouette IoUs; --psnr at the same poses prints the PSNR of the rig drawn unlit (its texture or
vertex colours) against the avatar's own render, both on black.  One JSON line goes to stdout.

    python tools/extract_mesh.py -s DATA -m MODEL --epoch N --format glb --topology body --subdiv 1 --smpl_model SMPL_NEUTRAL.pkl --out rig

--topology body (default tsdf) writes the rig in the body model's own topology instead (rig.extract_body_rig): the --uv_template
(default PROJECT/assets/template_mesh_{body}_uv.obj) subdivided --subdiv times (0, 1 or 2; default 1) and fitted through the
Gaussians, the body model's skin weights and the decoder's colour map as its texture.  It needs --smpl_model.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("-s", "--source_path", required=True)
    ap.add_argument("-m", "--model_path", required=True)
    ap.add_argument("--project_path", default=os.getcwd(), help="folder holding assets/ (UV masks, LBS maps)")
    ap.add_argument("--epoch", type=int, required=True)
    ap.add_argument("--stage", type=int, choices=(1, 2), default=1)
    ap.add_argument("--body", choices=("smpl", "smplx"), default="smpl")
    ap.add_argument("--smpl_model", default=None, help="SMPL_{GENDER}.pkl / SMPLX_{GENDER}.npz (its folder is the model path)")
    ap.add_argument("--smpl_gender", default="neutral")
    ap.add_argument("--uv_template", default=None, help="stage 2: the body's UV template OBJ")
    ap.add_argument("--query_posmap_size", type=int, default=512)
    ap.add_argument("--inp_posmap_size", type=int, default=128)
    ap.add_argument("--nf", type=int, default=32, help="stage 2: the pose encoder's base width")
    ap.add_argument("--frame", type=int, action="append", default=None, help="a training frame's pose (repeatable)")
    ap.add_argument("--motion", default=None, help="an AMASS .npz or a smpl_parms.pth, one mesh per output frame")
    ap.add_argument("--clip_fps", type=float, default=None, help="the clip's frame rate (required for a .pth)")
    ap.add_argument("--fps", type=float, default=None, help="output frame rate of --motion")
    ap.add_argument("--align_to", type=int, default=None, help="map clip frame 0 onto this training frame")
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--views", type=int, default=64)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--trunc", type=float, default=4.0, help="truncation distance in voxels")
    ap.add_argument("--min_carve", type=int, default=1)
    ap.add_argument("--format", choices=("ply", "obj", "glb"), default="ply")
    ap.add_argument("--influences", type=int, choices=(4, 8), default=None, help="glb: joints per vertex (default 4)")
    ap.add_argument("--up", choices=("y", "z", "-y"), default=None, help="glb: the clip world's up axis")
    ap.add_argument("--antialiasing", action="store_true", help="render the avatar's views with 3DGS's antialiasing setting (for an "
                    "avatar trained with it)")
    ap.add_argument("--out", required=True)
    ap.add_argument("--iou", action="store_true")
    ap.add_argument("--psnr", action="store_true", help="glb: the unlit rig's PSNR against the avatar's render")
    ap.add_argument("--topology", choices=("tsdf", "body"), default="tsdf", help="glb: the TSDF mesh or the body model's own topology")
    ap.add_argument("--subdiv", type=int, choices=(0, 1, 2), default=None, help="--topology body: midpoint subdivisions (default 1)")
    a = ap.parse_args(argv)
    if a.format != "glb" and (a.influences is not None or a.up is not None or a.psnr or a.topology != "tsdf"):
        ap.error("--influences, --up, --psnr and --topology go with --format glb")
    if a.subdiv is not None and a.topology != "body":
        ap.error("--subdiv goes with --topology body")
    if a.topology == "body" and not a.smpl_model:
        ap.error("--topology body needs --smpl_model (the body model's skin weights and canonical mesh)")
    if a.format == "glb":
        if a.frame is not None and a.motion is not None:
            ap.error("give --frame K (repeatable) or --motion CLIP, not both")
        if a.up is not None and a.motion is None:
            ap.error("--up goes with --motion")
    elif (a.frame is None) == (a.motion is None):
        ap.error("give --frame K (repeatable) or --motion CLIP, not both")
    if a.motion is None and (a.fps is not None or a.align_to is not None or a.clip_fps is not None):
        ap.error("--fps, --clip_fps and --align_to go with --motion")
    if a.motion is not None and a.fps is None:
        ap.error("--motion needs --fps")
    if a.fps is not None and not a.fps > 0:
        ap.error(f"--fps {a.fps} must be positive")
    if not 2 <= a.res <= 512:
        ap.error(f"--res {a.res} outside 2..512")
    if a.views < 1 or a.size < 1 or not a.trunc > 0 or a.min_carve < 1:
        ap.error("--views, --size, --trunc and --min_carve must be positive")
    if a.stage == 2 and not (a.smpl_model and a.uv_template):
        ap.error("--stage 2 needs --smpl_model and --uv_template for the input position maps")
    return a


def dataset_camera(src):
    """The dataset's camera at its image size: ([1,40] camera rows, H, W)."""
    from PIL import Image
    from gaussianavatar_b200.camera import make_camera
    from gaussianavatar_b200.mesh_render import cameras
    cam = np.load(os.path.join(src, "train", "cam_parms.npz"))
    K, E = np.array(cam["intrinsic"], np.float32).reshape(3, 3), np.asarray(cam["extrinsic"], np.float64)
    img_dir = os.path.join(src, "train", "images")
    W, H = Image.open(os.path.join(img_dir, sorted(os.listdir(img_dir))[0])).size
    return cameras([make_camera(K, E, H, W)]), H, W


def main(argv=None):
    a = parse(argv)
    if a.format == "glb":
        return main_glb(a)
    from animate import load_actor
    from gaussianavatar_b200 import animate as an
    from gaussianavatar_b200.mesh_extract import extract_mesh, silhouette_iou, write_obj, write_ply

    spec = dict(source_path=a.source_path, model_path=a.model_path, epoch=a.epoch, stage=a.stage, body=a.body, clip=None, speed=1.0,
                align_to=a.align_to, smpl_model=a.smpl_model, smpl_gender=a.smpl_gender, uv_template=a.uv_template,
                query_posmap_size=a.query_posmap_size, inp_posmap_size=a.inp_posmap_size, nf=a.nf, white_background=True,
                antialiasing=a.antialiasing)
    actor = load_actor(spec, a.project_path, None)
    model, body, dev = actor.model, actor.model.body, actor.model.device
    F = int(model.pose.weight.shape[0])
    jobs = []                     # (name, pose, transl, rest_pose)
    if a.frame is not None:
        rest = None
        if body.rest_width:
            train = an.MotionClip.load(os.path.join(a.source_path, "train", "smpl_parms.pth"), body.name, fps=30.0)
            rest = body.split(train.pose)[1]
        for k in a.frame:
            if not 0 <= k < F:
                raise SystemExit(f"--frame {k}: the model has training frames 0..{F - 1}")
            jobs.append((f"frame_{k:05d}", model.pose.weight[k].detach(), model.transl.weight[k].detach(), None if rest is None else rest[k]))
    else:
        clip = an.MotionClip.load(a.motion, body.name, fps=a.clip_fps)
        times = an.sample_times(clip.num_keys, clip.fps, a.fps)
        align = an.Ensemble._alignment(model, clip, a.align_to)
        pose, trans = an.motion_sample(clip.pose.to(dev).contiguous(), clip.trans.to(dev).contiguous(), torch.from_numpy(times).to(dev),
                                       torch.from_numpy(align).to(dev))
        pose, rest = body.split(pose)
        jobs = [(f"{i:05d}", pose[i], trans[i], None if rest is None else rest[i]) for i in range(pose.shape[0])]
    os.makedirs(a.out, exist_ok=True)
    cam = dataset_camera(a.source_path) if a.iou else None
    write = write_ply if a.format == "ply" else write_obj
    for name, pose, transl, rest in jobs:
        t0 = time.perf_counter()
        verts, faces, colors = extract_mesh(model, pose, transl, rest, res=a.res, views=a.views, size=a.size, trunc_voxels=a.trunc,
                                            min_carve=a.min_carve, pose_mapper=actor.pose_mapper)
        torch.cuda.synchronize()
        path = os.path.join(a.out, f"{name}.{a.format}")
        write(path, verts, faces, colors)
        rec = dict(mesh=path, vertices=int(verts.shape[0]), faces=int(faces.shape[0]), seconds=round(time.perf_counter() - t0, 4))
        if cam is not None:
            rec["iou"] = round(silhouette_iou(model, pose, transl, verts, faces, cam[0], cam[1], cam[2], rest, actor.pose_mapper)[0], 5)
        print(json.dumps(rec), flush=True)
    return 0


def main_glb(a):
    from animate import load_actor
    from gaussianavatar_b200 import animate as an
    from gaussianavatar_b200 import rig as rg
    from gaussianavatar_b200.mesh_extract import silhouette_iou

    spec = dict(source_path=a.source_path, model_path=a.model_path, epoch=a.epoch, stage=a.stage, body=a.body, clip=None, speed=1.0,
                align_to=a.align_to, smpl_model=a.smpl_model, smpl_gender=a.smpl_gender, uv_template=a.uv_template,
                query_posmap_size=a.query_posmap_size, inp_posmap_size=a.inp_posmap_size, nf=a.nf, white_background=True,
                antialiasing=a.antialiasing)
    actor = load_actor(spec, a.project_path, None)
    model, body = actor.model, actor.model.body
    F = int(model.pose.weight.shape[0])
    for k in a.frame or []:
        if not 0 <= k < F:
            raise SystemExit(f"--frame {k}: the model has training frames 0..{F - 1}")
    t0 = time.perf_counter()
    if a.topology == "body":
        from gaussianavatar_b200.body import load_model
        from gaussianavatar_b200.posmap import BodyPoser
        poser = actor.pose_mapper or BodyPoser(load_model(a.smpl_model), model.betas[0].cpu(), device=model.device, body=body)
        uv = a.uv_template or os.path.join(a.project_path, "assets", f"template_mesh_{body.name}_uv.obj")
        rig = rg.extract_body_rig(model, uv, 1 if a.subdiv is None else a.subdiv, a.influences or 4, pose_mapper=poser)
    else:
        rig = rg.extract_rigged_mesh(model, res=a.res, views=a.views, size=a.size, trunc_voxels=a.trunc, min_carve=a.min_carve,
                                     influences=a.influences or 4, pose_mapper=actor.pose_mapper)
    motion = None
    if a.motion is not None:
        clip = an.MotionClip.load(a.motion, body.name, fps=a.clip_fps)
        motion = rg.bake_motion(model, clip, a.fps, a.align_to, a.up, clip_path=a.motion)
    torch.cuda.synchronize()
    os.makedirs(a.out, exist_ok=True)
    path = os.path.join(a.out, "avatar.glb")
    rg.write_glb(path, rig, motion)
    rec = dict(mesh=path, vertices=int(rig.verts.shape[0]), faces=int(rig.faces.shape[0]), joints=len(rig.parents),
               frames=0 if motion is None else motion.frames, seconds=round(time.perf_counter() - t0, 4))
    if rig.fit is not None:
        rec["fit"] = rig.fit
    if a.iou or a.psnr:
        cam = dataset_camera(a.source_path)
        if motion is not None:        # the baked frames, carried back from glTF's +Y up into the clip's world
            poses = [(motion, i) for i in range(motion.frames)]
            pose, trans = an.motion_sample(clip.pose.to(model.device).contiguous(), clip.trans.to(model.device).contiguous(),
                                           torch.from_numpy(an.sample_times(clip.num_keys, clip.fps, a.fps)).to(model.device),
                                           torch.from_numpy(an.Ensemble._alignment(model, clip, a.align_to)).to(model.device))
            pose, rest = body.split(pose)
        else:
            pose, rest = None, None
            if body.rest_width:
                train = an.MotionClip.load(os.path.join(a.source_path, "train", "smpl_parms.pth"), body.name, fps=30.0)
                rest = body.split(train.pose)[1][a.frame or []].to(model.device)
            pose = model.pose.weight.detach()[a.frame or []]
            trans = model.transl.weight.detach()[a.frame or []]
            full = body.join(pose, rest) if body.rest_width else pose
            poses = [(rg.bake_poses(model._rest_joints, full[i:i + 1], trans[i:i + 1], 1.0, "y"), 0) for i in range(len(a.frame or []))]
        ious, psnrs = [], []
        for i, (m, f) in enumerate(poses):
            v = torch.from_numpy(rg.pose_rig(rig, m, f) @ m.up_rotation).float().to(model.device)
            r = None if rest is None else rest[i]
            if a.iou:
                ious.append(round(silhouette_iou(model, pose[i], trans[i], v, rig.faces, cam[0], cam[1], cam[2], r, actor.pose_mapper)[0], 5))
            if a.psnr:
                psnrs.append(round(rg.unlit_psnr(model, rig, v, pose[i], trans[i], cam[0], cam[1], cam[2], r, actor.pose_mapper)[0], 4))
        if a.iou:
            rec["iou"] = ious
        if a.psnr:
            rec["psnr"] = psnrs
    print(json.dumps(rec), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
