"""Draw the posed SMPL / SMPL-X body over every image of a data folder, on the GPU (the reference's scripts/render_pred_smpl.py
without pyrender, trimesh, cv2 or an OpenGL context).

    python tools/body_overlay.py DATA/train --body smpl --smpl_model SMPL_NEUTRAL.pkl --out OUT
    python tools/body_overlay.py DATA/train --body smplx --smpl_model SMPLX_NEUTRAL.npz --out OUT --iou

Poses come from FOLDER/smpl_parms_pred.pth if it exists, else smpl_parms.pth (or --params): row i of body_pose / trans belongs to
the i-th image in sorted order; with --body smplx body_pose [165] splits into the pose [:66] and the jaw, eye and hand pose [66:].
Cameras come from FOLDER/cam_parms.npz at each image's own size.  Writes OUT/pred_smpl_render/<image name> as PNG: the shade where
the body is drawn (floor(255 c + 0.5)), the input image's bytes everywhere else.  --iou also prints one JSON line with each
frame's IoU of the drawn silhouette against masks/<name> (>= 128 is the subject, as the datasets read it) and their mean, so that
running it on smpl_parms.pth and then smpl_parms_pred.pth measures what the stage-1 pose refinement did.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gaussianavatar_b200.body import body_of, load_model  # noqa: E402
from gaussianavatar_b200.camera import make_camera  # noqa: E402
from gaussianavatar_b200.mesh_render import COLORS, MAX_FRAMES_PER_CALL, MeshRenderer, cameras, coverage_iou  # noqa: E402
from gaussianavatar_b200.posmap import BodyPoser  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("folder")
    ap.add_argument("--body", choices=("smpl", "smplx"), default="smpl")
    ap.add_argument("--smpl_model", required=True, help="SMPL_{GENDER}.pkl (--body smplx: SMPLX_{GENDER}.npz)")
    ap.add_argument("--params", default=None, help="parameter file in FOLDER (default: smpl_parms_pred.pth, else smpl_parms.pth)")
    ap.add_argument("--color", default="white", choices=sorted(COLORS))
    ap.add_argument("--out", required=True)
    ap.add_argument("--iou", action="store_true", help="print the silhouette IoU against masks/ as one JSON line")
    a = ap.parse_args(argv)
    params = a.params or ("smpl_parms_pred.pth" if os.path.exists(os.path.join(a.folder, "smpl_parms_pred.pth")) else "smpl_parms.pth")
    prm = torch.load(os.path.join(a.folder, params), map_location="cpu", weights_only=False)
    body = body_of(a.body)
    pose = torch.as_tensor(prm["body_pose"]).float()
    transl = torch.as_tensor(prm["trans"]).float()
    beta = torch.as_tensor(prm["beta"]).float().reshape(-1, 10)[0]
    poser = BodyPoser(load_model(a.smpl_model), beta, body=body)
    renderer = MeshRenderer(poser.faces, poser.V, device=poser.device, color=a.color)
    cam_npz = np.load(os.path.join(a.folder, "cam_parms.npz"))
    K, extr = np.asarray(cam_npz["intrinsic"]).reshape(3, 3), np.asarray(cam_npz["extrinsic"])
    names = sorted(os.listdir(os.path.join(a.folder, "images")))
    if len(names) > pose.shape[0]:
        raise ValueError(f"{len(names)} images but {pose.shape[0]} poses in {params}")
    out_dir = os.path.join(a.out, "pred_smpl_render")
    os.makedirs(out_dir, exist_ok=True)
    ious = []
    for s in range(0, len(names), MAX_FRAMES_PER_CALL):
        chunk = names[s:s + MAX_FRAMES_PER_CALL]
        verts = poser.posed(*body.split(pose[s:s + len(chunk)]), transl[s:s + len(chunk)])
        images = [np.array(Image.open(os.path.join(a.folder, "images", n)).convert("RGB")) for n in chunk]
        sizes = {im.shape[:2] for im in images}
        # frames of one size go to the device together
        for H, W in sorted(sizes):
            idx = [i for i, im in enumerate(images) if im.shape[:2] == (H, W)]
            cams = cameras([make_camera(K, extr, H, W) for _ in idx])
            rgb, face_id, _ = renderer.render(verts[idx], cams, H, W)
            shade = torch.floor(rgb * 255.0 + 0.5).clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).cpu().numpy()
            drawn = (face_id >= 0).cpu().numpy()
            for j, i in enumerate(idx):
                img = np.where(drawn[j][..., None], shade[j], images[i])
                Image.fromarray(img, "RGB").save(os.path.join(out_dir, os.path.splitext(chunk[i])[0] + ".png"))
                if a.iou:
                    stem = os.path.splitext(chunk[i])[0]
                    mdir = os.path.join(a.folder, "masks")
                    mname = next(n for n in sorted(os.listdir(mdir)) if os.path.splitext(n)[0] == stem)
                    m = np.array(Image.open(os.path.join(mdir, mname)))
                    m = (m if m.ndim == 2 else m[..., 0]) >= 128
                    ious.append((s + i, coverage_iou(drawn[j], m)))
    if a.iou:
        ious.sort()
        per = [v for _, v in ious]
        print(json.dumps(dict(params=params, frames=len(per), iou=per, mean_iou=float(np.mean(per)) if per else None)))
    return 0


if __name__ == "__main__":
    sys.exit(main())
