"""Synthetic SMPL / SMPL-X subjects whose template mesh is a surface, for the body-topology rig.

`synthetic.make_body` samples its vertices at random on bone capsules, so the UV grid of `make_uv_template` joins them into a triangle
soup.  Here vertex (r, c) of the same grid (53 x 130 for SMPL, 50 x 209 for SMPL-X) sits on a tube around the synthetic spine: rows
along its height, columns around it, so that the last column coincides in position with the first (the tube's seam is welded in
space, not in index).  Skin weights come from `synthetic._skin_weights` of those points, the joint regressor from the points near
each synthetic joint.  The avatar assets are `posmap.canonical_assets` of that model (the query map is B x0 on the template's own
layout), loaded through `AvatarModel.from_assets`."""
from __future__ import annotations

import math

import numpy as np
import torch

from gaussianavatar_b200 import synthetic as syn

TUBE_RADIUS = 0.16
TUBE_Y = (-1.12, 0.52)          # feet to the top of the head of the synthetic skeleton


def tube_points(rows: int, cols: int) -> np.ndarray:
    y = np.linspace(TUBE_Y[0], TUBE_Y[1], rows)
    th = 2.0 * math.pi * np.arange(cols) / (cols - 1)
    r = TUBE_RADIUS * (1.0 + 0.25 * np.cos(3.0 * np.pi * (y - TUBE_Y[0]) / (TUBE_Y[1] - TUBE_Y[0])))[:, None]
    return np.stack([r * np.sin(th)[None], y[:, None].repeat(cols, 1), r * np.cos(th)[None]], -1).reshape(-1, 3)


def tube_model(body: str = "smpl", seed: int = 0):
    """(body-model fields as posmap.PoseMapper takes them, the UV template, betas [10])."""
    smplx = body == "smplx"
    base = syn.make_smplx_body(seed) if smplx else syn.make_body(seed)
    template = syn.make_smplx_uv_template(seed) if smplx else syn.make_uv_template(seed)
    R, C = syn.UV_GRID_X if smplx else syn.UV_GRID
    V = base.v_template.shape[0]
    v = np.zeros((V, 3))
    v[:R * C] = tube_points(R, C)
    v[R * C:] = [0.0, TUBE_Y[1], 0.0]                    # SMPL-X's last 25 vertices belong to no face
    joints, parents, _ = syn._SKELETON[body]
    pts = torch.from_numpy(v)
    W = syn._skin_weights(pts, joints=joints, parents=parents)
    d2 = ((torch.tensor(joints)[:, None] - pts[None]) ** 2).sum(-1)
    Jr = torch.softmax(-d2 / 0.002, dim=1)
    tube = syn.SyntheticBody(pts.float(), base.shapedirs, base.posedirs, Jr.float(), base.parents, W.float(), base.betas)
    template = (v, template[1], template[2], template[3])
    model = syn.smplx_mesh_model(tube, template, syn.smplx_posedirs(seed)) if smplx else syn.smpl_mesh_model(tube, template)
    return model, template, base.betas[0]


def tube_avatar(body: str = "smpl", stage: int = 1, S: int = 256, inp: int = 32, seed: int = 0, device="cuda"):
    """(model, the body's PoseMapper at the input-map size, template, pose, transl, rest_pose | None) of an untrained avatar on the
    tube: the decoder's weights are the seeded initialisation, its opacity head biased as tests/test_mesh_extract_gpu.py biases it."""
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.body import body_of
    from gaussianavatar_b200.config import NetworkParams
    from gaussianavatar_b200.posmap import PoseMapper, canonical_assets
    from gaussianavatar_b200.workload import load_poses
    model, template, betas = tube_model(body, seed)
    dev = torch.device(device)
    ca = canonical_assets(model, betas, template, S, body, device=dev)
    valid = (ca.face_id.reshape(-1) >= 0).cpu()
    assets = dict(valid_idx=valid, query_points=ca.posmap.reshape(-1, 3)[valid.to(dev)].cpu(),
                  query_lbs=ca.lbs_map.reshape(S * S, -1)[valid.to(dev)].cpu(), cano_joint_mats=ca.joint_mats.cpu(),
                  rest_joints=PoseMapper(model, betas, template, 1, device=dev, body=body_of(body)).rest_joints.cpu(), betas=betas, S=S,
                  smpl_type=body)
    pose, transl, _ = load_poses(4)
    if body == "smplx":
        pose = pose[:, :66].contiguous()
    fields = dict(train_stage=2, inp_posmap_size=inp) if stage == 2 else {}
    torch.manual_seed(0)
    m = AvatarModel.from_assets(assets, [], pose, transl, batch_size=1, train=False, net_parms=NetworkParams(nf=8), device=dev, **fields)
    with torch.no_grad():
        sd = m.net.state_dict()
        sd["decoder.conv8N.bias"] = torch.tensor([-5.3])
        m.net.load_state_dict(sd, strict=False)
    mapper = PoseMapper(model, betas, template, inp, device=dev, body=body_of(body))
    rest = syn.synthetic_smplx_poses(1, seed=0)[1].to(dev) if body == "smplx" else None
    return m, mapper, template, pose[1].to(dev), transl[1].to(dev), rest
