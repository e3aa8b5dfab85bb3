"""The two body models this library poses, SMPL (24 joints) and SMPL-X (55 joints), as data: every module that needs to know a
pose width, a joint count, a kinematic tree or which C entry point poses which body reads it from here.

SMPL-X poses follow the reference's smplx.SMPLX(use_pca=False, flat_hand_mean=True) split: the trained pose [B,66] (global + 21
body joints) and the frame's rest_pose [B,99] (jaw, left / right eye, 15 + 15 finger joints), 165 columns in all.  SMPL has no
rest_pose: its full pose is the trained pose [B,72].
"""
from __future__ import annotations

import os
from dataclasses import dataclass

import numpy as np
import torch

SMPL_PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21]
# SMPL-X: joint order global, 21 body, jaw, left eye, right eye, 15 left-hand, 15 right-hand (index, middle, pinky, ring, thumb;
# three segments each), kintree_table[0] of SMPLX_*.npz
SMPLX_PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 15, 15, 15, 20, 25, 26, 20, 28, 29, 20,
                 31, 32, 20, 34, 35, 20, 37, 38, 21, 40, 41, 21, 43, 44, 21, 46, 47, 21, 49, 50, 21, 52, 53]
SMPL_JOINT_NAMES = ("pelvis", "left_hip", "right_hip", "spine1", "left_knee", "right_knee", "spine2", "left_ankle", "right_ankle", "spine3",
                    "left_foot", "right_foot", "neck", "left_collar", "right_collar", "head", "left_shoulder", "right_shoulder",
                    "left_elbow", "right_elbow", "left_wrist", "right_wrist", "left_hand", "right_hand")
SMPLX_JOINT_NAMES = SMPL_JOINT_NAMES[:22] + ("jaw", "left_eye", "right_eye") + tuple(
    f"{side}_{finger}{s}" for side in ("left", "right") for finger in ("index", "middle", "pinky", "ring", "thumb") for s in (1, 2, 3))

MESH_FIELDS = ("v_template", "shapedirs", "posedirs", "weights", "f", "J_regressor")


@dataclass(frozen=True)
class Body:
    name: str                   # smpl_type, and the suffix of the reference's per-body file names
    label: str                  # for messages
    joints: int
    pose_width: int             # pose columns a model trains (the pose table's width)
    rest_width: int             # columns the frame supplies and nothing trains (SMPL-X's rest_pose)
    pose_features: int          # pose-blend features: 9 per non-root joint
    lbs_ld: int                 # row width of the skinning table the LBS kernel reads (SMPL-X: 55 padded to whole float4s)
    parents: tuple
    model_dir: str              # the ModelParams field naming the directory of the body-model file
    model_file: str             # the body-model file in it, {gender} upper case
    cano2live: str              # C entry points: joint transforms, their backward,
    cano2live_bwd: str
    vertices: str               # posed vertices, their backward and that backward's workspace size
    vertices_bwd: str
    vertices_bwd_ws: str

    @property
    def full_width(self) -> int:
        return self.pose_width + self.rest_width

    def pose_args(self, pose, rest_pose) -> tuple:
        """The pose arguments the body's C entry points take: (pose,) or (pose, rest_pose)."""
        return (pose, rest_pose)[:1 + (self.rest_width > 0)]

    def split(self, full):
        """A full pose [F,full_width] -> (pose [F,pose_width], rest_pose [F,rest_width] or None), both contiguous."""
        full = torch.as_tensor(full)
        if full.dim() != 2 or full.shape[1] != self.full_width:
            raise ValueError(f"pose {tuple(full.shape)}: expected [F,{self.full_width}] for {self.label}")
        pose, rest_pose = full[:, :self.pose_width].contiguous(), full[:, self.pose_width:].contiguous()
        return pose, (rest_pose if self.rest_width else None)

    def join(self, pose, rest_pose):
        """The inverse of `split`."""
        return torch.cat([pose, rest_pose], 1) if self.rest_width else pose

    def check_model(self, fields):
        """Raises ValueError unless the body-model fields hold the whole mesh model and the kinematic tree the kernels are built for."""
        missing = [k for k in MESH_FIELDS if k not in fields]
        if missing:
            raise ValueError(f"the {self.label} model has no {', '.join(missing)}: device position maps need the full mesh model")
        self._check_tree(fields)

    def _check_tree(self, fields):
        if "kintree_table" not in fields:
            raise ValueError(f"the {self.label} model has no kintree_table")
        kt = np.asarray(fields["kintree_table"]).astype(np.int64)[0].copy()
        kt[0] = -1
        if kt.shape != (self.joints,) or not np.array_equal(kt, np.asarray(self.parents)):
            raise ValueError(f"{self.label} model: kintree_table[0] is not the {self.joints}-joint {self.label} tree this library is "
                             "built for")

    def rest_joints(self, fields, betas) -> torch.Tensor:
        """Rest joints J = J_regressor (v_template + shapedirs[:, :, :len(betas)] betas) [J,3] fp32, formed in fp64.  The shape
        directions past the betas (SMPL-X's expression) drop out.  The model's kintree_table must be this body's tree."""
        self._check_tree(fields)
        Jr = fields["J_regressor"]
        Jr = torch.as_tensor(np.asarray(Jr.todense() if hasattr(Jr, "todense") else Jr)).double()
        return (Jr @ shaped_vertices(fields, betas)).float()


def shaped_vertices(fields, betas) -> torch.Tensor:
    """v_template + shapedirs[:, :, :len(betas)] betas [V,3] fp64."""
    beta = torch.as_tensor(betas).double().reshape(-1)
    v_t = torch.as_tensor(np.asarray(fields["v_template"])).double()
    sd = torch.as_tensor(np.asarray(fields["shapedirs"])[:, :, :beta.numel()]).double()
    return v_t + torch.einsum("l,mkl->mk", beta, sd)


SMPL = Body("smpl", "SMPL", 24, 72, 0, 207, 24, tuple(SMPL_PARENTS), "smpl_model_path", "SMPL_{gender}.pkl",
            "ga_smpl_forward", "ga_smpl_backward",
            "ga_smpl_vertices", "ga_smpl_vertices_backward", "ga_smpl_vertices_backward_workspace_bytes")
SMPLX = Body("smplx", "SMPL-X", 55, 66, 99, 486, 56, tuple(SMPLX_PARENTS), "smplx_model_path", "SMPLX_{gender}.npz",
             "ga_smplx_forward", "ga_smplx_backward",
             "ga_smplx_vertices", "ga_smplx_vertices_backward", "ga_smplx_vertices_backward_workspace_bytes")
BODIES = {b.name: b for b in (SMPL, SMPLX)}


def body_of(name: str) -> Body:
    """The body of a smpl_type / --body name."""
    if name not in BODIES:
        raise ValueError(f"body {name!r} is neither 'smpl' nor 'smplx'")
    return BODIES[name]


def load_model(path):
    """The fields of a body-model file as a dict: SMPL_{GENDER}.pkl (a pickle) or SMPLX_{GENDER}.npz."""
    if not os.path.exists(path):
        raise FileNotFoundError(f"body model {path} not found")
    if str(path).endswith(".npz"):
        with np.load(path, allow_pickle=True) as z:
            return {k: z[k] for k in z.files}
    import pickle
    with open(path, "rb") as fh:
        return dict(pickle.load(fh, encoding="latin1"))
