"""ORACLE — TEST INFRASTRUCTURE ONLY.

SMPL-X (55 joints) counterpart of `oracle.avatar_oracle.smpl_joint_transforms`: plain-torch CPU restatement (fp32 or fp64) of
`SMPLX.forward(...).A` as model/avatar_model.py:281-289 calls it (use_pca=False, flat_hand_mean=True: no pose mean, no
expression).  Pinned against the reference's own `smplx.SMPLX` by oracle/gen_golden_smplx.py (tests/golden/smplx_A.npz);
tests/test_smplx_cpu.py re-checks it against that fixture on every run.

Only tests/ may import this module.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle.avatar_oracle import batch_rodrigues

# SMPL-X kintree_table[0]: global, 21 body, jaw, left eye, right eye, 15 left-hand, 15 right-hand joints
SMPLX_PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 15, 15, 15, 20, 25, 26, 20, 28, 29, 20,
                 31, 32, 20, 34, 35, 20, 37, 38, 21, 40, 41, 21, 43, 44, 21, 46, 47, 21, 49, 50, 21, 52, 53]


def joint_transforms(J: torch.Tensor, pose: torch.Tensor, transl: torch.Tensor, parents=SMPLX_PARENTS) -> torch.Tensor:
    """A [B,J,4,4] of lbs(..., return_affine_mat=True) (submodules/smplx/lbs.py:152-252) reduced to what feeds A — Rodrigues
    (:299-333), kinematic chain (:349-405), `G - pad(G J)` (:402-403) — plus `A[:,:,:3,3] += transl` (body_models.py).
    J [nj,3] rest joints; pose [B, 3 nj]: for SMPL-X the full pose [pose (66) | rest_pose (99)]."""
    B, nj = pose.shape[0], len(parents)
    R = batch_rodrigues(pose.reshape(-1, 3)).view(B, nj, 3, 3)
    rel = J.clone()
    rel[1:] = J[1:] - J[torch.tensor(parents[1:])]
    local = torch.zeros(B, nj, 4, 4, dtype=pose.dtype)
    local[:, :, :3, :3] = R
    local[:, :, :3, 3] = rel[None]
    local[:, :, 3, 3] = 1
    chain = [local[:, 0]]
    for i in range(1, nj):
        chain.append(torch.matmul(chain[parents[i]], local[:, i]))
    G = torch.stack(chain, dim=1)
    Jh = F.pad(J, [0, 1])[None, :, :, None].to(pose.dtype)                       # [1,nj,4,1]
    A = G - F.pad(torch.matmul(G, Jh), [3, 0])
    A = A.clone()
    A[:, :, :3, 3] = A[:, :, :3, 3] + transl[:, None, :]
    return A


def smplx_joint_transforms(J: torch.Tensor, pose66: torch.Tensor, rest99: torch.Tensor, transl: torch.Tensor) -> torch.Tensor:
    """`SMPLX.forward(global_orient=pose[:, :3], body_pose=pose[:, 3:66], jaw/leye/reye/left_hand/right_hand = rest_pose split,
    transl=transl).A` [B,55,4,4] (model/avatar_model.py:281-289)."""
    return joint_transforms(J, torch.cat([pose66, rest99], 1), transl, SMPLX_PARENTS)
