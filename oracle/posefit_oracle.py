"""ORACLE — TEST INFRASTRUCTURE ONLY.  An fp64 torch restatement of vertex posing (SMPL and SMPL-X) and of the position-map fill, so
that torch autograd gives the reference gradients for the backward kernels of csrc/posmap.cu (ga_smpl_vertices_backward,
ga_smplx_vertices_backward, ga_posmap_fill_backward):

  vertices   posed vertices [B,V,3]: shape blend shapes, pose blend shapes (R_j - I, j >= 1), joint chain, LBS, transl, with the
             reference's Rodrigues (theta = |r + 1e-8|); SMPL-X takes the full pose [pose 66 | rest_pose 99];
  fill       the maps [B,3,S,S] = sum_i w_i x[f_i], 0 where no face covers the texel.

tests/test_posefit_cpu.py checks its forward against oracle/posmap_oracle.py and oracle/cano_oracle.py (pinned to the golden
fixtures) and its gradients against central differences.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle.cano_oracle import SMPLX_PARENTS
from oracle.posmap_oracle import PARENTS as SMPL_PARENTS


def _dense(x):
    return np.asarray(x.todense() if hasattr(x, "todense") else x, np.float64)


class Body:
    """The constant part of a body model in fp64: v_shaped [V,3], rest joints [J,3], posedirs [V,3,nf], weights [V,J]."""

    def __init__(self, model, betas):
        betas = np.asarray(betas, np.float64).reshape(-1)
        v_t = np.asarray(model["v_template"], np.float64)
        sd = np.asarray(model["shapedirs"], np.float64)[:, :, :betas.size]
        v_shaped = v_t + sd @ betas
        self.v_shaped = torch.from_numpy(v_shaped)
        self.J = torch.from_numpy(_dense(model["J_regressor"]) @ v_shaped)
        self.posedirs = torch.from_numpy(np.asarray(model["posedirs"], np.float64))
        self.weights = torch.from_numpy(np.asarray(model["weights"], np.float64))
        self.parents = SMPL_PARENTS if self.J.shape[0] == 24 else SMPLX_PARENTS


def rotations(aa):
    """[n,3] axis-angle -> [n,3,3] (differentiable)."""
    theta = torch.linalg.norm(aa + 1e-8, dim=1, keepdim=True)
    d = aa / theta
    z = torch.zeros_like(d[:, 0])
    K = torch.stack([z, -d[:, 2], d[:, 1], d[:, 2], z, -d[:, 0], -d[:, 1], d[:, 0], z], 1).reshape(-1, 3, 3)
    s, c = torch.sin(theta)[:, :, None], torch.cos(theta)[:, :, None]
    return torch.eye(3, dtype=aa.dtype, device=aa.device) + s * K + (1.0 - c) * (K @ K)


def vertices(body: Body, full_pose, transl):
    """full_pose [B,3J] (SMPL: 72; SMPL-X: pose 66 | rest_pose 99), transl [B,3] -> [B,V,3], all fp64 torch on the body's device."""
    nj = len(body.parents)
    out = []
    for b in range(full_pose.shape[0]):
        R = rotations(full_pose[b].reshape(nj, 3))
        feat = (R[1:] - torch.eye(3, dtype=R.dtype, device=R.device)).reshape(-1)
        v_posed = body.v_shaped + body.posedirs @ feat
        G = []
        for j in range(nj):
            p = body.parents[j]
            t = body.J[j] - (body.J[p] if p >= 0 else 0.0)
            L = torch.cat([torch.cat([R[j], t[:, None]], 1), torch.tensor([[0.0, 0.0, 0.0, 1.0]], dtype=R.dtype, device=R.device)], 0)
            G.append(L if p < 0 else G[p] @ L)
        G = torch.stack(G)
        A = torch.cat([G[:, :3, :3], (G[:, :3, 3] - torch.einsum("jab,jb->ja", G[:, :3, :3], body.J))[:, :, None]], 2)   # [J,3,4]
        T = torch.einsum("vj,jab->vab", body.weights, A)
        out.append(torch.einsum("vab,vb->va", T[:, :, :3], v_posed) + T[:, :, 3] + transl[b])
    return torch.stack(out)


def fill(verts, faces, face_id, bary):
    """verts [B,V,3] (fp64 torch), faces [F,3], face_id [S,S], bary [S,S,3] (numpy) -> [B,3,S,S] fp64 torch."""
    S = face_id.shape[0]
    cov = torch.from_numpy(np.asarray(face_id).reshape(-1) >= 0)
    tri = torch.from_numpy(np.asarray(faces, np.int64)[np.asarray(face_id).reshape(-1)[cov.numpy()]])          # [n,3]
    w = torch.from_numpy(np.asarray(bary, np.float64).reshape(-1, 3)[cov.numpy()])                               # [n,3]
    x = torch.einsum("ni,bnic->bnc", w, verts[:, tri])                                                           # [B,n,3]
    out = torch.zeros(verts.shape[0], S * S, 3, dtype=verts.dtype)
    out[:, cov] = x
    return out.permute(0, 2, 1).reshape(verts.shape[0], 3, S, S)
