"""ORACLE — TEST INFRASTRUCTURE ONLY.  An independent numpy restatement of the canonical-asset kernels of csrc/posmap.cu, next to
oracle/posmap_oracle.py (whose Rodrigues it reuses and which it leaves unchanged):

  smplx_vertices  posed SMPL-X vertices in fp64 (ga_smplx_vertices): shape blend shapes, pose blend shapes (R_j - I, j >= 1) over
                  486 features, the 55-joint chain, LBS, transl (submodules/smplx/lbs.py:lbs + body_models.py:1206-1275 of the
                  reference: full pose = [pose 66 | rest_pose 99], flat hands, no expression);
  weight_map      the texel skinning weights [S,S,J] (ga_posmap_weights): sum_i w_i W[f_i] (fp64; utils/general_utils.py:245-259),
                  0 where no face covers the texel.

Pinned against the reference's own outputs by oracle/gen_golden_cano.py; tests/test_cano_assets_cpu.py re-checks it on every run.
"""
from __future__ import annotations

import numpy as np

from oracle.posmap_oracle import _rotations

SMPLX_PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 15, 15, 15, 20, 25, 26, 20, 28, 29, 20,
                 31, 32, 20, 34, 35, 20, 37, 38, 21, 40, 41, 21, 43, 44, 21, 46, 47, 21, 49, 50, 21, 52, 53]


def smplx_vertices(model, betas, pose66, rest99, transl):
    """model: v_template [V,3], shapedirs [V,3,>=10], posedirs [V,3,486], weights [V,55], J_regressor [55,V].  pose66 [B,66],
    rest99 [B,99], transl [B,3] -> [B,V,3] float64."""
    betas = np.asarray(betas, np.float64).reshape(-1)
    v_t = np.asarray(model["v_template"], np.float64)
    sd = np.asarray(model["shapedirs"], np.float64)[:, :, :betas.size]
    pd = np.asarray(model["posedirs"], np.float64)                       # [V,3,486]
    W = np.asarray(model["weights"], np.float64)
    Jr = model["J_regressor"]
    Jr = np.asarray(Jr.todense() if hasattr(Jr, "todense") else Jr, np.float64)
    v_shaped = v_t + sd @ betas
    J = Jr @ v_shaped
    nj = len(SMPLX_PARENTS)
    pose = np.concatenate([np.asarray(pose66, np.float64).reshape(-1, 66), np.asarray(rest99, np.float64).reshape(-1, 99)], 1)
    transl = np.asarray(transl, np.float64).reshape(-1, 3)
    out = np.empty((pose.shape[0], v_t.shape[0], 3))
    for b in range(pose.shape[0]):
        R = _rotations(pose[b].reshape(nj, 3))
        feat = (R[1:] - np.eye(3)).reshape(-1)
        v_posed = v_shaped + pd @ feat
        G = np.zeros((nj, 4, 4))
        for j in range(nj):
            L = np.eye(4)
            L[:3, :3] = R[j]
            L[:3, 3] = J[j] - (J[SMPLX_PARENTS[j]] if j else 0.0)
            G[j] = L if j == 0 else G[SMPLX_PARENTS[j]] @ L
        A = G.copy()
        A[:, :3, 3] -= np.einsum("jab,jb->ja", G[:, :3, :3], J)
        T = np.einsum("vj,jab->vab", W, A)
        out[b] = np.einsum("vab,vb->va", T[:, :3, :3], v_posed) + T[:, :3, 3] + transl[b]
    return out


def weight_map(weights, faces, face_id, bary):
    """weights [V,J], faces [F,3], face_id [S,S], bary [S,S,3] -> [S,S,J] float64."""
    W = np.asarray(weights, np.float64)
    S = face_id.shape[0]
    out = np.zeros((S, S, W.shape[1]))
    cov = face_id >= 0
    tri = np.asarray(faces)[face_id[cov]]                       # [n,3]
    out[cov] = np.einsum("ni,nij->nj", bary[cov].astype(np.float64), W[tri])
    return out
