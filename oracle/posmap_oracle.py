"""ORACLE — TEST INFRASTRUCTURE ONLY.  An independent numpy restatement of the device position maps (csrc/posmap.cu):

  smpl_vertices   posed SMPL vertices in fp64: shape blend shapes, pose blend shapes (R_j - I, j >= 1), joint chain, LBS, transl
                  (submodules/smplx/lbs.py:lbs + body_models.py:380-382 of the reference);
  layout          which face covers each texel centre of an S x S map and its barycentric weights, with the library's coverage
                  rules: corners snapped to 1/256 texel (round half to even), exact integer edge functions, one tie rule (an edge
                  owns the centres on it when, walked counter-clockwise with y up, it goes down, or left when horizontal), no
                  culling, lowest face index wins, faces of zero area and faces with a non-finite corner or a coordinate above 4096
                  in magnitude cover nothing; output row r samples v = 1 - (r + 0.5) / S;
  fill            the maps [B,3,S,S]: sum_i w_i x[f_i] (fp64), 0 where no face covers the texel.
"""
from __future__ import annotations

import numpy as np

PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21]


def _rotations(aa):
    """[n,3] axis-angle -> [n,3,3], theta = |r + 1e-8| as the reference's batch_rodrigues."""
    theta = np.linalg.norm(aa + 1e-8, axis=1)
    k = aa / theta[:, None]
    out = np.empty((aa.shape[0], 3, 3))
    for i in range(aa.shape[0]):
        x, y, z = k[i]
        K = np.array([[0.0, -z, y], [z, 0.0, -x], [-y, x, 0.0]])
        out[i] = np.eye(3) + np.sin(theta[i]) * K + (1.0 - np.cos(theta[i])) * (K @ K)
    return out


def smpl_vertices(smpl, betas, pose, transl):
    """smpl: v_template [V,3], shapedirs [V,3,>=10], posedirs [V,3,207], weights [V,24], J_regressor [24,V].  pose [B,72],
    transl [B,3] -> [B,V,3] float64."""
    betas = np.asarray(betas, np.float64).reshape(-1)
    v_t = np.asarray(smpl["v_template"], np.float64)
    sd = np.asarray(smpl["shapedirs"], np.float64)[:, :, :betas.size]
    pd = np.asarray(smpl["posedirs"], np.float64)                       # [V,3,207]
    W = np.asarray(smpl["weights"], np.float64)
    Jr = smpl["J_regressor"]
    Jr = np.asarray(Jr.todense() if hasattr(Jr, "todense") else Jr, np.float64)
    v_shaped = v_t + sd @ betas
    J = Jr @ v_shaped
    pose = np.asarray(pose, np.float64).reshape(-1, 72)
    transl = np.asarray(transl, np.float64).reshape(-1, 3)
    out = np.empty((pose.shape[0], v_t.shape[0], 3))
    for b in range(pose.shape[0]):
        R = _rotations(pose[b].reshape(24, 3))
        feat = (R[1:] - np.eye(3)).reshape(-1)
        v_posed = v_shaped + pd @ feat
        G = np.zeros((24, 4, 4))
        for j in range(24):
            L = np.eye(4)
            L[:3, :3] = R[j]
            L[:3, 3] = J[j] - (J[PARENTS[j]] if j else 0.0)
            G[j] = L if j == 0 else G[PARENTS[j]] @ L
        A = G.copy()
        A[:, :3, 3] -= np.einsum("jab,jb->ja", G[:, :3, :3], J)
        T = np.einsum("vj,jab->vab", W, A)
        out[b] = np.einsum("vab,vb->va", T[:, :3, :3], v_posed) + T[:, :3, 3] + transl[b]
    return out


def _snap(corners, S):
    c = np.asarray(corners, np.float32).astype(np.float64)
    ok = np.all(np.isfinite(c) & (np.abs(c) <= 4096.0), axis=(1, 2))
    q = np.zeros(c.shape, np.int64)
    q[ok] = np.rint(c[ok] * (256.0 * S)).astype(np.int64)
    return q, ok


def _cross(o, a, p):
    """(a - o) x (p - o), z component; o, a: int64 [2]; p: int64 [...,2]."""
    return (a[0] - o[0]) * (p[..., 1] - o[1]) - (a[1] - o[1]) * (p[..., 0] - o[0])


def _face_texels(p, S):
    """Texel centres face p (snapped int64 [3,2]) covers: (rows, cols, window points [n,2]), empty for a face of zero area."""
    none = (np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros((0, 2), np.int64))
    area = _cross(p[0], p[1], p[2])
    if area == 0:
        return none
    loop = [0, 1, 2] if area > 0 else [0, 2, 1]              # counter-clockwise traversal
    centre = 256 * np.arange(S, dtype=np.int64) + 128          # window coordinate of column c / window row k
    xs = centre[(centre >= p[:, 0].min()) & (centre <= p[:, 0].max())]
    ks = np.nonzero((centre >= p[:, 1].min()) & (centre <= p[:, 1].max()))[0]
    if xs.size == 0 or ks.size == 0:
        return none
    P = np.stack(np.meshgrid(xs, centre[ks], indexing="xy"), -1)     # [k, x, 2]
    inside = np.ones(P.shape[:2], bool)
    for e in range(3):
        a, b = p[loop[e]], p[loop[(e + 1) % 3]]
        d = b - a
        val = _cross(a, b, P)
        owns_tie = d[1] < 0 or (d[1] == 0 and d[0] < 0)
        inside &= (val > 0) | ((val == 0) & owns_tie)
    rows = (S - 1 - ks)[:, None].repeat(xs.size, 1)            # window row k is output row S-1-k
    cols = ((xs - 128) // 256)[None, :].repeat(ks.size, 0)
    return rows[inside], cols[inside], P[inside]


def coverage_count(corners, S):
    """[S,S] number of faces covering each texel centre (before the lowest index is picked)."""
    q, ok = _snap(corners, S)
    count = np.zeros((S, S), np.int64)
    for f in np.nonzero(ok)[0]:
        r, c, _ = _face_texels(q[f], S)
        np.add.at(count, (r, c), 1)
    return count


def layout(corners, S):
    """corners [F,3,2] UV -> (face_id [S,S] int32 with -1 for none, bary [S,S,3] float32)."""
    q, ok = _snap(corners, S)
    face_id = np.full((S, S), -1, np.int64)
    bary = np.zeros((S, S, 3), np.float32)
    for f in np.nonzero(ok)[0]:
        p = q[f]
        r, c, pts = _face_texels(p, S)
        sel = face_id[r, c] < 0                                  # faces come in index order: the first one wins
        r, c, pts = r[sel], c[sel], pts[sel]
        face_id[r, c] = f
        area = float(_cross(p[0], p[1], p[2]))
        for i in range(3):
            e = _cross(p[(i + 1) % 3], p[(i + 2) % 3], pts)
            bary[r, c, i] = (e.astype(np.float64) / area).astype(np.float32)
    return face_id.astype(np.int32), bary


def fill(verts, faces, face_id, bary):
    """verts [B,V,3], faces [F,3], face_id [S,S], bary [S,S,3] -> [B,3,S,S] float64."""
    verts = np.asarray(verts, np.float64)
    S = face_id.shape[0]
    out = np.zeros((verts.shape[0], 3, S, S))
    cov = face_id >= 0
    tri = np.asarray(faces)[face_id[cov]]                       # [n,3]
    w = bary[cov].astype(np.float64)
    for b in range(verts.shape[0]):
        x = np.einsum("ni,nic->nc", w, verts[b][tri])
        out[b][:, cov] = x.T
    return out
