"""Deterministic synthetic stand-ins for the licensed / un-shipped assets of the reference (SURVEY.md §8d).

The reference needs the SMPL model pickle, UV masks, an LBS-weight map and canonical position maps from a OneDrive
archive (/root/reference README.md:41-54) that is not available offline.  This module produces tensors with the SAME
contracts (shapes, dtypes, value ranges, sparsity) so every kernel runs on realistic sizes:

  body      SMPL topology constants (24 joints, kinematic parents), a procedural 1.7 m T-pose skeleton, 6890
            pseudo-vertices on bone capsules, shapedirs / posedirs / J_regressor / lbs_weights of the right shapes
            (what submodules/smplx/lbs.py:152-163 consumes)
  avatar    N canonical "query" points in the star pose (arguments/__init__.py:44-53), their [N,24] skinning weights
            (<= 4 non-zeros per point like barycentric-interpolated SMPL weights, utils/general_utils.py:245-259), an
            S x S UV validity mask with exactly N valid pixels, inv(A_cano) (model/avatar_model.py:64,89)

The same for SMPL-X (55 joints: the 22 body joints of the SMPL skeleton, jaw, two eyes and three-segment fingers from the
wrists; 10475 pseudo-vertices): `make_avatar_assets(..., body="smplx")`, and `write_smplx_model_npz` writes a model file in the
layout of SMPLX_{GENDER}.npz that the reference's `smplx.SMPLX` loads.

Asset generation is one-off host work (numpy / torch CPU, float64 where it matters), not part of the per-frame path.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

from .body import SMPL_PARENTS, SMPLX_PARENTS

NUM_JOINTS = 24
NUM_VERTS = 6890

# approximate SMPL-neutral rest joints (metres; y up, +x = subject's left)
_REST_JOINTS = np.array([
    [0.00, -0.22, 0.03], [0.07, -0.31, 0.02], [-0.07, -0.31, 0.02], [0.00, -0.11, 0.00],
    [0.10, -0.70, 0.02], [-0.10, -0.70, 0.02], [0.00, 0.02, 0.02], [0.09, -1.10, -0.02],
    [-0.09, -1.10, -0.02], [0.00, 0.08, 0.00], [0.11, -1.16, 0.10], [-0.11, -1.16, 0.10],
    [0.00, 0.29, -0.02], [0.08, 0.20, 0.00], [-0.08, 0.20, 0.00], [0.00, 0.37, 0.03],
    [0.18, 0.23, -0.01], [-0.18, 0.23, -0.01], [0.44, 0.23, -0.03], [-0.44, 0.23, -0.03],
    [0.69, 0.23, -0.02], [-0.69, 0.23, -0.02], [0.78, 0.22, -0.02], [-0.78, 0.22, -0.02]], dtype=np.float64)

# capsule radius of the bone ending at joint j (bone = parent(j) -> j); joint 0 gets a pelvis blob
_BONE_RADIUS = np.array([0.12, 0.10, 0.10, 0.13, 0.075, 0.075, 0.14, 0.05, 0.05, 0.14, 0.04, 0.04,
                         0.06, 0.08, 0.08, 0.095, 0.06, 0.06, 0.045, 0.045, 0.035, 0.035, 0.03, 0.03], dtype=np.float64)

# ---- SMPL-X
SMPLX_NUM_JOINTS = 55
SMPLX_NUM_VERTS = 10475      # the reference's vertex-joint selector indexes SMPL-X vertex ids


def _smplx_rest_joints() -> np.ndarray:
    J = np.zeros((SMPLX_NUM_JOINTS, 3))
    J[:22] = _REST_JOINTS[:22]
    J[22] = J[15] + [0.00, -0.04, 0.07]           # jaw
    J[23] = J[15] + [0.03, 0.05, 0.08]            # left eye
    J[24] = J[15] + [-0.03, 0.05, 0.08]           # right eye
    # fingers: base offset from the wrist (y, z) and segment length; +x is the left hand's outward direction
    fingers = [(0.010, 0.025, 0.030), (0.0, 0.008, 0.032), (-0.012, -0.030, 0.022), (-0.006, -0.012, 0.028), (-0.015, 0.045, 0.026)]
    for side, wrist, base in ((1.0, 20, 25), (-1.0, 21, 40)):
        for k, (dy, dz, seg) in enumerate(fingers):
            start = J[wrist] + [side * (0.08 if k < 4 else 0.03), dy, dz]
            for s in range(3):
                J[base + 3 * k + s] = start + [side * seg * s, 0.0, 0.0]
    return J


_REST_JOINTS_X = _smplx_rest_joints()
_BONE_RADIUS_X = np.concatenate([_BONE_RADIUS[:22], [0.04, 0.012, 0.012], np.full(30, 0.009)])


def star_pose() -> np.ndarray:
    """Canonical pose of the reference: legs opened by 30 degrees (arguments/__init__.py:44-53)."""
    p = np.zeros(72, dtype=np.float64)
    p[5] = 30.0 / 180.0 * math.pi
    p[8] = -30.0 / 180.0 * math.pi
    return p


CANO_TRANSL = np.array([0.0, 0.30, 0.0], dtype=np.float64)   # scripts/gen_pose_map_cano_smpl.py:60-70


def rodrigues_np(r: np.ndarray) -> np.ndarray:
    """Axis-angle [J,3] -> [J,3,3] with the reference's shifted-norm convention (submodules/smplx/lbs.py:317)."""
    angle = np.linalg.norm(r + 1e-8, axis=1, keepdims=True)
    d = r / angle
    c, s = np.cos(angle)[:, :, None], np.sin(angle)[:, :, None]
    K = np.zeros((r.shape[0], 3, 3))
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 0], K[:, 1, 2], K[:, 2, 0], K[:, 2, 1] = -d[:, 2], d[:, 1], d[:, 2], -d[:, 0], -d[:, 1], d[:, 0]
    return np.eye(3)[None] + s * K + (1 - c) * (K @ K)


def joint_transforms_np(J: np.ndarray, pose72: np.ndarray, transl: np.ndarray | None = None, parents=SMPL_PARENTS) -> np.ndarray:
    """Relative joint transforms A [J,4,4] (float64) — closed form of lbs(..., return_affine_mat=True)
    (SURVEY.md Appendix B.3; submodules/smplx/lbs.py:349-405, body_models.py:380-383).  Host-side, asset generation only.
    pose72 is the full pose, 3 per joint of `parents` (SMPL-X: [pose 66 | rest_pose 99])."""
    nj = len(parents)
    R = rodrigues_np(pose72.reshape(nj, 3).astype(np.float64))
    G = np.zeros((nj, 4, 4))
    for j in range(nj):
        L = np.eye(4)
        L[:3, :3] = R[j]
        L[:3, 3] = J[j] if j == 0 else J[j] - J[parents[j]]
        G[j] = L if j == 0 else G[parents[j]] @ L
    A = G.copy()
    for j in range(nj):
        A[j, :3, 3] = G[j, :3, 3] - G[j, :3, :3] @ J[j]
    if transl is not None:
        A[:, :3, 3] += transl[None]
    return A


@dataclass
class SyntheticBody:
    """Tensor contract of the SMPL buffers `smplx.lbs.lbs` takes (submodules/smplx/lbs.py:152-163).  SMPL-X: 10475 vertices,
    55 joints, shapedirs [V,3,20] (10 shape + 10 expression directions; only the shape part is used), posedirs empty."""
    v_template: torch.Tensor    # [6890,3]
    shapedirs: torch.Tensor     # [6890,3,10]
    posedirs: torch.Tensor      # [207, 20670]
    J_regressor: torch.Tensor   # [24,6890]
    parents: torch.Tensor       # [24] long
    lbs_weights: torch.Tensor   # [6890,24]
    betas: torch.Tensor         # [1,10]

    def rest_joints(self) -> torch.Tensor:
        """J = J_regressor (v_template + shapedirs beta): constant per subject (betas are fixed, avatar_model.py:95-98)."""
        sd = self.shapedirs.double()[:, :, :self.betas.shape[1]]
        v = self.v_template.double() + torch.einsum("l,mkl->mk", self.betas[0].double(), sd)
        return (self.J_regressor.double() @ v).float()


def _sample_on_capsules(n: int, g: torch.Generator, joints=_REST_JOINTS, parents=SMPL_PARENTS, radius=_BONE_RADIUS):
    """n points on the T-pose bone capsules (+ bone id and position), roughly area-uniform."""
    bones = [(parents[j], j) for j in range(1, len(parents))]
    length = np.array([np.linalg.norm(joints[b] - joints[a]) for a, b in bones])
    rad = np.array([radius[b] for _, b in bones])
    area = 2 * math.pi * rad * (length + 2 * rad)
    prob = torch.tensor(area / area.sum())
    bid = torch.multinomial(prob, n, replacement=True, generator=g)
    t = torch.rand(n, generator=g, dtype=torch.float64) * 1.2 - 0.1          # slight overshoot: rounded ends
    th = torch.rand(n, generator=g, dtype=torch.float64) * 2 * math.pi
    a = torch.tensor(joints)[torch.tensor([x for x, _ in bones])[bid]]
    b = torch.tensor(joints)[torch.tensor([y for _, y in bones])[bid]]
    axis = (b - a) / (b - a).norm(dim=1, keepdim=True)
    ref = torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64).expand(n, 3).clone()
    par = (axis * ref).sum(1).abs() > 0.9
    ref[par] = torch.tensor([1.0, 0.0, 0.0], dtype=torch.float64)
    u = torch.linalg.cross(axis, ref)
    u = u / u.norm(dim=1, keepdim=True)
    v = torch.linalg.cross(axis, u)
    r = torch.tensor(rad)[bid]
    end = ((t < 0) | (t > 1)).double()
    r_eff = r * torch.sqrt(torch.clamp(1 - end * ((t.clamp(0, 1) - t).abs() * (b - a).norm(dim=1) / r) ** 2, min=0.05))
    pts = a + (b - a) * t[:, None] + r_eff[:, None] * (torch.cos(th)[:, None] * u + torch.sin(th)[:, None] * v)
    return pts, bid


def _skin_weights(pts: torch.Tensor, tau: float = 0.0035, k: int = 4, joints=_REST_JOINTS, parents=SMPL_PARENTS) -> torch.Tensor:
    """softmax(-d^2/tau) over the k nearest bones; a bone's weight goes to its PARENT-side joint (the joint that moves it)."""
    bones = [(parents[j], j) for j in range(1, len(parents))]
    J = torch.tensor(joints)
    a = J[torch.tensor([x for x, _ in bones])]
    b = J[torch.tensor([y for _, y in bones])]
    ab = b - a
    t = ((pts[:, None] - a[None]) * ab[None]).sum(-1) / (ab * ab).sum(-1)[None]
    q = a[None] + t.clamp(0, 1)[..., None] * ab[None]
    d2 = ((pts[:, None] - q) ** 2).sum(-1)                                    # [n, 23]
    near = torch.topk(-d2, k, dim=1)
    w = torch.softmax(near.values / tau, dim=1)
    W = torch.zeros(pts.shape[0], len(parents), dtype=torch.float64)
    owner = torch.tensor([x for x, _ in bones])                               # parent-side joint of each bone
    W.scatter_add_(1, owner[near.indices], w)
    return W


def make_body(seed: int = 0) -> SyntheticBody:
    g = torch.Generator().manual_seed(1000 + seed)
    v, _ = _sample_on_capsules(NUM_VERTS, g)
    W = _skin_weights(v)
    # J_regressor: softmax rows concentrated around each joint, then corrected so that J_regressor @ v_template
    # reproduces the rest skeleton closely (the regressor of the real model has the same property)
    d2 = ((torch.tensor(_REST_JOINTS)[:, None] - v[None]) ** 2).sum(-1)
    Jr = torch.softmax(-d2 / 0.002, dim=1)
    shapedirs = torch.randn(NUM_VERTS, 3, 10, generator=g, dtype=torch.float64) * 0.01
    posedirs = torch.randn(207, NUM_VERTS * 3, generator=g, dtype=torch.float64) * 0.001
    betas = torch.tensor([[-0.4732, -0.8652, 0.3936, 0.0133, -1.2825, -0.9797, -0.1731, 0.0270, -0.0786, -0.1593]])
    return SyntheticBody(v.float(), shapedirs.float(), posedirs.float(), Jr.float(), torch.tensor(SMPL_PARENTS, dtype=torch.long),
                         W.float(), betas.float())


_SKELETON = {"smpl": (_REST_JOINTS, SMPL_PARENTS, _BONE_RADIUS), "smplx": (_REST_JOINTS_X, SMPLX_PARENTS, _BONE_RADIUS_X)}


def make_smplx_body(seed: int = 0) -> SyntheticBody:
    """The SMPL-X counterpart of make_body: 10475 vertices on the 55-joint skeleton's capsules, a J_regressor concentrated around
    each joint, shapedirs [V,3,20], skinning weights [V,55]."""
    sk = _SKELETON["smplx"]
    g = torch.Generator().manual_seed(5000 + seed)
    v, _ = _sample_on_capsules(SMPLX_NUM_VERTS, g, *sk)
    W = _skin_weights(v, joints=sk[0], parents=sk[1])
    d2 = ((torch.tensor(sk[0])[:, None] - v[None]) ** 2).sum(-1)
    Jr = torch.softmax(-d2 / 0.002, dim=1)
    shapedirs = torch.randn(SMPLX_NUM_VERTS, 3, 20, generator=g, dtype=torch.float64) * 0.01
    betas = torch.tensor([[-0.4732, -0.8652, 0.3936, 0.0133, -1.2825, -0.9797, -0.1731, 0.0270, -0.0786, -0.1593]])
    return SyntheticBody(v.float(), shapedirs.float(), torch.zeros(0), Jr.float(), torch.tensor(SMPLX_PARENTS, dtype=torch.long),
                         W.float(), betas.float())


def write_smplx_model_npz(path: str, body: SyntheticBody, seed: int = 0, posedirs=None, faces=None) -> None:
    """SMPLX_{GENDER}.npz in the layout the reference's `smplx.SMPLX(..., use_pca=False, flat_hand_mean=True)` loads: faces,
    template, shape / pose directions, dense J_regressor, kintree_table, skinning weights, hand PCA placeholders and the landmark
    embedding.  By default the pose directions are zero and the faces random; posedirs [486, 3V] (smplx_posedirs) and faces [F,3]
    (a template's, make_smplx_uv_template) make a model whose mesh can be posed and drawn into position maps."""
    rng = np.random.default_rng(seed)
    V, nj = body.v_template.shape[0], len(SMPLX_PARENTS)
    kt = np.zeros((2, nj), np.int64)
    kt[0] = SMPLX_PARENTS
    kt[0, 0] = 4294967295          # uint32 -1, as the released model files store it
    kt[1] = np.arange(nj)
    f = rng.integers(0, V, (20908, 3)).astype(np.int64)
    if faces is not None:
        f = np.asarray(faces, np.int64)
    pd = np.zeros((V, 3, 486), np.float32) if posedirs is None else _posedirs_per_vertex(posedirs, V, 486)
    np.savez_compressed(path, f=f, v_template=body.v_template.double().numpy(),
                        shapedirs=body.shapedirs.double().numpy(), posedirs=pd,
                        J_regressor=body.J_regressor.double().numpy(), kintree_table=kt, weights=body.lbs_weights.double().numpy(),
                        hands_componentsl=np.eye(45), hands_componentsr=np.eye(45), hands_meanl=rng.normal(size=45) * 0.1,
                        hands_meanr=rng.normal(size=45) * 0.1, lmk_faces_idx=np.arange(51, dtype=np.int64),
                        lmk_bary_coords=np.full((51, 3), 1.0 / 3.0))


@dataclass
class SyntheticAvatarAssets:
    body: SyntheticBody
    S: int                       # query_posmap_size
    N: int                       # valid UV pixels == Gaussians
    valid_idx: torch.Tensor      # [S*S] bool, exactly N True
    query_points: torch.Tensor   # [N,3] canonical (star-pose) positions
    query_lbs: torch.Tensor      # [N,24] (SMPL-X: [N,55])
    cano_joint_mats: torch.Tensor  # [24,4,4] A_cano  (smpl_cano_joint_mat.pth; SMPL-X: [55,4,4])
    rest_joints: torch.Tensor    # [24,3] (SMPL-X: [55,3])
    smpl_type: str = "smpl"      # the body: "smpl" or "smplx"


def make_avatar_assets(N: int, S: int, seed: int = 0, body: str = "smpl") -> SyntheticAvatarAssets:
    """body: "smpl" (24 joints) or "smplx" (55 joints, canonical pose = the star pose with zero hand / face pose)."""
    assert N <= S * S and body in _SKELETON
    joints, parents, radius = _SKELETON[body]
    smpl_type, smplx = body, body == "smplx"
    body = make_smplx_body(seed) if smplx else make_body(seed)
    g = torch.Generator().manual_seed(2000 + seed)
    pts, _ = _sample_on_capsules(N, g, joints, parents, radius)
    W = _skin_weights(pts, joints=joints, parents=parents)
    J = body.rest_joints().double().numpy()
    cano_pose = np.concatenate([star_pose()[:66], np.zeros(99)]) if smplx else star_pose()
    A_cano = joint_transforms_np(J, cano_pose, CANO_TRANSL, parents)
    M = torch.einsum("nj,jxy->nxy", W, torch.tensor(A_cano))
    cano = torch.einsum("nxy,ny->nx", M[:, :3, :3], pts) + M[:, :3, 3]
    valid = torch.zeros(S * S, dtype=torch.bool)
    valid[torch.randperm(S * S, generator=g)[:N]] = True
    return SyntheticAvatarAssets(body, S, N, valid, cano.float().contiguous(), W.float().contiguous(),
                                 torch.tensor(A_cano).float(), torch.tensor(J).float(), smpl_type)


# BASELINE.json configs -> (N, S, image side)   (BASELINE.md §4)
CONFIGS = {1: (10_000, 128, 256), 2: (50_000, 256, 512), 3: (200_000, 512, 1024), 4: (200_000, 512, 1024), 5: (500_000, 768, 2048)}


def synthetic_poses(n: int, seed: int = 0) -> tuple[torch.Tensor, torch.Tensor]:
    """Smooth random SMPL poses / translations in the range of assets/test_pose/smpl_parms.pth (used when the
    committed subset in tests/golden/ is not wanted)."""
    g = torch.Generator().manual_seed(3000 + seed)
    pose = torch.randn(n, 72, generator=g) * 0.15
    pose[:, :3] = torch.randn(n, 3, generator=g) * 0.05
    transl = torch.tensor([0.0012, 0.168, -0.021]) + torch.randn(n, 3, generator=g) * 0.01
    return pose.float(), transl.float()


UV_GRID = (53, 130)      # rows x columns of the synthetic UV template's vertex grid: 53 * 130 = 6890 vertices


def make_uv_template(seed: int = 0, jitter: float = 0.2):
    """A UV template for the 6890 synthetic vertices, in the form `posmap.load_uv_template_obj` returns: (verts, faces, uvs,
    faces_uv).  Vertex r * 130 + c sits at row r, column c of a grid; each grid cell gives two triangles (the diagonal alternates),
    row-major, 13416 faces.  The atlas has two islands side by side: columns 0..64 in u 0.02..0.48 and columns 64..129 in u
    0.52..0.98, so column 64 has two texture coordinates (a seam) and the vt indices differ from the v indices.  Interior texture
    coordinates are jittered by up to `jitter` of a cell."""
    return _grid_uv_template(UV_GRID, 64, np.random.default_rng(4000 + seed), jitter, make_body(seed).v_template.double().numpy())


UV_GRID_X = (50, 209)    # the SMPL-X template's grid: 10450 of the 10475 vertices (the last 25 belong to no face)


def make_smplx_uv_template(seed: int = 0, jitter: float = 0.2):
    """The SMPL-X counterpart of make_uv_template: a 50 x 209 grid over the first 10450 synthetic SMPL-X vertices (the other 25
    belong to no face), 20384 faces, two islands with the seam at column 104."""
    return _grid_uv_template(UV_GRID_X, 104, np.random.default_rng(4500 + seed), jitter, make_smplx_body(seed).v_template.double().numpy())


def _grid_uv_template(grid, seam, g, jitter, verts):
    R, C = grid
    islands = [(np.arange(0, seam + 1), 0.02, 0.48), (np.arange(seam, C), 0.52, 0.98)]
    uvs, vt_of = [], []
    for cols, u0, u1 in islands:
        n = cols.size
        u = np.linspace(u0, u1, n)[None, :].repeat(R, 0)
        v = np.linspace(0.02, 0.98, R)[:, None].repeat(n, 1)
        du, dv = (u1 - u0) / (n - 1), 0.96 / (R - 1)
        inner = np.zeros((R, n), bool)
        inner[1:-1, 1:-1] = True
        u = u + inner * g.uniform(-jitter, jitter, (R, n)) * du
        v = v + inner * g.uniform(-jitter, jitter, (R, n)) * dv
        base = sum(len(x) for x in uvs)
        vt_of.append({int(c): base + np.arange(R) * n + k for k, c in enumerate(cols)})
        uvs.append(np.stack([u, v], -1).reshape(-1, 2))
    uvs = np.concatenate(uvs)
    faces, faces_uv = [], []
    for r in range(R - 1):
        for c in range(C - 1):
            isl = vt_of[0] if c < seam else vt_of[1]
            a, b, cc, d = (r, c), (r, c + 1), (r + 1, c + 1), (r + 1, c)
            tris = [(a, b, cc), (a, cc, d)] if (r + c) % 2 == 0 else [(a, b, d), (b, cc, d)]
            for t in tris:
                faces.append([i * C + j for i, j in t])
                faces_uv.append([int(isl[j][i]) for i, j in t])
    faces, faces_uv = np.asarray(faces, np.int64), np.asarray(faces_uv, np.int64)
    p = uvs[faces_uv]
    area = (p[:, 1, 0] - p[:, 0, 0]) * (p[:, 2, 1] - p[:, 0, 1]) - (p[:, 1, 1] - p[:, 0, 1]) * (p[:, 2, 0] - p[:, 0, 0])
    assert (area > 0).all(), "jitter folded a triangle"
    return verts, faces, uvs, faces_uv


def write_uv_template_obj(path: str, template) -> None:
    """Write (verts, faces, uvs, faces_uv) as an OBJ with `v`, `vt` and `f v/vt` lines (the layout of template_mesh_smpl_uv.obj)."""
    verts, faces, uvs, faces_uv = template
    with open(path, "w") as fh:
        fh.writelines(f"v {x:.6f} {y:.6f} {z:.6f}\n" for x, y, z in verts)
        fh.writelines(f"vt {u!r} {v!r}\n" for u, v in uvs.tolist())
        fh.writelines(f"f {a + 1}/{ta + 1} {b + 1}/{tb + 1} {c + 1}/{tc + 1}\n" for (a, b, c), (ta, tb, tc) in zip(faces.tolist(), faces_uv.tolist()))


def smpl_mesh_model(body: SyntheticBody, template) -> dict:
    """The fields of SMPL_{GENDER}.pkl the position maps need, for a synthetic body: v_template, shapedirs, posedirs [V,3,207],
    weights, f (the template's faces), J_regressor, kintree_table."""
    V = body.v_template.shape[0]
    return dict(v_template=body.v_template.numpy(), shapedirs=body.shapedirs.numpy(), J_regressor=body.J_regressor.numpy(),
                posedirs=body.posedirs.T.reshape(V, 3, 207).contiguous().numpy(), weights=body.lbs_weights.numpy(),
                f=np.asarray(template[1], np.uint32), kintree_table=np.stack([np.array(SMPL_PARENTS), np.arange(24)]))


def smplx_posedirs(seed: int = 0) -> torch.Tensor:
    """Non-zero SMPL-X pose blend shapes [486, 3 * 10475] (the layout smplx.SMPLX keeps), of the scale of make_body's."""
    g = torch.Generator().manual_seed(5500 + seed)
    return (torch.randn(486, SMPLX_NUM_VERTS * 3, generator=g, dtype=torch.float64) * 0.001).float()


def _posedirs_per_vertex(posedirs, V, n) -> np.ndarray:
    """[n, 3V] -> [V,3,n], the layout of the model files."""
    return torch.as_tensor(posedirs).T.reshape(V, 3, n).contiguous().numpy()


def smplx_mesh_model(body: SyntheticBody, template, posedirs) -> dict:
    """The fields of SMPLX_{GENDER}.npz the position maps need, for a synthetic SMPL-X body: v_template, shapedirs, posedirs
    [V,3,486], weights [V,55], f (the template's faces), J_regressor, kintree_table."""
    V = body.v_template.shape[0]
    return dict(v_template=body.v_template.numpy(), shapedirs=body.shapedirs.numpy(), J_regressor=body.J_regressor.numpy(),
                posedirs=_posedirs_per_vertex(posedirs, V, 486), weights=body.lbs_weights.numpy(),
                f=np.asarray(template[1], np.int64), kintree_table=np.stack([np.array(SMPLX_PARENTS), np.arange(55)]))


def synthetic_smplx_poses(n: int, seed: int = 0) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Smooth random SMPL-X poses: pose [n,66] (global + body), rest_pose [n,99] (jaw, eyes, fingers curled up to ~0.5 rad), transl."""
    g = torch.Generator().manual_seed(3500 + seed)
    pose = torch.randn(n, 66, generator=g) * 0.15
    pose[:, :3] = torch.randn(n, 3, generator=g) * 0.05
    rest = torch.randn(n, 99, generator=g) * 0.1
    rest[:, 9:] += 0.3 * torch.rand(n, 90, generator=g)
    transl = torch.tensor([0.0012, 0.168, -0.021]) + torch.randn(n, 3, generator=g) * 0.01
    return pose.float(), rest.float(), transl.float()
