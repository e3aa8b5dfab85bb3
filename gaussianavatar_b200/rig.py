"""A trained avatar as a rigged mesh: its canonical surface, the body skeleton, per-vertex skin weights taken from its own Gaussians,
and optionally a baked motion, written as a glTF 2.0 binary (.glb) that DCC tools and game engines load.

    rig = extract_rigged_mesh(model)                                  # canonical mesh + skeleton + skin weights (device)
    motion = bake_motion(model, MotionClip.load("walk.npz", "smpl"), fps=30)
    write_glb("avatar.glb", rig, motion)

Stage 1 is pure linear blend skinning: a Gaussian is posed by sum_j w_j cano2live_j with cano2live_j = A_j(pose) Cano_j^-1.  The glTF
skin reproduces that exactly: with the rest joints J_j and the canonical joint matrices Cano_j,
  inverse bind matrix   IBM_j = T(-J_j) Cano_j^-1
  bind-local rotation   R_parent(Cano)^T R_j(Cano)          (the root: R_0(Cano))
  node translation      J_j - J_parent                     (the root: Cano_0 J_0)
so that G_j(bind) IBM_j = I and, with each joint's local rotation set to the pose's Rodrigues matrix and the root's translation to
J_0 + transl, G_j(pose) IBM_j = cano2live_j(pose).  The mesh is the TSDF mesh of the canonical Gaussians (`mesh_extract`), and its
skin weights are blended from the k nearest Gaussians' skinning rows (`ga_skin_weights`, csrc/skin.cu).  Stage 2's pose-dependent
offsets are not carried: its rig is the canonical-pose decoder output.  Everything but the file writer runs on the current CUDA
stream; the model's parameters and BatchNorm statistics are left as they were.

    rig = extract_body_rig(model, "template_mesh_smpl_uv.obj", subdiv=1, pose_mapper=poser)   # the body model's own topology

`extract_body_rig` builds the rig in the body model's topology instead: the UV template subdivided by midpoints, fitted through the
Gaussians on the template's own UV layout (every Gaussian is a texel of it), skinned with the body model's weights and textured with
the decoder's colour map (DESIGN.md §2).  `render_rig_unlit` / `unlit_psnr` draw either kind of rig without lighting.
"""
from __future__ import annotations

import json
import math
import struct
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from ._lib import ptr
from .avatar_model import kept_state
from .body import SMPL_JOINT_NAMES, SMPLX, SMPLX_JOINT_NAMES
from .mesh_extract import mesh_gaussians
from .ops import LbsAssemble
from .synthetic import rodrigues_np

MAX_NEIGHBOURS, MAX_INFLUENCES = 16, 8       # ga_skin_weights: k, K
# the rotation taking a clip world's up axis to glTF's +Y
UP_ROTATIONS = {"y": np.eye(3), "z": np.array([[1.0, 0, 0], [0, 0, 1], [0, -1, 0]]), "-y": np.diag([1.0, -1.0, -1.0])}


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def skin_weights(verts, means, lbs, J: int, k: int = 8, K: int = 4):
    """ga_skin_weights on the current stream: verts [V,3], means [N,3], lbs [N,ld] (fp32, device) -> (joints [V,K] uint8, weights
    [V,K] fp32), heaviest first."""
    verts, means, lbs = (t.float().contiguous() for t in (verts, means, lbs))
    V, N, ld = int(verts.shape[0]), int(means.shape[0]), int(lbs.shape[1])
    joints = torch.empty(V, int(K), dtype=torch.uint8, device=verts.device)
    weights = torch.empty(V, int(K), dtype=torch.float32, device=verts.device)
    _lib.check(_lib.lib().ga_skin_weights(V, N, int(J), ld, int(k), int(K), ptr(verts), ptr(means), ptr(lbs), ptr(joints), ptr(weights),
                                          _stream()), "ga_skin_weights")
    return joints, weights


# ---- rotations --------------------------------------------------------------------------------------------------------------------
def quat_from_matrix(R) -> np.ndarray:
    """[...,3,3] rotation matrices -> [...,4] unit quaternions (x, y, z, w; glTF's order), w >= 0, fp64."""
    R = np.asarray(R, np.float64)
    m = R.reshape(-1, 3, 3)
    q = np.empty((m.shape[0], 4))
    tr = m[:, 0, 0] + m[:, 1, 1] + m[:, 2, 2]
    case = np.argmax(np.stack([tr, m[:, 0, 0], m[:, 1, 1], m[:, 2, 2]], 1), 1)
    for c in range(4):
        s_ = case == c
        a = m[s_]
        if c == 0:
            s = 2.0 * np.sqrt(np.maximum(1.0 + tr[s_], 1e-300))
            q[s_] = np.stack([(a[:, 2, 1] - a[:, 1, 2]) / s, (a[:, 0, 2] - a[:, 2, 0]) / s, (a[:, 1, 0] - a[:, 0, 1]) / s, 0.25 * s], 1)
        else:
            i, j, k = c - 1, c % 3, (c + 1) % 3
            s = 2.0 * np.sqrt(np.maximum(1.0 + a[:, i, i] - a[:, j, j] - a[:, k, k], 1e-300))
            v = np.empty((a.shape[0], 4))
            v[:, i] = 0.25 * s
            v[:, j] = (a[:, j, i] + a[:, i, j]) / s
            v[:, k] = (a[:, k, i] + a[:, i, k]) / s
            v[:, 3] = (a[:, k, j] - a[:, j, k]) / s
            q[s_] = v
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    q[q[:, 3] < 0] *= -1.0
    return q.reshape(R.shape[:-2] + (4,))


def matrix_from_quat(q) -> np.ndarray:
    """[...,4] quaternions (x, y, z, w) -> [...,3,3] rotation matrices (fp64; q is normalised first)."""
    q = np.asarray(q, np.float64)
    q = q / np.linalg.norm(q, axis=-1, keepdims=True)
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
                     np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
                     np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)], -2)


# ---- skeleton ---------------------------------------------------------------------------------------------------------------------
@dataclass
class RiggedMesh:
    """A canonical mesh with its skeleton.  Mesh on the device: verts [V,3], faces [F,3] int32, colors [V,3], joints [V,K] uint8,
    weights [V,K] (K = 4 or 8 influences, heaviest first).  Skeleton on the host (fp64): parents [J] (-1 for the root), names [J],
    translations [J,3] (node translations: rest-local, the root's Cano_0 J_0), rotations [J,4] (bind-local, x y z w), ibm [J,4,4]
    (inverse bind matrices) and rest_joints [J,3].  A textured rig (`extract_body_rig`) also carries uvs [T,2] (the template's
    convention, v up), uv_faces [F,3] (face f's corners in uvs), texture [S,S,3] uint8 on the device (row 0 first: row r is
    v = 1 - (r + 0.5) / S) and `fit`, the report of its geometry fit."""
    verts: torch.Tensor
    faces: torch.Tensor
    colors: torch.Tensor
    joints: torch.Tensor
    weights: torch.Tensor
    parents: tuple
    names: tuple
    translations: np.ndarray
    rotations: np.ndarray
    ibm: np.ndarray
    rest_joints: np.ndarray
    uvs: np.ndarray | None = None
    uv_faces: np.ndarray | None = None
    texture: torch.Tensor | None = None
    fit: dict | None = None


def skeleton(rest_joints, inv_cano, parents) -> dict:
    """The glTF skeleton of a subject: rest joints J [J,3], Cano^-1 [J,4,4] (`AvatarModel._inv_cano`) and the kinematic tree ->
    dict(translations, rotations, ibm, rest_joints), fp64."""
    Jr = np.asarray(torch.as_tensor(rest_joints).detach().cpu().double().numpy() if torch.is_tensor(rest_joints) else rest_joints, np.float64)
    inv = np.asarray(torch.as_tensor(inv_cano).detach().cpu().double().numpy() if torch.is_tensor(inv_cano) else inv_cano, np.float64)
    cano = np.linalg.inv(inv)
    nj = len(parents)
    T = np.tile(np.eye(4), (nj, 1, 1))
    T[:, :3, 3] = -Jr
    ibm = T @ inv
    Rg = cano[:, :3, :3]
    rot = np.empty((nj, 3, 3))
    trans = np.empty((nj, 3))
    for j, p in enumerate(parents):
        if p < 0:
            rot[j] = Rg[j]
            trans[j] = cano[j, :3, :3] @ Jr[j] + cano[j, :3, 3]
        else:
            rot[j] = Rg[p].T @ Rg[j]
            trans[j] = Jr[j] - Jr[p]
    return dict(translations=trans, rotations=quat_from_matrix(rot), ibm=ibm, rest_joints=Jr)


def node_globals(parents, translations, rotations) -> np.ndarray:
    """World matrices [J,4,4] (fp64) of the joint nodes from their local translations [J,3] and rotations [J,4] (parents first)."""
    R = matrix_from_quat(rotations)
    G = np.empty((len(parents), 4, 4))
    for j, p in enumerate(parents):
        L = np.eye(4)
        L[:3, :3], L[:3, 3] = R[j], translations[j]
        G[j] = L if p < 0 else G[p] @ L
    return G


# ---- motion -----------------------------------------------------------------------------------------------------------------------
@dataclass
class Motion:
    """A baked motion at `fps`: per frame the root node's translation [F,3] and every joint node's local rotation [F,J,4] (x y z w),
    with the up-axis rotation `up_rotation` [3,3] (clip world -> glTF, +Y up) folded into the root's two channels."""
    fps: float
    root_translation: np.ndarray
    rotations: np.ndarray
    up_rotation: np.ndarray

    @property
    def frames(self) -> int:
        return int(self.rotations.shape[0])

    @property
    def times(self) -> np.ndarray:
        return np.arange(self.frames, dtype=np.float64) / self.fps


def bake_poses(rest_joints, full_pose, transl, fps: float, up: str = "y") -> Motion:
    """Motion of full poses [F,J*3] (SMPL-X: pose 66 | rest_pose 99) and translations [F,3] in a world whose up axis is `up`: each
    joint's rotation is the shifted-norm Rodrigues matrix the library poses with, as a quaternion; the root's translation J_0 + t."""
    if up not in UP_ROTATIONS:
        raise ValueError(f"up {up!r}: one of {sorted(UP_ROTATIONS)}")
    if not (fps > 0 and math.isfinite(fps)):
        raise ValueError(f"fps {fps} must be positive")
    host = lambda a: np.asarray(a.detach().cpu().double().numpy() if torch.is_tensor(a) else a, np.float64)
    Jr, pose, t = host(rest_joints), host(full_pose), host(transl).reshape(-1, 3)
    F, nj = pose.shape[0], Jr.shape[0]
    if pose.shape[1] != 3 * nj or t.shape[0] != F:
        raise ValueError(f"pose {pose.shape} / transl {t.shape}: expected [F,{3 * nj}] / [F,3]")
    U = UP_ROTATIONS[up]
    R = rodrigues_np(pose.astype(np.float32).astype(np.float64).reshape(F * nj, 3)).reshape(F, nj, 3, 3)
    R[:, 0] = U[None] @ R[:, 0]
    q = quat_from_matrix(R)
    for f in range(1, F):                       # sign-continuous, so LINEAR sampling takes the short way
        flip = (q[f] * q[f - 1]).sum(-1) < 0
        q[f, flip] *= -1.0
    root = (Jr[0][None] + t) @ U.T
    return Motion(float(fps), root, q, U.copy())


def default_up(clip_path: str | None, align_to) -> str:
    """A clip world's up axis: the dataset camera frame's -y for a smpl_parms.pth or an aligned clip, else z (AMASS)."""
    return "-y" if align_to is not None or (clip_path is not None and not str(clip_path).endswith(".npz")) else "z"


def bake_motion(model, clip, fps: float, align_to=None, up=None, clip_path=None) -> Motion:
    """A `MotionClip` sampled at `fps` on the device (`animate.motion_sample`, clip frame 0 mapped onto training frame `align_to`),
    baked for the model's skeleton.  up: the clip world's up axis, 'y', 'z' or '-y' (default `default_up(clip_path, align_to)`)."""
    from .animate import Ensemble, motion_sample, sample_times
    Ensemble._check_clip(model, clip)
    dev = model.device
    times = sample_times(clip.num_keys, clip.fps, fps)
    align = Ensemble._alignment(model, clip, align_to)
    pose, trans = motion_sample(clip.pose.to(dev).contiguous(), clip.trans.to(dev).contiguous(), torch.from_numpy(times).to(dev),
                                torch.from_numpy(align).to(dev))
    return bake_poses(model._rest_joints, pose, trans, fps, up or default_up(clip_path, align_to))


def pose_rig(rig: RiggedMesh, motion: Motion | None = None, i: int = 0) -> np.ndarray:
    """The rig's vertices [V,3] (fp64, host) at frame i of `motion` (the bind pose without one), by plain LBS of the glTF data."""
    if motion is None:
        G = node_globals(rig.parents, rig.translations, rig.rotations)
    else:
        t = rig.translations.copy()
        t[0] = motion.root_translation[i]
        G = node_globals(rig.parents, t, motion.rotations[i])
    M = G @ rig.ibm
    v = rig.verts.detach().cpu().double().numpy()
    j = rig.joints.detach().cpu().long().numpy()
    w = rig.weights.detach().cpu().double().numpy()
    Mv = np.einsum("vk,vkab->vab", w, M[j])
    return np.einsum("vab,vb->va", Mv[:, :3, :3], v) + Mv[:, :3, 3]


# ---- extraction -------------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def canonical_gaussians(model, pose_mapper=None):
    """means, scales, colors [1,N,3] of the avatar in canonical space: the decoder output placed by `LbsAssemble` with identity
    cano2live rows, i.e. query_points + offsets.  Stage 1 uses the frame-invariant decoder; stage 2 evaluates it on the position maps
    of the canonical pose (`posmap.canonical_pose`, CANO_TRANSL).  Call under `kept_state`."""
    from .posmap import CANO_TRANSL, canonical_pose
    dev, body = model.device, model.body
    eye = torch.zeros(1, body.joints, 12, device=dev)
    eye[..., 0] = eye[..., 5] = eye[..., 10] = 1.0
    if int(model.model_parms.train_stage) == 2:
        mapper = pose_mapper if pose_mapper is not None else getattr(model, "pose_mapper", None)
        if mapper is None:
            raise ValueError("stage 2 needs a pose_mapper (posmap.PoseMapper / SmplxPoseMapper) for the input position maps")
        pose, rest = body.split(canonical_pose(body.name).to(dev))
        transl = torch.tensor([CANO_TRANSL], dtype=torch.float32, device=dev)
        feat = model.pose_encoder(mapper.maps(pose, rest, transl))
        dec = model.net.forward_packed_frames(model.geo_feature, feat, int(model.model_parms.query_posmap_size))
        return LbsAssemble.apply(dec, eye, model.valid_index, model._query_points, model._query_lbs, 1.0, True)
    return LbsAssemble.apply(model._stage1_decoder(1), eye, model.valid_index, model._query_points, model._query_lbs, 1.0, False)


@torch.no_grad()
def extract_rigged_mesh(model, res: int = 256, views: int = 64, size: int = 512, trunc_voxels: float = 4, min_carve: int = 1, k: int = 8,
                        influences: int = 4, pose_mapper=None) -> RiggedMesh:
    """The avatar's canonical mesh (`mesh_extract.mesh_gaussians` of `canonical_gaussians` with the same res / views / size /
    trunc_voxels / min_carve as `extract_mesh`), its skin weights from the k nearest canonical Gaussians (`influences` 4 or 8 joints
    per vertex) and the model's skeleton.  The model's state is left as it was."""
    if int(influences) not in (4, 8):
        raise ValueError(f"influences {influences}: 4 or 8")
    if not 1 <= int(k) <= MAX_NEIGHBOURS:
        raise ValueError(f"k {k} outside 1..{MAX_NEIGHBOURS}")
    with kept_state(model):
        means, scales, colors = canonical_gaussians(model, pose_mapper)
    verts, faces, cols = mesh_gaussians(model, means, scales, colors, res, views, size, trunc_voxels, min_carve)
    if verts.shape[0] == 0:
        raise RuntimeError("the canonical mesh is empty")
    body = model.body
    joints, weights = skin_weights(verts, means[0], model._query_lbs, body.joints, int(k), int(influences))
    names = SMPLX_JOINT_NAMES if body is SMPLX else SMPL_JOINT_NAMES
    return RiggedMesh(verts, faces, cols, joints, weights, tuple(body.parents), tuple(names),
                      **skeleton(model._rest_joints, model._inv_cano, body.parents))


# ---- the body model's own topology ---------------------------------------------------------------------------------------------------
# The fit's regulariser weight and its fixed number of preconditioned CG iterations (DESIGN.md §2 reports the residual they reach).
FIT_LAMBDA = 0.1
FIT_ITERATIONS = 200


def _midpoint_split(faces: np.ndarray, n: int):
    """One midpoint split of faces [F,3] over indices 0..n-1: (faces [4F,3], edges [E,2]).  The midpoint of edge k, numbered in
    ascending (min, max) order, is index n + k; face (a, b, c) becomes (a, ab, ca), (ab, b, bc), (ca, bc, c), (ab, bc, ca)."""
    F = faces.shape[0]
    e = np.sort(np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]), axis=1)
    edges, inv = np.unique(e, axis=0, return_inverse=True)
    ab, bc, ca = (n + inv.reshape(3, F)).astype(np.int64)
    a, b, c = faces.T
    out = np.stack([np.stack([a, ab, ca], 1), np.stack([ab, b, bc], 1), np.stack([ca, bc, c], 1), np.stack([ab, bc, ca], 1)], 1)
    return out.reshape(-1, 3), edges.astype(np.int64)


@dataclass
class BodyTopology:
    """A UV template subdivided `levels` times by midpoints (host): faces [F,3], uvs [T,2] (fp64), uv_faces [F,3], skin weights [V,J]
    (fp64, each new vertex the mean of its edge's ends), the edges whose midpoints were added, level by level, and the vertex
    adjacency CSR (offsets [V+1], adj) int32, neighbours ascending.  3D midpoints are keyed by vertex-index edges, so a UV seam stays
    welded in 3D; UV midpoints by UV-index edges."""
    faces: np.ndarray
    uvs: np.ndarray
    uv_faces: np.ndarray
    weights: np.ndarray
    splits: list
    offsets: np.ndarray
    adj: np.ndarray

    @property
    def V(self) -> int:
        return int(self.weights.shape[0])


def body_topology(uv_template, weights, levels: int = 1) -> BodyTopology:
    """`BodyTopology` of a UV template (a path or what `posmap.load_uv_template_obj` returns) whose vertices carry the body model's
    skin weights [V,J], subdivided levels in {0, 1, 2} times."""
    from .posmap import load_uv_template_obj
    if int(levels) not in (0, 1, 2):
        raise ValueError(f"subdivision levels {levels}: 0, 1 or 2")
    if isinstance(uv_template, (str, bytes)) or hasattr(uv_template, "__fspath__"):
        uv_template = load_uv_template_obj(uv_template)
    _, faces, uvs, uv_faces = uv_template
    w = np.asarray(weights.detach().cpu().double().numpy() if torch.is_tensor(weights) else weights, np.float64)
    faces, uv_faces, uvs = np.asarray(faces, np.int64), np.asarray(uv_faces, np.int64), np.asarray(uvs, np.float64)
    if faces.size and (faces.min() < 0 or faces.max() >= w.shape[0]):
        raise ValueError(f"the UV template indexes a vertex outside the body model's 0..{w.shape[0] - 1}")
    splits = []
    for _ in range(int(levels)):
        faces, e = _midpoint_split(faces, w.shape[0])
        uv_faces, et = _midpoint_split(uv_faces, uvs.shape[0])
        w = np.concatenate([w, 0.5 * (w[e[:, 0]] + w[e[:, 1]])])
        uvs = np.concatenate([uvs, 0.5 * (uvs[et[:, 0]] + uvs[et[:, 1]])])
        splits.append(e)
    V = w.shape[0]
    e = np.unique(np.sort(np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]), axis=1), axis=0)
    both = np.concatenate([e, e[:, ::-1]])
    both = both[np.lexsort((both[:, 1], both[:, 0]))]
    offsets = np.zeros(V + 1, np.int64)
    np.cumsum(np.bincount(both[:, 0], minlength=V), out=offsets[1:])
    return BodyTopology(faces, uvs, uv_faces, w, splits, offsets.astype(np.int32), both[:, 1].astype(np.int32))


def top_influences(weights, K: int):
    """(joints [V,K] uint8, weights [V,K] fp32): each row's K largest weights (equal ones to the lower joint), renormalised in fp64."""
    w = np.asarray(weights, np.float64)
    j = np.argsort(-w, axis=1, kind="stable")[:, :K]
    v = np.take_along_axis(w, j, 1)
    s = v.sum(1, keepdims=True)
    return j.astype(np.uint8), (v / np.where(s > 0, s, 1.0)).astype(np.float32)


def subdivide_points(x: torch.Tensor, topo: BodyTopology) -> torch.Tensor:
    """x [V0,3] on the original vertices -> [V,3] with every added vertex at its edge's midpoint, level by level."""
    for e in topo.splits:
        a, b = (torch.from_numpy(e[:, k]).to(x.device) for k in (0, 1))
        x = torch.cat([x, (x[a] + x[b]) * 0.5])
    return x.contiguous()


def mesh_laplacian(offsets: torch.Tensor, adj: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """ga_mesh_laplacian on the current stream: y [V,3] = deg_v x_v - sum of the neighbours' x (fp32, device)."""
    x = x.float().contiguous()
    y = torch.empty_like(x)
    _lib.check(_lib.lib().ga_mesh_laplacian(int(x.shape[0]), ptr(offsets), ptr(adj), ptr(x), ptr(y), _stream()), "ga_mesh_laplacian")
    return y


def texture_pushpull(image: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """ga_texture_pushpull on the current stream: image [C,S,S] fp32 with its covered texels mask [S,S] (nonzero) -> [C,S,S], every
    uncovered texel filled from the covered ones around it, the covered ones unchanged."""
    image = image.float().contiguous()
    C, S = int(image.shape[0]), int(image.shape[1])
    mask = mask.to(torch.uint8).contiguous()
    L = _lib.lib()
    n = L.ga_texture_pushpull_workspace_bytes(S, C)
    ws = torch.empty(max(n, 1), dtype=torch.uint8, device=image.device)
    out = torch.empty_like(image)
    _lib.check(L.ga_texture_pushpull(S, C, ptr(image), ptr(mask), ptr(ws), n, ptr(out), _stream()), "ga_texture_pushpull")
    return out


class UVLayout:
    """The position-map operator B of a mesh's UV layout at map size S (1..512), on the device: `fill` x [V,3] -> [3,S,S] (the
    texels' barycentric blends, `ga_posmap_fill`) and `fill_t` its transpose [3,S,S] -> [V,3] (`ga_posmap_fill_backward`)."""

    def __init__(self, faces, uvs, uv_faces, V: int, S: int, device):
        self.S, self.V, self.device = int(S), int(V), torch.device(device)
        dev = self.device
        self.faces = torch.from_numpy(np.asarray(faces, np.int32)).to(dev).contiguous()
        corners = torch.from_numpy(np.asarray(uvs, np.float32)[np.asarray(uv_faces)]).to(dev).contiguous()
        F, S = int(self.faces.shape[0]), self.S
        self.face_id = torch.empty(S, S, dtype=torch.int32, device=dev)
        self.bary = torch.empty(S, S, 3, dtype=torch.float32, device=dev)
        L = _lib.lib()
        _lib.check(L.ga_posmap_layout(F, S, ptr(corners), ptr(self.face_id), ptr(self.bary), _stream()), "ga_posmap_layout")
        self.offsets = torch.empty(self.V + 1, dtype=torch.int32, device=dev)
        self.entries = torch.empty(3 * S * S, dtype=torch.int32, device=dev)
        _lib.check(L.ga_posmap_vertex_csr(S, self.V, ptr(self.faces), ptr(self.face_id), ptr(self.offsets), ptr(self.entries), _stream()),
                   "ga_posmap_vertex_csr")

    def fill(self, x: torch.Tensor) -> torch.Tensor:
        out = torch.empty(1, 3, self.S, self.S, dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib().ga_posmap_fill(1, self.S, self.V, ptr(x.float().contiguous()), ptr(self.faces), ptr(self.face_id),
                                             ptr(self.bary), ptr(out), _stream()), "ga_posmap_fill")
        return out[0]

    def fill_t(self, m: torch.Tensor) -> torch.Tensor:
        out = torch.empty(1, self.V, 3, dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib().ga_posmap_fill_backward(1, self.S, self.V, ptr(self.offsets), ptr(self.entries), ptr(self.bary),
                                                      ptr(m.float().contiguous()), ptr(out), _stream()), "ga_posmap_fill_backward")
        return out[0]

    def diagonal(self, mask: torch.Tensor) -> torch.Tensor:
        """diag(B^T M B) [V] (fp32): sum over each vertex's texels t in the mask of bary[t, corner]^2, summed on the host in fp64."""
        off = self.offsets.cpu().numpy().astype(np.int64)
        e = self.entries.cpu().numpy()[:off[-1]].astype(np.int64)
        t, i = e // 3, e % 3
        val = mask.reshape(-1).double().cpu().numpy()[t] * self.bary.reshape(-1, 3).double().cpu().numpy()[t, i] ** 2
        d = np.bincount(np.repeat(np.arange(self.V), np.diff(off)), weights=val, minlength=self.V)
        return torch.from_numpy(d).float().to(self.device)


@torch.no_grad()
def fit_body_mesh(layout: UVLayout, topo: BodyTopology, x0: torch.Tensor, target: torch.Tensor, mask: torch.Tensor,
                  lam: float = FIT_LAMBDA, iterations: int = FIT_ITERATIONS):
    """x = x0 + d [V,3] minimising sum_{t in mask} |(B(x0 + d))_t - target_t|^2 + lam d^T L d (L the uniform graph Laplacian), by
    `iterations` steps of Jacobi-preconditioned conjugate gradients from the normalised scatter d0 = B^T M r / B^T M 1, r = target -
    B x0 (0 where the denominator is 0).  target [3,S,S], mask [S,S] (1 in M, else 0).  On the device with no host read-back in the
    loop, bit-reproducible.  Returns (x, relative residual |b - A d| / |b| of the normal equations, a 0-d device tensor)."""
    dev = x0.device
    mask = mask.float()
    offsets, adj = (torch.from_numpy(a).to(dev) for a in (topo.offsets, topo.adj))
    lam = float(lam)
    A = lambda p: layout.fill_t(layout.fill(p) * mask) + lam * mesh_laplacian(offsets, adj, p)
    b = layout.fill_t((target - layout.fill(x0)) * mask)
    den = layout.fill_t(mask.expand(3, -1, -1))
    d = torch.where(den > 0, b / torch.where(den > 0, den, 1.0), 0.0)
    diag = layout.diagonal(mask) + lam * torch.from_numpy(np.diff(topo.offsets).astype(np.float32)).to(dev)
    minv = torch.where(diag > 0, 1.0 / torch.where(diag > 0, diag, 1.0), 0.0)[:, None]
    dot = lambda u, v: (u.double() * v.double()).sum()
    r = b - A(d)
    z = minv * r
    p = z
    rz = dot(r, z)
    for _ in range(int(iterations)):
        Ap = A(p)
        pAp = dot(p, Ap)
        alpha = torch.where(pAp > 0, rz / torch.where(pAp > 0, pAp, 1.0), 0.0).float()
        d = d + alpha * p
        r = r - alpha * Ap
        z = minv * r
        rz_new = dot(r, z)
        beta = torch.where(rz > 0, rz_new / torch.where(rz > 0, rz, 1.0), 0.0).float()
        p = z + beta * p
        rz = rz_new
    bn = b.double().norm()
    rel = torch.where(bn > 0, (b - A(d)).double().norm() / torch.where(bn > 0, bn, 1.0), 0.0)
    return x0 + d, rel


@torch.no_grad()
def extract_body_rig(model, uv_template, subdiv: int = 1, influences: int = 4, pose_mapper=None, lam: float = FIT_LAMBDA,
                     iterations: int = FIT_ITERATIONS) -> RiggedMesh:
    """The avatar as a rig in its body model's own topology: the UV template (a path or what `posmap.load_uv_template_obj` returns)
    subdivided `subdiv` times, fitted through the canonical Gaussians on the template's UV layout at the model's query_posmap_size
    (`fit_body_mesh`), textured with the decoder's colour map (gaps filled by `texture_pushpull`, quantised as ga_frame_pack does),
    skinned with the body model's weights (the K = `influences` heaviest) and the model's skeleton.  pose_mapper: a
    `posmap.BodyPoser` (or PoseMapper) of the subject's body model, default the model's own; stage 2 also takes its input maps from
    it.  The rig's `fit` holds the fit's report: the RMS of B x - g over M, CG's final relative residual, |M|, lam, iterations.  The
    model's state is left as it was."""
    from .animate import frame_pack
    from .posmap import CANO_TRANSL, canonical_pose
    if int(influences) not in (4, 8):
        raise ValueError(f"influences {influences}: 4 or 8")
    poser = pose_mapper if pose_mapper is not None else getattr(model, "pose_mapper", None)
    if poser is None:
        raise ValueError("extract_body_rig needs the subject's body model: pass a posmap.BodyPoser / PoseMapper as pose_mapper")
    dev, body, S = model.device, model.body, int(model.model_parms.query_posmap_size)
    if poser.body is not body:
        raise ValueError(f"the pose_mapper poses {poser.body.label}, the model is {body.label}")
    topo = body_topology(uv_template, poser.weights, subdiv)
    pose, rest = body.split(canonical_pose(body.name).to(dev))
    x0 = subdivide_points(poser.posed(pose, rest, torch.tensor([CANO_TRANSL], dtype=torch.float32, device=dev))[0], topo)
    with kept_state(model):
        means, _, colors = canonical_gaussians(model, pose_mapper)
    layout = UVLayout(topo.faces, topo.uvs, topo.uv_faces, topo.V, S, dev)
    idx = model.valid_index.long()
    has = torch.zeros(S * S, dtype=torch.uint8, device=dev)
    has[idx] = 1
    target = torch.zeros(3, S * S, device=dev)
    target[:, idx] = means[0].t()
    cmap = torch.zeros(3, S * S, device=dev)
    cmap[:, idx] = colors[0].t()
    M = ((layout.face_id.reshape(-1) >= 0) & (has > 0)).float().reshape(S, S)
    target, cmap = target.reshape(3, S, S), cmap.reshape(3, S, S)
    x, rel = fit_body_mesh(layout, topo, x0, target, M, lam, iterations)
    fitted = layout.fill(x)
    rms = ((((fitted - target) ** 2).sum(0) * M).sum() / M.sum().clamp(min=1)).sqrt()
    texture = frame_pack(texture_pushpull(cmap, has.reshape(S, S))[None])[0]
    den = layout.fill_t(M.expand(3, -1, -1))
    vcol = torch.where(den > 0, layout.fill_t(cmap * M) / torch.where(den > 0, den, 1.0), 0.0)
    joints, weights = top_influences(topo.weights[:, :body.joints], int(influences))
    names = SMPLX_JOINT_NAMES if body is SMPLX else SMPL_JOINT_NAMES
    return RiggedMesh(x.contiguous(), torch.from_numpy(topo.faces.astype(np.int32)).to(dev), vcol, torch.from_numpy(joints).to(dev),
                      torch.from_numpy(weights).to(dev), tuple(body.parents), tuple(names),
                      **skeleton(model._rest_joints, model._inv_cano, body.parents), uvs=topo.uvs, uv_faces=topo.uv_faces, texture=texture,
                      fit=dict(residual_rms=float(rms), cg_relative_residual=float(rel), texels=int(M.sum()), lam=float(lam),
                               iterations=int(iterations)))


def seam_split(rig: RiggedMesh):
    """The textured rig's vertices split at UV seams into unique (vertex, uv) pairs: (vertex [V',] int64, the welded vertex of each,
    texcoord [V',2] fp32 in glTF's convention (u, 1 - v), faces [F,3] over the pairs)."""
    f = np.asarray(rig.faces.detach().cpu().numpy() if torch.is_tensor(rig.faces) else rig.faces, np.int64).reshape(-1)
    t = np.asarray(rig.uv_faces, np.int64).reshape(-1)
    pairs, inv = np.unique(np.stack([f, t], 1), axis=0, return_inverse=True)
    uv = np.asarray(rig.uvs, np.float64)[pairs[:, 1]]
    tex = np.stack([uv[:, 0], 1.0 - uv[:, 1]], 1).astype(np.float32)
    return pairs[:, 0], tex, inv.reshape(-1, 3).astype(np.int64)


@torch.no_grad()
def render_rig_unlit(rig: RiggedMesh, verts, cams, H: int, W: int, background=None):
    """The rig, posed at verts [B,V,3] (its own vertex order), drawn unlit from the camera rows cams [B,40]: with its texture when it
    has one, else its vertex colours (`MeshRenderer.render_unlit`).  Returns (rgb [B,3,H,W], face_id [B,H,W])."""
    from .mesh_render import MeshRenderer
    verts = torch.as_tensor(verts).float()
    dev = verts.device
    if rig.texture is None:
        mr = MeshRenderer(rig.faces, int(rig.verts.shape[0]), device=dev)
        rgb, fid, _ = mr.render_unlit(verts, cams, H, W, colors=rig.colors, background=background)
        return rgb, fid
    vid, tex, faces = seam_split(rig)
    mr = MeshRenderer(faces, len(vid), device=dev)
    texture = rig.texture.to(dev).float() / 255.0
    rgb, fid, _ = mr.render_unlit(verts[:, torch.from_numpy(vid).to(dev)], cams, H, W, uvs=torch.from_numpy(tex), texture=texture,
                                  background=background)
    return rgb, fid


@torch.no_grad()
def unlit_psnr(model, rig: RiggedMesh, verts, pose, transl, cams, H: int, W: int, rest_pose=None, pose_mapper=None) -> list:
    """Per camera row of cams [B,40]: the PSNR (dB, peak 1) of the rig posed at verts [V,3], drawn unlit on black, against the avatar's
    own render (bg 0) in the same pose, both H x W."""
    from .mesh_extract import posed_gaussians, render_views
    from .metrics import ssim_sse
    with kept_state(model):
        means, scales, colors = posed_gaussians(model, pose, transl, rest_pose, pose_mapper)
    cams = torch.as_tensor(cams).to(device=means.device, dtype=torch.float32)
    verts = torch.as_tensor(verts).to(device=means.device, dtype=torch.float32).reshape(1, -1, 3)
    out = []
    for s, e, img, _, _ in render_views(model, means, scales, colors, cams, H, W):
        rgb, _ = render_rig_unlit(rig, verts.expand(e - s, -1, -1), cams[s:e], H, W)
        _, sse = ssim_sse(rgb.contiguous(), img.contiguous().clamp(0.0, 1.0))
        mse = sse.cpu().numpy() / (3 * H * W)
        out += [float(10.0 * np.log10(1.0 / max(m, 1e-20))) for m in mse]
    return out


# ---- glTF 2.0 binary --------------------------------------------------------------------------------------------------------------
_FLOAT, _UBYTE, _UINT = 5126, 5121, 5125
_ARRAY_BUFFER, _ELEMENT_ARRAY_BUFFER = 34962, 34963
_LINEAR, _CLAMP_TO_EDGE = 9729, 33071
_UNLIT = "KHR_materials_unlit"


def encode_png(rgb: np.ndarray) -> bytes:
    """rgb [H,W,3] uint8 as a PNG: 8-bit RGB, filter 0 on every row, one zlib stream."""
    import zlib
    rgb = np.ascontiguousarray(rgb, np.uint8)
    H, W, _ = rgb.shape
    raw = np.concatenate([np.zeros((H, 1), np.uint8), rgb.reshape(H, 3 * W)], 1).tobytes()
    chunk = lambda tag, data: struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)
    return (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, 8, 2, 0, 0, 0)) + chunk(b"IDAT", zlib.compress(raw, 6))
            + chunk(b"IEND", b""))


class _Bin:
    """The BIN chunk under construction: one bufferView per accessor, each at an offset aligned to 4 bytes."""

    def __init__(self):
        self.data, self.views, self.accessors = bytearray(), [], []

    def add(self, arr, ctype, atype, target=None, minmax=False) -> int:
        arr = np.ascontiguousarray(arr)
        self.data += b"\0" * (-len(self.data) % 4)
        view = {"buffer": 0, "byteOffset": len(self.data), "byteLength": arr.nbytes}
        if target is not None:
            view["target"] = target
        self.views.append(view)
        self.data += arr.tobytes()
        acc = {"bufferView": len(self.views) - 1, "componentType": ctype, "count": int(arr.shape[0]), "type": atype}
        if minmax:
            flat = arr.reshape(arr.shape[0], -1)
            acc["min"], acc["max"] = [float(x) for x in flat.min(0)], [float(x) for x in flat.max(0)]
        self.accessors.append(acc)
        return len(self.accessors) - 1


def write_glb(path, rig: RiggedMesh, motion: Motion | None = None) -> None:
    """The rig (and the motion, as one animation with LINEAR samplers) as a glTF 2.0 binary: node 0 the skinned mesh, nodes 1..J the
    joints in the skeleton's order, one skin, column-major inverse bind matrices.  A rig with a texture is split at its UV seams
    (`seam_split`) and written with TEXCOORD_0, the texture as an embedded PNG, and one unlit material (KHR_materials_unlit); one
    without is written with per-vertex COLOR_0."""
    host = lambda t: t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)
    v = host(rig.verts).astype(np.float32).reshape(-1, 3)
    f = host(rig.faces).astype(np.uint32).reshape(-1)
    jo, w = host(rig.joints).astype(np.uint8), host(rig.weights).astype(np.float32)
    K = jo.shape[1]
    if K not in (4, 8):
        raise ValueError(f"{K} influences per vertex: 4 or 8")
    nj = len(rig.parents)
    b = _Bin()
    textured = rig.texture is not None
    if textured:
        vid, tex, faces = seam_split(rig)
        v, jo, w, f = v[vid], jo[vid], w[vid], faces.astype(np.uint32).reshape(-1)
        attrs = {"POSITION": b.add(v, _FLOAT, "VEC3", _ARRAY_BUFFER, minmax=True), "TEXCOORD_0": b.add(tex, _FLOAT, "VEC2", _ARRAY_BUFFER)}
    else:
        c = np.clip(host(rig.colors).astype(np.float32).reshape(-1, 3), 0.0, 1.0)
        attrs = {"POSITION": b.add(v, _FLOAT, "VEC3", _ARRAY_BUFFER, minmax=True), "COLOR_0": b.add(c, _FLOAT, "VEC3", _ARRAY_BUFFER)}
    for s in range(K // 4):
        attrs[f"JOINTS_{s}"] = b.add(jo[:, 4 * s:4 * s + 4], _UBYTE, "VEC4", _ARRAY_BUFFER)
        attrs[f"WEIGHTS_{s}"] = b.add(w[:, 4 * s:4 * s + 4], _FLOAT, "VEC4", _ARRAY_BUFFER)
    indices = b.add(f, _UINT, "SCALAR", _ELEMENT_ARRAY_BUFFER)
    ibm = b.add(np.transpose(rig.ibm, (0, 2, 1)).astype(np.float32).reshape(nj, 16), _FLOAT, "MAT4")   # column-major
    nodes = [{"name": "avatar", "mesh": 0, "skin": 0}]
    for j in range(nj):
        node = {"name": rig.names[j], "translation": [float(x) for x in rig.translations[j]],
                "rotation": [float(x) for x in rig.rotations[j]]}
        kids = [1 + i for i, p in enumerate(rig.parents) if p == j]
        if kids:
            node["children"] = kids
        nodes.append(node)
    prim = {"attributes": attrs, "indices": indices, "mode": 4}
    gltf = {"asset": {"version": "2.0", "generator": "gaussianavatar_b200.rig"}, "scene": 0, "scenes": [{"nodes": [0, 1]}], "nodes": nodes,
            "meshes": [{"name": "avatar", "primitives": [prim]}],
            "skins": [{"joints": list(range(1, nj + 1)), "inverseBindMatrices": ibm, "skeleton": 1}]}
    if textured:
        # the colours carry the capture's lighting already: an unlit material, so that a viewer does not light them again
        png = encode_png(host(rig.texture).astype(np.uint8))
        b.data += b"\0" * (-len(b.data) % 4)
        b.views.append({"buffer": 0, "byteOffset": len(b.data), "byteLength": len(png)})
        b.data += png
        prim["material"] = 0
        gltf.update(images=[{"bufferView": len(b.views) - 1, "mimeType": "image/png"}],
                    samplers=[{"magFilter": _LINEAR, "minFilter": _LINEAR, "wrapS": _CLAMP_TO_EDGE, "wrapT": _CLAMP_TO_EDGE}],
                    textures=[{"sampler": 0, "source": 0}],
                    materials=[{"name": "avatar", "pbrMetallicRoughness": {"baseColorTexture": {"index": 0}, "metallicFactor": 0.0},
                                "extensions": {_UNLIT: {}}}],
                    extensionsUsed=[_UNLIT])
    if motion is not None:
        if motion.rotations.shape[1] != nj:
            raise ValueError(f"the motion has {motion.rotations.shape[1]} joints, the rig {nj}")
        t_in = b.add(motion.times.astype(np.float32), _FLOAT, "SCALAR", minmax=True)
        samplers = [{"input": t_in, "output": b.add(motion.root_translation.astype(np.float32), _FLOAT, "VEC3"), "interpolation": "LINEAR"}]
        channels = [{"sampler": 0, "target": {"node": 1, "path": "translation"}}]
        for j in range(nj):
            samplers.append({"input": t_in, "output": b.add(motion.rotations[:, j].astype(np.float32), _FLOAT, "VEC4"), "interpolation": "LINEAR"})
            channels.append({"sampler": j + 1, "target": {"node": 1 + j, "path": "rotation"}})
        gltf["animations"] = [{"name": "motion", "samplers": samplers, "channels": channels}]
    b.data += b"\0" * (-len(b.data) % 4)
    gltf.update(accessors=b.accessors, bufferViews=b.views, buffers=[{"byteLength": len(b.data)}])
    js = json.dumps(gltf, separators=(",", ":")).encode()
    js += b" " * (-len(js) % 4)
    total = 12 + 8 + len(js) + 8 + len(b.data)
    with open(path, "wb") as fh:
        fh.write(struct.pack("<III", 0x46546C67, 2, total))
        fh.write(struct.pack("<II", len(js), 0x4E4F534A) + js)
        fh.write(struct.pack("<II", len(b.data), 0x004E4942) + bytes(b.data))
