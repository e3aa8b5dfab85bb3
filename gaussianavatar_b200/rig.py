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
    (inverse bind matrices) and rest_joints [J,3]."""
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


# ---- glTF 2.0 binary --------------------------------------------------------------------------------------------------------------
_FLOAT, _UBYTE, _UINT = 5126, 5121, 5125
_ARRAY_BUFFER, _ELEMENT_ARRAY_BUFFER = 34962, 34963


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
    joints in the skeleton's order, one skin, column-major inverse bind matrices."""
    host = lambda t: t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)
    v = host(rig.verts).astype(np.float32).reshape(-1, 3)
    f = host(rig.faces).astype(np.uint32).reshape(-1)
    c = np.clip(host(rig.colors).astype(np.float32).reshape(-1, 3), 0.0, 1.0)
    jo, w = host(rig.joints).astype(np.uint8), host(rig.weights).astype(np.float32)
    K = jo.shape[1]
    if K not in (4, 8):
        raise ValueError(f"{K} influences per vertex: 4 or 8")
    nj = len(rig.parents)
    b = _Bin()
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
    gltf = {"asset": {"version": "2.0", "generator": "gaussianavatar_b200.rig"}, "scene": 0, "scenes": [{"nodes": [0, 1]}], "nodes": nodes,
            "meshes": [{"name": "avatar", "primitives": [{"attributes": attrs, "indices": indices, "mode": 4}]}],
            "skins": [{"joints": list(range(1, nj + 1)), "inverseBindMatrices": ibm, "skeleton": 1}]}
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
