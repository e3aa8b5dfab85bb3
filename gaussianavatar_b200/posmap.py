"""Position maps built on the device from SMPL / SMPL-X poses: the stage-2 input maps of every frame and a subject's canonical assets.

The reference makes `inp_map/inp_posemap_{S}_{idx:08d}.npz` offline (scripts/gen_pose_map_our_smpl.py): the smplx forward pass,
one OBJ per frame, then an OpenGL render of each mesh in UV space.  Because that render happens in UV space, which face covers which
texel (and with which barycentric weights) does not depend on the pose: `PoseMapper` computes that layout once on the device
(`ga_posmap_layout`), and a frame costs the posed vertices (`ga_smpl_vertices`) and a gather (`ga_posmap_fill`).  The coverage
rules are the library's own statement of what the GL rasterizer does (csrc/posmap.cu; DESIGN.md, PARITY UNPINNED).
`SmplxPoseMapper` does the same for SMPL-X (`ga_smplx_vertices`).  Both are differentiable with respect to pose and transl
(test-time pose fitting, `posefit.py`).  Their vertex-posing half, which needs no UV template, is `BodyPoser` / `SmplxBodyPoser`;
the mesh overlay (`mesh_render`) uses it too.

`canonical_assets` builds, from the same pieces, the per-subject and per-size files the reference makes with OpenGL
(scripts/gen_pose_map_cano_smpl.py) or ships pre-rendered: the canonical query map and joint matrices, the UV face-id mask, the
texel skinning-weight map (`ga_posmap_weights`) and the barycentric map.
"""
from __future__ import annotations

import math
import os
from typing import NamedTuple

import numpy as np
import torch

from . import _lib
from ._lib import ptr

SMPL_MESH_FIELDS = ("v_template", "shapedirs", "posedirs", "weights", "f", "J_regressor")
MAX_FRAMES_PER_CALL = 8          # ga_smpl_vertices / ga_smplx_vertices and their backward


def load_uv_template_obj(path):
    """Parse a UV template OBJ: `v x y z`, `vt u v`, and `f` entries `v/vt` or `v/vt/vn` (triangles or quads).  A quad (a, b, c, d)
    becomes the triangles (a, b, c) and (c, d, a), in that order, because the face order is the primitive id of the map.

    Returns (verts [Nv,3] float64, faces [F,3] int64, uvs [Nt,2] float64, faces_uv [F,3] int64), indices 0-based."""
    verts, uvs, faces, faces_uv = [], [], [], []
    with open(path, "r") as fh:
        for ln, line in enumerate(fh, 1):
            tok = line.split()
            if not tok or tok[0].startswith("#"):
                continue
            if tok[0] == "v":
                verts.append([float(x) for x in tok[1:4]])
            elif tok[0] == "vt":
                uvs.append([float(x) for x in tok[1:3]])
            elif tok[0] == "f":
                corners = tok[1:]
                if len(corners) not in (3, 4):
                    raise ValueError(f"{path}:{ln}: a face has {len(corners)} corners; only triangles and quads are supported")
                vi, ti = [], []
                for c in corners:
                    parts = c.split("/")
                    if len(parts) < 2 or not parts[1]:
                        raise ValueError(f"{path}:{ln}: face corner {c!r} has no texture coordinate (v/vt or v/vt/vn expected)")
                    vi.append(int(parts[0]) - 1)
                    ti.append(int(parts[1]) - 1)
                order = [(0, 1, 2)] if len(corners) == 3 else [(0, 1, 2), (2, 3, 0)]
                for tri in order:
                    faces.append([vi[k] for k in tri])
                    faces_uv.append([ti[k] for k in tri])
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    faces_uv = np.asarray(faces_uv, np.int64).reshape(-1, 3)
    uvs = np.asarray(uvs, np.float64).reshape(-1, 2)
    if faces_uv.size and (faces_uv.min() < 0 or faces_uv.max() >= len(uvs)):
        raise ValueError(f"{path}: a face indexes a texture coordinate outside 1..{len(uvs)}")
    return np.asarray(verts, np.float64).reshape(-1, 3), faces, uvs, faces_uv


def _dense(x):
    return np.asarray(x.todense() if hasattr(x, "todense") else x)


class BodyPoser:
    """Posed SMPL vertices [B,V,3] on the device, from the body model alone (no UV template): the vertex-posing half of `PoseMapper`,
    which the position maps and the mesh overlay (`mesh_render`) share.

    smpl: the SMPL model as stored in SMPL_{GENDER}.pkl (any mapping with v_template [V,3], shapedirs [V,3,>=10], posedirs
    [V,3,207], weights [V,24], f [F,3], J_regressor [24,V] dense or sparse); betas [10].  Everything runs on the current CUDA
    stream under no_grad."""

    BODY, JOINTS, POSE_FEATURES, POSE_WIDTH = "SMPL", 24, 207, 72
    # the C entry points of vertex posing, its backward and the backward's workspace size
    _VERTICES, _VERTICES_BWD, _VERTICES_BWD_WS = ("ga_smpl_vertices", "ga_smpl_vertices_backward",
                                                  "ga_smpl_vertices_backward_workspace_bytes")

    def __init__(self, smpl, betas, device="cuda"):
        missing = [k for k in SMPL_MESH_FIELDS if k not in smpl]
        if missing:
            raise ValueError(f"the {self.BODY} model has no {', '.join(missing)}: device position maps need the full mesh model")
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError(f"{type(self).__name__} runs on CUDA only (no CPU fallback)")
        self._check_model(smpl)
        v_t = np.asarray(smpl["v_template"], np.float64)
        V = v_t.shape[0]
        nj, nf, body = self.JOINTS, self.POSE_FEATURES, self.BODY
        beta = np.asarray(torch.as_tensor(betas).double().reshape(-1))
        sd = np.asarray(smpl["shapedirs"])[:, :, :beta.size].astype(np.float64)
        posedirs = np.asarray(smpl["posedirs"], np.float32)
        weights = np.asarray(smpl["weights"], np.float32)
        faces = np.asarray(smpl["f"]).astype(np.int64)
        Jr = _dense(smpl["J_regressor"]).astype(np.float64)
        if posedirs.shape != (V, 3, nf) or weights.shape != (V, nj) or Jr.shape != (nj, V) or faces.ndim != 2 or faces.shape[1] != 3:
            raise ValueError(f"{body} model: posedirs {posedirs.shape}, weights {weights.shape}, J_regressor {Jr.shape}, f {faces.shape}; "
                             f"expected [{V},3,{nf}], [{V},{nj}], [{nj},{V}], [F,3]")
        if faces.size and (faces.min() < 0 or faces.max() >= V):
            raise ValueError(f"{body} model: a face indexes a vertex outside 0..{V - 1}")
        v_shaped = v_t + np.einsum("l,mkl->mk", beta, sd)
        dev = self.device
        self.V, self.F = V, faces.shape[0]
        self.rest_joints = torch.from_numpy(Jr @ v_shaped).float().to(dev).contiguous()                 # [J,3]
        self.v_shaped = torch.from_numpy(v_shaped).float().to(dev).contiguous()                         # [V,3]
        self.posedirs = torch.from_numpy(posedirs.reshape(V * 3, nf).T.copy()).to(dev)                  # [207 / 486, 3V] as smplx keeps it
        self.weights = torch.from_numpy(weights).to(dev).contiguous()                                   # [V,J]
        self.faces = torch.from_numpy(faces.astype(np.int32)).to(dev).contiguous()                      # [F,3]

    def _check_model(self, model):
        pass

    @staticmethod
    def _stream() -> int:
        return torch.cuda.current_stream().cuda_stream

    def _inputs(self, pose, transl):
        pose = torch.as_tensor(pose).to(device=self.device, dtype=torch.float32).reshape(-1, self.POSE_WIDTH).contiguous()
        transl = torch.as_tensor(transl).to(device=self.device, dtype=torch.float32).reshape(-1, 3).contiguous()
        if pose.shape[0] != transl.shape[0]:
            raise ValueError(f"pose {tuple(pose.shape)} and transl {tuple(transl.shape)} have different frame counts")
        return pose, transl

    @staticmethod
    def _poses(pose, rest_pose):
        """The pose arguments the entry points take: pose (SMPL has no rest_pose)."""
        return (pose,)

    def _vertices(self, poses, transl) -> torch.Tensor:
        """Posed vertices [B,V,3] of checked poses, (pose,) or (pose, rest_pose), and transl: MAX_FRAMES_PER_CALL frames per call."""
        B = transl.shape[0]
        out = torch.empty(B, self.V, 3, dtype=torch.float32, device=self.device)
        fn = getattr(_lib.lib(), self._VERTICES)
        for s in range(0, B, MAX_FRAMES_PER_CALL):
            e = min(B, s + MAX_FRAMES_PER_CALL)
            _lib.check(fn(e - s, self.V, *(ptr(p[s:e]) for p in poses), ptr(transl[s:e]), ptr(self.rest_joints), ptr(self.v_shaped),
                          ptr(self.posedirs), ptr(self.weights), ptr(out[s:e]), self._stream()), self._VERTICES)
        return out

    @torch.no_grad()
    def vertices(self, pose, transl) -> torch.Tensor:
        """Posed SMPL vertices [B,V,3] for pose [B,72] and transl [B,3] (the reference's `SMPL.forward(...).vertices`)."""
        pose, transl = self._inputs(pose, transl)
        return self._vertices((pose,), transl)


class SmplxBodyPoser(BodyPoser):
    """The SMPL-X counterpart of `BodyPoser`: the model as stored in SMPLX_{GENDER}.npz (v_template, shapedirs [V,3,>=10] of which
    the first len(betas) columns are used, posedirs [V,3,486], weights [V,55], f, J_regressor [55,V], kintree_table, which must be
    the 55-joint tree of `synthetic.SMPLX_PARENTS`).  Poses are the reference's smplx.SMPLX(use_pca=False, flat_hand_mean=True)
    split: pose [B,66] (global + 21 body joints) and rest_pose [B,99] (jaw, left / right eye, 15 + 15 finger joints)."""

    BODY, JOINTS, POSE_FEATURES, POSE_WIDTH = "SMPL-X", 55, 486, 66
    _VERTICES, _VERTICES_BWD, _VERTICES_BWD_WS = ("ga_smplx_vertices", "ga_smplx_vertices_backward",
                                                  "ga_smplx_vertices_backward_workspace_bytes")

    def _check_model(self, smplx):
        from .synthetic import SMPLX_PARENTS
        if "kintree_table" not in smplx:
            raise ValueError("the SMPL-X model has no kintree_table")
        kt = np.asarray(smplx["kintree_table"]).astype(np.int64)[0].copy()
        kt[0] = -1
        if kt.shape != (len(SMPLX_PARENTS),) or not np.array_equal(kt, np.asarray(SMPLX_PARENTS)):
            raise ValueError("SMPL-X model: kintree_table[0] is not the 55-joint SMPL-X tree this library is built for")

    @staticmethod
    def _poses(pose, rest_pose):
        return (pose, rest_pose)

    def _inputs(self, pose, rest_pose, transl):
        pose, transl = super()._inputs(pose, transl)
        rest_pose = torch.as_tensor(rest_pose).to(device=self.device, dtype=torch.float32).reshape(-1, 99).contiguous()
        if rest_pose.shape[0] != pose.shape[0]:
            raise ValueError(f"pose {tuple(pose.shape)} and rest_pose {tuple(rest_pose.shape)} have different frame counts")
        return pose, rest_pose, transl

    @torch.no_grad()
    def vertices(self, pose, rest_pose, transl) -> torch.Tensor:
        """Posed SMPL-X vertices [B,V,3] for pose [B,66], rest_pose [B,99] and transl [B,3] (`SMPLX.forward(...).vertices`)."""
        pose, rest_pose, transl = self._inputs(pose, rest_pose, transl)
        return self._vertices((pose, rest_pose), transl)


class PoseMapper(BodyPoser):
    """Posed-body position maps [B,3,S,S] from SMPL poses, channel-first as the pose encoder takes them.

    smpl, betas: as `BodyPoser` takes them; uv_template: a path to the UV template OBJ or what `load_uv_template_obj` returns; S: map
    size (1..512).  Face i of the map is the mesh face f[i] drawn at the UV corners of template face i, so the template must have
    exactly F faces.  Everything runs on the current CUDA stream; calling the mapper with grad on and a pose or transl that requires
    grad makes the maps differentiable with respect to both (`ga_posmap_fill_backward`, then the vertex-posing backward)."""

    def __init__(self, smpl, betas, uv_template, S: int, device="cuda"):
        BodyPoser.__init__(self, smpl, betas, device)
        self.S = int(S)
        if not 1 <= self.S <= 512:
            raise ValueError(f"map size {S} outside 1..512")
        if isinstance(uv_template, (str, os.PathLike)):
            uv_template = load_uv_template_obj(uv_template)
        _, _, uvs, faces_uv = uv_template
        if faces_uv.shape[0] != self.F:
            raise ValueError(f"the UV template has {faces_uv.shape[0]} faces, the {self.BODY} mesh {self.F}: face i of one must be face i of "
                             "the other")
        dev = self.device
        corners = torch.from_numpy(np.asarray(uvs, np.float32)[faces_uv]).to(dev).contiguous()        # [F,3,2]
        self.face_id = torch.empty(self.S, self.S, dtype=torch.int32, device=dev)
        self.bary = torch.empty(self.S, self.S, 3, dtype=torch.float32, device=dev)
        _lib.check(_lib.lib().ga_posmap_layout(self.F, self.S, ptr(corners), ptr(self.face_id), ptr(self.bary), self._stream()),
                   "ga_posmap_layout")

    @torch.no_grad()
    def fill(self, verts: torch.Tensor) -> torch.Tensor:
        """Position maps [B,3,S,S] of posed vertices [B,V,3]; 0 where no face covers a texel."""
        verts = verts.to(device=self.device, dtype=torch.float32).contiguous()
        if verts.dim() != 3 or tuple(verts.shape[1:]) != (self.V, 3):
            raise ValueError(f"vertices {tuple(verts.shape)}: expected [B,{self.V},3]")
        B = verts.shape[0]
        out = torch.empty(B, 3, self.S, self.S, dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib().ga_posmap_fill(B, self.S, self.V, ptr(verts), ptr(self.faces), ptr(self.face_id), ptr(self.bary), ptr(out),
                                             self._stream()), "ga_posmap_fill")
        return out

    def __call__(self, pose, transl) -> torch.Tensor:
        """pose [B,72], transl [B,3] -> position maps [B,3,S,S], differentiable with respect to pose and transl when grad is on."""
        if _wants_grad(pose, transl):
            return _PoseMap.apply(self, pose, None, transl)
        return self.fill(self.vertices(pose, transl))

    def vertex_csr(self):
        """(offsets [V+1], entries [3 S^2]) int32: each vertex's (texel, corner) pairs, entry 3 t + i, ascending per vertex
        (`ga_posmap_vertex_csr`); what the fill's backward runs over.  Built on first use, once per mapper."""
        if getattr(self, "_csr", None) is None:
            offsets = torch.empty(self.V + 1, dtype=torch.int32, device=self.device)
            entries = torch.empty(3 * self.S * self.S, dtype=torch.int32, device=self.device)
            _lib.check(_lib.lib().ga_posmap_vertex_csr(self.S, self.V, ptr(self.faces), ptr(self.face_id), ptr(offsets), ptr(entries),
                                                       self._stream()), "ga_posmap_vertex_csr")
            self._csr = (offsets, entries)
        return self._csr

    def fill_backward(self, d_maps: torch.Tensor) -> torch.Tensor:
        """d_verts [B,V,3] of position-map gradients d_maps [B,3,S,S] (`ga_posmap_fill_backward`)."""
        d_maps = d_maps.to(device=self.device, dtype=torch.float32).contiguous()
        B = d_maps.shape[0]
        offsets, entries = self.vertex_csr()
        out = torch.empty(B, self.V, 3, dtype=torch.float32, device=self.device)
        for s in range(0, B, MAX_FRAMES_PER_CALL):
            e = min(B, s + MAX_FRAMES_PER_CALL)
            _lib.check(_lib.lib().ga_posmap_fill_backward(e - s, self.S, self.V, ptr(offsets), ptr(entries), ptr(self.bary), ptr(d_maps[s:e]),
                                                          ptr(out[s:e]), self._stream()), "ga_posmap_fill_backward")
        return out

    @torch.no_grad()
    def weight_map(self) -> torch.Tensor:
        """Texel skinning weights [S,S,J] = sum_i bary_i weights[f_i] (the reference's gen_lbs_weight_from_ori), 0 where no face covers
        a texel."""
        out = torch.empty(self.S, self.S, self.JOINTS, dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib().ga_posmap_weights(self.S, self.JOINTS, ptr(self.weights), ptr(self.faces), ptr(self.face_id), ptr(self.bary),
                                                ptr(out), self._stream()), "ga_posmap_weights")
        return out


class SmplxPoseMapper(SmplxBodyPoser, PoseMapper):
    """The SMPL-X counterpart of `PoseMapper`: the model and poses as `SmplxBodyPoser` takes them."""

    def __init__(self, smplx, betas, uv_template, S: int, device="cuda"):
        PoseMapper.__init__(self, smplx, betas, uv_template, S, device)

    def __call__(self, pose, rest_pose, transl) -> torch.Tensor:
        """pose [B,66], rest_pose [B,99], transl [B,3] -> position maps [B,3,S,S], differentiable with respect to pose and transl
        (not rest_pose) when grad is on."""
        if _wants_grad(pose, transl):
            return _PoseMap.apply(self, pose, rest_pose, transl)
        return self.fill(self.vertices(pose, rest_pose, transl))


def _wants_grad(*ts) -> bool:
    return torch.is_grad_enabled() and any(torch.is_tensor(t) and t.requires_grad for t in ts)


def vertices_backward(poser, pose, rest_pose, d_verts):
    """(d_pose [B,72|66], d_transl [B,3]) of vertex gradients d_verts [B,V,3] at pose (and SMPL-X rest_pose), through
    `ga_smpl_vertices_backward` / `ga_smplx_vertices_backward`."""
    d_verts = d_verts.to(device=poser.device, dtype=torch.float32).contiguous()
    B = pose.shape[0]
    d_pose = torch.empty(B, poser.POSE_WIDTH, dtype=torch.float32, device=poser.device)
    d_transl = torch.empty(B, 3, dtype=torch.float32, device=poser.device)
    L = _lib.lib()
    ws = torch.empty(getattr(L, poser._VERTICES_BWD_WS)(min(B, MAX_FRAMES_PER_CALL), poser.V), dtype=torch.uint8, device=poser.device)
    fn, poses = getattr(L, poser._VERTICES_BWD), poser._poses(pose, rest_pose)
    for s in range(0, B, MAX_FRAMES_PER_CALL):
        e = min(B, s + MAX_FRAMES_PER_CALL)
        _lib.check(fn(e - s, poser.V, *(ptr(p[s:e]) for p in poses), ptr(poser.rest_joints), ptr(poser.v_shaped), ptr(poser.posedirs),
                      ptr(poser.weights), ptr(d_verts[s:e]), ptr(ws), ws.numel(), ptr(d_pose[s:e]), ptr(d_transl[s:e]), poser._stream()),
                   poser._VERTICES_BWD)
    return d_pose, d_transl


class _PoseMap(torch.autograd.Function):
    """(pose, [rest_pose,] transl) -> position maps [B,3,S,S] of a `PoseMapper` / `SmplxPoseMapper`: the forward kernels as the mapper
    launches them, and backward through `ga_posmap_fill_backward` then the vertex-posing backward.  rest_pose is data."""

    @staticmethod
    def forward(ctx, mapper, pose, rest_pose, transl):
        if rest_pose is None:
            pose, transl = mapper._inputs(pose, transl)
            verts = mapper.vertices(pose, transl)
        else:
            pose, rest_pose, transl = mapper._inputs(pose, rest_pose, transl)
            verts = mapper.vertices(pose, rest_pose, transl)
        ctx.mapper = mapper
        ctx.save_for_backward(pose, rest_pose)
        return mapper.fill(verts)

    @staticmethod
    def backward(ctx, d_maps):
        pose, rest_pose = ctx.saved_tensors
        mapper = ctx.mapper
        d_pose, d_transl = vertices_backward(mapper, pose, rest_pose, mapper.fill_backward(d_maps))
        return None, d_pose, None, d_transl


def load_body_model(path):
    """The fields of a body-model file as a dict: SMPL_{GENDER}.pkl (a pickle) or SMPLX_{GENDER}.npz."""
    if not os.path.exists(path):
        raise FileNotFoundError(f"body model {path} not found")
    if str(path).endswith(".npz"):
        with np.load(path, allow_pickle=True) as z:
            return {k: z[k] for k in z.files}
    import pickle
    with open(path, "rb") as fh:
        return dict(pickle.load(fh, encoding="latin1"))


# The reference's canonical pose (arguments/__init__.py:44-53, smpl_cpose_param / smplx_cpose_param: legs at +-30 degrees, every other
# joint zero, so SMPL-X hands are flat) and translation (scripts/gen_pose_map_cano_smpl.py:60-70).
CANO_LEG_ANGLE = 30.0 / 180.0 * math.pi
CANO_TRANSL = (0.0, 0.30, 0.0)


def canonical_pose(body: str) -> torch.Tensor:
    """The canonical pose [1,72] (SMPL) or [1,165] (SMPL-X: pose 66 | rest_pose 99)."""
    p = torch.zeros(1, 72 if body == "smpl" else 165)
    p[0, 5] = CANO_LEG_ANGLE
    p[0, 8] = -CANO_LEG_ANGLE
    return p


class CanonicalAssets(NamedTuple):
    posmap: torch.Tensor        # [S,S,3] canonical query map (query_posemap_{S}_cano_{body}.npz), 0 where no face covers a texel
    joint_mats: torch.Tensor    # [J,4,4] canonical joint transforms A ({body}_cano_joint_mat.pth), transl included
    face_id: torch.Tensor       # [S,S] int32, -1 for background (uv_mask{S}_with_faceid_{body}.npy)
    lbs_map: torch.Tensor       # [S,S,J] texel skinning weights (lbs_map_{body}_{S}.npy)
    bary: torch.Tensor          # [S,S,3] barycentric weights of each texel in its face (bary_coords_{body}_uv{S}.npy)


@torch.no_grad()
def canonical_assets(model, betas, uv_template, S: int, body: str = "smpl", device="cuda") -> CanonicalAssets:
    """A subject's canonical assets, built on the device: what the reference's scripts/gen_pose_map_cano_smpl.py renders with OpenGL
    plus the UV mask, skinning-weight map and barycentric map it ships per map size.  model: the body-model fields (a dict, or a path
    to SMPL_{GENDER}.pkl / SMPLX_{GENDER}.npz); betas [10]; uv_template: a path or what `load_uv_template_obj` returns; body: "smpl"
    or "smplx".  The mesh is posed at `canonical_pose(body)` with transl CANO_TRANSL; the joint matrices are the same pose's A."""
    if body not in ("smpl", "smplx"):
        raise ValueError(f"body {body!r} is neither 'smpl' nor 'smplx'")
    if isinstance(model, (str, os.PathLike)):
        model = load_body_model(model)
    smplx = body == "smplx"
    mapper = (SmplxPoseMapper if smplx else PoseMapper)(model, betas, uv_template, S, device=device)
    dev = mapper.device
    pose = canonical_pose(body).to(dev)
    transl = torch.tensor([CANO_TRANSL], dtype=torch.float32, device=dev)
    if smplx:
        verts = mapper.vertices(pose[:, :66], pose[:, 66:], transl)
    else:
        verts = mapper.vertices(pose, transl)
    posmap = mapper.fill(verts)[0].permute(1, 2, 0).contiguous()
    J = mapper.JOINTS
    eye = torch.eye(4, device=dev).expand(J, 4, 4).contiguous()         # inv_cano = I: cano2live is A itself
    C = torch.empty(1, J, 12, device=dev)
    G = torch.empty(1, J, 12, device=dev)
    L = _lib.lib()
    if smplx:
        p66, r99 = pose[:, :66].contiguous(), pose[:, 66:].contiguous()
        _lib.check(L.ga_smplx_forward(1, ptr(p66), ptr(r99), ptr(transl), ptr(mapper.rest_joints), ptr(eye), ptr(C), ptr(G),
                                      mapper._stream()), "ga_smplx_forward")
    else:
        _lib.check(L.ga_smpl_forward(1, ptr(pose), ptr(transl), ptr(mapper.rest_joints), ptr(eye), ptr(C), ptr(G), mapper._stream()),
                   "ga_smpl_forward")
    A = torch.cat([C.reshape(J, 3, 4), eye[:, 3:4]], 1)
    return CanonicalAssets(posmap, A, mapper.face_id.clone(), mapper.weight_map(), mapper.bary.clone())
