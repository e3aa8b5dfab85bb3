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
from .body import SMPL, SMPLX, Body, body_of, shaped_vertices
from .body import load_model as load_body_model
from .ops import Cano2Live
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


class BodyPoser:
    """Posed vertices [B,V,3] on the device, from the body model alone (no UV template): the vertex-posing half of `PoseMapper`,
    which the position maps and the mesh overlay (`mesh_render`) share.

    smpl: the body model as stored in SMPL_{GENDER}.pkl or SMPLX_{GENDER}.npz (any mapping with v_template [V,3], shapedirs
    [V,3,>=len(betas)], posedirs [V,3,207|486], weights [V,J], f [F,3], J_regressor [J,V] dense or sparse, kintree_table);
    betas [10]; body: `body.SMPL` or `body.SMPLX`.  Everything runs on the current CUDA stream under no_grad."""

    def __init__(self, smpl, betas, device="cuda", body: Body = SMPL):
        self.body = body
        body.check_model(smpl)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError(f"{type(self).__name__} runs on CUDA only (no CPU fallback)")
        v_shaped = shaped_vertices(smpl, betas)
        V = v_shaped.shape[0]
        nj, nf = body.joints, body.pose_features
        posedirs = np.asarray(smpl["posedirs"], np.float32)
        weights = np.asarray(smpl["weights"], np.float32)
        faces = np.asarray(smpl["f"]).astype(np.int64)
        Jr = smpl["J_regressor"]
        Jr_shape = tuple(Jr.shape)
        if posedirs.shape != (V, 3, nf) or weights.shape != (V, nj) or Jr_shape != (nj, V) or faces.ndim != 2 or faces.shape[1] != 3:
            raise ValueError(f"{body.label} model: posedirs {posedirs.shape}, weights {weights.shape}, J_regressor {Jr_shape}, "
                             f"f {faces.shape}; expected [{V},3,{nf}], [{V},{nj}], [{nj},{V}], [F,3]")
        if faces.size and (faces.min() < 0 or faces.max() >= V):
            raise ValueError(f"{body.label} model: a face indexes a vertex outside 0..{V - 1}")
        dev = self.device
        self.V, self.F = V, faces.shape[0]
        self.rest_joints = body.rest_joints(smpl, betas).to(dev).contiguous()                           # [J,3]
        self.v_shaped = v_shaped.float().to(dev).contiguous()                                           # [V,3]
        self.posedirs = torch.from_numpy(posedirs.reshape(V * 3, nf).T.copy()).to(dev)                  # [207 / 486, 3V] as smplx keeps it
        self.weights = torch.from_numpy(weights).to(dev).contiguous()                                   # [V,J]
        self.faces = torch.from_numpy(faces.astype(np.int32)).to(dev).contiguous()                      # [F,3]

    @property
    def JOINTS(self) -> int:
        return self.body.joints

    @staticmethod
    def _stream() -> int:
        return torch.cuda.current_stream().cuda_stream

    def _rows(self, t, width):
        return torch.as_tensor(t).to(device=self.device, dtype=torch.float32).reshape(-1, width).contiguous()

    def _inputs(self, pose, rest_pose, transl):
        """pose, rest_pose (None for SMPL) and transl as contiguous fp32 rows on the device, with one frame count."""
        b = self.body
        pose, transl = self._rows(pose, b.pose_width), self._rows(transl, 3)
        rest_pose = self._rows(rest_pose, b.rest_width) if b.rest_width else None
        for name, t in (("transl", transl), ("rest_pose", rest_pose)):
            if t is not None and t.shape[0] != pose.shape[0]:
                raise ValueError(f"pose {tuple(pose.shape)} and {name} {tuple(t.shape)} have different frame counts")
        return pose, rest_pose, transl

    def _vertices(self, pose, rest_pose, transl) -> torch.Tensor:
        """Posed vertices [B,V,3] of checked inputs: MAX_FRAMES_PER_CALL frames per call."""
        B = transl.shape[0]
        out = torch.empty(B, self.V, 3, dtype=torch.float32, device=self.device)
        name = self.body.vertices
        fn = getattr(_lib.lib(), name)
        poses = self.body.pose_args(pose, rest_pose)
        for s in range(0, B, MAX_FRAMES_PER_CALL):
            e = min(B, s + MAX_FRAMES_PER_CALL)
            _lib.check(fn(e - s, self.V, *(ptr(p[s:e]) for p in poses), ptr(transl[s:e]), ptr(self.rest_joints), ptr(self.v_shaped),
                          ptr(self.posedirs), ptr(self.weights), ptr(out[s:e]), self._stream()), name)
        return out

    @torch.no_grad()
    def posed(self, pose, rest_pose, transl) -> torch.Tensor:
        """Posed vertices [B,V,3] for pose [B,pose_width], rest_pose [B,rest_width] (None for SMPL) and transl [B,3]."""
        return self._vertices(*self._inputs(pose, rest_pose, transl))

    def vertices(self, pose, transl, rest_pose=None) -> torch.Tensor:
        """Posed vertices [B,V,3] for pose [B,72] and transl [B,3] (the reference's `SMPL.forward(...).vertices`); SMPL-X also takes
        rest_pose [B,99]."""
        return self.posed(pose, rest_pose, transl)


class SmplxBodyPoser(BodyPoser):
    """`BodyPoser` of `body.SMPLX`: the model as stored in SMPLX_{GENDER}.npz, poses split as the reference's
    smplx.SMPLX(use_pca=False, flat_hand_mean=True) splits them: pose [B,66] and rest_pose [B,99]."""

    def __init__(self, smplx, betas, device="cuda"):
        super().__init__(smplx, betas, device, SMPLX)

    def vertices(self, pose, rest_pose, transl) -> torch.Tensor:
        """Posed SMPL-X vertices [B,V,3] for pose [B,66], rest_pose [B,99] and transl [B,3] (`SMPLX.forward(...).vertices`)."""
        return self.posed(pose, rest_pose, transl)


class PoseMapper(BodyPoser):
    """Posed-body position maps [B,3,S,S] from poses, channel-first as the pose encoder takes them.

    smpl, betas, body: as `BodyPoser` takes them; uv_template: a path to the UV template OBJ or what `load_uv_template_obj` returns;
    S: map size (1..512).  Face i of the map is the mesh face f[i] drawn at the UV corners of template face i, so the template must
    have exactly F faces.  Everything runs on the current CUDA stream; calling the mapper with grad on and a pose or transl that
    requires grad makes the maps differentiable with respect to both (`ga_posmap_fill_backward`, then the vertex-posing backward)."""

    def __init__(self, smpl, betas, uv_template, S: int, device="cuda", body: Body = SMPL):
        super().__init__(smpl, betas, device, body)
        self.S = int(S)
        if not 1 <= self.S <= 512:
            raise ValueError(f"map size {S} outside 1..512")
        if isinstance(uv_template, (str, os.PathLike)):
            uv_template = load_uv_template_obj(uv_template)
        _, _, uvs, faces_uv = uv_template
        if faces_uv.shape[0] != self.F:
            raise ValueError(f"the UV template has {faces_uv.shape[0]} faces, the {body.label} mesh {self.F}: face i of one must be "
                             "face i of the other")
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

    def maps(self, pose, rest_pose, transl) -> torch.Tensor:
        """pose [B,pose_width], rest_pose [B,rest_width] (None for SMPL), transl [B,3] -> position maps [B,3,S,S], differentiable
        with respect to pose and transl (not rest_pose) when grad is on."""
        if _wants_grad(pose, transl):
            return _PoseMap.apply(self, pose, rest_pose, transl)
        return self.fill(self.posed(pose, rest_pose, transl))

    def __call__(self, pose, transl, rest_pose=None) -> torch.Tensor:
        """pose [B,72], transl [B,3] (SMPL-X also rest_pose [B,99]) -> position maps [B,3,S,S] (`maps`)."""
        return self.maps(pose, rest_pose, transl)

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
        J = self.JOINTS
        out = torch.empty(self.S, self.S, J, dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib().ga_posmap_weights(self.S, J, ptr(self.weights), ptr(self.faces), ptr(self.face_id), ptr(self.bary),
                                                ptr(out), self._stream()), "ga_posmap_weights")
        return out


class SmplxPoseMapper(PoseMapper):
    """`PoseMapper` of `body.SMPLX`: the model and poses as `SmplxBodyPoser` takes them."""

    def __init__(self, smplx, betas, uv_template, S: int, device="cuda"):
        super().__init__(smplx, betas, uv_template, S, device, SMPLX)

    def vertices(self, pose, rest_pose, transl) -> torch.Tensor:
        """As `SmplxBodyPoser.vertices`."""
        return self.posed(pose, rest_pose, transl)

    def __call__(self, pose, rest_pose, transl) -> torch.Tensor:
        """pose [B,66], rest_pose [B,99], transl [B,3] -> position maps [B,3,S,S] (`maps`)."""
        return self.maps(pose, rest_pose, transl)


def _wants_grad(*ts) -> bool:
    return torch.is_grad_enabled() and any(torch.is_tensor(t) and t.requires_grad for t in ts)


def vertices_backward(poser, pose, rest_pose, d_verts):
    """(d_pose [B,pose_width], d_transl [B,3]) of vertex gradients d_verts [B,V,3] at pose (and SMPL-X's rest_pose), through the
    body's vertex-posing backward (`ga_smpl_vertices_backward` / `ga_smplx_vertices_backward`)."""
    d_verts = d_verts.to(device=poser.device, dtype=torch.float32).contiguous()
    B, body = pose.shape[0], poser.body
    d_pose = torch.empty(B, body.pose_width, dtype=torch.float32, device=poser.device)
    d_transl = torch.empty(B, 3, dtype=torch.float32, device=poser.device)
    L = _lib.lib()
    ws = torch.empty(getattr(L, body.vertices_bwd_ws)(min(B, MAX_FRAMES_PER_CALL), poser.V), dtype=torch.uint8, device=poser.device)
    fn, poses = getattr(L, body.vertices_bwd), body.pose_args(pose, rest_pose)
    for s in range(0, B, MAX_FRAMES_PER_CALL):
        e = min(B, s + MAX_FRAMES_PER_CALL)
        _lib.check(fn(e - s, poser.V, *(ptr(p[s:e]) for p in poses), ptr(poser.rest_joints), ptr(poser.v_shaped), ptr(poser.posedirs),
                      ptr(poser.weights), ptr(d_verts[s:e]), ptr(ws), ws.numel(), ptr(d_pose[s:e]), ptr(d_transl[s:e]), poser._stream()),
                   body.vertices_bwd)
    return d_pose, d_transl


class _PoseMap(torch.autograd.Function):
    """(pose, rest_pose | None, transl) -> position maps [B,3,S,S] of a `PoseMapper`: the forward kernels as the mapper launches them,
    and backward through `ga_posmap_fill_backward` then the vertex-posing backward.  rest_pose is data."""

    @staticmethod
    def forward(ctx, mapper, pose, rest_pose, transl):
        pose, rest_pose, transl = mapper._inputs(pose, rest_pose, transl)
        ctx.mapper = mapper
        ctx.save_for_backward(pose, rest_pose)
        return mapper.fill(mapper._vertices(pose, rest_pose, transl))

    @staticmethod
    def backward(ctx, d_maps):
        pose, rest_pose = ctx.saved_tensors
        mapper = ctx.mapper
        d_pose, d_transl = vertices_backward(mapper, pose, rest_pose, mapper.fill_backward(d_maps))
        return None, d_pose, None, d_transl


# The reference's canonical pose (arguments/__init__.py:44-53, smpl_cpose_param / smplx_cpose_param: legs at +-30 degrees, every other
# joint zero, so SMPL-X hands are flat) and translation (scripts/gen_pose_map_cano_smpl.py:60-70).
CANO_LEG_ANGLE = 30.0 / 180.0 * math.pi
CANO_TRANSL = (0.0, 0.30, 0.0)


def canonical_pose(body: str) -> torch.Tensor:
    """The canonical pose [1,72] (SMPL) or [1,165] (SMPL-X: pose 66 | rest_pose 99)."""
    p = torch.zeros(1, body_of(body).full_width)
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
    b = body_of(body)
    if isinstance(model, (str, os.PathLike)):
        model = load_body_model(model)
    mapper = PoseMapper(model, betas, uv_template, S, device=device, body=b)
    dev = mapper.device
    pose, rest_pose = b.split(canonical_pose(body).to(dev))
    transl = torch.tensor([CANO_TRANSL], dtype=torch.float32, device=dev)
    posmap = mapper.fill(mapper.posed(pose, rest_pose, transl))[0].permute(1, 2, 0).contiguous()
    J = b.joints
    eye = torch.eye(4, device=dev).expand(J, 4, 4).contiguous()         # inv_cano = I: cano2live is A itself
    C = Cano2Live.apply(b, pose, rest_pose, transl, mapper.rest_joints, eye)
    A = torch.cat([C.reshape(J, 3, 4), eye[:, 3:4]], 1)
    return CanonicalAssets(posmap, A, mapper.face_id.clone(), mapper.weight_map(), mapper.bary.clone())
