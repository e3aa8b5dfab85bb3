"""Stage-2 input position maps built on the device from each frame's SMPL pose.

The reference makes `inp_map/inp_posemap_{S}_{idx:08d}.npz` offline (scripts/gen_pose_map_our_smpl.py): the smplx forward pass,
one OBJ per frame, then an OpenGL render of each mesh in UV space.  Because that render happens in UV space, which face covers which
texel (and with which barycentric weights) does not depend on the pose: `PoseMapper` computes that layout once on the device
(`ga_posmap_layout`), and a frame costs the posed vertices (`ga_smpl_vertices`) and a gather (`ga_posmap_fill`).  The coverage
rules are the library's own statement of what the GL rasterizer does (csrc/posmap.cu; DESIGN.md, PARITY UNPINNED).
"""
from __future__ import annotations

import os

import numpy as np
import torch

from . import _lib
from ._lib import ptr

SMPL_MESH_FIELDS = ("v_template", "shapedirs", "posedirs", "weights", "f", "J_regressor")
MAX_FRAMES_PER_CALL = 8          # ga_smpl_vertices


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


class PoseMapper:
    """Posed-body position maps [B,3,S,S] from SMPL poses, channel-first as the pose encoder takes them.

    smpl: the SMPL model as stored in SMPL_{GENDER}.pkl (any mapping with v_template [V,3], shapedirs [V,3,>=10], posedirs
    [V,3,207], weights [V,24], f [F,3], J_regressor [24,V] dense or sparse); betas [10]; uv_template: a path to the UV template OBJ
    or what `load_uv_template_obj` returns; S: map size (1..512).  Face i of the map is the mesh face f[i] drawn at the UV corners
    of template face i, so the template must have exactly F faces.  Everything runs on the current CUDA stream under no_grad."""

    def __init__(self, smpl, betas, uv_template, S: int, device="cuda"):
        missing = [k for k in SMPL_MESH_FIELDS if k not in smpl]
        if missing:
            raise ValueError(f"the SMPL model has no {', '.join(missing)}: device position maps need the full mesh model")
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("PoseMapper runs on CUDA only (no CPU fallback)")
        self.S = int(S)
        if not 1 <= self.S <= 512:
            raise ValueError(f"map size {S} outside 1..512")
        if isinstance(uv_template, (str, os.PathLike)):
            uv_template = load_uv_template_obj(uv_template)
        _, _, uvs, faces_uv = uv_template
        v_t = np.asarray(smpl["v_template"], np.float64)
        V = v_t.shape[0]
        beta = np.asarray(torch.as_tensor(betas).double().reshape(-1))
        sd = np.asarray(smpl["shapedirs"])[:, :, :beta.size].astype(np.float64)
        posedirs = np.asarray(smpl["posedirs"], np.float32)
        weights = np.asarray(smpl["weights"], np.float32)
        faces = np.asarray(smpl["f"]).astype(np.int64)
        Jr = _dense(smpl["J_regressor"]).astype(np.float64)
        if posedirs.shape != (V, 3, 207) or weights.shape != (V, 24) or Jr.shape != (24, V) or faces.ndim != 2 or faces.shape[1] != 3:
            raise ValueError(f"SMPL model: posedirs {posedirs.shape}, weights {weights.shape}, J_regressor {Jr.shape}, f {faces.shape}; "
                             f"expected [{V},3,207], [{V},24], [24,{V}], [F,3]")
        if faces.size and (faces.min() < 0 or faces.max() >= V):
            raise ValueError(f"SMPL model: a face indexes a vertex outside 0..{V - 1}")
        if faces_uv.shape[0] != faces.shape[0]:
            raise ValueError(f"the UV template has {faces_uv.shape[0]} faces, the SMPL mesh {faces.shape[0]}: face i of one must be face i of "
                             "the other")
        v_shaped = v_t + np.einsum("l,mkl->mk", beta, sd)
        dev = self.device
        self.V, self.F = V, faces.shape[0]
        self.rest_joints = torch.from_numpy(Jr @ v_shaped).float().to(dev).contiguous()                 # [24,3]
        self.v_shaped = torch.from_numpy(v_shaped).float().to(dev).contiguous()                         # [V,3]
        self.posedirs = torch.from_numpy(posedirs.reshape(V * 3, 207).T.copy()).to(dev)                 # [207,3V] as smplx.SMPL keeps it
        self.weights = torch.from_numpy(weights).to(dev).contiguous()                                   # [V,24]
        self.faces = torch.from_numpy(faces.astype(np.int32)).to(dev).contiguous()                      # [F,3]
        corners = torch.from_numpy(np.asarray(uvs, np.float32)[faces_uv]).to(dev).contiguous()        # [F,3,2]
        self.face_id = torch.empty(self.S, self.S, dtype=torch.int32, device=dev)
        self.bary = torch.empty(self.S, self.S, 3, dtype=torch.float32, device=dev)
        _lib.check(_lib.lib().ga_posmap_layout(self.F, self.S, ptr(corners), ptr(self.face_id), ptr(self.bary), self._stream()),
                   "ga_posmap_layout")

    @staticmethod
    def _stream() -> int:
        return torch.cuda.current_stream().cuda_stream

    def _inputs(self, pose, transl):
        pose = torch.as_tensor(pose).to(device=self.device, dtype=torch.float32).reshape(-1, 72).contiguous()
        transl = torch.as_tensor(transl).to(device=self.device, dtype=torch.float32).reshape(-1, 3).contiguous()
        if pose.shape[0] != transl.shape[0]:
            raise ValueError(f"pose {tuple(pose.shape)} and transl {tuple(transl.shape)} have different frame counts")
        return pose, transl

    @torch.no_grad()
    def vertices(self, pose, transl) -> torch.Tensor:
        """Posed SMPL vertices [B,V,3] for pose [B,72] and transl [B,3] (the reference's `SMPL.forward(...).vertices`)."""
        pose, transl = self._inputs(pose, transl)
        B = pose.shape[0]
        out = torch.empty(B, self.V, 3, dtype=torch.float32, device=self.device)
        L = _lib.lib()
        for s in range(0, B, MAX_FRAMES_PER_CALL):
            e = min(B, s + MAX_FRAMES_PER_CALL)
            _lib.check(L.ga_smpl_vertices(e - s, self.V, ptr(pose[s:e]), ptr(transl[s:e]), ptr(self.rest_joints), ptr(self.v_shaped),
                                          ptr(self.posedirs), ptr(self.weights), ptr(out[s:e]), self._stream()), "ga_smpl_vertices")
        return out

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
        """pose [B,72], transl [B,3] -> position maps [B,3,S,S]."""
        return self.fill(self.vertices(pose, transl))
