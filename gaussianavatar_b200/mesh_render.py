"""Posed-body overlay on the device: a depth-tested, shaded triangle-mesh render with the cameras the avatar's Gaussians use.

The reference checks its stage-1 pose refinement by drawing the posed SMPL mesh over every training image with pyrender
(scripts/render_pred_smpl.py: OpenGL, a MetallicRoughnessMaterial, one directional light).  `MeshRenderer` draws the same mesh with
the library's own kernel (`ga_mesh_render`, csrc/mesh_render.cu): exact integer coverage at pixel centres, the nearest face per
pixel, the glTF metallic-roughness BRDF lit by a headlight.  The coverage and shading rules are the library's own statement of
what pyrender does (DESIGN.md §2, PARITY UNPINNED).  Vertices come from `posmap.BodyPoser` / `posmap.SmplxBodyPoser`.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import _lib
from ._lib import ptr
from .rasterizer import CAM_STRIDE, pack_cameras

MAX_FRAMES_PER_CALL = 8          # ga_mesh_render
MAX_SIDE = 16384

# render_pred_smpl.py's colors_dict (base colours of the material)
COLORS = {
    "red": (0.5, 0.2, 0.2),
    "pink": (0.7, 0.5, 0.5),
    "neutral": (0.7, 0.7, 0.6),
    "purple": (0.55, 0.4, 0.9),
    "green": (0.5, 0.55, 0.3),
    "sky": (0.3, 0.5, 0.55),
    "white": (1.0, 0.98, 0.94),
}


def vertex_face_csr(faces: np.ndarray, V: int):
    """The vertex -> face adjacency of faces [F,3] as CSR (offsets [V+1], faces [3F]) int32: the faces of vertex v, in ascending
    face order and once per corner they have at v, are faces[offsets[v]:offsets[v+1]]."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    F = faces.shape[0]
    vert = faces.reshape(-1)
    face = np.repeat(np.arange(F, dtype=np.int64), 3)
    order = np.lexsort((face, vert))
    offsets = np.zeros(V + 1, np.int64)
    np.cumsum(np.bincount(vert, minlength=V), out=offsets[1:])
    return offsets.astype(np.int32), face[order].astype(np.int32)


def coverage_iou(drawn, mask) -> float:
    """IoU of a drawn silhouette (face_id >= 0) and a subject mask (byte >= 128), boolean [H,W] numpy arrays or tensors; 1 when
    both are empty.  Integer counts, so the value does not depend on where it is computed."""
    union = int((mask | drawn).sum())
    return int((mask & drawn).sum()) / union if union else 1.0


def cameras(cams) -> torch.Tensor:
    """[B,40] camera block (ga_rasterb_* layout) of a list of `camera.Camera`."""
    view = torch.stack([c.world_view_transform.float().cpu() for c in cams])
    proj = torch.stack([c.full_proj_transform.float().cpu() for c in cams])
    center = torch.stack([c.camera_center.float().cpu() for c in cams])
    return pack_cameras(view, proj, [math.tan(c.FovX * 0.5) for c in cams], [math.tan(c.FovY * 0.5) for c in cams], "cpu", campos=center)


class MeshRenderer:
    """Draws a fixed triangle mesh, faces [F,3] over V vertices, on the device.

    `render(verts [B,V,3], cams [B,40], H, W, background=None)` returns (rgb [B,3,H,W] fp32, face_id [B,H,W] int32, depth
    [B,H,W] fp32): the shade where a face is drawn and the background (0 if None) elsewhere, the drawn face (-1: none) and its
    view-space depth (0: none).  color: the material's base colour, a name of `COLORS` or an RGB triple.  Runs on the current CUDA
    stream under no_grad; there is no CPU fallback."""

    def __init__(self, faces, V: int, device="cuda", color="white"):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("MeshRenderer runs on CUDA only (no CPU fallback)")
        f = np.asarray(faces.cpu() if torch.is_tensor(faces) else faces)
        if f.ndim != 2 or f.shape[1] != 3 or not np.issubdtype(f.dtype, np.integer):
            raise ValueError(f"faces {f.shape} {f.dtype}: expected an integer [F,3] array")
        self.V, self.F = int(V), f.shape[0]
        if not 1 <= self.V <= 1 << 24 or self.F > 1 << 24:
            raise ValueError(f"{self.V} vertices / {self.F} faces outside the kernel's range (1..2^24 / 0..2^24)")
        if f.size and (f.min() < 0 or f.max() >= self.V):
            raise ValueError(f"a face indexes a vertex outside 0..{self.V - 1}")
        rgb = COLORS[color] if isinstance(color, str) else tuple(float(c) for c in color)
        if len(rgb) != 3:
            raise ValueError(f"color {color!r}: expected a name of COLORS or three floats")
        self.color = tuple(float(np.float32(c)) for c in rgb)
        off, adj = vertex_face_csr(f, self.V)
        self.faces = torch.from_numpy(f.astype(np.int32)).to(self.device).contiguous()
        self.adj_offsets = torch.from_numpy(off).to(self.device)
        self.adj_faces = torch.from_numpy(adj).to(self.device)

    @torch.no_grad()
    def render(self, verts, cams, H: int, W: int, background=None):
        H, W = int(H), int(W)
        if not (1 <= H <= MAX_SIDE and 1 <= W <= MAX_SIDE):
            raise ValueError(f"frame {H} x {W} outside [1, {MAX_SIDE}]^2")
        verts = torch.as_tensor(verts).to(device=self.device, dtype=torch.float32).contiguous()
        if verts.dim() != 3 or tuple(verts.shape[1:]) != (self.V, 3):
            raise ValueError(f"vertices {tuple(verts.shape)}: expected [B,{self.V},3]")
        B = verts.shape[0]
        cams = torch.as_tensor(cams).to(device=self.device, dtype=torch.float32).contiguous()
        if tuple(cams.shape) != (B, CAM_STRIDE):
            raise ValueError(f"cameras {tuple(cams.shape)}: expected [{B},{CAM_STRIDE}]")
        if background is not None:
            background = torch.as_tensor(background).to(device=self.device, dtype=torch.float32).contiguous()
            if tuple(background.shape) != (B, 3, H, W):
                raise ValueError(f"background {tuple(background.shape)}: expected [{B},3,{H},{W}]")
        rgb = torch.empty(B, 3, H, W, dtype=torch.float32, device=self.device)
        face_id = torch.empty(B, H, W, dtype=torch.int32, device=self.device)
        depth = torch.empty(B, H, W, dtype=torch.float32, device=self.device)
        L = _lib.lib()
        ws = None
        stream = torch.cuda.current_stream().cuda_stream
        for s in range(0, B, MAX_FRAMES_PER_CALL):
            e = min(B, s + MAX_FRAMES_PER_CALL)
            if ws is None:
                ws = torch.empty(L.ga_mesh_render_workspace_bytes(e - s, self.V, self.F, H, W), dtype=torch.uint8, device=self.device)
            _lib.check(L.ga_mesh_render(e - s, self.V, self.F, H, W, ptr(verts[s:e]), ptr(self.faces), ptr(self.adj_offsets),
                                        ptr(self.adj_faces), ptr(cams[s:e]), *self.color,
                                        None if background is None else ptr(background[s:e]), ptr(ws), ptr(face_id[s:e]),
                                        ptr(depth[s:e]), ptr(rgb[s:e]), stream), "ga_mesh_render")
        return rgb, face_id, depth

    @torch.no_grad()
    def render_unlit(self, verts, cams, H: int, W: int, colors=None, uvs=None, texture=None, background=None):
        """The mesh drawn as `render` draws it, coloured without lighting (`ga_mesh_shade_unlit`): colors [V,3] interpolated, or
        texture [Th,Tw,3] (fp32, row 0 first) sampled bilinearly at uvs [V,2] (glTF's convention), clamped to the edge.  Returns
        (rgb [B,3,H,W], face_id [B,H,W], depth [B,H,W])."""
        if (colors is None) == (uvs is None or texture is None):
            raise ValueError("give colors, or uvs and texture")
        _, face_id, depth = self.render(verts, cams, H, W)
        H, W = int(H), int(W)
        dev = self.device
        verts = torch.as_tensor(verts).to(device=dev, dtype=torch.float32).contiguous()
        cams = torch.as_tensor(cams).to(device=dev, dtype=torch.float32).contiguous()
        B = verts.shape[0]
        f32 = lambda t, shape: None if t is None else _shaped(t, shape, dev)
        colors, uvs = f32(colors, (self.V, 3)), f32(uvs, (self.V, 2))
        Th = Tw = 0
        if texture is not None:
            texture = torch.as_tensor(texture).to(device=dev, dtype=torch.float32).contiguous()
            if texture.dim() != 3 or texture.shape[2] != 3:
                raise ValueError(f"texture {tuple(texture.shape)}: expected [Th,Tw,3]")
            Th, Tw = int(texture.shape[0]), int(texture.shape[1])
        if background is not None:
            background = _shaped(background, (B, 3, H, W), dev)
        rgb = torch.empty(B, 3, H, W, dtype=torch.float32, device=dev)
        stream = torch.cuda.current_stream().cuda_stream
        for s in range(0, B, MAX_FRAMES_PER_CALL):
            e = min(B, s + MAX_FRAMES_PER_CALL)
            _lib.check(_lib.lib().ga_mesh_shade_unlit(e - s, self.V, self.F, H, W, ptr(verts[s:e]), ptr(self.faces), ptr(cams[s:e]),
                                                      ptr(face_id[s:e]), ptr(colors), ptr(uvs), ptr(texture), Th, Tw,
                                                      None if background is None else ptr(background[s:e]), ptr(rgb[s:e]), stream),
                       "ga_mesh_shade_unlit")
        return rgb, face_id, depth


def _shaped(t, shape, device) -> torch.Tensor:
    t = torch.as_tensor(t).to(device=device, dtype=torch.float32).contiguous()
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"{tuple(t.shape)}: expected {list(shape)}")
    return t
