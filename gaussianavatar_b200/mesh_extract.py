"""A coloured, watertight mesh of a posed avatar, extracted on the device.

    verts, faces, colors = extract_mesh(model, model.pose.weight[:1], model.transl.weight[:1])
    write_ply("avatar.ply", verts, faces, colors)

The posed Gaussians are rendered from `views` cameras on a Fibonacci sphere around them (`rasterize_batch_depth`, bg 0), and each
view's median depth, colour and final transmittance are fused into a truncated signed distance field (`TsdfVolume`, csrc/tsdf.cu:
`ga_tsdf_integrate`): the method 2DGS and GOF use to mesh splats.  Its zero level set is extracted by marching tetrahedra on the
Kuhn split of every grid cube (`ga_tsdf_mesh_count` / `ga_tsdf_mesh_emit`), so the mesh is closed and 2-manifold without an
ambiguity table, its vertices welded exactly, and bit-reproducible from run to run.

Samples a view sees no surface through (median depth 0, alpha < 0.5) are carved: a sample carved by at least `min_carve` views is
outside.  Samples no view saw in front of are inside.  Parts thinner than about the truncation distance or one fusion pixel (fingers
at a low resolution) may be carved away; a larger `min_carve` keeps them.  The model's parameters and BatchNorm statistics are left
as they were.  Everything runs on the current CUDA stream; there is no CPU fallback.
"""
from __future__ import annotations

import ctypes
import math

import numpy as np
import torch

from . import _lib
from ._lib import ptr
from .animate import final_transmittance
from .avatar_model import kept_state
from .camera import make_camera
from .rasterizer import CAM_STRIDE, MAX_FRAMES_PER_CALL, RasterBatchPlan, rasterize_batch_depth

MAX_SIDE = 512                   # ga_tsdf_*: samples per axis
PLANES = ("sdf", "weight", "carve", "r", "g", "b", "cw")


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


class TsdfVolume:
    """A TSDF grid on the device: samples at origin + voxel (i, j, k) for dims (nx, ny, nz) (each 2..512), truncation `trunc` in
    world units.  The state is 28 bytes per sample (`fields()`)."""

    def __init__(self, origin, voxel: float, dims, trunc: float, device="cuda"):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("TsdfVolume runs on CUDA only (no CPU fallback)")
        nx, ny, nz = (int(n) for n in dims)
        self.dims = (nx, ny, nz)
        self.origin = tuple(float(np.float32(o)) for o in origin)
        self.voxel, self.trunc = float(np.float32(voxel)), float(np.float32(trunc))
        self.desc = _lib.GaTsdfDesc(nx, ny, nz, (ctypes.c_float * 3)(*self.origin), self.voxel, self.trunc)
        L = _lib.lib()
        nbytes = L.ga_tsdf_state_bytes(ctypes.byref(self.desc))
        if nbytes == 0:
            raise ValueError(L.ga_last_error().decode())
        self.state = torch.empty(nbytes // 4, dtype=torch.int32, device=self.device)
        self.device = self.state.device
        self.reset()

    def reset(self):
        _lib.check(_lib.lib().ga_tsdf_reset(ctypes.byref(self.desc), ptr(self.state), _stream()), "ga_tsdf_reset")

    def fields(self) -> dict:
        """Views [nz,ny,nx] of the state planes: sdf (fp32, units of trunc), weight, carve (int32), r, g, b (fp32 colour sums) and
        cw (int32 colour weight)."""
        nx, ny, nz = self.dims
        planes = self.state.view(len(PLANES), nz, ny, nx)
        return {k: (planes[i].view(torch.float32) if k in ("sdf", "r", "g", "b") else planes[i]) for i, k in enumerate(PLANES)}

    @torch.no_grad()
    def integrate(self, depth, image, final_T, cams):
        """Fuses B views: depth [B,2,H,W] (its median plane), image [B,3,H,W] rendered with bg 0, final_T [B,H,W], cams [B,40], in
        launches of up to 8 views.  The result does not depend on how the views are split."""
        B, _, H, W = (int(n) for n in depth.shape)
        want = {"depth": (depth, (B, 2, H, W)), "image": (image, (B, 3, H, W)), "final_T": (final_T, (B, H, W)), "cams": (cams, (B, CAM_STRIDE))}
        args = {}
        for name, (t, shape) in want.items():
            if not torch.is_tensor(t) or t.device != self.device or t.dtype != torch.float32 or tuple(t.shape) != shape:
                raise ValueError(f"{name}: expected a float32 tensor {list(shape)} on {self.device}")
            args[name] = t.contiguous()
        L = _lib.lib()
        for s in range(0, B, MAX_FRAMES_PER_CALL):
            e = min(B, s + MAX_FRAMES_PER_CALL)
            _lib.check(L.ga_tsdf_integrate(ctypes.byref(self.desc), e - s, H, W, ptr(args["cams"][s:e]), ptr(args["depth"][s:e]),
                                           ptr(args["image"][s:e]), ptr(args["final_T"][s:e]), ptr(self.state), _stream()),
                       "ga_tsdf_integrate")

    @torch.no_grad()
    def mesh(self, min_carve: int = 1):
        """(verts [V,3] fp32, faces [F,3] int32, colors [V,3] fp32) of the zero level set.  Reads the two totals on the host (one
        synchronise)."""
        if int(min_carve) < 1:
            raise ValueError(f"min_carve {min_carve} must be >= 1")
        L = _lib.lib()
        d = ctypes.byref(self.desc)
        ws = torch.empty(L.ga_tsdf_mesh_workspace_bytes(d), dtype=torch.uint8, device=self.device)
        totals = torch.zeros(2, dtype=torch.int32, device=self.device)
        _lib.check(L.ga_tsdf_mesh_count(d, ptr(self.state), int(min_carve), ptr(ws), ws.numel(), ptr(totals), _stream()), "ga_tsdf_mesh_count")
        V, F = (int(n) for n in totals.cpu())
        verts = torch.empty(V, 3, dtype=torch.float32, device=self.device)
        colors = torch.empty(V, 3, dtype=torch.float32, device=self.device)
        faces = torch.empty(F, 3, dtype=torch.int32, device=self.device)
        _lib.check(L.ga_tsdf_mesh_emit(d, ptr(self.state), int(min_carve), ptr(ws), ws.numel(), V, F, ptr(verts) if V else None,
                                       ptr(colors) if V else None, ptr(faces) if F else None, _stream()), "ga_tsdf_mesh_emit")
        return verts, faces, colors


def fibonacci_directions(n: int) -> np.ndarray:
    """[n,3] unit vectors spread evenly over the sphere (fp64)."""
    k = np.arange(n, dtype=np.float64) + 0.5
    y = 1.0 - 2.0 * k / n
    rad = np.sqrt(np.maximum(0.0, 1.0 - y * y))
    phi = k * math.pi * (3.0 - math.sqrt(5.0))
    return np.stack([np.cos(phi) * rad, y, np.sin(phi) * rad], 1)


def look_at_extrinsic(eye, target) -> np.ndarray:
    """World -> camera 4x4 (x right, y down, z forward, as the datasets' cameras) looking from eye at target."""
    f = np.asarray(target, np.float64) - np.asarray(eye, np.float64)
    f /= np.linalg.norm(f)
    up = np.array([0.0, 1.0, 0.0]) if abs(f[1]) < 0.9 else np.array([0.0, 0.0, 1.0])     # not along the view at the poles
    right = np.cross(f, up)
    right /= np.linalg.norm(right)
    down = np.cross(f, right)
    E = np.eye(4)
    E[:3, :3] = np.stack([right, down, f])
    E[:3, 3] = -E[:3, :3] @ np.asarray(eye, np.float64)
    return E


def fusion_cameras(center, radius: float, n_views: int, size: int) -> torch.Tensor:
    """[n_views,40] camera rows (host fp32, `pack_cameras` layout) of size x size views from n_views directions on a Fibonacci sphere,
    each looking at `center`.  The ball of `radius` around it fills the view with a 10 % margin, and every point of the ball is at
    least max(1.5 radius, 0.5) in front of each camera, beyond the rasterizer's z = 0.2 cull."""
    from .mesh_render import cameras as camera_block
    radius, size = float(radius), int(size)
    if not (radius > 0 and math.isfinite(radius)) or n_views < 1 or size < 1:
        raise ValueError(f"radius {radius}, n_views {n_views} and size {size} must be positive")
    dist = max(2.5 * radius, radius + 0.5)
    s = 1.1 * radius / dist
    f = 0.5 * size / (s / math.sqrt(1.0 - s * s))
    K = np.array([[f, 0.0, 0.5 * size], [0.0, f, 0.5 * size], [0.0, 0.0, 1.0]], np.float32)
    c = np.asarray(center, np.float64).reshape(3)
    return camera_block([make_camera(K, look_at_extrinsic(c + dist * d, c), size, size, zfar=max(100.0, 4 * dist))
                         for d in fibonacci_directions(int(n_views))])


def posed_gaussians(model, pose, transl, rest_pose=None, pose_mapper=None):
    """means, scales, colors [1,N,3] of the avatar in one pose, as the animation player poses them: stage 1 the frame-invariant decoder
    and `_assemble`, stage 2 `_stage2_from_pose` with pose_mapper (default: the model's).  Call under no_grad and `kept_state`."""
    dev = model.device
    pose = torch.as_tensor(pose).to(device=dev, dtype=torch.float32).reshape(1, -1).contiguous()
    transl = torch.as_tensor(transl).to(device=dev, dtype=torch.float32).reshape(1, 3).contiguous()
    if rest_pose is not None:
        rest_pose = torch.as_tensor(rest_pose).to(device=dev, dtype=torch.float32).reshape(1, -1).contiguous()
    if int(model.model_parms.train_stage) == 2:
        mapper = pose_mapper if pose_mapper is not None else getattr(model, "pose_mapper", None)
        if mapper is None:
            raise ValueError("stage 2 needs a pose_mapper (posmap.PoseMapper / SmplxPoseMapper) for the input position maps")
        return model._stage2_from_pose(mapper, pose, transl, rest_pose)[:3]
    return model._assemble(model._stage1_decoder(1), pose, transl, rest_pose)


def render_views(model, means, scales, colors, cams, H: int, W: int):
    """Yields (s, e, images [b,3,H,W], depth [b,2,H,W], final_T [b,H,W]) for the camera rows cams[s:e] in chunks of up to 8, rendered
    with bg 0 (`rasterize_batch_depth`) in the model's antialiasing mode; a chunk whose binning buffer overflowed is rendered again after it grew.  final_T is a view
    of the chunk's raster buffers: use it before the next chunk is drawn."""
    dev = means.device
    bg = torch.zeros(3, dtype=torch.float32, device=dev)
    P = int(means.shape[1])
    plans = {}
    for s in range(0, cams.shape[0], MAX_FRAMES_PER_CALL):
        e = min(cams.shape[0], s + MAX_FRAMES_PER_CALL)
        b = e - s
        if b not in plans:
            plans[b] = RasterBatchPlan(b, P, H, W, dev, antialiasing=getattr(model, "antialiasing", False))
        plan = plans[b]
        args = (means.expand(b, -1, -1), colors.expand(b, -1, -1), scales.expand(b, -1, -1), model.fix_rotation, model.fix_opacity,
                cams[s:e].contiguous(), bg, plan)
        (img, depth), _ = plan.render_checked(lambda: rasterize_batch_depth(*args), "mesh extraction")
        yield s, e, img, depth, final_transmittance(plan)


def fusion_grid(means, scales, res: int, trunc_voxels: float):
    """(origin, voxel, dims, trunc) of a grid holding the Gaussians' means +- 3 max scale, padded by trunc + 2 voxels on every side,
    with `res` samples along its longest side."""
    m = means.reshape(-1, 3).double()
    r = 3.0 * scales.reshape(-1, 3).double().max(1).values[:, None]
    lo, hi = (m - r).min(0).values.cpu().numpy(), (m + r).max(0).values.cpu().numpy()
    pad_voxels = float(trunc_voxels) + 2.0
    inner = int(res) - 1 - 2.0 * pad_voxels
    if not 2 <= int(res) <= MAX_SIDE or inner <= 0:
        raise ValueError(f"res {res} outside 2..{MAX_SIDE} or too small for trunc_voxels {trunc_voxels}")
    voxel = float(np.float32(max(float((hi - lo).max()), 1e-6) / inner))
    origin = lo - pad_voxels * voxel
    dims = [int(min(res, max(2, math.ceil((hi[a] - lo[a]) / voxel + 2.0 * pad_voxels - 1e-9) + 1))) for a in range(3)]
    return origin, voxel, dims, float(trunc_voxels) * voxel


@torch.no_grad()
def extract_mesh(model, pose, transl, rest_pose=None, res: int = 256, views: int = 64, size: int = 512, trunc_voxels: float = 4,
                 min_carve: int = 1, pose_mapper=None):
    """The avatar in one pose (pose [72|66], transl [3], SMPL-X's rest_pose [99]) as (verts [V,3] fp32, faces [F,3] int32, colors
    [V,3] fp32 in [0,1]) on the device: `views` size x size depth passes fused into a grid with `res` samples along its longest side
    and truncation trunc_voxels voxels, meshed with `min_carve`.  The model's state is left as it was."""
    with kept_state(model):
        means, scales, colors = posed_gaussians(model, pose, transl, rest_pose, pose_mapper)
    return mesh_gaussians(model, means, scales, colors, res, views, size, trunc_voxels, min_carve)


@torch.no_grad()
def mesh_gaussians(model, means, scales, colors, res: int = 256, views: int = 64, size: int = 512, trunc_voxels: float = 4,
                   min_carve: int = 1):
    """The mesh of a set of the model's Gaussians, means, scales, colors [1,N,3] on the device (rendered with its rotations and
    opacities), as `extract_mesh` returns it."""
    origin, voxel, dims, trunc = fusion_grid(means, scales, res, trunc_voxels)
    vol = TsdfVolume(origin, voxel, dims, trunc, device=means.device)
    center = np.asarray(vol.origin) + 0.5 * voxel * (np.asarray(dims) - 1)
    radius = 0.5 * voxel * float(np.linalg.norm(np.asarray(dims) - 1))
    cams = fusion_cameras(center, radius, views, size).to(means.device)
    for s, e, img, depth, final_T in render_views(model, means, scales, colors, cams, size, size):
        vol.integrate(depth, img, final_T, cams[s:e])
    return vol.mesh(min_carve)


@torch.no_grad()
def silhouette_iou(model, pose, transl, verts, faces, cams, H: int, W: int, rest_pose=None, pose_mapper=None) -> list:
    """Per camera row of cams [B,40]: the IoU of the mesh's drawn pixels (`MeshRenderer` face_id >= 0) and the avatar's own surface
    (median depth > 0, i.e. alpha >= 0.5) in the same pose, both H x W."""
    from .mesh_render import MeshRenderer, coverage_iou
    with kept_state(model):
        means, scales, colors = posed_gaussians(model, pose, transl, rest_pose, pose_mapper)
    cams = torch.as_tensor(cams).to(device=means.device, dtype=torch.float32)
    mr = MeshRenderer(faces, int(verts.shape[0]), device=means.device)
    out = []
    for s, e, _, depth, _ in render_views(model, means, scales, colors, cams, H, W):
        _, face_id, _ = mr.render(verts.reshape(1, -1, 3).expand(e - s, -1, -1), cams[s:e], H, W)
        out += [coverage_iou(face_id[b] >= 0, depth[b, 1] > 0) for b in range(e - s)]
    return out


def quantize(colors) -> np.ndarray:
    """uint8 colours as ga_frame_pack quantises: clamp(fp32(fp32(x 255) + 0.5), 0, 255), truncated, NaN -> 0."""
    x = np.asarray(colors, np.float32)
    with np.errstate(invalid="ignore"):
        q = (x * np.float32(255)) + np.float32(0.5)
    return np.clip(np.nan_to_num(q, nan=0.0), 0, 255).astype(np.uint8)


def _host(verts, faces, colors):
    t = lambda a: a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    return t(verts).astype(np.float32).reshape(-1, 3), t(faces).astype(np.int32).reshape(-1, 3), t(colors).astype(np.float32).reshape(-1, 3)


def write_ply(path, verts, faces, colors) -> None:
    """Binary little-endian PLY: float x, y, z and uchar red, green, blue per vertex; faces as uchar-counted int lists."""
    v, f, c = _host(verts, faces, colors)
    vert = np.empty(len(v), dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    vert["x"], vert["y"], vert["z"] = v[:, 0], v[:, 1], v[:, 2]
    q = quantize(c)
    vert["red"], vert["green"], vert["blue"] = q[:, 0], q[:, 1], q[:, 2]
    face = np.empty(len(f), dtype=[("n", "u1"), ("v", "<i4", (3,))])
    face["n"], face["v"] = 3, f
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {len(v)}\nproperty float x\nproperty float y\nproperty float z\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\n"
              f"element face {len(f)}\nproperty list uchar int vertex_indices\nend_header\n")
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(vert.tobytes())
        fh.write(face.tobytes())


def write_obj(path, verts, faces, colors) -> None:
    """OBJ with per-vertex colours: `v x y z r g b` (colours in [0,1]) and 1-based `f a b c`."""
    v, f, c = _host(verts, faces, colors)
    with open(path, "w") as fh:
        for p, col in zip(v, c):
            fh.write("v %.9g %.9g %.9g %.6g %.6g %.6g\n" % (p[0], p[1], p[2], col[0], col[1], col[2]))
        for t in f + 1:
            fh.write("f %d %d %d\n" % (t[0], t[1], t[2]))
