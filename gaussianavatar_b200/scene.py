"""A 3D Gaussian Splatting scene to render an avatar in, and where the avatar stands in it.

    scene = GaussianScene.load_ply("output/room/point_cloud/iteration_30000/point_cloud.ply").to("cuda")
    place = Placement.from_axis_angle(0.9, [0, 0, 0], [0.2, -1.1, 3.0])       # x_scene = s R x_avatar + t
    anim = Animator(model, cameras, H, W, scene=scene, placement=place)

`GaussianScene.load_ply` reads the file 3DGS's `GaussianModel.save_ply` writes and applies its activations.  The rasterizer splats
the scene's Gaussians and the avatar's in one sort per tile (`rasterizer.rasterize_batch_scene`), so each hides the other where it
is in front.  `Placement` moves the avatar into the scene by folding [sR | t] into the per-joint cano2live transforms and s into the
skinning kernel's scale multiplier, and carries a camera defined around the avatar into the scene so that it frames the avatar
exactly as before.
"""
from __future__ import annotations

import json
import os
import re
from dataclasses import dataclass, field

import numpy as np
import torch

from .camera import Camera, make_camera

# f_rest_* properties per SH degree: 3 channels x ((D + 1)^2 - 1) coefficients
SH_DEGREE_OF_REST = {0: 0, 9: 1, 24: 2, 45: 3}

_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2", "uint16": "u2",
              "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4", "double": "f8", "float64": "f8"}


def _read_ply_vertices(path):
    """The `vertex` element of a binary little-endian PLY as a numpy structured array (properties by name)."""
    with open(path, "rb") as f:
        data = f.read()
    if not data.startswith(b"ply\n"):
        raise ValueError(f"{path}: not a PLY file (no 'ply' magic line)")
    end = data.find(b"end_header\n")
    if end < 0:
        raise ValueError(f"{path}: PLY header has no 'end_header' line")
    header = data[:end].decode("ascii", errors="replace").splitlines()
    body = end + len(b"end_header\n")
    fmt, elements, cur = None, [], None
    for line in header[1:]:
        tok = line.split()
        if not tok or tok[0] in ("comment", "obj_info"):
            continue
        if tok[0] == "format":
            fmt = tok[1] if len(tok) > 1 else ""
        elif tok[0] == "element":
            cur = (tok[1], int(tok[2]), [])
            elements.append(cur)
        elif tok[0] == "property":
            if cur is None:
                raise ValueError(f"{path}: PLY property before any element")
            if tok[1] == "list":
                raise ValueError(f"{path}: element '{cur[0]}' has a list property ('{tok[-1]}'); a 3DGS scene has none")
            if tok[1] not in _PLY_TYPES:
                raise ValueError(f"{path}: PLY property '{tok[2]}' has unknown type '{tok[1]}'")
            cur[2].append((tok[2], _PLY_TYPES[tok[1]]))
    if fmt != "binary_little_endian":
        raise ValueError(f"{path}: PLY format '{fmt}' is not supported; 3DGS writes binary_little_endian (ASCII and big-endian are not read)")
    if not elements or elements[0][0] != "vertex":
        raise ValueError(f"{path}: the first PLY element must be 'vertex'")
    _, n, props = elements[0]
    dtype = np.dtype([(name, "<" + t) for name, t in props])
    if len(data) - body < n * dtype.itemsize:
        raise ValueError(f"{path}: truncated: the header declares {n} vertices of {dtype.itemsize} bytes, the file holds "
                         f"{(len(data) - body) // max(dtype.itemsize, 1)}")
    return np.frombuffer(data, dtype=dtype, count=n, offset=body)


@dataclass
class GaussianScene:
    """Ps static Gaussians, activated: means3D [Ps,3], scales [Ps,3], rotations [Ps,4] (w, x, y, z, unit), opacities [Ps], and SH
    coefficients shs [Ps,M,3] (k = 0 the DC term, M = (sh_degree + 1)^2), all fp32 and contiguous.

    antialiasing: the scene was trained with 3DGS's `antialiasing` setting (Mip-Splatting's screen-space filter) and renders
    with it.  A PLY does not record this, so it is the caller's to say (the player's `--scene_antialiasing`)."""
    means3D: torch.Tensor
    scales: torch.Tensor
    rotations: torch.Tensor
    opacities: torch.Tensor
    shs: torch.Tensor
    sh_degree: int
    antialiasing: bool = False

    def __len__(self) -> int:
        return int(self.means3D.shape[0])

    def to(self, device) -> "GaussianScene":
        f = lambda t: t.to(device=device, dtype=torch.float32).contiguous()
        return GaussianScene(f(self.means3D), f(self.scales), f(self.rotations), f(self.opacities).reshape(-1), f(self.shs), int(self.sh_degree),
                             bool(self.antialiasing))

    @classmethod
    def load_ply(cls, path, antialiasing: bool = False) -> "GaussianScene":
        """The `point_cloud.ply` of 3DGS's `GaussianModel.save_ply`: binary little-endian, element `vertex` with x y z, f_dc_0..2,
        f_rest_0..K-1 (channel-major: f_rest_{c (M-1) + k}), opacity, scale_0..2, rot_0..3 (w first).  Properties are read by name
        and others (nx ny nz, ...) ignored; K + 3 = 3M fixes the degree.  opacity -> sigmoid, scale -> exp, rot -> normalised."""
        path = os.fspath(path)
        v = _read_ply_vertices(path)
        names = set(v.dtype.names)
        need = ["x", "y", "z", "f_dc_0", "f_dc_1", "f_dc_2", "opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
        missing = [p for p in need if p not in names]
        if missing:
            raise ValueError(f"{path}: missing vertex propert{'y' if len(missing) == 1 else 'ies'} {', '.join(missing)}")
        rest = sorted(int(m.group(1)) for p in names if (m := re.fullmatch(r"f_rest_(\d+)", p)))
        if rest != list(range(len(rest))):
            raise ValueError(f"{path}: f_rest properties are not numbered 0..{len(rest) - 1}")
        if len(rest) not in SH_DEGREE_OF_REST:
            raise ValueError(f"{path}: {len(rest)} f_rest properties fit no SH degree (0, 9, 24 or 45 for degrees 0..3)")
        D = SH_DEGREE_OF_REST[len(rest)]
        M = (D + 1) ** 2
        col = lambda *ps: np.stack([np.asarray(v[p], np.float64) for p in ps], 1)
        P = len(v)
        shs = np.zeros((P, M, 3), np.float64)
        shs[:, 0, :] = col("f_dc_0", "f_dc_1", "f_dc_2")
        if M > 1:
            fr = col(*[f"f_rest_{i}" for i in range(len(rest))]).reshape(P, 3, M - 1)     # [P, channel, k]
            shs[:, 1:, :] = fr.transpose(0, 2, 1)
        rot = col("rot_0", "rot_1", "rot_2", "rot_3")
        rot = rot / np.maximum(np.linalg.norm(rot, axis=1, keepdims=True), 1e-12)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32))
        return cls(t(col("x", "y", "z")), t(np.exp(col("scale_0", "scale_1", "scale_2"))), t(rot),
                   t(1.0 / (1.0 + np.exp(-np.asarray(v["opacity"], np.float64)))), t(shs), D, bool(antialiasing))


def _rodrigues(rvec) -> np.ndarray:
    r = np.asarray(rvec, np.float64).reshape(3)
    th = float(np.linalg.norm(r))
    if th < 1e-15:
        return np.eye(3)
    k = r / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * (Kx @ Kx)


@dataclass
class Placement:
    """The avatar's world in the scene: x_scene = scale rotation x_avatar + translation (fp64 on the host)."""
    scale: float = 1.0
    rotation: np.ndarray = field(default_factory=lambda: np.eye(3))
    translation: np.ndarray = field(default_factory=lambda: np.zeros(3))

    def __post_init__(self):
        self.scale = float(self.scale)
        self.rotation = np.asarray(self.rotation, np.float64).reshape(3, 3)
        self.translation = np.asarray(self.translation, np.float64).reshape(3)
        if not self.scale > 0:
            raise ValueError(f"placement scale {self.scale} must be positive")
        if not np.allclose(self.rotation @ self.rotation.T, np.eye(3), atol=1e-6) or np.linalg.det(self.rotation) < 0:
            raise ValueError("placement rotation is not a rotation matrix")
        self._rows = {}

    @classmethod
    def from_axis_angle(cls, scale, axis_angle, translation) -> "Placement":
        return cls(scale, _rodrigues(axis_angle), translation)

    def matrix(self) -> np.ndarray:
        """[3,4] = [s R | t]."""
        return np.concatenate([self.scale * self.rotation, self.translation[:, None]], 1)

    def fold(self, cano2live: torch.Tensor) -> torch.Tensor:
        """[B,J,12] cano2live rows (3x4 per joint) -> [s R | t] composed with each: a 3x4 product per joint on the device."""
        dev = cano2live.device
        if dev not in self._rows:         # built once, outside any graph capture (the player's eager warm-up runs first)
            M = torch.from_numpy(self.matrix()).to(device=dev, dtype=torch.float32)
            self._rows[dev] = (M[:, :3].contiguous(), M[:, 3].contiguous())
        A, t = self._rows[dev]
        B, J = cano2live.shape[0], cano2live.shape[1]
        out = torch.matmul(A, cano2live.reshape(B, J, 3, 4))
        out[..., 3] += t
        return out.reshape(B, J, 12)

    def extrinsic(self, E) -> np.ndarray:
        """A world->camera extrinsic [4,4] of the avatar's world -> the same camera in the scene: R_c' = R_c R^T, C' = s R C + t, so
        a placed point's camera coordinates are s x the unplaced ones (same pixel and 2D covariance, depth x s)."""
        E = np.asarray(E, np.float64)
        Rc, tc = E[:3, :3], E[:3, 3]
        C = -Rc.T @ tc
        Rn = Rc @ self.rotation.T
        Cn = self.scale * self.rotation @ C + self.translation
        out = np.eye(4)
        out[:3, :3] = Rn
        out[:3, 3] = -Rn @ Cn
        return out

    def camera(self, K, E, H: int, W: int) -> Camera:
        return make_camera(K, self.extrinsic(E), H, W)

    def carry(self, cam: Camera) -> Camera:
        """`extrinsic` applied to a `camera.Camera` (its view matrix and centre; the projection is kept)."""
        wvt = cam.world_view_transform.double().cpu()
        proj_t = torch.linalg.solve(wvt, cam.full_proj_transform.double().cpu())          # transposed projection
        wvt_n = torch.from_numpy(self.extrinsic(wvt.T.numpy())).T
        center = torch.from_numpy(self.scale * self.rotation @ cam.camera_center.double().cpu().numpy() + self.translation)
        return Camera(cam.FovX, cam.FovY, cam.height, cam.width, wvt_n.float().contiguous(), (wvt_n @ proj_t).float().contiguous(),
                      center.float().contiguous())


@dataclass
class SceneCamera:
    """One entry of 3DGS's cameras.json: intrinsics K (principal point at the image centre), world->camera extrinsic E."""
    K: np.ndarray
    E: np.ndarray
    width: int
    height: int
    name: str = ""

    def camera(self, H: int | None = None, W: int | None = None) -> Camera:
        """The `camera.Camera` at H x W (default: the entry's size; the intrinsics scale with it)."""
        H, W = int(H or self.height), int(W or self.width)
        K = self.K.copy()
        K[0] *= W / self.width
        K[1] *= H / self.height
        return make_camera(K, self.E, H, W)


def load_scene_cameras(path) -> list[SceneCamera]:
    """3DGS's cameras.json: entries with width, height, position (the camera centre), rotation (3x3 camera->world), fx, fy."""
    path = os.fspath(path)
    with open(path) as f:
        entries = json.load(f)
    if not isinstance(entries, list) or not entries:
        raise ValueError(f"{path}: expected a non-empty JSON list of cameras")
    out = []
    for i, e in enumerate(entries):
        missing = [k for k in ("width", "height", "position", "rotation", "fx", "fy") if k not in e]
        if missing:
            raise ValueError(f"{path}: camera {i} has no {', '.join(missing)}")
        Rcw = np.asarray(e["rotation"], np.float64).reshape(3, 3)
        C = np.asarray(e["position"], np.float64).reshape(3)
        w, h = int(e["width"]), int(e["height"])
        E = np.eye(4)
        E[:3, :3] = Rcw.T
        E[:3, 3] = -Rcw.T @ C
        K = np.array([[float(e["fx"]), 0.0, w / 2.0], [0.0, float(e["fy"]), h / 2.0], [0.0, 0.0, 1.0]])
        out.append(SceneCamera(K, E, w, h, str(e.get("img_name", i))))
    return out


def scene_cameras_path(ply_path) -> str:
    """cameras.json of the 3DGS model folder that holds point_cloud/iteration_*/point_cloud.ply."""
    return os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(ply_path)))), "cameras.json")
