"""Animation player: a trained avatar driven by a motion clip, rendered on the device and streamed out as bytes.

    clip = MotionClip.load("walk.npz", body="smpl")                 # AMASS SMPL+H / SMPL-X .npz, or a smpl_parms.pth (fps=...)
    anim = Animator(model, camera_item(K, E, 1024, 1024), 1024, 1024, chunk=8)
    for first, frames in anim.frames(clip, fps_out=30, align_to=0):   # frames: uint8 [b,H,W,C] in pinned host memory
        sink.write(frames.numpy().tobytes())

Per output frame the clip is sampled at a fractional key index (`ga_motion_sample`: per-joint slerp in fp64, the root and the
translation moved by a rigid alignment), posed, skinned and rasterized, and packed into interleaved bytes (`ga_frame_pack`:
torchvision's save_image quantisation, straight alpha from the rasterizer's final transmittance with `channels=4`).

Stage 1 evaluates the frame-invariant decoder once and replays one CUDA graph per chunk of up to 8 frames
(sample -> cano2live -> LBS -> batched rasterizer -> pack).  The bytes leave through two pinned buffers on a copy stream, so chunk
j+1 renders while the caller consumes chunk j; the rasterizer's overflow status travels with the bytes, and a chunk whose binning
buffer overflowed is re-rendered after the buffer has grown (and the graphs are re-captured) before it is yielded.  Stage 2 runs
eagerly, one frame per forward, with the sampled pose for both the input position map and the skeleton.  The model's parameters
and BatchNorm statistics are left exactly as they were.

With a scene (`scene.GaussianScene`) both stages render through the composite forward instead, which splats the avatar and the
scene in one sort per tile; a `scene.Placement` moves the avatar (and the cameras given around it) into the scene.

Several avatars play together through `Ensemble`, of which `Animator` is the one-actor case:

    cast = [Actor(model_a, walk), Actor(model_b, dance, placement=Placement.from_axis_angle(1, [0, 0, 0], [0.8, 0, 0]))]
    for first, frames, mattes in Ensemble(cast, cameras, 1080, 1920, mattes=True).frames(fps_out=30):   # mattes: uint8 [b,K,H,W]
        ...

Their Gaussians are concatenated into one dynamic set and splatted together (and with the scene), so they occlude each other;
with `mattes` each actor's visible matte comes from the same compositing pass (`rasterizer.rasterize_batch_mattes`).  With
`depth` the same pass also writes each frame's mean and median view depth (`rasterizer.rasterize_batch_depth`):

    for first, frames, mattes, depth in Ensemble(cast, cameras, 1080, 1920, depth=True).frames(fps_out=30):  # depth: fp32 [b,2,H,W]
        ...
"""
from __future__ import annotations

import contextlib
import math
import os
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from ._lib import ptr
from .avatar_model import kept_state
from .body import body_of
from .camera import Camera, make_camera
from .dataset import _rodrigues, rotate_camera_by_frame_idx
from .rasterizer import (MAX_FRAMES_PER_CALL, MAX_SETS, RasterBatchPlan, rasterize_batch, rasterize_batch_depth, rasterize_batch_mattes,
                         rasterize_batch_scene)
from .scene import SceneCamera

SCENE_CHUNK = 2                 # the player's default chunk with a scene
IDENTITY_ALIGN = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], np.float64)


# ---- C ABI wrappers ---------------------------------------------------------------------------------------------------------------
def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def motion_sample(key_pose, key_trans, times, align, pose_out=None, trans_out=None):
    """ga_motion_sample on the current stream: key_pose [T,J*3], key_trans [T,3] fp32, times [n] and align [12] fp64, all on the
    device -> (pose [n,J*3], trans [n,3]) fp32."""
    T, width = int(key_pose.shape[0]), int(key_pose.shape[1])
    n = int(times.shape[0])
    dev = key_pose.device
    if pose_out is None:
        pose_out = torch.empty(n, width, dtype=torch.float32, device=dev)
    if trans_out is None:
        trans_out = torch.empty(n, 3, dtype=torch.float32, device=dev)
    _lib.check(_lib.lib().ga_motion_sample(T, width // 3, ptr(key_pose), ptr(key_trans), n, ptr(times), ptr(align), ptr(pose_out),
                                           ptr(trans_out), _stream()), "ga_motion_sample")
    return pose_out, trans_out


def frame_pack(images, final_T=None, bg=None, channels=3, out=None):
    """ga_frame_pack on the current stream: images [B,3,H,W] fp32 (+ final_T [B,H,W] and bg [3] for channels=4) -> uint8 [B,H,W,C]."""
    B, _, H, W = map(int, images.shape)
    if out is None:
        out = torch.empty(B, H, W, channels, dtype=torch.uint8, device=images.device)
    _lib.check(_lib.lib().ga_frame_pack(B, H, W, int(channels), ptr(images), ptr(final_T), ptr(bg), ptr(out), _stream()), "ga_frame_pack")
    return out


def matte_pack(mattes, out=None):
    """ga_matte_pack on the current stream: mattes [B,K,H,W] fp32 -> uint8 [B,K,H,W] (ga_frame_pack's quantisation)."""
    if out is None:
        out = torch.empty(mattes.shape, dtype=torch.uint8, device=mattes.device)
    _lib.check(_lib.lib().ga_matte_pack(mattes.numel(), ptr(mattes), ptr(out), _stream()), "ga_matte_pack")
    return out


def final_transmittance(plan) -> torch.Tensor:
    """[B,H,W] view of a RasterBatchPlan's final transmittance (the rasterizer's image buffer; the address comes from ga_raster_views,
    nothing is read on the host)."""
    v = _lib.GaRasterViews()
    _lib.check(_lib.lib().ga_raster_views(plan.B, plan.P, plan.H, plan.W, plan.capacity, None, None, ptr(plan.img), v), "ga_raster_views")
    off = int(v.final_T) - plan.img.data_ptr()
    n = plan.B * plan.H * plan.W
    return plan.img[off:off + 4 * n].view(torch.float32).view(plan.B, plan.H, plan.W)


# ---- clips, time and alignment --------------------------------------------------------------------------------------------------
@dataclass
class MotionClip:
    """pose [T,72] (SMPL) or [T,165] (SMPL-X: global + 21 body joints | jaw, eyes | 2 x 15 finger joints), trans [T,3], fp32 on the
    host, and the clip's frame rate."""
    pose: torch.Tensor
    trans: torch.Tensor
    fps: float
    body: str

    @property
    def num_keys(self) -> int:
        return int(self.pose.shape[0])

    @classmethod
    def load(cls, path, body: str, fps: float | None = None) -> "MotionClip":
        """A reference `smpl_parms.pth` (`body_pose` [T,72|165] and `trans`; fps must be given), an AMASS SMPL+H `.npz` (`poses`
        [T,156], `trans`, `mocap_framerate`) or an AMASS SMPL-X `.npz` (`poses` [T,165], `trans`, `mocap_frame_rate` or
        `mocap_framerate`).  `fps` overrides a file's rate.  The clip's betas are ignored: only rotations and translations transfer."""
        width = body_of(body).full_width
        path = os.fspath(path)
        if path.endswith(".npz"):
            with np.load(path, allow_pickle=False) as z:
                d = {k: z[k] for k in z.files}
            for key in ("poses", "trans"):
                if key not in d:
                    raise ValueError(f"{path}: no '{key}' array (an AMASS clip has 'poses', 'trans' and its frame rate)")
            poses = np.asarray(d["poses"], np.float64)
            if poses.ndim != 2 or poses.shape[1] not in (156, 165):
                raise ValueError(f"{path}: 'poses' {poses.shape}; expected [T,156] (SMPL+H) or [T,165] (SMPL-X)")
            rate_keys = ("mocap_framerate",) if poses.shape[1] == 156 else ("mocap_frame_rate", "mocap_framerate")
            if fps is None:
                rate = next((d[k] for k in rate_keys if k in d), None)
                if rate is None:
                    raise ValueError(f"{path}: no frame rate ({' or '.join(rate_keys)}); pass fps")
                fps = float(rate)
            pose = amass_pose(poses, body)
            trans = np.asarray(d["trans"], np.float64)
        else:
            if fps is None:
                raise ValueError(f"{path}: a smpl_parms.pth carries no frame rate; pass fps")
            d = torch.load(path, map_location="cpu", weights_only=False)
            for key in ("body_pose", "trans"):
                if key not in d:
                    raise ValueError(f"{path}: no '{key}' entry")
            pose = np.asarray(torch.as_tensor(d["body_pose"]).double().numpy())
            if pose.ndim != 2 or pose.shape[1] != width:
                raise ValueError(f"{path}: 'body_pose' {pose.shape}; expected [T,{width}] for body={body!r}")
            trans = np.asarray(torch.as_tensor(d["trans"]).double().numpy())
        if pose.shape[0] < 1 or trans.shape != (pose.shape[0], 3):
            raise ValueError(f"{path}: 'trans' {trans.shape}; expected [{pose.shape[0]},3] (one row per pose, at least one)")
        fps = float(fps)
        if not fps > 0 or not math.isfinite(fps):
            raise ValueError(f"{path}: frame rate {fps} is not positive")
        return cls(torch.from_numpy(pose.astype(np.float32)), torch.from_numpy(trans.astype(np.float32)), fps, body)


def amass_pose(poses: np.ndarray, body: str) -> np.ndarray:
    """AMASS `poses` [T,156] (SMPL+H: global, 21 body joints, 2 x 15 hand joints) or [T,165] (SMPL-X) -> [T,72] or [T,165].
    SMPL keeps the first 22 joints and zeros joints 22 / 23 (SMPL's hands); SMPL-X from SMPL+H zeros the jaw and eyes and takes the
    hands as they are (flat_hand_mean=True)."""
    T = poses.shape[0]
    if body == "smpl":
        return np.concatenate([poses[:, :66], np.zeros((T, 6))], 1)
    if poses.shape[1] == 165:
        return poses
    return np.concatenate([poses[:, :66], np.zeros((T, 9)), poses[:, 66:156]], 1)


def sample_times(num_keys: int, fps_clip: float, fps_out: float, speed: float = 1.0) -> np.ndarray:
    """Fractional key indices tau_k = k speed fps_clip / fps_out (fp64) for k < floor((T-1) fps_out / (speed fps_clip)) + 1."""
    if not (fps_out > 0 and speed > 0 and fps_clip > 0):
        raise ValueError(f"fps_out {fps_out}, speed {speed} and the clip's rate {fps_clip} must be positive")
    step = float(speed) * float(fps_clip) / float(fps_out)
    n = int(math.floor((num_keys - 1) / step)) + 1
    return np.arange(n, dtype=np.float64) * step


def alignment(root0, trans0, target_root, target_trans) -> np.ndarray:
    """align [12] (row-major R_a, then c) mapping clip frame 0 (root axis-angle, translation) exactly onto a target frame:
    R_a = R_k R_c0^T, c = t_k - R_a t_c0 (fp64).  The pelvis rest joint cancels out, so any up-axis convention works."""
    Rc = _rodrigues(np.asarray(root0, np.float64).reshape(3))
    Rk = _rodrigues(np.asarray(target_root, np.float64).reshape(3))
    Ra = Rk @ Rc.T
    c = np.asarray(target_trans, np.float64).reshape(3) - Ra @ np.asarray(trans0, np.float64).reshape(3)
    return np.concatenate([Ra.reshape(9), c])


@dataclass
class OrbitCamera:
    """The free-view orbit of `dataset.rotate_camera_by_frame_idx` (intrinsics K, extrinsic of frame 0) around the aligned clip's
    frame-0 pelvis, one turn over the clip."""
    K: np.ndarray
    extrinsic: np.ndarray
    rotate_axis: str = "y"
    inv_angle: bool = False


@dataclass
class Schedule:
    times: np.ndarray        # [n] fractional key indices (fp64)
    align: np.ndarray        # [12] R_a (row-major), c (fp64)
    cams: torch.Tensor       # [n,40] camera block (host fp32)




def cast_times(num_keys, fps_clip, speeds, fps_out: float) -> np.ndarray:
    """Fractional key indices [K, n] of K clips played together: actor k samples tau = min(j speed_k fps_k / fps_out, T_k - 1), so a
    shorter clip holds its last pose, and the playback lasts as long as the longest (n = the most `sample_times` frames)."""
    steps = [float(v) * float(f) / float(fps_out) for v, f in zip(speeds, fps_clip)]
    n = max(len(sample_times(T, f, fps_out, v)) for T, f, v in zip(num_keys, fps_clip, speeds))
    j = np.arange(n, dtype=np.float64)
    return np.stack([np.minimum(j * st, float(T - 1)) for T, st in zip(num_keys, steps)])


@dataclass
class Actor:
    """One avatar of an `Ensemble`: an inference `AvatarModel` (stage 1 or 2) driven by `clip` (of the model's body) at `speed`,
    clip frame 0 mapped onto training frame `align_to` (None: the clip as it is), and `placement` (a `scene.Placement`, None =
    identity) mapping the avatar's world into the shared one.  pose_mapper: stage 2's position mapper (default: the model's own)."""
    model: object
    clip: MotionClip | None
    placement: object = None
    align_to: int | None = None
    speed: float = 1.0
    pose_mapper: object = None


# ---- the player -------------------------------------------------------------------------------------------------------------------
class Ensemble:
    """Renders up to 8 actors (`Actor`) together, each along its own clip, splatted in one sort per tile so that each hides the
    others (and the scene) where it is in front.

    cameras: a `dataset.camera_item` dict (one camera for every frame), an `OrbitCamera` (around actor 0's aligned frame-0 pelvis),
    or with a scene a `scene.SceneCamera` (in the scene's world, used as it is).  Dict and orbit cameras are given in actor 0's world
    and carried through actor 0's placement, so the shared world is the scene's with a scene and otherwise actor 0's.  H, W: frame
    size.  chunk: frames per rasterizer call (1..8; default 8, with a scene SCENE_CHUNK).  channels: 3 (RGB) or 4 (straight-alpha
    RGBA, alpha = 1 - final transmittance over everything splatted).  mattes: also return each actor's visibility matte, the weight
    its Gaussians added to each pixel (`rasterize_batch_mattes`), as bytes.  capacity: initial binning capacity of the rasterizer
    (instances); it grows on overflow.  graphs: replay CUDA graphs when every actor is in stage 1 (False runs the same launches
    eagerly).  scene: a `scene.GaussianScene` the actors are rendered in.  depth: also return each frame's depth pass, fp32
    [b,2,H,W] (`rasterize_batch_depth`: plane 0 the mean, plane 1 the median view depth in the shared world's units, 0 where there
    is no surface), from the same compositing launch; it leaves through two pinned slots of 8 x 2 x H x W floats each, about 265 MB
    of pinned host memory at 1920 x 1080 (and as much on the device).

    With every actor in stage 1 each distinct model's decoder is evaluated once and one CUDA graph per (chunk size, output slot)
    replays sample -> cano2live -> LBS per actor, their concatenation, the rasterizer and the packing.  Any stage-2 actor makes the
    player render eagerly, one frame per rasterizer call.  Every model's parameters and BatchNorm statistics are left as they were."""

    def __init__(self, actors, cameras, H: int, W: int, chunk: int | None = None, channels: int = 3, mattes: bool = False,
                 capacity=None, graphs: bool = True, scene=None, depth: bool = False):
        self.actors = list(actors)
        if not 1 <= len(self.actors) <= MAX_SETS:
            raise ValueError(f"{len(self.actors)} actors: 1..{MAX_SETS}")
        self.H, self.W = int(H), int(W)
        if not (1 <= self.H <= 16384 and 1 <= self.W <= 16384):
            raise ValueError(f"frame {self.H} x {self.W} outside [1, 16384]^2")
        if chunk is None:        # with a scene, chunks beyond 2 frames render no faster (DESIGN.md §7) and need far more memory
            chunk = MAX_FRAMES_PER_CALL if scene is None else SCENE_CHUNK
        if not 1 <= int(chunk) <= MAX_FRAMES_PER_CALL:
            raise ValueError(f"chunk {chunk} outside 1..{MAX_FRAMES_PER_CALL}")
        if int(channels) not in (3, 4):
            raise ValueError(f"channels {channels}: 3 (RGB) or 4 (RGBA)")
        self.chunk, self.channels = int(chunk), int(channels)
        if isinstance(cameras, dict):
            h, w = int(cameras.get("height", self.H)), int(cameras.get("width", self.W))
            if (h, w) != (self.H, self.W):
                raise ValueError(f"the camera was built for {w} x {h}, the frames are {self.W} x {self.H}")
        elif isinstance(cameras, SceneCamera):
            if scene is None:
                raise ValueError("a scene camera (cameras.json) needs the scene")
        elif not isinstance(cameras, OrbitCamera):
            raise TypeError("cameras: a camera_item dict, an OrbitCamera or a scene.SceneCamera")
        self.cameras = cameras
        m0 = self.actors[0].model
        self.dev = m0.device
        self._stages, self._mappers = [], []
        for k, a in enumerate(self.actors):
            if a.clip is not None:
                self._check_clip(a.model, a.clip, k)
            if not torch.equal(a.model.background.to(self.dev), m0.background):
                raise ValueError(f"actor {k}'s background {a.model.background.tolist()} differs from actor 0's {m0.background.tolist()}")
            if getattr(a.model, "antialiasing", False) != getattr(m0, "antialiasing", False):
                raise ValueError(f"actor {k} renders with antialiasing={getattr(a.model, 'antialiasing', False)}, actor 0 with "
                                 f"antialiasing={getattr(m0, 'antialiasing', False)}: the actors of a cast must share the mode")
            stage = 2 if int(a.model.model_parms.train_stage) == 2 else 1
            mapper = a.pose_mapper if a.pose_mapper is not None else getattr(a.model, "pose_mapper", None)
            if stage == 2 and mapper is None:
                raise ValueError("stage 2 needs a pose_mapper (posmap.PoseMapper / SmplxPoseMapper) for the input position maps")
            self._stages.append(stage)
            self._mappers.append(mapper)
        self._models = list({id(a.model): a.model for a in self.actors}.values())
        sizes = [int(a.model._query_points.shape[0]) for a in self.actors]
        self.first = [0] + np.cumsum(sizes).tolist()          # actor k's Gaussians in the concatenated dynamic set
        self.antialiasing = bool(getattr(m0, "antialiasing", False))    # the actors' (shared) mode; a scene's is its own
        one = len(self.actors) == 1                             # rotations / opacities shared by every frame, concatenated
        self._rot = m0.fix_rotation if one else torch.cat([a.model.fix_rotation for a in self.actors])
        self._opac = m0.fix_opacity if one else torch.cat([a.model.fix_opacity for a in self.actors])
        self.mattes, self.depth = bool(mattes), bool(depth)
        self.scene = None if scene is None else scene.to(self.dev)
        self.capacity = capacity
        self.use_graphs = bool(graphs)
        self.captures = 0          # CUDA graphs captured
        self.recaptures = 0        # ... of them because a chunk overflowed the binning buffer
        self.overflows = 0         # chunks rendered again after an overflow
        self._plans, self._graphs, self._clip_key = {}, {}, None
        C, K, dev = self.channels, len(self.actors), self.dev
        self._out_dev = [torch.empty(MAX_FRAMES_PER_CALL, self.H, self.W, C, dtype=torch.uint8, device=dev) for _ in range(2)]
        self._out_host = [torch.empty(MAX_FRAMES_PER_CALL, self.H, self.W, C, dtype=torch.uint8).pin_memory() for _ in range(2)]
        if self.mattes:
            self._mattes_dev = [torch.empty(MAX_FRAMES_PER_CALL, K, self.H, self.W, dtype=torch.uint8, device=dev) for _ in range(2)]
            self._mattes_host = [torch.empty(MAX_FRAMES_PER_CALL, K, self.H, self.W, dtype=torch.uint8).pin_memory() for _ in range(2)]
        if self.depth:
            self._depth_dev = [torch.empty(MAX_FRAMES_PER_CALL, 2, self.H, self.W, dtype=torch.float32, device=dev) for _ in range(2)]
            self._depth_host = [torch.empty(MAX_FRAMES_PER_CALL, 2, self.H, self.W, dtype=torch.float32).pin_memory() for _ in range(2)]
        self._status_dev = [torch.zeros(16, dtype=torch.int32, device=dev) for _ in range(2)]      # eager rendering leaves them at 0
        self._status_host = [torch.zeros(16, dtype=torch.int32).pin_memory() for _ in range(2)]
        self._keys_pose, self._keys_trans = [None] * K, [None] * K
        self._align = [torch.zeros(12, dtype=torch.float64, device=dev) for _ in range(K)]
        self._times_dev = [torch.zeros(MAX_FRAMES_PER_CALL, dtype=torch.float64, device=dev) for _ in range(K)]
        self._cams_dev = torch.zeros(MAX_FRAMES_PER_CALL, 40, dtype=torch.float32, device=dev)
        self._copy_stream = torch.cuda.Stream(device=dev)
        self._rendered = [torch.cuda.Event() for _ in range(2)]
        self._copied = [torch.cuda.Event() for _ in range(2)]
        self._slot_used = [False, False]

    # ---- host-side schedule ------------------------------------------------------------------------------------------------------
    @staticmethod
    def _check_clip(model, clip, k=0):
        if clip.body != model.body.name or clip.pose.shape[1] != model.body.full_width:
            who = "the avatar" if k == 0 else f"actor {k}'s avatar"
            raise ValueError(f"clip for body {clip.body!r} ({tuple(clip.pose.shape)}), {who} is {model.body.name!r}")

    @staticmethod
    def _alignment(model, clip, align_to):
        if align_to is None:
            return IDENTITY_ALIGN.copy()
        k = int(align_to)
        F = int(model.pose.weight.shape[0])
        if not 0 <= k < F:
            raise ValueError(f"align_to {k}: the model has training frames 0..{F - 1}")
        return alignment(clip.pose[0, :3].double().numpy(), clip.trans[0].double().numpy(),
                         model.pose.weight[k, :3].detach().double().cpu().numpy(), model.transl.weight[k].detach().double().cpu().numpy())

    def _camera_rows(self, n, clip, align):
        """[n,40] camera rows (host fp32): dict and orbit cameras from actor 0 (its clip, alignment and placement)."""
        from .mesh_render import cameras as camera_block
        cam, a0 = self.cameras, self.actors[0]
        place = (lambda c: c) if a0.placement is None else a0.placement.carry
        if isinstance(cam, SceneCamera):                  # already in the scene's world
            return camera_block([cam.camera(self.H, self.W)]).expand(n, -1).contiguous()
        if isinstance(cam, dict):
            one = Camera(float(cam["FovX"]), float(cam["FovY"]), self.H, self.W, torch.as_tensor(cam["world_view_transform"]),
                         torch.as_tensor(cam["full_proj_transform"]), torch.as_tensor(cam["camera_center"]))
            return camera_block([place(one)]).expand(n, -1).contiguous()
        R, c = align[:9].reshape(3, 3), align[9:]
        t0 = R @ clip.trans[0].double().numpy() + c
        pelvis = a0.model._rest_joints[0].double().cpu().numpy() + t0        # the root rotates about the rest pelvis
        rows = [place(make_camera(cam.K, rotate_camera_by_frame_idx(cam.extrinsic, k, trans=pelvis, rotate_axis=cam.rotate_axis, period=n,
                                                                   inv_angle=cam.inv_angle), self.H, self.W)) for k in range(n)]
        return camera_block(rows)

    def _playback(self, fps_out):
        """Per-actor times [K,n] and alignments [K][12], and the camera rows [n,40] of a playback."""
        for k, a in enumerate(self.actors):
            if a.clip is None:
                raise ValueError(f"actor {k} has no clip")
            self._check_clip(a.model, a.clip, k)
        times = cast_times([a.clip.num_keys for a in self.actors], [a.clip.fps for a in self.actors], [a.speed for a in self.actors],
                           fps_out)
        aligns = [self._alignment(a.model, a.clip, a.align_to) for a in self.actors]
        return times, aligns, self._camera_rows(times.shape[1], self.actors[0].clip, aligns[0])

    def _kept(self):
        stack = contextlib.ExitStack()
        for m in self._models:
            stack.enter_context(kept_state(m))
        return stack

    # ---- playback ---------------------------------------------------------------------------------------------------------------
    def frames(self, fps_out: float):
        """Yields (index of the chunk's first frame, uint8 [b,H,W,C], uint8 [b,K,H,W] mattes or None) in order, and with depth a
        fourth item, the fp32 [b,2,H,W] depth pass.  The arrays live in two pinned buffers and are overwritten two chunks later: copy
        them to keep them."""
        times, aligns, cams = self._playback(fps_out)
        n = times.shape[1]
        starts = list(range(0, n, self.chunk))
        with torch.no_grad(), self._kept():
            setup = self._stage1_setup if all(s == 1 for s in self._stages) else self._eager_setup
            render = setup(times, aligns, cams)
        self._enqueue(render, starts[0], min(n, starts[0] + self.chunk), 0)
        for j, s in enumerate(starts):
            e = min(n, s + self.chunk)
            if j + 1 < len(starts):
                self._enqueue(render, starts[j + 1], min(n, starts[j + 1] + self.chunk), (j + 1) % 2)
            slot = j % 2
            self._copied[slot].synchronize()
            tries = 0
            while int(self._status_host[slot][1]) != 0:          # the binning buffer overflowed: grow it, render the chunk again
                tries += 1
                if tries > 3:
                    raise RuntimeError("animation: the rasterizer's binning buffer overflowed again after growing")
                self.overflows += 1
                self._grow(e - s, int(self._status_host[slot][0]))
                self._enqueue(render, s, e, slot)
                self._copied[slot].synchronize()
            out = (s, self._out_host[slot][:e - s], self._mattes_host[slot][:e - s] if self.mattes else None)
            yield out + (self._depth_host[slot][:e - s],) if self.depth else out
        torch.cuda.current_stream().wait_stream(self._copy_stream)

    def _enqueue(self, render, s, e, slot):
        """Renders frames s..e-1 into the slot's device buffers and copies them, with the overflow status, to its pinned buffers."""
        main = torch.cuda.current_stream()
        if self._slot_used[slot]:
            main.wait_event(self._copied[slot])          # the previous copy out of this slot has finished reading it
        with torch.no_grad(), self._kept():
            render(s, e, slot)
        self._rendered[slot].record(main)
        self._slot_used[slot] = True
        with torch.cuda.stream(self._copy_stream):
            self._copy_stream.wait_event(self._rendered[slot])
            self._out_host[slot][:e - s].copy_(self._out_dev[slot][:e - s], non_blocking=True)
            if self.mattes:
                self._mattes_host[slot][:e - s].copy_(self._mattes_dev[slot][:e - s], non_blocking=True)
            if self.depth:
                self._depth_host[slot][:e - s].copy_(self._depth_dev[slot][:e - s], non_blocking=True)
            self._status_host[slot].copy_(self._status_dev[slot], non_blocking=True)
            self._copied[slot].record(self._copy_stream)

    def _plan(self, b):
        if b not in self._plans:
            self._plans[b] = RasterBatchPlan(b, self.first[-1], self.H, self.W, self.dev, capacity=self.capacity,
                                             static_P=0 if self.scene is None else len(self.scene), antialiasing=self.antialiasing)
        return self._plans[b]

    def _render(self, parts, cams, plan):
        """Concatenates the actors' (means, scales, colours) and rasterizes them: (images, mattes or None, depth or None)."""
        means, scales, colors = parts[0] if len(parts) == 1 else [torch.cat(t, 1) for t in zip(*parts)]
        bg = self.actors[0].model.background
        mattes = depth = None
        if self.depth:
            out = rasterize_batch_depth(means, colors, scales, self._rot, self._opac, cams, bg, plan, self.scene,
                                        self.first if self.mattes else None)
            img, depth = out[0], out[-1]
            mattes = out[1] if self.mattes else None
        elif self.mattes:
            img, mattes = rasterize_batch_mattes(means, colors, scales, self._rot, self._opac, cams, bg, plan, self.first, self.scene)
        elif self.scene is None:
            img = rasterize_batch(means, colors, scales, self._rot, self._opac, cams, bg, plan)
        else:
            img = rasterize_batch_scene(means, colors, scales, self._rot, self._opac, cams, bg, plan, self.scene)
        return img, mattes, depth

    def _pack(self, img, mattes, depth, plan, slot, lo, hi):
        """Packs images (and mattes) into frames lo..hi-1 of the slot's device buffers, and copies depth there."""
        frame_pack(img, final_transmittance(plan), self.actors[0].model.background, self.channels, self._out_dev[slot][lo:hi])
        if mattes is not None:
            matte_pack(mattes, self._mattes_dev[slot][lo:hi])
        if depth is not None:
            self._depth_dev[slot][lo:hi].copy_(depth)

    def _grow(self, b, needed):
        if self._graphs:
            torch.cuda.current_stream().synchronize()     # no replay still reads the buffers about to go
        self._plan(b).grow(needed)
        for key in [k for k in self._graphs if k[0] == b]:       # the graphs hold the old binning buffer's address
            del self._graphs[key]
            self.recaptures += 1

    # ---- every actor in stage 1: one graph per (chunk size, slot) ----------------------------------------------------------------
    def _stage1_setup(self, times, aligns, cams):
        decs = {}
        for m in self._models:
            decs[id(m)] = m._stage1_decoder(1)
        key = []
        for k, a in enumerate(self.actors):
            T, width = a.clip.num_keys, int(a.clip.pose.shape[1])
            if self._keys_pose[k] is None or self._keys_pose[k].shape[0] < T or self._keys_pose[k].shape[1] != width:
                self._keys_pose[k] = torch.empty(T, width, dtype=torch.float32, device=self.dev)
                self._keys_trans[k] = torch.empty(T, 3, dtype=torch.float32, device=self.dev)
                self._graphs = {}
            self._keys_pose[k][:T].copy_(a.clip.pose)
            self._keys_trans[k][:T].copy_(a.clip.trans)
            self._align[k].copy_(torch.from_numpy(aligns[k]))
            key.append((T, decs[id(a.model)].data_ptr()))
        # the graphs take each clip's key count as a kernel argument and the decoder outputs by address
        if key != self._clip_key:
            self._graphs, self._clip_key = {}, key
        times_all = torch.from_numpy(times).to(self.dev)
        cams_all = cams.to(self.dev)

        def body(b, slot):
            plan = self._plan(b)
            parts = []
            for k, a in enumerate(self.actors):
                T = a.clip.num_keys
                pose, trans = motion_sample(self._keys_pose[k][:T], self._keys_trans[k][:T], self._times_dev[k][:b], self._align[k])
                pose, rest = a.model.body.split(pose)
                parts.append(a.model._assemble(decs[id(a.model)], pose, trans, rest, placement=a.placement))
            self._pack(*self._render(parts, self._cams_dev[:b], plan), plan, slot, 0, b)
            self._status_dev[slot].copy_(plan.status_dev)

        def render(s, e, slot):
            b = e - s
            for k in range(len(self.actors)):
                self._times_dev[k][:b].copy_(times_all[k, s:e])
            self._cams_dev[:b].copy_(cams_all[s:e])
            if not self.use_graphs:
                body(b, slot)
                return
            g = self._graphs.get((b, slot))
            if g is None:
                body(b, slot)                           # eager warm-up: allocations and one-time attributes outside the capture
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    body(b, slot)
                self._graphs[(b, slot)] = g
                self.captures += 1
            g.replay()
        return render

    # ---- any actor in stage 2: eager, one frame per forward -----------------------------------------------------------------------
    def _eager_setup(self, times, aligns, cams):
        sampled, decs = [], {}
        for k, a in enumerate(self.actors):
            sampled.append(motion_sample(a.clip.pose.to(self.dev).contiguous(), a.clip.trans.to(self.dev).contiguous(),
                                         torch.from_numpy(times[k]).to(self.dev), torch.from_numpy(aligns[k]).to(self.dev)))
            if self._stages[k] == 1 and id(a.model) not in decs:
                decs[id(a.model)] = a.model._stage1_decoder(1)
        cams_all = cams.to(self.dev)

        def render(s, e, slot):
            for i in range(s, e):
                parts = []
                for k, a in enumerate(self.actors):
                    m = a.model
                    p, rest = m.body.split(sampled[k][0][i:i + 1])
                    t = sampled[k][1][i:i + 1]
                    if self._stages[k] == 2:
                        parts.append(m._stage2_from_pose(self._mappers[k], p, t, rest, placement=a.placement)[:3])
                    else:
                        parts.append(m._assemble(decs[id(m)], p, t, rest, placement=a.placement))
                plan = self._plan(1)       # as _render_batched: a frame whose binning buffer overflowed is rendered again after it grew
                out, again = plan.render_checked(lambda: self._render(parts, cams_all[i:i + 1], plan), "animation")
                self.overflows += int(again)
                self._pack(*out, plan, slot, i - s, i - s + 1)
        return render


class Animator(Ensemble):
    """Renders one inference `AvatarModel` (stage 1 or 2) along motion clips: the one-actor `Ensemble`.

    cameras, H, W, chunk, channels, capacity, graphs, scene and depth as for `Ensemble`; pose_mapper: stage 2's `posmap.PoseMapper` /
    `SmplxPoseMapper` (default: the model's own).  scene: a `scene.GaussianScene` the avatar is rendered in, splatted together
    with it (`rasterize_batch_scene`) so that either hides the other; placement: the `scene.Placement` of the avatar's world in
    it.  The cameras are given in the avatar's world and carried into the scene through the placement; alpha (channels=4) is
    1 - final transmittance over both sets."""

    def __init__(self, model, cameras, H: int, W: int, chunk: int | None = None, channels: int = 3, pose_mapper=None,
                 capacity=None, graphs: bool = True, scene=None, placement=None, depth: bool = False):
        super().__init__([Actor(model, None, placement, pose_mapper=pose_mapper)], cameras, H, W, chunk=chunk, channels=channels,
                         capacity=capacity, graphs=graphs, scene=scene, depth=depth)
        self.model, self.body, self.placement = model, model.body, placement
        self.stage, self.pose_mapper = self._stages[0], self._mappers[0]

    def schedule(self, clip: MotionClip, fps_out: float, speed: float = 1.0, align_to=None) -> Schedule:
        """Sample times, alignment and camera rows of a playback (all built on the host in fp64, cameras narrowed to fp32)."""
        self._cast(clip, speed, align_to)
        times, aligns, cams = self._playback(fps_out)
        return Schedule(times[0], aligns[0], cams)

    @torch.no_grad()
    def sample(self, clip: MotionClip, sched: Schedule):
        """All sampled poses [n,72|165] and translations [n,3] of a playback, on the device."""
        keys_p, keys_t = clip.pose.to(self.dev).contiguous(), clip.trans.to(self.dev).contiguous()
        times = torch.from_numpy(sched.times).to(self.dev)
        align = torch.from_numpy(sched.align).to(self.dev)
        return motion_sample(keys_p, keys_t, times, align)

    def frames(self, clip: MotionClip, fps_out: float, speed: float = 1.0, align_to=None):
        """Yields (index of the chunk's first frame, uint8 [b,H,W,C]) in order, with depth (..., fp32 [b,2,H,W] depth).  The arrays
        live in two pinned buffers and are overwritten two chunks later: copy them to keep them."""
        self._cast(clip, speed, align_to)
        for s, frames, _, *depth in super().frames(fps_out):
            yield (s, frames, *depth)

    def _cast(self, clip, speed, align_to):
        self.actors[0] = Actor(self.model, clip, self.placement, align_to, speed, self.actors[0].pose_mapper)
        self._check_clip(self.model, clip)
