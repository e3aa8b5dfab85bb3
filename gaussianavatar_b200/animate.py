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
"""
from __future__ import annotations

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
from .rasterizer import MAX_FRAMES_PER_CALL, RasterBatchPlan, rasterize_batch, rasterize_batch_scene
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


# ---- the player -------------------------------------------------------------------------------------------------------------------
class Animator:
    """Renders an inference `AvatarModel` (stage 1 or 2) along motion clips.

    cameras: a `dataset.camera_item` dict (one camera for every frame), an `OrbitCamera`, or with a scene a `scene.SceneCamera` (one of
    the scene's own cameras, in the scene's world).  H, W: frame size.  chunk: frames per
    rasterizer call (1..8; default 8, with a scene SCENE_CHUNK).  channels: 3 (RGB) or 4 (straight-alpha RGBA).  pose_mapper: stage 2's `posmap.PoseMapper` /
    `SmplxPoseMapper` (default: the model's own).  capacity: initial binning capacity of the rasterizer (instances); it grows on
    overflow.  graphs: replay CUDA graphs in stage 1 (False runs the same launches eagerly, e.g. for per-kernel profiling).
    scene: a `scene.GaussianScene` the avatar is rendered in, splatted together with it (`rasterize_batch_scene`) so that either
    hides the other; placement: the `scene.Placement` of the avatar's world in it.  The cameras are given in the avatar's world
    and carried into the scene through the placement; alpha (channels=4) is 1 - final transmittance over both sets."""

    def __init__(self, model, cameras, H: int, W: int, chunk: int | None = None, channels: int = 3, pose_mapper=None,
                 capacity=None, graphs: bool = True, scene=None, placement=None):
        self.model = model
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
        self.stage = 2 if int(model.model_parms.train_stage) == 2 else 1
        self.body = model.body
        self.pose_mapper = pose_mapper if pose_mapper is not None else getattr(model, "pose_mapper", None)
        if self.stage == 2 and self.pose_mapper is None:
            raise ValueError("stage 2 needs a pose_mapper (posmap.PoseMapper / SmplxPoseMapper) for the input position maps")
        self.dev = model.device
        self.scene = None if scene is None else scene.to(self.dev)
        self.placement = placement
        self.capacity = capacity
        self.use_graphs = bool(graphs)
        self.captures = 0          # CUDA graphs captured
        self.recaptures = 0        # ... of them because a chunk overflowed the binning buffer
        self.overflows = 0         # chunks rendered again after an overflow
        self._plans, self._graphs, self._clip_key = {}, {}, None
        C, dev = self.channels, self.dev
        self._out_dev = [torch.empty(MAX_FRAMES_PER_CALL, self.H, self.W, C, dtype=torch.uint8, device=dev) for _ in range(2)]
        self._out_host = [torch.empty(MAX_FRAMES_PER_CALL, self.H, self.W, C, dtype=torch.uint8).pin_memory() for _ in range(2)]
        self._status_dev = [torch.zeros(16, dtype=torch.int32, device=dev) for _ in range(2)]      # stage 2 leaves them at 0
        self._status_host = [torch.zeros(16, dtype=torch.int32).pin_memory() for _ in range(2)]
        self._keys_pose = self._keys_trans = self._dec = None
        self._align = torch.zeros(12, dtype=torch.float64, device=dev)
        self._times_dev = torch.zeros(MAX_FRAMES_PER_CALL, dtype=torch.float64, device=dev)
        self._cams_dev = torch.zeros(MAX_FRAMES_PER_CALL, 40, dtype=torch.float32, device=dev)
        self._copy_stream = torch.cuda.Stream(device=dev)
        self._rendered = [torch.cuda.Event() for _ in range(2)]
        self._copied = [torch.cuda.Event() for _ in range(2)]
        self._slot_used = [False, False]

    # ---- host-side schedule ------------------------------------------------------------------------------------------------------
    def schedule(self, clip: MotionClip, fps_out: float, speed: float = 1.0, align_to=None) -> Schedule:
        """Sample times, alignment and camera rows of a playback (all built on the host in fp64, cameras narrowed to fp32)."""
        self._check_clip(clip)
        times = sample_times(clip.num_keys, clip.fps, fps_out, speed)
        if align_to is None:
            align = IDENTITY_ALIGN.copy()
        else:
            k = int(align_to)
            F = int(self.model.pose.weight.shape[0])
            if not 0 <= k < F:
                raise ValueError(f"align_to {k}: the model has training frames 0..{F - 1}")
            align = alignment(clip.pose[0, :3].double().numpy(), clip.trans[0].double().numpy(),
                              self.model.pose.weight[k, :3].detach().double().cpu().numpy(),
                              self.model.transl.weight[k].detach().double().cpu().numpy())
        return Schedule(times, align, self._camera_rows(len(times), clip, align))

    def _camera_rows(self, n, clip, align):
        from .mesh_render import cameras as camera_block
        cam = self.cameras
        place = (lambda c: c) if self.placement is None else self.placement.carry
        if isinstance(cam, SceneCamera):                  # already in the scene's world
            return camera_block([cam.camera(self.H, self.W)]).expand(n, -1).contiguous()
        if isinstance(cam, dict):
            one = Camera(float(cam["FovX"]), float(cam["FovY"]), self.H, self.W, torch.as_tensor(cam["world_view_transform"]),
                         torch.as_tensor(cam["full_proj_transform"]), torch.as_tensor(cam["camera_center"]))
            return camera_block([place(one)]).expand(n, -1).contiguous()
        R, c = align[:9].reshape(3, 3), align[9:]
        t0 = R @ clip.trans[0].double().numpy() + c
        pelvis = self.model._rest_joints[0].double().cpu().numpy() + t0        # the root rotates about the rest pelvis
        rows = [place(make_camera(cam.K, rotate_camera_by_frame_idx(cam.extrinsic, k, trans=pelvis, rotate_axis=cam.rotate_axis, period=n,
                                                                   inv_angle=cam.inv_angle), self.H, self.W)) for k in range(n)]
        return camera_block(rows)

    def _check_clip(self, clip):
        if clip.body != self.body.name or clip.pose.shape[1] != self.body.full_width:
            raise ValueError(f"clip for body {clip.body!r} ({tuple(clip.pose.shape)}), the avatar is {self.body.name!r}")

    @torch.no_grad()
    def sample(self, clip: MotionClip, sched: Schedule):
        """All sampled poses [n,72|165] and translations [n,3] of a playback, on the device."""
        keys_p, keys_t = clip.pose.to(self.dev).contiguous(), clip.trans.to(self.dev).contiguous()
        times = torch.from_numpy(sched.times).to(self.dev)
        align = torch.from_numpy(sched.align).to(self.dev)
        return motion_sample(keys_p, keys_t, times, align)

    # ---- playback ---------------------------------------------------------------------------------------------------------------
    def frames(self, clip: MotionClip, fps_out: float, speed: float = 1.0, align_to=None):
        """Yields (index of the chunk's first frame, uint8 [b,H,W,C]) in order.  The array lives in one of two pinned buffers and is
        overwritten two chunks later: copy it to keep it."""
        sched = self.schedule(clip, fps_out, speed, align_to)
        n = len(sched.times)
        starts = list(range(0, n, self.chunk))
        with torch.no_grad(), kept_state(self.model):
            render = self._stage1_setup(clip, sched) if self.stage == 1 else self._stage2_setup(clip, sched)
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
            yield s, self._out_host[slot][:e - s]
        torch.cuda.current_stream().wait_stream(self._copy_stream)

    def _enqueue(self, render, s, e, slot):
        """Renders frames s..e-1 into the slot's device buffer and copies them, with the overflow status, to its pinned buffers."""
        main = torch.cuda.current_stream()
        if self._slot_used[slot]:
            main.wait_event(self._copied[slot])          # the previous copy out of this slot has finished reading it
        with torch.no_grad(), kept_state(self.model):
            render(s, e, slot)
        self._rendered[slot].record(main)
        self._slot_used[slot] = True
        with torch.cuda.stream(self._copy_stream):
            self._copy_stream.wait_event(self._rendered[slot])
            self._out_host[slot][:e - s].copy_(self._out_dev[slot][:e - s], non_blocking=True)
            self._status_host[slot].copy_(self._status_dev[slot], non_blocking=True)
            self._copied[slot].record(self._copy_stream)

    # ---- stage 1: one graph per (chunk size, slot) -------------------------------------------------------------------------------
    def _plan(self, b):
        if b not in self._plans:
            self._plans[b] = RasterBatchPlan(b, int(self.model._query_points.shape[0]), self.H, self.W, self.dev, capacity=self.capacity,
                                             static_P=0 if self.scene is None else len(self.scene))
        return self._plans[b]

    def _raster(self, means, scales, colors, cams, plan):
        m = self.model
        if self.scene is None:
            return rasterize_batch(means, colors, scales, m.fix_rotation, m.fix_opacity, cams, m.background, plan)
        return rasterize_batch_scene(means, colors, scales, m.fix_rotation, m.fix_opacity, cams, m.background, plan, self.scene)

    def _grow(self, b, needed):
        if self._graphs:
            torch.cuda.current_stream().synchronize()     # no replay still reads the buffers about to go
        self._plan(b).grow(needed)
        for key in [k for k in self._graphs if k[0] == b]:       # the graphs hold the old binning buffer's address
            del self._graphs[key]
            self.recaptures += 1

    def _stage1_setup(self, clip, sched):
        m = self.model
        T, width = clip.num_keys, int(clip.pose.shape[1])
        dec = m._stage1_decoder(1)
        if self._keys_pose is None or self._keys_pose.shape[0] < T:
            self._keys_pose = torch.empty(T, width, dtype=torch.float32, device=self.dev)
            self._keys_trans = torch.empty(T, 3, dtype=torch.float32, device=self.dev)
            self._graphs = {}
        # the graphs take the clip's key count as a kernel argument and the decoder output by address
        key = (T, dec.data_ptr())
        if key != self._clip_key:
            self._graphs, self._clip_key = {}, key
        self._dec = dec
        self._keys_pose[:T].copy_(clip.pose)
        self._keys_trans[:T].copy_(clip.trans)
        self._align.copy_(torch.from_numpy(sched.align))
        times_all = torch.from_numpy(sched.times).to(self.dev)
        cams_all = sched.cams.to(self.dev)

        def body(b, slot):
            plan = self._plan(b)
            pose, trans = motion_sample(self._keys_pose[:T], self._keys_trans[:T], self._times_dev[:b], self._align)
            pose, rest = self.body.split(pose)
            means, scales, colors = m._assemble(self._dec, pose, trans, rest, placement=self.placement)
            img = self._raster(means, scales, colors, self._cams_dev[:b], plan)
            frame_pack(img, final_transmittance(plan), m.background, self.channels, self._out_dev[slot][:b])
            self._status_dev[slot].copy_(plan.status_dev)

        def render(s, e, slot):
            b = e - s
            self._times_dev[:b].copy_(times_all[s:e])
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

    # ---- stage 2: eager, one frame per forward ------------------------------------------------------------------------------------
    def _stage2_setup(self, clip, sched):
        m = self.model
        pose, trans = self.sample(clip, sched)
        cams_all = sched.cams.to(self.dev)

        def render(s, e, slot):
            for i in range(s, e):
                p, rest = self.body.split(pose[i:i + 1])
                means, scales, colors, _, _ = m._stage2_from_pose(self.pose_mapper, p, trans[i:i + 1], rest, placement=self.placement)
                if self.scene is None:
                    batch = {"_cams": cams_all[i:i + 1], "height": [self.H], "width": [self.W]}
                    img = m._render_frames(batch, means, scales, colors)
                    plan = m._last_plan
                else:                # as _render_batched: a frame whose binning buffer overflowed is rendered again after it grew
                    plan = self._plan(1)
                    img = self._raster(means, scales, colors, cams_all[i:i + 1], plan)
                    if not plan.check(wait=True):
                        self.overflows += 1
                        img = self._raster(means, scales, colors, cams_all[i:i + 1], plan)
                        if not plan.check(wait=True):
                            raise RuntimeError("animation: the rasterizer's binning buffer overflowed again after growing")
                frame_pack(img, final_transmittance(plan), m.background, self.channels, self._out_dev[slot][i - s:i - s + 1])
        return render
