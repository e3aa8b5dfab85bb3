"""Synthetic stage-1 training workloads at the sizes BASELINE.json names (SURVEY.md §8d): procedural body + UV layout
(synthetic.py), the reference's shipped poses / camera (committed subset of assets/test_pose under tests/golden/),
reference-default net initialisation with `decoder.conv8N.bias = -5.3` (sigmoid ~ 0.005 m Gaussians), white background,
ground-truth images rendered from a perturbed copy of the model so that losses and gradients are non-degenerate."""
from __future__ import annotations

import os

import numpy as np
import torch

from . import synthetic as syn
from .avatar_model import AvatarModel
from .body import body_of
from .camera import TEST_POSE_EXTRINSIC, TEST_POSE_K, make_camera, scaled_intrinsics
from .config import OptimizationParams

_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def load_poses(num: int = 32):
    path = os.path.join(_REPO, "tests", "golden", "test_pose_subset.npz")
    if os.path.exists(path):
        d = np.load(path)
        return torch.tensor(d["body_pose"][:num]), torch.tensor(d["trans"][:num]), "assets/test_pose subset (tests/golden/test_pose_subset.npz)"
    pose, transl = syn.synthetic_poses(num)
    return pose, transl, "synthetic poses"


class Stage1Workload:
    """body="smplx": the same workload on the synthetic 55-joint body; the body pose is the shipped poses' first 66 values and every
    frame carries a synthetic hand / face pose (`rest_pose` [99]) in its batch."""
    def __init__(self, config: int = 3, frames_per_gpu: int = 2, device="cuda:0", seed: int = 0, N=None, S=None, side=None,
                 inp_posmap_size: int = 128, num_frames: int = 32, body: str = "smpl"):
        cN, cS, cside = syn.CONFIGS[config]
        self.N, self.S, self.side = N or cN, S or cS, side or cside
        self.B = frames_per_gpu
        self.device = torch.device(device)
        assets = syn.make_avatar_assets(self.N, self.S, seed=seed, body=body)
        pose, transl, self.pose_source = load_poses(num_frames)
        self.num_frames = pose.shape[0]
        b = body_of(body)
        pose = pose[:, :b.pose_width].contiguous()
        self.rest_dev = syn.synthetic_smplx_poses(self.num_frames, seed=seed)[1].to(self.device) if b.rest_width else None
        cam = make_camera(scaled_intrinsics(TEST_POSE_K, self.side), TEST_POSE_EXTRINSIC, self.side, self.side)
        self.cam = cam
        frames = [dict(pose_idx=i) for i in range(self.num_frames)]
        torch.manual_seed(seed)                      # utils/general_utils.py:126-128 seeds 0
        self.model = AvatarModel.from_assets(assets, frames, pose, transl, batch_size=self.B, opt_parms=OptimizationParams(), device=device)
        if inp_posmap_size != self.model.model_parms.inp_posmap_size:
            self.model.model_parms.inp_posmap_size = inp_posmap_size
            self.model.net_set(1)
        with torch.no_grad():
            sd = self.model.net.state_dict()
            sd["decoder.conv8N.bias"] = torch.tensor([-5.3])
            self.model.net.load_state_dict(sd, strict=False)
        self._cam_dev = cam.to(self.device)
        self.gt_host = None      # [F,3,H,W] pinned
        self.gt_dev = None

    # ------------------------------------------------------------------------------------------------------------------
    def camera_fields(self, B):
        c = self._cam_dev
        return dict(FovX=[c.FovX] * B, FovY=[c.FovY] * B, height=[c.height] * B, width=[c.width] * B,
                    world_view_transform=c.world_view_transform[None].expand(B, -1, -1),
                    full_proj_transform=c.full_proj_transform[None].expand(B, -1, -1), camera_center=c.camera_center[None].expand(B, -1))

    @torch.no_grad()
    def make_ground_truth(self, keep_on_device: bool = True, pin: bool = True):
        """GT = render of a perturbed copy of the model (different geo_feature draw), one image per pose."""
        m = self.model
        g = torch.Generator(device="cpu").manual_seed(1)
        geo_backup = m.geo_feature.data.clone()
        m.geo_feature.data.copy_((torch.randn(geo_backup.shape, generator=g) * 0.03).to(self.device))
        run_backup = m.net.bn_running.clone()
        imgs = []
        for f0 in range(0, self.num_frames, self.B):
            idx = torch.arange(f0, min(self.num_frames, f0 + self.B), device=self.device)
            while idx.numel() < self.B:
                idx = torch.cat([idx, idx[-1:]])
            batch = dict(pose_idx=idx, **self.camera_fields(self.B))
            if self.rest_dev is not None:
                batch["rest_pose"] = self.rest_dev[idx]
            imgs.append(m.render_free_stage1(batch, 59400)[: min(self.B, self.num_frames - f0)].clone())
        m.geo_feature.data.copy_(geo_backup)
        m.net.bn_running.copy_(run_backup)
        gt = torch.cat(imgs, 0).contiguous()
        self.gt_dev = gt if keep_on_device else None
        host = gt.cpu()
        self.gt_host = host.pin_memory() if pin else host
        return gt

    def frame_ids(self, step: int, rank: int = 0, world: int = 1):
        """Global batch = world * B distinct frames per step, sharded one slice per rank (BASELINE config 4 semantics)."""
        base = (step * world + rank) * self.B
        return [(base + j) % self.num_frames for j in range(self.B)]

    def device_batch(self, ids):
        """Batch dict (scene/dataset_mono.py:238-255 keys) with inputs already resident in HBM."""
        # the index tensors live on the device (one per distinct id tuple): building one per step from host data costs either a
        # stream-synchronising pageable copy or a pinned allocation, both of which stall the enqueueing thread
        cache = self.__dict__.setdefault("_idx_cache", {})
        key = tuple(ids)
        if key not in cache:
            cache[key] = torch.tensor(ids, device=self.device)
        idx = cache[key]
        B = len(ids)
        img = self.gt_dev[ids[0]:ids[0] + B] if all(ids[j] == ids[0] + j for j in range(B)) else self.gt_dev[idx]     # a view when contiguous
        out = dict(pose_idx=idx, original_image=img, **self.camera_fields(B))
        if self.rest_dev is not None:
            out["rest_pose"] = self.rest_dev[idx]
        return out

    def host_batch(self, ids):
        """The same batch as HOST tensors (pinned), as a DataLoader would hand it over (train.py:63-66)."""
        c = self.cam
        B = len(ids)
        if all(ids[j] == ids[0] + j for j in range(B)):
            img = self.gt_host[ids[0]:ids[0] + B]              # view of the pinned pool: no host-side copy
        else:
            img = self.gt_host[ids].pin_memory()
        return dict(pose_idx=torch.tensor(ids), original_image=img,
                    FovX=[c.FovX] * B, FovY=[c.FovY] * B, height=[c.height] * B, width=[c.width] * B,
                    world_view_transform=c.world_view_transform[None].expand(B, -1, -1).contiguous(),
                    full_proj_transform=c.full_proj_transform[None].expand(B, -1, -1).contiguous(),
                    camera_center=c.camera_center[None].expand(B, -1).contiguous())


def to_cuda(batch, device):
    """utils/general_utils.py:129-163 `to_cuda`: tensors go to the device (non_blocking from pinned memory), scalars stay.
    Returns (batch_on_device, bytes_copied)."""
    out, nbytes = {}, 0
    for k, v in batch.items():
        if torch.is_tensor(v):
            if not v.is_cuda:
                nbytes += v.numel() * v.element_size()
            out[k] = v.to(device, non_blocking=True)
        else:
            out[k] = v
    return out, nbytes
