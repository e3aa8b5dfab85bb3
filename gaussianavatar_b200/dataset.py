"""The reference's dataset folder contract (/root/reference scene/dataset_mono.py:83-96) read into the batch-dict vocabulary the
hot path consumes (`original_image FovX FovY width height pose_idx world_view_transform projection_matrix
full_proj_transform camera_center [pose_data transl_data inp_pos_map rest_pose]`, dataset_mono.py:225-257,498-522,638-676).

    <source_path>/{train,test}/images/<name>.<ext>          RGB frames
                              /masks/<name>.<ext>           foreground masks (>= 128 = subject); absent with no_mask
                              /cam_parms.npz                {intrinsic [3,3], extrinsic [4,4]}   (cam_static)
                              /cam_parms/<name>.npz         per-frame cameras                    (not cam_static)
                              /smpl_parms.pth               {beta [1,10], body_pose [F,72], trans [F,3]}  (stage 2: smpl_parms_pred.pth)
                              /inp_map/inp_posemap_<S>_<idx:08d>.npz   stage-2 posed position maps ['posmap<S>']
    <test_folder>/smpl_parms.pth, cam_parms.npz             novel-pose sequences (assets/test_pose in the reference)

Four datasets with the reference's names: MonoDataset_train / _test (dataset_mono.py:98-417), MonoDataset_novel_pose (:419-522),
MonoDataset_novel_view (:524-676).  Host work only (PIL + numpy); `device_decode=True` hands the raw uint8 image and mask to the
caller instead, so that the white-background compositing and the /255 happen on the GPU after a 4x smaller H2D copy
(`composite_on_device`)."""
from __future__ import annotations

import math
import os
from os.path import join

import numpy as np
import torch
from torch.utils.data import Dataset

from .camera import make_camera, projection_from_K


def _torch_load(path):
    return torch.load(path, weights_only=False)


def _as_tensor(x):
    return x if torch.is_tensor(x) else torch.from_numpy(np.asarray(x))


def camera_item(K, extrinsic, height, width, znear=0.01, zfar=100.0) -> dict:
    """The camera fields of a batch item (dataset_mono.py:238-255)."""
    cam = make_camera(np.asarray(K, np.float32).reshape(3, 3), np.asarray(extrinsic, np.float64), height, width, znear, zfar)
    proj = projection_from_K(znear, zfar, np.asarray(K, np.float32).reshape(3, 3), height, width).transpose(0, 1).contiguous()
    return dict(FovX=cam.FovX, FovY=cam.FovY, width=int(width), height=int(height), world_view_transform=cam.world_view_transform,
                projection_matrix=proj, full_proj_transform=cam.full_proj_transform, camera_center=cam.camera_center)


def composite_host(image_u8: np.ndarray, mask_u8: np.ndarray | None) -> torch.Tensor:
    """dataset_mono.py:207-236: threshold the mask at 128, white background, [3,H,W] float in [0,1]."""
    img = np.asarray(image_u8)
    if mask_u8 is not None:
        m = np.array(mask_u8)
        if m.ndim < 3:
            m = m[..., None]
        m = (m >= 128).astype(np.uint8)
        img = (img * m + (1 - m) * 255).astype(np.uint8)          # the reference narrows through np.byte and PIL: same 8 bits
    t = torch.from_numpy(np.ascontiguousarray(img)) / 255.0
    t = t.permute(2, 0, 1) if t.dim() == 3 else t.unsqueeze(-1).permute(2, 0, 1)
    return t.clamp(0.0, 1.0)


def composite_on_device(image_u8: torch.Tensor, mask_u8: torch.Tensor | None) -> torch.Tensor:
    """The same arithmetic on the GPU for a batch of raw frames: image_u8 [B,H,W,3] uint8, mask_u8 [B,H,W] or [B,H,W,C] uint8 ->
    [B,3,H,W] float32.  Bit-identical to composite_host (integer select, one division)."""
    img = image_u8
    if mask_u8 is not None:
        m = mask_u8 if mask_u8.dim() == 4 else mask_u8.unsqueeze(-1)
        img = torch.where(m >= 128, img, torch.full_like(img, 255))
    return (img.permute(0, 3, 1, 2).to(torch.float32) / 255.0).clamp_(0.0, 1.0).contiguous()


class _MonoFolder(Dataset):
    """Common part of the four datasets: SMPL parameters, frame names, cameras."""
    split = "train"

    def __init__(self, dataset_parms, device=None, device_decode: bool = False):
        super().__init__()
        self.dataset_parms = dataset_parms
        self.data_folder = self._folder(dataset_parms)
        self.device = device
        self.device_decode = bool(device_decode)
        self.gender = dataset_parms.smpl_gender
        self.zfar, self.znear = 100.0, 0.01
        self.no_mask = bool(dataset_parms.no_mask)
        self.smpl_data = _torch_load(join(self.data_folder, self._smpl_file(dataset_parms)))
        self._index_frames()
        pose, trans = _as_tensor(self.smpl_data["body_pose"]), _as_tensor(self.smpl_data["trans"])
        n = self.data_length
        if dataset_parms.smpl_type == "smplx":
            self.pose_data, self.rest_pose_data = pose[:n, :66], pose[:n, 66:]
        else:
            self.pose_data, self.rest_pose_data = pose[:n], None
        self.transl_data = trans[:n, :]
        if dataset_parms.cam_static:
            cam = np.load(join(self.data_folder, "cam_parms.npz"))
            self.extr_npy = np.asarray(cam["extrinsic"])
            self.intrinsic = np.array(cam["intrinsic"], np.float32).reshape(3, 3)

    def _folder(self, p):
        return join(p.source_path, self.split)

    def _smpl_file(self, p):
        return "smpl_parms.pth" if p.train_stage == 1 else "smpl_parms_pred.pth"

    def _index_frames(self):
        names = sorted(os.listdir(join(self.data_folder, "images")))
        self.data_length = len(names)
        self.name_list = [(i, n.split(".")[0]) for i, n in enumerate(names)]
        self.image_fix = names[0].split(".")[-1]
        if not self.no_mask:
            self.mask_fix = sorted(os.listdir(join(self.data_folder, "masks")))[0].split(".")[-1]

    def __len__(self):
        return self.data_length

    def _reads_inp_map(self):
        """Stage 2 reads inp_map/ unless the model builds the maps from the pose (ModelParams.inp_posmap_from_pose)."""
        p = self.dataset_parms
        return p.train_stage == 2 and not getattr(p, "inp_posmap_from_pose", False)

    def _inp_posmap(self, pose_idx):
        S = self.dataset_parms.inp_posmap_size
        d = np.load(join(self.data_folder, "inp_map", "inp_posemap_%s_%s.npz" % (str(S), str(pose_idx).zfill(8))))
        return d["posmap" + str(S)].transpose(2, 0, 1)

    def _camera(self, name):
        if self.dataset_parms.cam_static:
            return self.intrinsic, self.extr_npy
        cam = np.load(join(self.data_folder, "cam_parms", name + ".npz"))
        return np.array(cam["intrinsic"], np.float32).reshape(3, 3), np.asarray(cam["extrinsic"])

    def _image_item(self, name):
        from PIL import Image
        image = Image.open(join(self.data_folder, "images", name + "." + self.image_fix)).convert("RGB")
        width, height = image.size
        mask = None if self.no_mask else np.array(Image.open(join(self.data_folder, "masks", name + "." + self.mask_fix)))
        if self.device_decode:
            item = dict(image_u8=torch.from_numpy(np.array(image)))
            if mask is not None:
                item["mask_u8"] = torch.from_numpy(mask if mask.ndim == 2 else mask[..., 0])
        else:
            item = dict(original_image=composite_host(np.array(image), mask))
        return item, width, height


class MonoDataset_train(_MonoFolder):
    split = "train"

    def __getitem__(self, index, ignore_list=None):
        pose_idx, name = self.name_list[index]
        item, width, height = self._image_item(name)
        if self._reads_inp_map():
            item["inp_pos_map"] = self._inp_posmap(pose_idx)
        K, E = self._camera(name)
        item.update(camera_item(K, E, height, width, self.znear, self.zfar))
        item["pose_idx"] = pose_idx
        if self.rest_pose_data is not None:
            item["rest_pose"] = self.rest_pose_data[pose_idx]
        return item


class MonoDataset_test(MonoDataset_train):
    split = "test"

    def __getitem__(self, index, ignore_list=None):
        item = super().__getitem__(index)
        pose_idx = item["pose_idx"]
        item["pose_data"], item["transl_data"] = self.pose_data[pose_idx], self.transl_data[pose_idx]      # dataset_mono.py:398-399
        return item


class MonoDataset_novel_pose(_MonoFolder):
    """Poses from <test_folder>/smpl_parms.pth rendered through the static camera at 1024^2 (dataset_mono.py:419-522)."""

    def _folder(self, p):
        return p.test_folder

    def _smpl_file(self, p):
        return "smpl_parms.pth"

    def _index_frames(self):
        self.data_length = int(_as_tensor(self.smpl_data["body_pose"]).shape[0])
        self.name_list = [(i, str(i)) for i in range(self.data_length)]

    def __getitem__(self, index, ignore_list=None):
        item = {}
        if self._reads_inp_map():
            item["inp_pos_map"] = self._inp_posmap(index)
        item.update(camera_item(self.intrinsic, self.extr_npy, 1024, 1024, self.znear, self.zfar))         # size hard-coded at :492
        item.update(pose_idx=index, pose_data=self.pose_data[index], transl_data=self.transl_data[index])
        if self.rest_pose_data is not None:
            item["rest_pose"] = self.rest_pose_data[index]
        return item


def _rodrigues(v):
    th = float(np.linalg.norm(v))
    if th < 1e-12:
        return np.eye(3)
    k = np.asarray(v, np.float64) / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + math.sin(th) * K + (1 - math.cos(th)) * (K @ K)


def rotate_camera_by_frame_idx(extrinsics, frame_idx, trans=None, rotate_axis="y", period=196, inv_angle=False):
    """Free-view orbit of dataset_mono.py:10-81 (after humannerf): rotate the camera about `rotate_axis` through `trans`."""
    angle = 2 * np.pi * (frame_idx / period)
    if inv_angle:
        angle = -angle
    inv_E = np.linalg.inv(np.asarray(extrinsics, np.float64))
    camrot, campos = inv_E[:3, :3], inv_E[:3, 3].copy()
    if trans is not None:
        campos -= trans
    if camrot.T[1, 1] < 0.0:
        angle = -angle
    vec = np.zeros(3)
    vec[{"x": 0, "y": 1, "z": 2}[rotate_axis]] = angle
    R = _rodrigues(vec).astype(np.float32)
    rot_campos, rot_camrot = R.dot(campos), R.dot(camrot)
    if trans is not None:
        rot_campos += trans
    E = np.identity(4)
    E[:3, :3] = rot_camrot.T
    E[:3, 3] = -rot_camrot.T.dot(rot_campos)
    return E


class MonoDataset_novel_view(_MonoFolder):
    """One training pose seen from an orbiting camera (dataset_mono.py:524-676).  `update_smpl(pose_idx, frame_num, pelvis)` fixes
    the pose and the orbit centre; the reference takes the T-pose pelvis from a numpy SMPL model, here it is passed in (the
    avatar model knows its rest joints)."""
    split = "test"
    ROT_CAM_PARAMS = {"zju_mocap": {"rotate_axis": "z", "inv_angle": True}, "wild": {"rotate_axis": "y", "inv_angle": False}}

    def __init__(self, dataset_parms, device=None, device_decode=False):
        super().__init__(dataset_parms, device, device_decode)
        self.src_type = "wild"
        self.fix_pose_idx, self.Th = 0, np.zeros(3)

    def update_smpl(self, pose_idx, frame_num, pelvis_pos=None):
        pelvis = np.zeros(3) if pelvis_pos is None else np.asarray(pelvis_pos, np.float64)
        self.Th = pelvis + _as_tensor(self.smpl_data["trans"])[pose_idx].numpy().astype(np.float64)
        self.data_length = int(frame_num)
        self.fix_pose_idx = int(pose_idx)

    def __getitem__(self, index):
        from PIL import Image
        pose_idx = self.fix_pose_idx
        _, name = self.name_list[0]
        width, height = Image.open(join(self.data_folder, "images", name + "." + self.image_fix)).size
        E = rotate_camera_by_frame_idx(self.extr_npy, index, trans=self.Th, period=self.data_length, **self.ROT_CAM_PARAMS[self.src_type])
        item = {}
        if self._reads_inp_map():
            item["inp_pos_map"] = self._inp_posmap(pose_idx)
        item.update(camera_item(self.intrinsic, E, height, width, self.znear, self.zfar))
        item.update(pose_idx=pose_idx, pose_data=self.pose_data[pose_idx], transl_data=self.transl_data[pose_idx])
        if self.rest_pose_data is not None:
            item["rest_pose"] = self.rest_pose_data[pose_idx]
        return item
