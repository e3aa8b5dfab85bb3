"""`AvatarModel` with the reference's public surface (/root/reference model/avatar_model.py:19-649) over the fused
sm_90a kernels: SMPL / SMPL-X pose -> cano2live (one kernel), feature net (once per step), fused LBS + attribute assembly,
tile rasterizer per frame.  `smpl_type='smplx'` (55 joints) takes the hand / face pose of every frame from the batch's
`rest_pose` [B,99], as the reference does (model/avatar_model.py:279-289).

Same methods / attributes as the reference: train_stage1, render_free_stage1, training_setup, zero_grad, step, save,
load, stage_load, getTrainDataloader ..., `.net .pose .transl .geo_feature .model_path`.  Stage 2 (pose encoder U-Net,
SURVEY.md §8f rank 2) is not built yet and raises NotImplementedError.

Two ways to construct:
  AvatarModel(model_parms, net_parms, opt_parms, train=True)   reference signature; reads the dataset folder contract
                                                               of scene/dataset_mono.py:83-96 + assets/ (needs the
                                                               licensed SMPL / UV assets the reference needs)
  AvatarModel.from_assets(assets, frames, ...)                 tensors in memory (synthetic assets, benchmarks, tests)
"""
from __future__ import annotations

import os
from os.path import join

import numpy as np
import torch
import torch.nn as nn

from .config import ModelParams, NetworkParams, OptimizationParams
from .network import POP_no_unet
from .ops import LbsAssemble, SmplCano2Live, SmplxCano2Live
from .renderer import render_batch


class _FrameSet(torch.utils.data.Dataset):
    """In-memory stand-in for MonoDataset_train (scene/dataset_mono.py:98-257): yields the same dict keys."""

    def __init__(self, frames):
        self.frames = frames

    def __len__(self):
        return len(self.frames)

    def __getitem__(self, i):
        return self.frames[i]


class AvatarModel:
    def __init__(self, model_parms, net_parms, opt_parms, load_iteration=None, train=True, _assets=None, _frames=None,
                 _pose_data=None, _transl_data=None, device="cuda"):
        self.model_parms, self.net_parms, self.opt_parms = model_parms, net_parms, opt_parms
        self.model_path = model_parms.model_path
        self.loaded_iter = None
        self.train = train
        self.train_mode = model_parms.train_mode
        self.gender = model_parms.smpl_gender
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("AvatarModel runs on CUDA only (no CPU fallback)")
        self.batch_size = model_parms.batch_size if train else 1      # avatar_model.py:31-34
        assert model_parms.smpl_type in ["smplx", "smpl"]
        self.smplx = model_parms.smpl_type == "smplx"
        self.num_joints = 55 if self.smplx else 24
        if model_parms.train_stage not in (0, 1, 2):
            raise ValueError(f"train_stage {model_parms.train_stage} is not one of 1, 2")
        self.posmap_from_pose = model_parms.train_stage == 2 and bool(getattr(model_parms, "inp_posmap_from_pose", False))
        if self.posmap_from_pose and self.smplx:
            raise NotImplementedError("inp_posmap_from_pose: device position maps are built for the SMPL mesh only (smpl_type='smpl')")

        if _assets is None:
            _assets, _frames, _pose_data, _transl_data = self._load_reference_assets(model_parms, train)
        self._from_folder = not isinstance(_frames, list)
        S = int(model_parms.query_posmap_size)
        assert _assets["valid_idx"].numel() == S * S
        dev = self.device
        self.valid_idx = _assets["valid_idx"].to(dev)                                   # bool [S*S]
        self.valid_index = torch.nonzero(self.valid_idx).reshape(-1).to(torch.int32).contiguous()   # order of the boolean mask
        qp = _assets["query_points"].to(dev).float().contiguous()                      # [N,3]
        self._query_points = qp
        self.query_points = qp[None].expand(self.batch_size, -1, -1)                    # avatar_model.py:75-77
        N = qp.shape[0]
        self.fix_opacity = torch.ones((N, 1), device=dev)                               # avatar_model.py:80-83
        rots = torch.zeros((N, 4), device=dev)
        rots[:, 0] = 1
        self.fix_rotation = rots
        J = self.num_joints
        lbs = _assets["query_lbs"].to(dev).float()
        if tuple(lbs.shape) != (N, J):
            raise ValueError(f"query_lbs {tuple(lbs.shape)}: expected [{N},{J}] for smpl_type={model_parms.smpl_type!r}")
        if self.smplx:      # 220-byte rows -> 224: whole float4s for the LBS kernel's TMA copy and row reads (zero last column)
            lbs = torch.nn.functional.pad(lbs, (0, 1))
        self._query_lbs = lbs.contiguous()                                              # [N,24] / [N,56], ONE copy for all frames
        self.query_lbs = self._query_lbs[None, :, :J].expand(self.batch_size, -1, -1)  # view only (reference materialises B copies, :86-87)
        cano = _assets["cano_joint_mats"].to(dev).float()
        if tuple(cano.shape) != (J, 4, 4) or tuple(_assets["rest_joints"].shape) != (J, 3):
            raise ValueError(f"cano_joint_mats {tuple(cano.shape)} / rest_joints {tuple(_assets['rest_joints'].shape)}: expected [{J},4,4] / [{J},3]")
        self._inv_cano = torch.linalg.inv(cano).contiguous()                            # [J,4,4]  avatar_model.py:89
        self.inv_mats = self._inv_cano[None].expand(self.batch_size, -1, -1, -1)
        self._rest_joints = _assets["rest_joints"].to(dev).float().contiguous()        # J(beta): constant per subject
        self.betas = _assets["betas"].to(dev).float()[None].expand(self.batch_size, -1) if "betas" in _assets else None

        self.train_dataset = _FrameSet(_frames) if isinstance(_frames, list) else _frames
        num_training_frames = _pose_data.shape[0]
        pose_dim = 66 if self.smplx else 72          # SMPL-X: global + 21 body joints are trained, the rest comes with the frame
        if _pose_data.shape[1] != pose_dim:
            raise ValueError(f"pose data {tuple(_pose_data.shape)}: expected [F,{pose_dim}] for smpl_type={model_parms.smpl_type!r}")
        self.pose = torch.nn.Embedding(num_training_frames, pose_dim, _weight=_pose_data.clone().float(), sparse=True).to(dev)
        self.transl = torch.nn.Embedding(num_training_frames, 3, _weight=_transl_data.clone().float(), sparse=True).to(dev)
        self.optimizer_pose = torch.optim.SparseAdam(list(self.pose.parameters()) + list(self.transl.parameters()), 5.0e-3)
        bg_color = [1, 1, 1] if model_parms.white_background else [0, 0, 0]
        self.background = torch.tensor(bg_color, dtype=torch.float32, device=dev)
        self.optimizer = None
        self.scheduler = None
        self.cache_decoder = not train     # inference models evaluate the frame-invariant stage-1 net once (see render_free_stage1)
        self._dec_cache = None
        self.net_set(model_parms.train_stage)
        self.pose_mapper = None
        if self.posmap_from_pose:         # stage-2 input maps from the pose, on the device (posmap.py)
            from .posmap import PoseMapper
            if "smpl_mesh" not in _assets or "uv_template" not in _assets:
                raise ValueError("inp_posmap_from_pose: the assets carry no 'smpl_mesh' / 'uv_template' (the SMPL mesh model and its UV template)")
            self.pose_mapper = PoseMapper(_assets["smpl_mesh"], _assets["betas"], _assets["uv_template"], int(model_parms.inp_posmap_size),
                                          device=dev)

    # ------------------------------------------------------------------------------------------------------------------
    @classmethod
    def from_assets(cls, assets, frames, pose_data, transl_data, batch_size=2, train=True, opt_parms=None, device="cuda", net_parms=None,
                    **model_fields):
        """assets: gaussianavatar_b200.synthetic.SyntheticAvatarAssets (or a dict with the same fields).  55 rest joints make an
        SMPL-X model (its frames then carry `rest_pose`).  model_fields override ModelParams fields (e.g. train_stage=2,
        inp_posmap_size, inp_posmap_from_pose=True; the last needs the dict keys `smpl_mesh`, the SMPL_{GENDER}.pkl fields, and
        `uv_template`, a path or what posmap.load_uv_template_obj returns)."""
        if not isinstance(assets, dict):
            assets = dict(valid_idx=assets.valid_idx, query_points=assets.query_points, query_lbs=assets.query_lbs,
                          cano_joint_mats=assets.cano_joint_mats, rest_joints=assets.rest_joints, betas=assets.body.betas[0], S=assets.S)
        smpl_type = "smplx" if assets["rest_joints"].shape[0] == 55 else "smpl"
        mp = ModelParams(batch_size=batch_size, query_posmap_size=int(assets["S"]), smpl_type=smpl_type, **model_fields)
        return cls(mp, net_parms or NetworkParams(), opt_parms or OptimizationParams(), train=train, _assets=assets, _frames=frames,
                   _pose_data=pose_data, _transl_data=transl_data, device=device)

    def _load_reference_assets(self, mp, train):
        """Folder contract of the reference (model/avatar_model.py:41-98; scene/dataset_mono.py:83-160): the training dataset (always
        built, even for evaluation, avatar_model.py:41), the UV mask / canonical position map / LBS map / canonical joint
        matrices, and the SMPL model pickle for the rest joints J(beta).  Exercised against a synthetic folder written in the
        same layout (tests/test_dataset_cpu.py, tests/test_avatar_gpu.py)."""
        from .dataset import MonoDataset_train
        split = "train" if train else "test"
        dataset = MonoDataset_train(mp)
        S = int(mp.query_posmap_size)
        if mp.smpl_type == "smplx":
            return self._load_reference_assets_smplx(mp, split, dataset, S)
        mask = np.load(join(mp.project_path, "assets", "uv_masks", f"uv_mask{S}_with_faceid_smpl.npy")).reshape(S, S)
        valid = torch.from_numpy(mask != -1).reshape(-1)
        qmap = torch.from_numpy(np.load(join(mp.source_path, split, f"query_posemap_{S}_cano_smpl.npz"))[f"posmap{S}"]).reshape(-1, 3)
        lbs = torch.from_numpy(np.load(join(mp.project_path, "assets", f"lbs_map_smpl_{S}.npy"))).reshape(S * S, 24)
        cano = torch.load(join(mp.source_path, split, "smpl_cano_joint_mat.pth"), weights_only=False).reshape(24, 4, 4)
        cano = torch.as_tensor(cano).float()
        smpl_data = dataset.smpl_data
        beta = torch.as_tensor(smpl_data["beta"][0]).float()
        import pickle
        with open(join(mp.smpl_model_path, f"SMPL_{mp.smpl_gender.upper()}.pkl"), "rb") as f:
            sm = pickle.load(f, encoding="latin1")
        v_t = torch.as_tensor(np.asarray(sm["v_template"])).double()
        sd = torch.as_tensor(np.asarray(sm["shapedirs"])[:, :, :10]).double()
        Jr = torch.as_tensor(np.asarray(sm["J_regressor"].todense() if hasattr(sm["J_regressor"], "todense") else sm["J_regressor"])).double()
        rest = (Jr @ (v_t + torch.einsum("l,mkl->mk", beta.double(), sd))).float()
        pose = dataset.pose_data.float()
        transl = dataset.transl_data.float()
        assets = dict(valid_idx=valid, query_points=qmap[valid].float(), query_lbs=lbs[valid].float(), cano_joint_mats=cano, rest_joints=rest,
                      betas=beta, S=S)
        if mp.train_stage == 2 and getattr(mp, "inp_posmap_from_pose", False):
            # the mesh comes from the same SMPL_{GENDER}.pkl as the rest joints; the UV template from where the reference's scripts read it
            from .posmap import SMPL_MESH_FIELDS
            missing = [k for k in SMPL_MESH_FIELDS if k not in sm]
            if missing:
                raise ValueError(f"{f.name}: no {', '.join(missing)}; inp_posmap_from_pose needs the full SMPL mesh model")
            template = join(mp.project_path, "assets", "template_mesh_smpl_uv.obj")
            if not os.path.exists(template):
                raise FileNotFoundError(f"inp_posmap_from_pose: UV template {template} not found")
            assets.update(smpl_mesh=sm, uv_template=template)
        return assets, dataset, pose, transl

    def _load_reference_assets_smplx(self, mp, split, dataset, S):
        """The SMPL-X branch of the folder contract (model/avatar_model.py:45-53): `uv_mask{S}_with_faceid_smplx.npy`,
        `query_posemap_{S}_cano_smplx.npz`, `lbs_map_smplx_{S}.npy` [S*S,55], `smplx_cano_joint_mat.pth` [55,4,4], and the rest joints
        from `SMPLX_{GENDER}.npz` under smplx_model_path (the shape directions past the 10 betas are expression: the reference passes
        none, so they drop out)."""
        from .synthetic import SMPLX_PARENTS
        mask = np.load(join(mp.project_path, "assets", "uv_masks", f"uv_mask{S}_with_faceid_smplx.npy")).reshape(S, S)
        valid = torch.from_numpy(mask != -1).reshape(-1)
        qmap = torch.from_numpy(np.load(join(mp.source_path, split, f"query_posemap_{S}_cano_smplx.npz"))[f"posmap{S}"]).reshape(-1, 3)
        lbs = torch.from_numpy(np.load(join(mp.project_path, "assets", f"lbs_map_smplx_{S}.npy"))).reshape(S * S, 55)
        cano = torch.as_tensor(torch.load(join(mp.source_path, split, "smplx_cano_joint_mat.pth"), weights_only=False)).reshape(55, 4, 4).float()
        beta = torch.as_tensor(dataset.smpl_data["beta"][0]).float()
        rest = smplx_rest_joints(join(mp.smplx_model_path, f"SMPLX_{mp.smpl_gender.upper()}.npz"), beta, SMPLX_PARENTS)
        assets = dict(valid_idx=valid, query_points=qmap[valid].float(), query_lbs=lbs[valid].float(), cano_joint_mats=cano, rest_joints=rest,
                      betas=beta, S=S)
        return assets, dataset, dataset.pose_data.float(), dataset.transl_data.float()

    # ------------------------------------------------------------------------------------------------------------------
    def net_set(self, mode):
        assert mode in [0, 1, 2]
        self._dec_cache = None
        npm = self.net_parms
        self.net = POP_no_unet(c_geom=npm.c_geom, geom_layer_type=npm.geom_layer_type, nf=npm.nf, hsize=npm.hsize, up_mode=npm.up_mode,
                               use_dropout=bool(npm.use_dropout), uv_feat_dim=2).to(self.device)
        inp = self.model_parms.inp_posmap_size
        geo = torch.ones(1, npm.c_geom, inp, inp).normal_(mean=0., std=0.01).float().to(self.device)      # avatar_model.py:136
        self.geo_feature = nn.Parameter(geo.requires_grad_(True))
        if self.model_parms.train_stage == 2:                                                              # avatar_model.py:138-146
            from .pose_encoder import UnetNoCond5DS
            if npm.c_pose != npm.c_geom:
                raise NotImplementedError("c_pose must equal c_geom: the two maps are ADDED (model/network.py:58)")
            self.pose_encoder = UnetNoCond5DS(input_nc=3, output_nc=npm.c_pose, nf=npm.nf, up_mode=npm.up_mode, use_dropout=False).to(self.device)

    def training_setup(self):
        # avatar_model.py:148-162: stage 1 trains the net and geo_feature; stage 2 the net at a tenth of the rate and the pose encoder
        if self.model_parms.train_stage == 2:
            self.optimizer = torch.optim.Adam([{"params": self.net.parameters(), "lr": self.opt_parms.lr_net * 0.1},
                                               {"params": self.pose_encoder.parameters(), "lr": self.opt_parms.lr_net}])
        else:
            self.optimizer = torch.optim.Adam([{"params": self.net.parameters(), "lr": self.opt_parms.lr_net},
                                               {"params": self.geo_feature, "lr": self.opt_parms.lr_geomfeat}])
        self.scheduler = torch.optim.lr_scheduler.MultiStepLR(self.optimizer, self.opt_parms.sched_milestones, gamma=0.1)

    def save(self, iteration):
        path = os.path.join(self.model_path, "net/iteration_{}".format(iteration))
        os.makedirs(path, exist_ok=True)
        if self.model_parms.train_stage == 2:                      # avatar_model.py:177-186
            torch.save({"pose_encoder": self.pose_encoder.state_dict(), "geo_feature": self.geo_feature, "pose": self.pose.state_dict(),
                        "transl": self.transl.state_dict(), "net": self.net.state_dict(), "optimizer": self.optimizer.state_dict(),
                        "scheduler": self.scheduler.state_dict()}, os.path.join(path, "pose_encoder.pth"))
            return
        torch.save({"net": self.net.state_dict(), "geo_feature": self.geo_feature, "pose": self.pose.state_dict(),
                    "transl": self.transl.state_dict(), "optimizer": self.optimizer.state_dict(),
                    "scheduler": self.scheduler.state_dict()}, os.path.join(path, "net.pth"))

    def load(self, iteration, test=False):
        self._dec_cache = None
        path = os.path.join(self.model_path, "net/iteration_{}".format(iteration))
        saved = torch.load(os.path.join(path, "net.pth"), weights_only=False)
        self.net.load_state_dict(saved["net"], strict=False)
        if self.model_parms.train_stage == 1:                      # avatar_model.py:197-202
            if not test:
                self.pose.load_state_dict(saved["pose"], strict=False)
                self.transl.load_state_dict(saved["transl"], strict=False)
            self.geo_feature.data[...] = saved["geo_feature"].data[...]
        # optimizer state: written either by this implementation (ONE flat net parameter + geo_feature) or by the reference
        # (53 per-tensor Adam states + geo_feature, avatar_model.py:148-155): the latter is re-laid out into the flat buffer
        if self.optimizer is not None and "optimizer" in saved:
            self.optimizer.load_state_dict(self.translate_optimizer_state(saved["optimizer"]))
        if self.scheduler is not None and "scheduler" in saved:
            self.scheduler.load_state_dict(saved["scheduler"])

    def translate_optimizer_state(self, osd):
        """A `torch.optim.Adam.state_dict()` over the reference's parameter list -> the same over (net.flat, geo_feature).
        State dicts already in this implementation's layout pass through unchanged."""
        from .network import REFERENCE_PARAM_ORDER
        groups = osd["param_groups"]
        n_ref = len(REFERENCE_PARAM_ORDER)
        if not (len(groups) == 2 and len(groups[0]["params"]) == n_ref and len(groups[1]["params"]) == 1):
            return osd
        ids, geo_id = list(groups[0]["params"]), groups[1]["params"][0]
        state = osd.get("state", {})
        new_state = {}
        if all(i in state for i in ids):
            new_state[0] = {"step": state[ids[0]]["step"],
                            "exp_avg": self.net.flat_from_reference_tensors([state[i]["exp_avg"] for i in ids]),
                            "exp_avg_sq": self.net.flat_from_reference_tensors([state[i]["exp_avg_sq"] for i in ids])}
        if geo_id in state:
            new_state[1] = dict(state[geo_id])
        g0, g1 = dict(groups[0]), dict(groups[1])
        g0["params"], g1["params"] = [0], [1]
        return {"state": new_state, "param_groups": [g0, g1]}

    def stage_load(self, ckpt_path):
        self._dec_cache = None
        saved = torch.load(os.path.join(ckpt_path, "net.pth"), weights_only=False)
        self.net.load_state_dict(saved["net"], strict=False)
        self.pose.load_state_dict(saved["pose"], strict=False)
        self.transl.load_state_dict(saved["transl"], strict=False)
        self.geo_feature.data[...] = saved["geo_feature"].data[...]

    def stage2_load(self, epoch):
        """avatar_model.py:223-236: everything a stage-2 run saved (`pose_encoder.pth`)."""
        self._dec_cache = None
        path = os.path.join(self.model_parms.project_path, self.model_path, "net/iteration_{}".format(epoch))
        saved = torch.load(os.path.join(path, "pose_encoder.pth"), weights_only=False)
        self.net.load_state_dict(saved["net"], strict=False)
        self.pose.load_state_dict(saved["pose"], strict=False)
        self.transl.load_state_dict(saved["transl"], strict=False)
        self.geo_feature.data[...] = saved["geo_feature"].data[...]
        self.pose_encoder.load_state_dict(saved["pose_encoder"], strict=False)
        return getattr(self, "novel_view_dataset", None)

    def getTrainDataloader(self):
        # model/avatar_model.py:238-244 (4 workers when the frames come from disk)
        return torch.utils.data.DataLoader(self.train_dataset, batch_size=self.batch_size, shuffle=True,
                                           num_workers=4 if self._from_folder else 0, drop_last=True)

    def _need_folder(self, what):
        if not self._from_folder:
            raise RuntimeError(f"{what}: this AvatarModel was built from in-memory assets (from_assets); the dataset accessors read the "
                               "reference's folder layout (scene/dataset_mono.py:83-96) given by model_parms.source_path / test_folder")

    def getTestDataset(self):          # model/avatar_model.py:246-248
        from .dataset import MonoDataset_test
        self._need_folder("getTestDataset")
        self.test_dataset = MonoDataset_test(self.model_parms)
        return self.test_dataset

    def getNovelposeDataset(self):     # model/avatar_model.py:250-252
        from .dataset import MonoDataset_novel_pose
        self._need_folder("getNovelposeDataset")
        self.novel_pose_dataset = MonoDataset_novel_pose(self.model_parms)
        return self.novel_pose_dataset

    def getNovelviewDataset(self):     # model/avatar_model.py:254-256
        from .dataset import MonoDataset_novel_view
        self._need_folder("getNovelviewDataset")
        self.novel_view_dataset = MonoDataset_novel_view(self.model_parms)
        return self.novel_view_dataset

    def zero_grad(self, epoch):
        self.optimizer.zero_grad()
        if self.model_parms.train_stage == 1 and epoch > self.opt_parms.pose_op_start_iter:     # avatar_model.py:258-262
            self.optimizer_pose.zero_grad()

    def step(self, epoch):
        self.optimizer.step()
        self.scheduler.step()
        if self.model_parms.train_stage == 1 and epoch > self.opt_parms.pose_op_start_iter:     # avatar_model.py:263-270
            self.optimizer_pose.step()

    # ------------------------------------------------------------------------------------------------------------------
    def _cano2live(self, pose_batch, transl_batch, rest_pose=None):
        """[B,J,12] for the body model: SMPL from pose [B,72]; SMPL-X from pose [B,66] and the frames' rest_pose [B,99]."""
        if not self.smplx:
            return SmplCano2Live.apply(pose_batch, transl_batch, self._rest_joints, self._inv_cano)
        B = pose_batch.shape[0]
        if rest_pose is None:
            raise ValueError("smpl_type='smplx': the batch has no 'rest_pose' (jaw, eyes and hands, [B,99])")
        rest_pose = torch.as_tensor(rest_pose)
        if rest_pose.dim() != 2 or tuple(rest_pose.shape) != (B, 99):
            raise ValueError(f"smpl_type='smplx': rest_pose {tuple(rest_pose.shape)}, expected [{B},99] (jaw, eyes, 2 x 15 finger joints)")
        rest_pose = rest_pose.to(device=self.device, dtype=torch.float32)
        return SmplxCano2Live.apply(pose_batch, rest_pose, transl_batch, self._rest_joints, self._inv_cano)

    def _posed_gaussians(self, idx, iteration, ramp=True, rest_pose=None):
        """SMPL / SMPL-X -> cano2live -> net (once) -> fused LBS/assembly.  Returns means3D, scales, colors [B,N,3] and dec_out."""
        if getattr(self, "_detach_pose", False):      # pose optimisation inactive (epoch <= pose_op_start_iter): its gradients are never read
            pose_batch, transl_batch = self.pose.weight.detach()[idx], self.transl.weight.detach()[idx]
        else:
            pose_batch = self.pose(idx)
            transl_batch = self.transl(idx)
        B = pose_batch.shape[0]
        cano2live = self._cano2live(pose_batch, transl_batch, rest_pose)                                  # [B,J,12]
        S = int(self.model_parms.query_posmap_size)
        dec = self.net.forward_packed(self.geo_feature, S, B)                                             # [S*S, 8]
        scale_mul = 1e-3 * iteration if (ramp and iteration < 1000) else 1.0                              # avatar_model.py:316-319
        means, scales, colors = LbsAssemble.apply(dec, cano2live, self.valid_index, self._query_points, self._query_lbs, scale_mul)
        return means, scales, colors, dec

    def _render_one(self, batch_data, means, scales, colors, b):
        return render_batch(points=means[b], shs=None, colors_precomp=colors[b], rotations=self.fix_rotation,
                            scales=scales[b], opacity=self.fix_opacity, FovX=batch_data["FovX"][b], FovY=batch_data["FovY"][b],
                            height=batch_data["height"][b], width=batch_data["width"][b], bg_color=self.background,
                            world_view_transform=batch_data["world_view_transform"][b],
                            full_proj_transform=batch_data["full_proj_transform"][b], active_sh_degree=0,
                            camera_center=batch_data["camera_center"][b])

    # ---- batched rasterization: every frame of the step in one set of launches, no host read-back -------------------------------
    @staticmethod
    def _scalar_list(v, B):
        """Per-frame python numbers of a batch field (a list, or a CPU / CUDA tensor after the reference's collate + to_cuda)."""
        if torch.is_tensor(v):
            return v.reshape(-1)[:B].tolist()          # a CUDA tensor costs one host sync (the reference's own loop reads them too)
        return [float(x) for x in list(v)[:B]]

    def _batch_cameras(self, batch_data, B, dev):
        """[B,40] camera block for ga_rasterb_* (view, proj, tan(Fov/2)); the tangent pair is cached per Fov tuple."""
        import math
        from .rasterizer import CAM_STRIDE
        fx, fy = batch_data["FovX"], batch_data["FovY"]
        if torch.is_tensor(fx) and fx.is_cuda:
            tans = torch.stack([torch.tan(fx.double() * 0.5), torch.tan(fy.double() * 0.5)], 1).float()
        else:
            key = (tuple(self._scalar_list(fx, B)), tuple(self._scalar_list(fy, B)))
            cache = self.__dict__.setdefault("_tan_cache", {})
            tans = cache.get(key)
            if tans is None:
                tans = torch.tensor([[math.tan(a * 0.5), math.tan(b * 0.5)] for a, b in zip(*key)], dtype=torch.float32).to(dev)
                if len(cache) < 64:
                    cache[key] = tans
        cams = torch.zeros(B, CAM_STRIDE, dtype=torch.float32, device=dev)
        view, proj = batch_data["world_view_transform"], batch_data["full_proj_transform"]
        if not torch.is_tensor(view):
            view, proj = torch.stack(list(view)[:B]), torch.stack(list(proj)[:B])
        cams[:, 0:16] = view.reshape(B, 16)
        cams[:, 16:32] = proj.reshape(B, 16)
        cams[:, 32:34] = tans
        return cams

    def raster_plan(self, B, P, H, W):
        from .rasterizer import RasterBatchPlan
        plans = self.__dict__.setdefault("_raster_plans", {})
        key = (int(B), int(P), int(H), int(W))
        if key not in plans:
            plans[key] = RasterBatchPlan(B, P, H, W, self.device)
        return plans[key]

    def raster_ok(self, wait=True) -> bool:
        """False if the last batched render overflowed its binning buffer (the buffer has then been grown: run it again)."""
        plan = getattr(self, "_last_plan", None)
        return True if plan is None else plan.check(wait)

    def _render_batched(self, batch_data, means, scales, colors):
        from .rasterizer import rasterize_batch
        B, P = int(means.shape[0]), int(means.shape[1])
        H, W = int(self._scalar_list(batch_data["height"], 1)[0]), int(self._scalar_list(batch_data["width"], 1)[0])
        cams = batch_data["_cams"] if "_cams" in batch_data else self._batch_cameras(batch_data, B, means.device)
        plan = self.raster_plan(B, P, H, W)
        self._last_plan = plan
        images = rasterize_batch(means, colors, scales, self.fix_rotation, self.fix_opacity, cams, self.background, plan)
        if (not torch.is_grad_enabled() and not torch.cuda.is_current_stream_capturing() and not getattr(self, "defer_raster_check", False)
                and not plan.check(wait=True)):          # inference: make the result right before returning it (unless the caller checks later)
            images = rasterize_batch(means, colors, scales, self.fix_rotation, self.fix_opacity, cams, self.background, plan)
            if not plan.check(wait=True):
                raise RuntimeError("batched rasterizer: binning buffer overflowed twice in a row")
        return images

    def _uniform_frames(self, batch_data, B):
        h, w = self._scalar_list(batch_data["height"], B), self._scalar_list(batch_data["width"], B)
        return len(set(h)) == 1 and len(set(w)) == 1

    def _render_frames(self, batch_data, means, scales, colors):
        if means.is_cuda and means.shape[0] <= 8 and self._uniform_frames(batch_data, means.shape[0]):
            return self._render_batched(batch_data, means, scales, colors)
        return self._render_frames_one_by_one(batch_data, means, scales, colors)

    def _render_frames_one_by_one(self, batch_data, means, scales, colors):
        """The reference rasterizes the frames of a batch one after the other (avatar_model.py:332-365).  Frames are independent, and
        the compositing kernels end in a long tail of a few crowded tiles, so consecutive frames go to two alternating side
        streams: frame b+1's preprocess / sort (and, in the backward, its replay) fill the SMs frame b's tail leaves idle.
        autograd runs each frame's backward on the stream of its forward."""
        B = means.shape[0]
        if B < 2 or not means.is_cuda:
            return torch.stack([self._render_one(batch_data, means, scales, colors, b) for b in range(B)], dim=0)
        main = torch.cuda.current_stream()
        if getattr(self, "_frame_streams", None) is None:
            self._frame_streams = [torch.cuda.Stream(device=means.device) for _ in range(2)]
        ready = torch.cuda.Event()
        ready.record(main)
        images = []
        for b in range(B):
            s = self._frame_streams[b % 2]
            s.wait_event(ready)                       # means / scales / colours were produced on the main stream
            with torch.cuda.stream(s):
                img = self._render_one(batch_data, means, scales, colors, b)
            img.record_stream(main)
            images.append(img)
        for s in self._frame_streams[:min(B, 2)]:
            for t in (means, scales, colors):
                t.record_stream(s)
            main.wait_stream(s)
        return torch.stack(images, dim=0)

    def train_stage1(self, batch_data, iteration):
        """model/avatar_model.py:272-367: returns (images [B,3,H,W], full_pred [B,N,3], offset_loss, geo_loss, scale_loss)."""
        idx = batch_data["pose_idx"]
        means, scales, colors, dec = self._posed_gaussians(idx, iteration, rest_pose=batch_data.get("rest_pose"))
        # regularisers exactly as the reference forms them (avatar_model.py:328-330): mean over ALL S*S pixels of
        # (0.02 res)^2 (identical for every frame of the batch), mean of the repeated scales, mean of geo_feature^2
        offset_loss = torch.mean((dec[:, :3] * 0.02) ** 2)
        geo_loss = torch.mean(self.geo_feature ** 2)
        scale_loss = torch.mean(scales)
        self._last_gaussians = (means, scales, colors)      # parity tests read the rasterizer's inputs / their gradients here
        images = self._render_frames(batch_data, means, scales, colors)
        return images, means, offset_loss, geo_loss, scale_loss

    def _stage2_gaussians(self, batch_data):
        """Stage 2 (model/avatar_model.py:369-420 / :557-612): the pose encoder turns each frame's posed-body position map into a
        feature map that is ADDED to the geometry features, so the decoder runs per frame (B*S*S rows, BatchNorm statistics over all of
        them); no scale ramp in this stage."""
        inp = batch_data.get("inp_pos_map")
        inp = self._pose_map(batch_data) if inp is None else inp.to(self.device).float()
        idx = batch_data["pose_idx"]
        cano2live = self._cano2live(self.pose(idx), self.transl(idx), batch_data.get("rest_pose"))
        S = int(self.model_parms.query_posmap_size)
        pose_featmap = self.pose_encoder(inp)                                                         # [B,64,h,h]
        dec = self.net.forward_packed_frames(self.geo_feature, pose_featmap, S)                      # [B*S*S, 8]
        means, scales, colors = LbsAssemble.apply(dec, cano2live, self.valid_index, self._query_points, self._query_lbs, 1.0, True)
        return means, scales, colors, dec, pose_featmap

    def _pose_map(self, batch_data):
        """Input position maps [B,3,s,s] of a batch that carries none: from its `pose_data` / `transl_data` when it has them (test,
        novel pose), else from the model's pose / transl rows at `pose_idx` (in stage 2 those are smpl_parms_pred.pth, never stepped)."""
        if self.pose_mapper is None:
            raise KeyError("inp_pos_map: the batch has no stage-2 input position map (set ModelParams.inp_posmap_from_pose to build it "
                           "from the pose)")
        if "pose_data" in batch_data:
            pose, transl = batch_data["pose_data"], batch_data["transl_data"]
        else:
            idx = torch.as_tensor(batch_data["pose_idx"], device=self.device).long()
            pose, transl = self.pose.weight.detach()[idx], self.transl.weight.detach()[idx]
        return self.pose_mapper(pose, transl)

    def train_stage2(self, batch_data, iteration):
        """model/avatar_model.py:369-463: returns (images [B,3,H,W], full_pred [B,N,3], pose_loss, offset_loss)."""
        means, scales, colors, dec, pose_featmap = self._stage2_gaussians(batch_data)
        offset_loss = torch.mean((dec[:, :3] * 0.02) ** 2)          # mean over B x S*S x 3 (avatar_model.py:424)
        pose_loss = torch.mean(pose_featmap ** 2)
        self._last_gaussians = (means, scales, colors)
        images = self._render_frames(batch_data, means, scales, colors)
        return images, means, pose_loss, offset_loss

    def render_free_stage1(self, batch_data, iteration):
        """model/avatar_model.py:467-554: same forward minus the losses (BatchNorm still uses batch statistics).

        In stage 1 the feature net's inputs (geo_feature, the uv grid) do not depend on the frame, so its output is the same for every
        frame the reference renders (SURVEY.md §3.2 / §8e): a model built for inference (`train=False`, what eval.py /
        render_novel_pose.py construct) evaluates the net ONCE and reuses the packed output until parameters are loaded again
        (`cache_decoder`).  Per frame that leaves SMPL -> LBS -> rasterizer.  Only the BatchNorm running statistics (never used for
        normalisation by the reference's scripts) stop being updated by the skipped evaluations."""
        S = int(self.model_parms.query_posmap_size)
        if "pose_data" in batch_data:      # novel-pose datasets carry the pose instead of an embedding index
            pose_batch, transl_batch = batch_data["pose_data"].float(), batch_data["transl_data"].float()
        else:
            idx = batch_data["pose_idx"]
            pose_batch, transl_batch = self.pose(idx), self.transl(idx)
        B = pose_batch.shape[0]
        cano2live = self._cano2live(pose_batch, transl_batch, batch_data.get("rest_pose"))
        cached = getattr(self, "_dec_cache", None)
        if self.cache_decoder and not torch.is_grad_enabled() and cached is not None:
            dec = cached
        else:
            dec = self.net.forward_packed(self.geo_feature, S, B)
            if self.cache_decoder and not torch.is_grad_enabled():
                self._dec_cache = dec.detach()
        scale_mul = 1e-3 * iteration if iteration < 1000 else 1.0
        means, scales, colors = LbsAssemble.apply(dec, cano2live, self.valid_index, self._query_points, self._query_lbs, scale_mul)
        return self._render_frames(batch_data, means, scales, colors)

    def invalidate_decoder_cache(self):
        self._dec_cache = None

    def render_free_stage2(self, batch_data, iteration):
        """model/avatar_model.py:557-649: the stage-2 forward without the losses."""
        means, scales, colors, _, _ = self._stage2_gaussians(batch_data)
        return self._render_frames(batch_data, means, scales, colors)


def smplx_rest_joints(npz_path, beta, parents) -> torch.Tensor:
    """Rest joints J = J_regressor (v_template + shapedirs[:, :, :10] beta) [55,3] of an SMPLX_{GENDER}.npz.  The file's
    kintree_table must be the SMPL-X tree the joint-transform kernel is built for."""
    sm = np.load(npz_path, allow_pickle=True)
    kt = np.asarray(sm["kintree_table"]).astype(np.int64)[0].copy()
    kt[0] = -1
    if kt.shape != (len(parents),) or not np.array_equal(kt, np.asarray(parents)):
        raise ValueError(f"{npz_path}: kintree_table[0] is not the 55-joint SMPL-X tree this library is built for")
    beta = torch.as_tensor(beta).double().reshape(-1)
    v_t = torch.as_tensor(np.asarray(sm["v_template"])).double()
    sd = torch.as_tensor(np.asarray(sm["shapedirs"])[:, :, :beta.numel()]).double()
    Jr = sm["J_regressor"]
    Jr = torch.as_tensor(np.asarray(Jr.todense() if hasattr(Jr, "todense") else Jr)).double()
    return (Jr @ (v_t + torch.einsum("l,mkl->mk", beta, sd))).float()
