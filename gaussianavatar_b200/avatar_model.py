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

import contextlib
import os
from os.path import join

import numpy as np
import torch
import torch.nn as nn

from .body import SMPLX, body_of, load_model
from .config import ModelParams, NetworkParams, OptimizationParams
from .network import POP_no_unet
from .ops import Cano2Live, LbsAssemble
from .rasterizer import MAX_FRAMES_PER_CALL
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
        # every render of this avatar (training, render_free_*, the depth pass and the tools that take the model) uses the mode
        self.antialiasing = bool(getattr(model_parms, "antialiasing", False))
        self.body = body_of(model_parms.smpl_type)
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
        J = self.body.joints
        lbs = _assets["query_lbs"].to(dev).float()
        if tuple(lbs.shape) != (N, J):
            raise ValueError(f"query_lbs {tuple(lbs.shape)}: expected [{N},{J}] for smpl_type={model_parms.smpl_type!r}")
        lbs = torch.nn.functional.pad(lbs, (0, self.body.lbs_ld - J))                  # zero columns up to the LBS kernel's row width
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
        pose_dim = self.body.pose_width                 # SMPL-X: global + 21 body joints are trained, the rest comes with the frame
        if _pose_data.shape[1] != pose_dim:
            raise ValueError(f"pose data {tuple(_pose_data.shape)}: expected [F,{pose_dim}] for smpl_type={model_parms.smpl_type!r}")
        self.pose = torch.nn.Embedding(num_training_frames, pose_dim, _weight=_pose_data.clone().float(), sparse=True).to(dev)
        self.transl = torch.nn.Embedding(num_training_frames, 3, _weight=_transl_data.clone().float(), sparse=True).to(dev)
        self.optimizer_pose = torch.optim.SparseAdam(list(self.pose.parameters()) + list(self.transl.parameters()), 5.0e-3)
        # per-training-frame colour transform [A | t] (ModelParams.train_exposure), identity at the start; row 0 is the gauge anchor and
        # never moves (DESIGN.md §4)
        self.exposure = None
        self.exposure_optimizer = None
        if bool(getattr(model_parms, "train_exposure", False)):
            self.exposure = nn.Parameter(identity_exposure(num_training_frames, dev))
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
        """assets: gaussianavatar_b200.synthetic.SyntheticAvatarAssets (or a dict with the same fields; without `smpl_type` the body
        is SMPL).  An SMPL-X model's frames carry `rest_pose`.  model_fields override ModelParams fields (e.g. train_stage=2,
        inp_posmap_size, inp_posmap_from_pose=True; the last needs the dict keys `smpl_mesh`, the SMPL_{GENDER}.pkl fields, and
        `uv_template`, a path or what posmap.load_uv_template_obj returns)."""
        if not isinstance(assets, dict):
            assets = dict(valid_idx=assets.valid_idx, query_points=assets.query_points, query_lbs=assets.query_lbs,
                          cano_joint_mats=assets.cano_joint_mats, rest_joints=assets.rest_joints, betas=assets.body.betas[0], S=assets.S,
                          smpl_type=assets.smpl_type)
        mp = ModelParams(batch_size=batch_size, query_posmap_size=int(assets["S"]), smpl_type=assets.get("smpl_type", "smpl"), **model_fields)
        return cls(mp, net_parms or NetworkParams(), opt_parms or OptimizationParams(), train=train, _assets=assets, _frames=frames,
                   _pose_data=pose_data, _transl_data=transl_data, device=device)

    def _load_reference_assets(self, mp, train):
        """Folder contract of the reference (model/avatar_model.py:41-98; scene/dataset_mono.py:83-160): the training dataset (always
        built, even for evaluation, avatar_model.py:41), the UV mask / canonical position map / LBS map / canonical joint
        matrices of the body (`uv_mask{S}_with_faceid_{body}.npy`, `query_posemap_{S}_cano_{body}.npz`, `lbs_map_{body}_{S}.npy`,
        `{body}_cano_joint_mat.pth`), and the body-model file (SMPL_{GENDER}.pkl under smpl_model_path, SMPLX_{GENDER}.npz under
        smplx_model_path) for the rest joints J(beta).  Exercised against a synthetic folder written in the same layout
        (tests/test_dataset_cpu.py, tests/test_avatar_gpu.py)."""
        from .dataset import MonoDataset_train
        split = "train" if train else "test"
        dataset = MonoDataset_train(mp)
        S, body = int(mp.query_posmap_size), self.body
        n, J = body.name, body.joints
        mask = np.load(join(mp.project_path, "assets", "uv_masks", f"uv_mask{S}_with_faceid_{n}.npy")).reshape(S, S)
        valid = torch.from_numpy(mask != -1).reshape(-1)
        qmap = torch.from_numpy(np.load(join(mp.source_path, split, f"query_posemap_{S}_cano_{n}.npz"))[f"posmap{S}"]).reshape(-1, 3)
        lbs = torch.from_numpy(np.load(join(mp.project_path, "assets", f"lbs_map_{n}_{S}.npy"))).reshape(S * S, J)
        cano = torch.as_tensor(torch.load(join(mp.source_path, split, f"{n}_cano_joint_mat.pth"), weights_only=False)).reshape(J, 4, 4).float()
        beta = torch.as_tensor(dataset.smpl_data["beta"][0]).float()
        model = load_model(join(getattr(mp, body.model_dir), body.model_file.format(gender=mp.smpl_gender.upper())))
        assets = dict(valid_idx=valid, query_points=qmap[valid].float(), query_lbs=lbs[valid].float(), cano_joint_mats=cano,
                      rest_joints=body.rest_joints(model, beta), betas=beta, S=S)
        if mp.train_stage == 2 and getattr(mp, "inp_posmap_from_pose", False):
            # the mesh comes from the same model file as the rest joints; the UV template from where the reference's scripts read it
            body.check_model(model)
            template = join(mp.project_path, "assets", f"template_mesh_{n}_uv.obj")
            if not os.path.exists(template):
                raise FileNotFoundError(f"inp_posmap_from_pose: UV template {template} not found")
            assets.update(smpl_mesh=model, uv_template=template)
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
        self.exposure_setup()

    def exposure_schedule_steps(self, world: int = 1) -> int:
        """Steps of the stage one process takes: epochs x its batches per epoch (the frames split over `world` data-parallel ranks)."""
        batches = len(self.train_dataset) // max(int(self.batch_size) * max(int(world), 1), 1)
        return int(getattr(self.opt_parms, "epochs", 1)) * max(batches, 1)

    def exposure_setup(self, world: int = 1):
        """The exposure table's own Adam (ModelParams.train_exposure): its rate falls log-linearly over the stage's steps
        (`exposure_schedule_steps`)."""
        if self.exposure is None:
            return
        from .optim import ExposureAdam
        op = self.opt_parms
        self.exposure_optimizer = ExposureAdam(self.exposure, self.exposure_schedule_steps(world), float(getattr(op, "exposure_lr_init", 0.01)),
                                               float(getattr(op, "exposure_lr_final", 0.001)))

    def _exposure_state(self):
        """Checkpoint entries of the exposure table: {} when the model does not train one."""
        if self.exposure is None:
            return {}
        out = {"exposure": self.exposure.detach().clone()}
        if self.exposure_optimizer is not None:
            out["exposure_optimizer"] = self.exposure_optimizer.state_dict()
        return out

    def _load_exposure(self, saved, optimizer=True):
        """The checkpoint's exposure table, or identity when it has none (reference checkpoints, ones written without the table)."""
        if self.exposure is None:
            return
        table = saved.get("exposure")
        with torch.no_grad():
            if table is None:
                self.exposure.copy_(identity_exposure(self.exposure.shape[0], self.device))
            else:
                table = torch.as_tensor(table).detach().float()
                if tuple(table.shape) != tuple(self.exposure.shape):
                    raise ValueError(f"checkpoint exposure {tuple(table.shape)}: expected {tuple(self.exposure.shape)}")
                self.exposure.copy_(table)
        if optimizer and self.exposure_optimizer is not None and "exposure_optimizer" in saved:
            self.exposure_optimizer.load_state_dict(saved["exposure_optimizer"])

    def save(self, iteration):
        path = os.path.join(self.model_path, "net/iteration_{}".format(iteration))
        os.makedirs(path, exist_ok=True)
        if self.model_parms.train_stage == 2:                      # avatar_model.py:177-186
            torch.save({"pose_encoder": self.pose_encoder.state_dict(), "geo_feature": self.geo_feature, "pose": self.pose.state_dict(),
                        "transl": self.transl.state_dict(), "net": self.net.state_dict(), "optimizer": self.optimizer.state_dict(),
                        "scheduler": self.scheduler.state_dict(), **self._exposure_state()}, os.path.join(path, "pose_encoder.pth"))
            return
        torch.save({"net": self.net.state_dict(), "geo_feature": self.geo_feature, "pose": self.pose.state_dict(),
                    "transl": self.transl.state_dict(), "optimizer": self.optimizer.state_dict(),
                    "scheduler": self.scheduler.state_dict(), **self._exposure_state()}, os.path.join(path, "net.pth"))

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
            if not test:
                self._load_exposure(saved)
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
        self._load_exposure(saved, optimizer=False)      # stage 1's table carries into stage 2; its Adam state does not

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
        self._load_exposure(saved)
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
        if self.exposure is not None:
            self.exposure.grad = None
        if self.model_parms.train_stage == 1 and epoch > self.opt_parms.pose_op_start_iter:     # avatar_model.py:258-262
            self.optimizer_pose.zero_grad()

    def step(self, epoch):
        self.optimizer.step()
        self.scheduler.step()
        if self.exposure_optimizer is not None:         # from the first step on, not only after pose_op_start_iter
            self.exposure_optimizer.step()
        if self.model_parms.train_stage == 1 and epoch > self.opt_parms.pose_op_start_iter:     # avatar_model.py:263-270
            self.optimizer_pose.step()

    # ------------------------------------------------------------------------------------------------------------------
    @property
    def smplx(self) -> bool:
        return self.body is SMPLX

    def _cano2live(self, pose_batch, transl_batch, rest_pose=None):
        """[B,J,12] for the body model: SMPL from pose [B,72]; SMPL-X from pose [B,66] and the frames' rest_pose [B,99]."""
        return Cano2Live.apply(self.body, pose_batch, rest_pose, transl_batch, self._rest_joints, self._inv_cano)

    def _assemble(self, dec, pose, transl, rest_pose=None, scale_mul=1.0, per_frame=False, placement=None, exposure=None, exposure_idx=None):
        """Decoder output `dec` posed by pose / transl (and SMPL-X's rest_pose): cano2live, then the fused LBS / attribute assembly.
        Returns means3D, scales, colors [B,N,3].  per_frame: `dec` holds one [S*S,8] block per frame (stage 2).  placement: a
        `scene.Placement` folded into cano2live, its scale into the LBS scale multiplier (the Gaussians are isotropic).  exposure
        [F,3,4] with exposure_idx [B]: frame b's colours become A c + t, [A | t] = exposure[exposure_idx[b]] (None: identity)."""
        cano2live = self._cano2live(pose, transl, rest_pose)                                              # [B,J,12]
        if placement is not None:
            cano2live = placement.fold(cano2live)
            scale_mul = scale_mul * placement.scale
        return LbsAssemble.apply(dec, cano2live, self.valid_index, self._query_points, self._query_lbs, scale_mul, per_frame, exposure,
                                 exposure_idx)

    def _batch_exposure(self, batch_data):
        """(table [B,3,4], rows [B]) of a batch whose items carry a fitted `exposure` [3,4] (test frames), else (None, None)."""
        e = batch_data.get("exposure")
        if e is None:
            return None, None
        e = torch.as_tensor(e).to(device=self.device, dtype=torch.float32).reshape(-1, 3, 4).contiguous()
        return e, torch.arange(e.shape[0], device=self.device, dtype=torch.int32)

    def _stage1_decoder(self, batch):
        """Stage 1's frame-invariant decoder output [S*S,8], its BatchNorm statistics taken over `batch` frames.  With `cache_decoder`
        set and grad off it is evaluated once and reused until parameters are loaded again."""
        cache = self.cache_decoder and not torch.is_grad_enabled()
        if cache and self._dec_cache is not None:
            return self._dec_cache
        dec = self.net.forward_packed(self.geo_feature, int(self.model_parms.query_posmap_size), batch)
        if cache:
            self._dec_cache = dec.detach()
        return dec

    def _posed_gaussians(self, idx, iteration, ramp=True, rest_pose=None):
        """SMPL / SMPL-X -> cano2live -> net (once) -> fused LBS/assembly.  Returns means3D, scales, colors [B,N,3] and dec_out."""
        if getattr(self, "_detach_pose", False):      # pose optimisation inactive (epoch <= pose_op_start_iter): its gradients are never read
            pose_batch, transl_batch = self.pose.weight.detach()[idx], self.transl.weight.detach()[idx]
        else:
            pose_batch = self.pose(idx)
            transl_batch = self.transl(idx)
        S = int(self.model_parms.query_posmap_size)
        dec = self.net.forward_packed(self.geo_feature, S, pose_batch.shape[0])                           # [S*S, 8]
        scale_mul = 1e-3 * iteration if (ramp and iteration < 1000) else 1.0                              # avatar_model.py:316-319
        means, scales, colors = self._assemble(dec, pose_batch, transl_batch, rest_pose, scale_mul, exposure=self.exposure,
                                               exposure_idx=idx if self.exposure is not None else None)
        return means, scales, colors, dec

    def _render_one(self, batch_data, means, scales, colors, b):
        return render_batch(points=means[b], shs=None, colors_precomp=colors[b], rotations=self.fix_rotation,
                            scales=scales[b], opacity=self.fix_opacity, FovX=batch_data["FovX"][b], FovY=batch_data["FovY"][b],
                            height=batch_data["height"][b], width=batch_data["width"][b], bg_color=self.background,
                            world_view_transform=batch_data["world_view_transform"][b],
                            full_proj_transform=batch_data["full_proj_transform"][b], active_sh_degree=0,
                            camera_center=batch_data["camera_center"][b], antialiasing=self.antialiasing)

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
            plans[key] = RasterBatchPlan(B, P, H, W, self.device, antialiasing=self.antialiasing)
        return plans[key]

    def raster_ok(self, wait=True) -> bool:
        """False if the last batched render overflowed its binning buffer (the buffer has then been grown: run it again)."""
        plan = getattr(self, "_last_plan", None)
        return True if plan is None else plan.check(wait)

    def _render_batched(self, batch_data, means, scales, colors, depth=False):
        """depth: render through rasterize_batch_with_depth and keep its differentiable depth pass [B,2,H,W] in `last_depth`."""
        from .rasterizer import rasterize_batch, rasterize_batch_with_depth
        B, P = int(means.shape[0]), int(means.shape[1])
        H, W = int(self._scalar_list(batch_data["height"], 1)[0]), int(self._scalar_list(batch_data["width"], 1)[0])
        cams = batch_data["_cams"] if "_cams" in batch_data else self._batch_cameras(batch_data, B, means.device)
        plan = self.raster_plan(B, P, H, W)
        self._last_plan = plan

        def render():
            if not depth:
                return rasterize_batch(means, colors, scales, self.fix_rotation, self.fix_opacity, cams, self.background, plan)
            images, self.last_depth = rasterize_batch_with_depth(means, colors, scales, self.fix_rotation, self.fix_opacity, cams,
                                                                 self.background, plan)
            return images
        if torch.is_grad_enabled() or torch.cuda.is_current_stream_capturing() or getattr(self, "defer_raster_check", False):
            return render()
        return plan.render_checked(render, "AvatarModel")[0]    # inference: make the result right before returning it

    def _uniform_frames(self, batch_data, B):
        h, w = self._scalar_list(batch_data["height"], B), self._scalar_list(batch_data["width"], B)
        return len(set(h)) == 1 and len(set(w)) == 1

    def _render_frames(self, batch_data, means, scales, colors, depth=False):
        if means.is_cuda and means.shape[0] <= MAX_FRAMES_PER_CALL and self._uniform_frames(batch_data, means.shape[0]):
            return self._render_batched(batch_data, means, scales, colors, depth)
        if depth:
            raise RuntimeError(f"training against depth maps needs the batched rasterizer: at most {MAX_FRAMES_PER_CALL} CUDA frames of one "
                               "size per batch (the one-frame-at-a-time path renders no depth)")
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
        """model/avatar_model.py:272-367: returns (images [B,3,H,W], full_pred [B,N,3], offset_loss, geo_loss, scale_loss).  A batch
        with `depth` (ModelParams.depth_maps) also leaves the differentiable depth pass [B,2,H,W] in `last_depth`."""
        idx = batch_data["pose_idx"]
        means, scales, colors, dec = self._posed_gaussians(idx, iteration, rest_pose=batch_data.get("rest_pose"))
        # regularisers exactly as the reference forms them (avatar_model.py:328-330): mean over ALL S*S pixels of
        # (0.02 res)^2 (identical for every frame of the batch), mean of the repeated scales, mean of geo_feature^2
        offset_loss = torch.mean((dec[:, :3] * 0.02) ** 2)
        geo_loss = torch.mean(self.geo_feature ** 2)
        scale_loss = torch.mean(scales)
        self._last_gaussians = (means, scales, colors)      # parity tests read the rasterizer's inputs / their gradients here
        images = self._render_frames(batch_data, means, scales, colors, depth=batch_data.get("depth") is not None)
        return images, means, offset_loss, geo_loss, scale_loss

    def _stage2_gaussians(self, batch_data, pose=None, transl=None, placement=None, exposure=None, exposure_idx=None):
        """Stage 2 (model/avatar_model.py:369-420 / :557-612): the pose encoder turns each frame's posed-body position map into a
        feature map that is ADDED to the geometry features, so the decoder runs per frame (B*S*S rows, BatchNorm statistics over all of
        them); no scale ramp in this stage.  The skeleton is posed with the model's pose / transl rows at `pose_idx`, as the reference
        does, unless `pose` [B,72|66] and `transl` [B,3] are given (the animation player's sampled poses).  exposure / exposure_idx:
        as `_assemble` takes them."""
        inp = batch_data.get("inp_pos_map")
        inp = self._pose_map(batch_data) if inp is None else inp.to(self.device).float()
        if pose is None:
            idx = batch_data["pose_idx"]
            pose, transl = self.pose(idx), self.transl(idx)
        S = int(self.model_parms.query_posmap_size)
        pose_featmap = self.pose_encoder(inp)                                                         # [B,64,h,h]
        dec = self.net.forward_packed_frames(self.geo_feature, pose_featmap, S)                      # [B*S*S, 8]
        means, scales, colors = self._assemble(dec, pose, transl, batch_data.get("rest_pose"), per_frame=True, placement=placement,
                                               exposure=exposure, exposure_idx=exposure_idx)
        return means, scales, colors, dec, pose_featmap

    def _stage2_from_pose(self, mapper, pose, transl, rest_pose=None, placement=None, exposure=None, exposure_idx=None):
        """`_stage2_gaussians` of explicit poses [B,72|66] / transl [B,3] (and SMPL-X's rest_pose [B,99]): the input position maps are
        built from the same pose by `mapper` (a posmap.PoseMapper / SmplxPoseMapper, differentiable in pose and transl).  placement
        moves the posed Gaussians into a scene (`_assemble`); the position maps stay in the body's own frame."""
        inp = mapper.maps(pose, rest_pose, transl)
        return self._stage2_gaussians({"inp_pos_map": inp, "rest_pose": rest_pose}, pose=pose, transl=transl, placement=placement,
                                      exposure=exposure, exposure_idx=exposure_idx)

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
        """model/avatar_model.py:369-463: returns (images [B,3,H,W], full_pred [B,N,3], pose_loss, offset_loss); `last_depth` as
        train_stage1 leaves it."""
        if self.exposure is not None:
            means, scales, colors, dec, pose_featmap = self._stage2_gaussians(batch_data, exposure=self.exposure,
                                                                              exposure_idx=batch_data["pose_idx"])
        else:
            means, scales, colors, dec, pose_featmap = self._stage2_gaussians(batch_data)
        offset_loss = torch.mean((dec[:, :3] * 0.02) ** 2)          # mean over B x S*S x 3 (avatar_model.py:424)
        pose_loss = torch.mean(pose_featmap ** 2)
        self._last_gaussians = (means, scales, colors)
        images = self._render_frames(batch_data, means, scales, colors, depth=batch_data.get("depth") is not None)
        return images, means, pose_loss, offset_loss

    def render_free_stage1(self, batch_data, iteration):
        """model/avatar_model.py:467-554: same forward minus the losses (BatchNorm still uses batch statistics).

        In stage 1 the feature net's inputs (geo_feature, the uv grid) do not depend on the frame, so its output is the same for every
        frame the reference renders (SURVEY.md §3.2 / §8e): a model built for inference (`train=False`, what eval.py /
        render_novel_pose.py construct) evaluates the net ONCE and reuses the packed output until parameters are loaded again
        (`cache_decoder`).  Per frame that leaves SMPL -> LBS -> rasterizer.  Only the BatchNorm running statistics (never used for
        normalisation by the reference's scripts) stop being updated by the skipped evaluations."""
        if "pose_data" in batch_data:      # novel-pose datasets carry the pose instead of an embedding index
            pose_batch, transl_batch = batch_data["pose_data"].float(), batch_data["transl_data"].float()
        else:
            idx = batch_data["pose_idx"]
            pose_batch, transl_batch = self.pose(idx), self.transl(idx)
        dec = self._stage1_decoder(pose_batch.shape[0])
        scale_mul = 1e-3 * iteration if iteration < 1000 else 1.0
        table, rows = self._batch_exposure(batch_data)
        means, scales, colors = self._assemble(dec, pose_batch, transl_batch, batch_data.get("rest_pose"), scale_mul, exposure=table,
                                               exposure_idx=rows)
        return self._render_frames(batch_data, means, scales, colors)

    def invalidate_decoder_cache(self):
        self._dec_cache = None

    def render_free_stage2(self, batch_data, iteration):
        """model/avatar_model.py:557-649: the stage-2 forward without the losses."""
        table, rows = self._batch_exposure(batch_data)
        means, scales, colors, _, _ = self._stage2_gaussians(batch_data, exposure=table, exposure_idx=rows)
        return self._render_frames(batch_data, means, scales, colors)


def identity_exposure(frames: int, device="cuda") -> torch.Tensor:
    """[frames,3,4] of [I | 0]: every frame's colours as the decoder makes them."""
    return torch.eye(3, 4, device=device, dtype=torch.float32).repeat(int(frames), 1, 1).contiguous()


@contextlib.contextmanager
def kept_state(model):
    """Restores the model's BatchNorm statistics (running buffers and batch counts) on exit: rendering or fitting poses through a
    trained avatar must not change what `save()` writes."""
    net = model.net
    run = net.bn_running.detach().clone()
    counts = {k: st.num_batches_tracked for k, st in net._states.items()}
    enc = getattr(model, "pose_encoder", None)
    bufs = [(b, b.detach().clone()) for b in enc.buffers()] if enc is not None else []
    try:
        yield
    finally:
        with torch.no_grad():
            net.bn_running.copy_(run)
            for k, st in net._states.items():
                st.num_batches_tracked = counts.get(k, 0)
            for b, v in bufs:
                b.copy_(v)

