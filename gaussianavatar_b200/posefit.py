"""Test-time pose fitting: the SMPL / SMPL-X pose and translation of frames a trained avatar was not trained on, refined so that the
avatar's render matches each frame's image.

    fitter = PoseFitter(model, iters=100, lr=5e-3, pose_mapper=mapper)      # mapper: stage 2 only (posmap.PoseMapper / SmplxPoseMapper)
    pose, transl, report = fitter.fit([test_dataset[i] for i in range(len(test_dataset))])

Stage 1 refines only the training frames' poses; a test split keeps the poses it came with (raw estimates on a user's own capture),
so eval.py's metrics measure pose error as much as appearance.  The fit holds the avatar, the betas, the camera and SMPL-X's
rest_pose fixed and, per frame, runs plain Adam on pose (72, or SMPL-X's 66) and transl against the training image loss
(1 - lambda) L1 + lambda (1 - SSIM) (`losses.image_loss`, lambda = opt.lambda_dssim) on the model's background.  No prior, no
coupling between frames.  With `exposure=True` each frame's colour transform [A | t] (DESIGN.md §4) is fitted with its pose, from
identity, by its own Adam (the training table's learning-rate schedule over the fit's steps).  A frame's result is its lowest-loss iterate, counting the initial pose as iterate 0 and evaluating once
more after the last step, so its fitted loss is never above its initial loss.

Stage 1 evaluates the frame-invariant decoder once and fits chunks of up to 8 frames through cano2live -> LBS -> the batched
rasterizer; the Adam update (`ga_adam_step_dev`) takes the rasterizer's overflow word as its skip flag, and a chunk that overflowed
the binning buffer at any iteration is fitted again from its initial poses after the buffer has grown.  Stage 2 fits one frame per
decoder forward (its BatchNorm uses the batch's statistics): the input position map is built from the current pose by the
differentiable mapper, so the gradient reaches the pose through the map as well as through the skeleton.  The model's parameters,
BatchNorm statistics and batch counts are left as they were, and nothing is stored on the model but stage 1's decoder cache.
"""
from __future__ import annotations

import math

import torch

from . import _lib
from ._lib import ptr
from .avatar_model import kept_state
from .losses import image_loss
from .rasterizer import MAX_FRAMES_PER_CALL, RasterBatchPlan, rasterize_batch

BETAS = (0.9, 0.999)   # torch.optim.Adam's defaults, as the training pose optimiser uses them
EPS = 1e-8


class PoseFitter:
    """model: an `AvatarModel` (stage 1 or 2).  iters: Adam steps per frame.  lr: Adam's learning rate (the training pose optimiser's
    by default).  pose_mapper: stage 2's `posmap.PoseMapper` / `SmplxPoseMapper` (default: the model's own).  chunk: frames per
    stage-1 rasterizer call (1..8).  capacity: initial binning capacity of the rasterizer (instances); it grows on overflow.  exposure:
    also fit each frame's [A | t]; `fit` then returns the table [F,3,4] as a fourth value."""

    def __init__(self, model, iters: int = 100, lr: float = 5e-3, pose_mapper=None, chunk: int = MAX_FRAMES_PER_CALL, capacity=None,
                 exposure: bool = False):
        if int(iters) < 0:
            raise ValueError(f"iters {iters} is negative")
        if not (lr > 0 and math.isfinite(lr)):
            raise ValueError(f"lr {lr} is not a positive number")
        if not 1 <= int(chunk) <= MAX_FRAMES_PER_CALL:
            raise ValueError(f"chunk {chunk} outside 1..{MAX_FRAMES_PER_CALL}")
        self.model = model
        self.exposure = bool(exposure)
        self.iters, self.lr, self.chunk, self.capacity = int(iters), float(lr), int(chunk), capacity
        self.stage = 2 if int(model.model_parms.train_stage) == 2 else 1
        self.pose_mapper = pose_mapper if pose_mapper is not None else getattr(model, "pose_mapper", None)
        if self.stage == 2 and self.pose_mapper is None:
            raise ValueError("stage 2 needs a pose_mapper (posmap.PoseMapper / SmplxPoseMapper) for the input position maps")
        self.width = model.body.pose_width
        self.lam = float(model.opt_parms.lambda_dssim)
        self.dev = model.device
        self.overflows = 0         # chunks fitted again after a binning overflow
        self._plans = {}
        b1, b2 = BETAS
        k = torch.arange(1, self.iters + 1, dtype=torch.float64)
        hyper = torch.stack([torch.full_like(k, self.lr), torch.full_like(k, b1), torch.full_like(k, b2), torch.full_like(k, EPS),
                             1.0 - b1 ** k, torch.sqrt(1.0 - b2 ** k), torch.ones_like(k)], 1)
        self._hyper = hyper.float().to(self.dev).contiguous()        # row k: Adam's scalars of step k + 1
        if self.exposure:
            from .optim import ExposureAdam
            op = model.opt_parms
            ea = ExposureAdam(torch.empty(0), max(self.iters, 1), float(getattr(op, "exposure_lr_init", 0.01)),
                              float(getattr(op, "exposure_lr_final", 0.001)))
            self._hyper_e = ea._hyper_rows(max(self.iters, 1)).to(self.dev)

    # ---- public ---------------------------------------------------------------------------------------------------------------
    def fit(self, frames):
        """frames: `MonoDataset_test`-style items (original_image [3,H,W], the camera fields, pose_data [72|66], transl_data [3], and
        rest_pose [99] for SMPL-X).  Returns (pose [F,72|66], transl [F,3], report), fp32 on the host; report[i] holds frame i's
        initial_loss, fitted_loss and best_iter (0: the initial pose).  With exposure=True a fourth value: exposure [F,3,4]."""
        frames = list(frames)
        n = len(frames)
        pose = torch.empty(n, self.width)
        transl = torch.empty(n, 3)
        exposure = torch.eye(3, 4).repeat(n, 1, 1)
        report = [None] * n
        m = self.model
        with kept_state(m):
            if self.stage == 1:
                with torch.no_grad():
                    dec = m._stage1_decoder(1)
                groups = self._chunks(frames)
            else:
                dec = None
                groups = [[i] for i in range(n)]
            for idx in groups:
                items = [frames[i] for i in idx]
                objective = self._stage1_objective(items, dec) if self.stage == 1 else self._stage2_objective(items[0])
                p, t, e, init, best, it = self._fit_group(items, objective)
                pose[idx], transl[idx] = p.cpu(), t.cpu()
                if e is not None:
                    exposure[idx] = e.cpu().view(-1, 3, 4)
                for k, i in enumerate(idx):
                    report[i] = dict(frame=i, initial_loss=float(init[k]), fitted_loss=float(best[k]), best_iter=int(it[k]))
        return (pose, transl, report, exposure) if self.exposure else (pose, transl, report)

    # ---- the loop -------------------------------------------------------------------------------------------------------------
    def _chunks(self, frames):
        """Consecutive frames of one image size, at most `chunk` per group."""
        groups = []
        for i, it in enumerate(frames):
            size = _size(it)
            if groups and len(groups[-1]) < self.chunk and _size(frames[groups[-1][0]]) == size:
                groups[-1].append(i)
            else:
                groups.append([i])
        return groups

    def _plan(self, b, H, W):
        key = (b, H, W)
        if key not in self._plans:
            self._plans[key] = RasterBatchPlan(b, int(self.model._query_points.shape[0]), H, W, self.dev, capacity=self.capacity,
                                                  antialiasing=getattr(self.model, "antialiasing", False))
        return self._plans[key]

    def _fit_group(self, items, objective):
        """Adam on [pose | transl] (and [A | t]) of the group's frames; returns (best pose, best transl, best [b,12] exposure or None,
        initial losses, best losses, best iters)."""
        W = self.width
        p0 = torch.cat([torch.stack([torch.as_tensor(it["pose_data"]).float().reshape(W) for it in items]),
                        torch.stack([torch.as_tensor(it["transl_data"]).float().reshape(3) for it in items])], 1).to(self.dev)
        b = p0.shape[0]
        e0 = torch.eye(3, 4, device=self.dev).reshape(1, 12).repeat(b, 1) if self.exposure else None
        L = _lib.lib()
        stream = torch.cuda.current_stream().cuda_stream
        for _ in range(4):
            params = p0.clone().requires_grad_(True)
            exp_avg, exp_avg_sq = torch.zeros_like(p0), torch.zeros_like(p0)
            if e0 is not None:
                eparams = e0.clone().requires_grad_(True)
                e_avg, e_avg_sq = torch.zeros_like(e0), torch.zeros_like(e0)
                best_e = e0.clone()
            best, best_loss = p0.clone(), torch.full((b,), math.inf, device=self.dev)
            best_it = torch.zeros(b, dtype=torch.int64, device=self.dev)
            overflow = torch.zeros(2, dtype=torch.int32, device=self.dev)        # [max instances needed, any overflow]
            init = None
            for k in range(self.iters + 1):
                with torch.enable_grad():
                    losses, plan = objective(params[:, :W], params[:, W:], eparams if e0 is not None else None)
                status = plan.status_dev
                with torch.no_grad():
                    if init is None:
                        init = losses.detach().clone()
                    better = (losses < best_loss) & (status[1] == 0)
                    best_loss = torch.where(better, losses, best_loss)
                    best = torch.where(better[:, None], params, best)
                    if e0 is not None:
                        best_e = torch.where(better[:, None], eparams, best_e)
                    best_it = torch.where(better, torch.full_like(best_it, k), best_it)
                    torch.maximum(overflow, torch.stack([status[0], (status[1] != 0).int()]), out=overflow)
                if k == self.iters:
                    break
                if e0 is None:
                    g, = torch.autograd.grad(losses.sum(), params)
                else:
                    g, ge = torch.autograd.grad(losses.sum(), [params, eparams])
                    _lib.check(L.ga_adam_step_dev(eparams.numel(), ptr(eparams), ptr(ge.contiguous()), ptr(e_avg), ptr(e_avg_sq),
                                                  ptr(self._hyper_e[k]), ptr(status[1:2]), stream), "ga_adam_step_dev")
                _lib.check(L.ga_adam_step_dev(params.numel(), ptr(params), ptr(g.contiguous()), ptr(exp_avg), ptr(exp_avg_sq),
                                              ptr(self._hyper[k]), ptr(status[1:2]), stream), "ga_adam_step_dev")
            ovf = overflow.cpu()
            if int(ovf[1]) == 0:
                return best[:, :W], best[:, W:], best_e if e0 is not None else None, init, best_loss, best_it
            self.overflows += 1
            plan.grow(int(ovf[0]))
        raise RuntimeError("pose fitting: the rasterizer's binning buffer overflowed again after growing")

    # ---- objectives: (pose [b,W], transl [b,3], exposure [b,12] or None) -> (per-frame losses [b], the plan of the render) --------
    def _table(self, e):
        """The fitted rows behind an identity row 0: the kernel keeps row 0 (the gauge anchor) out of the gradient."""
        if e is None:
            return None, None
        b = e.shape[0]
        table = torch.cat([torch.eye(3, 4, device=self.dev)[None], e.view(b, 3, 4)], 0)
        return table, torch.arange(1, b + 1, device=self.dev, dtype=torch.int32)

    def _cameras(self, items):
        H, W = _size(items[0])
        batch = {k: [it[k] for it in items] for k in ("FovX", "FovY", "world_view_transform", "full_proj_transform")}
        return self.model._batch_cameras(batch, len(items), self.dev), H, W

    def _targets(self, items):
        return torch.stack([torch.as_tensor(it["original_image"]).float() for it in items]).to(self.dev).contiguous()

    def _rest(self, items):
        """The frames' rest_pose [b,rest_width] on the device (None for SMPL)."""
        body = self.model.body
        if not body.rest_width:
            return None
        if any("rest_pose" not in it for it in items):
            raise ValueError(f"smpl_type={body.name!r}: every frame needs its 'rest_pose' (jaw, eyes and hands, [{body.rest_width}])")
        return torch.stack([torch.as_tensor(it["rest_pose"]).float().reshape(body.rest_width) for it in items]).to(self.dev).contiguous()

    def _stage1_objective(self, items, dec):
        m = self.model
        cams, H, W = self._cameras(items)
        gt, rest = self._targets(items), self._rest(items)
        plan = self._plan(len(items), H, W)

        def objective(pose, transl, e=None):
            table, rows = self._table(e)
            means, scales, colors = m._assemble(dec, pose, transl, rest, exposure=table, exposure_idx=rows)
            img = rasterize_batch(means, colors, scales, m.fix_rotation, m.fix_opacity, cams, m.background, plan)
            return torch.stack([image_loss(img[i:i + 1], gt[i:i + 1], self.lam) for i in range(len(items))]), plan
        return objective

    def _stage2_objective(self, item):
        m = self.model
        cams, H, W = self._cameras([item])
        gt, rest = self._targets([item]), self._rest([item])
        plan = self._plan(1, H, W)

        def objective(pose, transl, e=None):
            table, rows = self._table(e)
            means, scales, colors, _, _ = m._stage2_from_pose(self.pose_mapper, pose, transl, rest, exposure=table, exposure_idx=rows)
            img = rasterize_batch(means, colors, scales, m.fix_rotation, m.fix_opacity, cams, m.background, plan)
            return image_loss(img, gt, self.lam).reshape(1), plan
        return objective


def _size(item):
    return int(item["height"]), int(item["width"])
