"""Fused Adam with torch.optim.Adam's semantics and state layout (reference: model/avatar_model.py:148-155 builds
`torch.optim.Adam` over net + geo_feature; `step()` at :264-267).  One kernel launch per parameter tensor; with the flat
parameter buffer of `POP_no_unet` that is two launches per step.  `grad_scale` folds the 1/world_size of the
data-parallel all-reduce(sum) into the update."""
from __future__ import annotations

import math

import torch

from . import _lib
from ._lib import ptr


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps))
        self.grad_scale = 1.0
        self.skip_flag = None      # device int32 tensor: a non-zero word makes the update a no-op (rasterizer overflow guard)

    @torch.no_grad()
    def step(self, closure=None):
        L = _lib.lib()
        st = torch.cuda.current_stream().cuda_stream
        for group in self.param_groups:
            b1, b2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                if not p.is_cuda or not p.is_contiguous() or p.dtype != torch.float32:
                    raise RuntimeError("FusedAdam needs contiguous fp32 CUDA parameters")
                s = self.state[p]
                if len(s) == 0:
                    s["step"] = 0
                    s["exp_avg"] = torch.zeros_like(p)
                    s["exp_avg_sq"] = torch.zeros_like(p)
                s["step"] = int(s["step"]) + 1
                g = p.grad if p.grad.is_contiguous() else p.grad.contiguous()
                _lib.check(L.ga_adam_step(p.numel(), ptr(p), ptr(g), ptr(s["exp_avg"]), ptr(s["exp_avg_sq"]), float(group["lr"]),
                                          float(b1), float(b2), float(group["eps"]), s["step"], float(self.grad_scale),
                                          ptr(self.skip_flag), st),
                           "ga_adam_step")
        return None


def log_linear_lr(step: int, total: int, lr_init: float, lr_final: float) -> float:
    """3DGS's get_expon_lr_func without delay: exp of the linear blend of log(lr_init) and log(lr_final), t = step / total in [0, 1]."""
    t = min(max(step / max(total, 1), 0.0), 1.0)
    return math.exp(math.log(lr_init) * (1.0 - t) + math.log(lr_final) * t)


class ExposureAdam:
    """Dense Adam on the per-frame exposure table with torch.optim.Adam's semantics (betas 0.9 / 0.999, eps 1e-8), its learning rate
    falling log-linearly from lr_init to lr_final over `total_steps`.  One `ga_adam_step_dev` launch per step; its scalars come from a
    device table of rows built on the host ahead of time, so a step reads nothing back.  `skip_flag` (device int32, the
    rasterizer's overflow word) turns a step into a no-op on the device; the caller then takes the host count back (`undo`)."""

    BETAS = (0.9, 0.999)
    EPS = 1e-8

    def __init__(self, param, total_steps: int, lr_init: float = 0.01, lr_final: float = 0.001):
        self.param = param
        self.total_steps, self.lr_init, self.lr_final = max(int(total_steps), 1), float(lr_init), float(lr_final)
        self.step_count = 0
        self.launched = False      # did the last step() launch an update (the one undo() takes back)
        self.exp_avg = torch.zeros_like(param)
        self.exp_avg_sq = torch.zeros_like(param)
        self.grad_scale = 1.0
        self.skip_flag = None
        self._hyper = None
        self._hyper_key = None

    def _hyper_rows(self, need: int):
        """Device rows [lr, beta1, beta2, eps, 1-beta1^k, sqrt(1-beta2^k), grad_scale] for steps k = 1..; rebuilt (doubled) on demand."""
        key = (self.grad_scale, self.total_steps)
        if self._hyper is None or self._hyper.shape[0] < need or self._hyper_key != key:
            n = max(need, self.total_steps, 2 * (0 if self._hyper is None else self._hyper.shape[0]))
            b1, b2 = self.BETAS
            k = torch.arange(1, n + 1, dtype=torch.float64)
            lr = torch.tensor([log_linear_lr(int(i) - 1, self.total_steps, self.lr_init, self.lr_final) for i in range(1, n + 1)],
                              dtype=torch.float64)
            rows = torch.stack([lr, torch.full_like(k, b1), torch.full_like(k, b2), torch.full_like(k, self.EPS), 1.0 - b1 ** k,
                                torch.sqrt(1.0 - b2 ** k), torch.full_like(k, self.grad_scale)], 1)
            self._hyper = rows.float().to(self.param.device).contiguous()
            self._hyper_key = key
        return self._hyper

    def lr(self, step: int) -> float:
        """The learning rate of update number `step` (1-based)."""
        return log_linear_lr(step - 1, self.total_steps, self.lr_init, self.lr_final)

    @torch.no_grad()
    def step(self):
        g = self.param.grad
        self.launched = False
        if g is None:
            return
        if not (self.param.is_cuda and self.param.is_contiguous() and self.param.dtype == torch.float32):
            raise RuntimeError("ExposureAdam needs a contiguous fp32 CUDA table")
        self.step_count += 1
        rows = self._hyper_rows(self.step_count)
        g = g if g.is_contiguous() else g.contiguous()
        _lib.check(_lib.lib().ga_adam_step_dev(self.param.numel(), ptr(self.param), ptr(g), ptr(self.exp_avg), ptr(self.exp_avg_sq),
                                               ptr(rows[self.step_count - 1]), ptr(self.skip_flag), torch.cuda.current_stream().cuda_stream),
                   "ga_adam_step_dev")
        self.launched = True

    def undo(self):
        """Host bookkeeping of a step the device skipped: the count goes back only if that step launched an update."""
        if self.launched:
            self.step_count -= 1
            self.launched = False

    def state_dict(self):
        return {"step": self.step_count, "exp_avg": self.exp_avg.detach().clone(), "exp_avg_sq": self.exp_avg_sq.detach().clone(),
                "total_steps": self.total_steps, "lr_init": self.lr_init, "lr_final": self.lr_final}

    def load_state_dict(self, sd):
        with torch.no_grad():
            self.exp_avg.copy_(torch.as_tensor(sd["exp_avg"]).reshape(self.exp_avg.shape))
            self.exp_avg_sq.copy_(torch.as_tensor(sd["exp_avg_sq"]).reshape(self.exp_avg_sq.shape))
        self.step_count = int(sd["step"])
