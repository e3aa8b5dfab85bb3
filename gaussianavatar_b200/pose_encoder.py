"""Stage-2 pose encoder with the reference's name and checkpoint layout: `UnetNoCond5DS` (reference: /root/reference
model/modules.py:185-232, blocks :62-111; built at model/avatar_model.py:139-146 with input_nc=3, output_nc=c_pose=64, nf=32,
up_mode='upconv', no dropout; called at :401,589).

    posed-body position map [B,3,128,128]
      -> 5 down steps   (LeakyReLU(0.2) ->) conv 4x4 stride 2 pad 1 (-> BatchNorm, no affine)        32,64,128,256,256 channels
      -> 5 up steps     ReLU -> transposed conv 4x4 stride 2 pad 1 (-> BatchNorm) -> concat skip      256,128,64,32 -> 64 (+bias)
      -> pose_featmap [B,64,128,128]

The whole network is one table of steps and one functional forward; parameters and BatchNorm running statistics are registered under
the reference's state-dict names (`conv{k}.conv.weight`, `conv{k}.bn.running_mean`, `upconv{k}.up.weight`, `upconv5.up.bias`, ...)
so `pose_encoder.pth` (avatar_model.py:177-186,223-236) loads unchanged.  One reference quirk shapes the numerics and is kept:
the down steps apply their LeakyReLU IN PLACE, i.e. to the tensor the previous step returned, so the skip tensors that reach the up
path are the leaky-ReLU'd activations, not the raw conv / BatchNorm outputs (SURVEY.md App. B.2; pinned by
tests/golden/unet5ds_nf8_s32.npz through oracle/avatar_oracle.py:unet5ds_forward).

Scope note: at 1.2 GFLOP per frame (the decoder behind it: 95 GFLOP per frame) these ten convolutions run on cuDNN — library kernels,
in TF32 like the reference's — not on hand-written ones; what this package hand-writes of stage 2 is everything downstream: the
per-frame decoder on the tensor cores (`POP_no_unet.forward_packed_frames`), per-frame LBS / assembly and the batched rasterizer.
BatchNorm here is written out (sums -> mean / variance -> normalise) so that the data-parallel variant is the same code with the
two sums all-reduced over the ranks (`sync_group`): exact global-batch statistics, as SURVEY.md §8e asks for stage 2."""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F


def _holder(**children) -> nn.Module:
    m = nn.Module()
    for k, v in children.items():
        setattr(m, k, v)
    return m


def _leaf(weight: torch.Tensor, bias: torch.Tensor | None = None) -> nn.Module:
    m = nn.Module()
    m.weight = nn.Parameter(weight)
    if bias is not None:
        m.bias = nn.Parameter(bias)
    return m


def _bn_buffers(channels: int) -> nn.Module:
    m = nn.Module()
    m.register_buffer("running_mean", torch.zeros(channels))
    m.register_buffer("running_var", torch.ones(channels))
    m.register_buffer("num_batches_tracked", torch.tensor(0, dtype=torch.long))
    return m


class UnetNoCond5DS(nn.Module):
    EPS, MOMENTUM, SLOPE = 1e-5, 0.1, 0.2

    def __init__(self, input_nc=3, output_nc=3, nf=64, up_mode="upconv", use_dropout=False, return_lowres=False, return_2branches=False):
        super().__init__()
        if up_mode != "upconv" or use_dropout or return_lowres or return_2branches:
            raise NotImplementedError("built for the configuration the reference instantiates (model/avatar_model.py:139-146): "
                                      "up_mode='upconv', no dropout, single output branch")
        # (name, in channels, out channels, BatchNorm?)
        self.down = (("conv1", input_nc, nf, False), ("conv2", nf, 2 * nf, True), ("conv3", 2 * nf, 4 * nf, True),
                     ("conv4", 4 * nf, 8 * nf, True), ("conv5", 8 * nf, 8 * nf, False))
        self.up = (("upconv1", 8 * nf, 8 * nf, True), ("upconv2", 16 * nf, 4 * nf, True), ("upconv3", 8 * nf, 2 * nf, True),
                   ("upconv4", 4 * nf, nf, True), ("upconv5", 2 * nf, output_nc, False))
        for name, ci, co, bn in self.down:          # nn.Conv2d's default initialisation (kaiming_uniform(a=sqrt(5)) = U(+-1/sqrt(fan_in)))
            w = torch.empty(co, ci, 4, 4).uniform_(-1.0, 1.0) / (ci * 16) ** 0.5
            setattr(self, name, _holder(conv=_leaf(w), **({"bn": _bn_buffers(co)} if bn else {})))
        for name, ci, co, bn in self.up:            # nn.ConvTranspose2d: weight [in, out, 4, 4], fan_in counted on dim 1
            w = torch.empty(ci, co, 4, 4).uniform_(-1.0, 1.0) / (co * 16) ** 0.5
            b = None if bn else torch.empty(co).uniform_(-1.0, 1.0) / (co * 16) ** 0.5
            setattr(self, name, _holder(up=_leaf(w, b), **({"bn": _bn_buffers(co)} if bn else {})))
        self.sync_group = None        # set to a process group (or True for the default group) for cross-rank BatchNorm statistics

    def _batch_norm(self, x, buffers):
        """Training-mode BatchNorm2d(affine=False): biased batch variance normalises, the unbiased one feeds the running statistics."""
        n = x.numel() // x.shape[1]
        sums = torch.cat([x.sum((0, 2, 3)), (x * x).sum((0, 2, 3))])
        if self.sync_group is not None and torch.distributed.is_initialized() and torch.distributed.get_world_size() > 1:
            import torch.distributed.nn.functional as dnn
            group = None if self.sync_group is True else self.sync_group
            sums = dnn.all_reduce(sums, group=group)
            n = n * torch.distributed.get_world_size(group)
        C = x.shape[1]
        mean = sums[:C] / n
        var = (sums[C:] / n - mean * mean).clamp_min(0.0)
        with torch.no_grad():
            buffers.running_mean.mul_(1 - self.MOMENTUM).add_(mean.detach(), alpha=self.MOMENTUM)
            buffers.running_var.mul_(1 - self.MOMENTUM).add_(var.detach() * (n / max(n - 1, 1)), alpha=self.MOMENTUM)
            buffers.num_batches_tracked += 1
        return (x - mean[None, :, None, None]) * torch.rsqrt(var + self.EPS)[None, :, None, None]

    def forward(self, x):
        skips = []
        t = x
        for k, (name, _, _, bn) in enumerate(self.down):
            m = getattr(self, name)
            t = F.conv2d(t, m.conv.weight, stride=2, padding=1)
            if bn:
                t = self._batch_norm(t, m.bn)
            if k < 4:
                t = F.leaky_relu(t, self.SLOPE)     # the NEXT step's in-place LeakyReLU: also what the skip connection carries
                skips.append(t)
        for k, (name, _, _, bn) in enumerate(self.up):
            m = getattr(self, name)
            t = F.conv_transpose2d(F.relu(t), m.up.weight, bias=getattr(m.up, "bias", None), stride=2, padding=1)
            if bn:
                t = self._batch_norm(t, m.bn)
            if k < 4:
                t = torch.cat([t, skips[3 - k]], 1)
        return t
