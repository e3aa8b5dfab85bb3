"""LPIPS perceptual distance (lpips.LPIPS(net='alex', version='0.1'), eval mode) on the library's sm_90a kernels, as train.py:89-91
adds it to the loss from epoch lpips_start_iter + 1 on.  Gradient to in0 only; the network's weights are frozen.

Weights are the user's own: ``load_alex_weights(lin_path, alexnet_path)`` builds lpips's state dict from lpips's
``weights/v0.1/alex.pth`` and torchvision's ``alexnet-owt-*.pth``.  Nothing is downloaded.
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import ptr

SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)
CHANNELS = (64, 192, 384, 256, 256)
IN_CHANNELS = (3, 64, 192, 384, 256)
KERNELS = (11, 5, 3, 3, 3)
_FEATURE_INDEX = (0, 3, 6, 8, 10)     # the convolutions of torchvision's alexnet().features, and their lpips slice positions


def _conv_keys(k):
    i = _FEATURE_INDEX[k]
    return f"net.slice{k + 1}.{i}.weight", f"net.slice{k + 1}.{i}.bias"


def _shapes() -> dict:
    out = {}
    for k in range(5):
        wk, bk = _conv_keys(k)
        out[wk] = (CHANNELS[k], IN_CHANNELS[k], KERNELS[k], KERNELS[k])
        out[bk] = (CHANNELS[k],)
        out[f"lin{k}.model.1.weight"] = (1, CHANNELS[k], 1, 1)
    return out


def _checked(sd: dict, key: str, shape: tuple, where: str) -> torch.Tensor:
    if key not in sd:
        raise KeyError(f"{where}: missing {key!r}")
    t = sd[key]
    if not torch.is_tensor(t) or tuple(t.shape) != tuple(shape):
        got = tuple(t.shape) if torch.is_tensor(t) else type(t).__name__
        raise ValueError(f"{where}: {key!r} has shape {got}, expected {tuple(shape)}")
    return t


def validate_state_dict(sd: dict) -> dict:
    """The 15 tensors the network needs, by lpips's names, after checking every key of `sd`: the conv and lin weights must be
    present with their shapes; lpips's `lins.K.*` duplicates must equal `linK.*` and the `scaling_layer` buffers must hold lpips's
    constants; any other key raises."""
    shapes = _shapes()
    out = {k: _checked(sd, k, s, "LPIPS state dict") for k, s in shapes.items()}
    for key, t in sd.items():
        if key in shapes:
            continue
        if key.startswith("lins.") and key.endswith(".model.1.weight"):
            k = key.split(".")[1]
            ref = out.get(f"lin{k}.model.1.weight")
            if ref is None or not torch.is_tensor(t) or t.shape != ref.shape or not torch.equal(t.cpu(), ref.cpu()):
                raise ValueError(f"LPIPS state dict: {key!r} differs from lin{k}.model.1.weight")
        elif key in ("scaling_layer.shift", "scaling_layer.scale"):
            ref = torch.tensor(SHIFT if key.endswith("shift") else SCALE).reshape(1, 3, 1, 1)
            if not torch.is_tensor(t) or t.shape != ref.shape or not torch.equal(t.detach().float().cpu(), ref):
                raise ValueError(f"LPIPS state dict: {key!r} is not lpips's {tuple(ref.flatten().tolist())}")
        else:
            raise KeyError(f"LPIPS state dict: unexpected key {key!r}")
    return out


def pack_weights(sd: dict, device) -> torch.Tensor:
    """The flat fp32 buffer ga_lpips_forward / ga_lpips_backward read (layout: include/gavatar.h)."""
    sd = validate_state_dict(sd)
    parts = []
    for k in range(5):
        wk, bk = _conv_keys(k)
        w = sd[wk].detach().to(device=device, dtype=torch.float32)
        wf = w.permute(0, 2, 3, 1).reshape(CHANNELS[k], -1)                          # [C_out][tap][C_in]
        if k == 0:
            wf = torch.nn.functional.pad(wf, (0, 384 - wf.shape[1]))
        parts += [wf.reshape(-1), sd[bk].detach().to(device=device, dtype=torch.float32).reshape(-1)]
    for k in range(1, 5):
        w = sd[_conv_keys(k)[0]].detach().to(device=device, dtype=torch.float32)
        parts.append(w.flip(2, 3).permute(1, 2, 3, 0).reshape(-1))                    # [C_in][flipped tap][C_out]
    for k in range(5):
        parts.append(sd[f"lin{k}.model.1.weight"].detach().to(device=device, dtype=torch.float32).reshape(-1))
    flat = torch.cat(parts).contiguous()
    n = _lib.lib().ga_lpips_weights_floats()
    if flat.numel() != n:
        raise RuntimeError(f"LPIPS weight packing: {flat.numel()} floats, the library expects {n}")
    return flat


def _stream():
    return torch.cuda.current_stream().cuda_stream


class _LpipsFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, in0, in1, flat, in_scale, in_shift):
        B, C, H, W = in0.shape
        L = _lib.lib()
        ws = torch.empty(L.ga_lpips_workspace_bytes(B, H, W), dtype=torch.uint8, device=in0.device)
        out = torch.empty(B, dtype=torch.float32, device=in0.device)
        _lib.check(L.ga_lpips_forward(B, H, W, ptr(flat), ptr(in0), ptr(in1), float(in_scale), float(in_shift), ptr(ws), ptr(out),
                                      _stream()), "ga_lpips_forward")
        ctx.save_for_backward(flat, ws)
        ctx.shape = (B, H, W)
        return out.view(B, 1, 1, 1)

    @staticmethod
    def backward(ctx, g):
        flat, ws = ctx.saved_tensors
        B, H, W = ctx.shape
        g = g.reshape(B).float().contiguous()
        d = torch.empty(B, 3, H, W, dtype=torch.float32, device=g.device)
        _lib.check(_lib.lib().ga_lpips_backward(B, H, W, ptr(flat), ptr(ws), ptr(g), ptr(d), _stream()), "ga_lpips_backward")
        return d, None, None, None, None


class LPIPS(torch.nn.Module):
    """lpips.LPIPS(net='alex', version='0.1') in eval mode, from a state dict in lpips's key names (``net.slice1.0.weight`` ...
    ``net.slice5.10.bias``, ``lin0.model.1.weight`` ... ``lin4.model.1.weight``; a full ``lpips.LPIPS().state_dict()`` is accepted
    too).  The weights are packed once on `device` into the library's layout; ``.to()`` moves them."""

    def __init__(self, state_dict: dict, device="cuda"):
        super().__init__()
        self.register_buffer("flat", pack_weights(state_dict, device), persistent=False)

    def forward(self, in0, in1, normalize: bool = False):
        """[B,1,1,1] distances of [B,3,H,W] images in [-1,1] (normalize=True: in [0,1]); the gradient flows to in0 only."""
        if not (torch.is_tensor(in0) and torch.is_tensor(in1)) or not (in0.is_cuda and in1.is_cuda):
            raise RuntimeError("LPIPS needs CUDA tensors (no CPU fallback)")
        if in1.requires_grad:
            raise ValueError("LPIPS: in1 must not require grad (the gradient is computed for in0 only)")
        if in0.dim() != 4 or in0.shape[1] != 3 or in0.shape != in1.shape:
            raise ValueError(f"LPIPS: in0 {tuple(in0.shape)} and in1 {tuple(in1.shape)} must both be [B,3,H,W]")
        H, W = in0.shape[-2:]
        if H < 31 or W < 31:
            raise ValueError(f"LPIPS: images of {H}x{W} are too small for AlexNet's two max pools (H, W >= 31)")
        if self.flat.device != in0.device:
            raise RuntimeError(f"LPIPS weights are on {self.flat.device}, the images on {in0.device}")
        scale, shift = (2.0, -1.0) if normalize else (1.0, 0.0)
        return _LpipsFn.apply(in0.float().contiguous(), in1.detach().float().contiguous(), self.flat, scale, shift)


def load_alex_weights(lin_path: str, alexnet_path: str) -> dict:
    """lpips's state dict from the two files a user of the reference has: lpips's ``weights/v0.1/alex.pth`` (``linK.model.1.weight``)
    and torchvision's ``alexnet-owt-*.pth`` (``features.{0,3,6,8,10}.weight`` / ``.bias``).  A missing key or wrong shape raises and
    names the key."""
    lin = torch.load(lin_path, map_location="cpu", weights_only=True)
    alex = torch.load(alexnet_path, map_location="cpu", weights_only=True)
    sd = {}
    for k in range(5):
        i = _FEATURE_INDEX[k]
        wk, bk = _conv_keys(k)
        sd[wk] = _checked(alex, f"features.{i}.weight", (CHANNELS[k], IN_CHANNELS[k], KERNELS[k], KERNELS[k]), alexnet_path)
        sd[bk] = _checked(alex, f"features.{i}.bias", (CHANNELS[k],), alexnet_path)
        key = f"lin{k}.model.1.weight"
        sd[key] = _checked(lin, key, (1, CHANNELS[k], 1, 1), lin_path)
    return sd
