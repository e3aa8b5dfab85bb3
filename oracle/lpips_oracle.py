"""Plain-torch restatement of lpips.LPIPS(net='alex', version='0.1') in eval mode, called with normalize=False (train.py:26,89-91).

The feature network is torchvision.models.alexnet(weights=None).features, sliced as lpips slices it ([0:2], [2:5], [5:8], [8:10],
[10:12]); the rest is restated from lpips, which is not vendored here (PARITY UNPINNED, DESIGN §2):
    x = (in - shift) / scale                      shift = (-.030, -.088, -.188), scale = (.458, .448, .450)
    f_k = relu_k(x),  fhat = f / (sqrt(sum_c f_c^2) + 1e-10)
    out = sum_k mean_px sum_c w_k,c (fhat0_c - fhat1_c)^2          [B,1,1,1]
Eval mode: lpips's Dropout in front of each lin layer is off (recent lpips builds the module with eval_mode=True; train.py never calls
.train() on it).  The gradient is torch autograd, so at a pixel whose feature vector is all zero the normalisation's NaN is dropped by
ReLU's threshold_backward, as in the reference.
"""
from __future__ import annotations

import torch
import torchvision

SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)
CHANNELS = (64, 192, 384, 256, 256)
IN_CHANNELS = (3, 64, 192, 384, 256)
KERNELS = (11, 5, 3, 3, 3)
FEATURE_INDEX = (0, 3, 6, 8, 10)          # the convolutions of alexnet().features
SLICES = ((0, 2), (2, 5), (5, 8), (8, 10), (10, 12))
EPS = 1e-10


def conv_keys():
    """lpips's names of the five convolutions' parameters: [(weight key, bias key, features index)]."""
    return [(f"net.slice{k + 1}.{i}.weight", f"net.slice{k + 1}.{i}.bias", i) for k, i in enumerate(FEATURE_INDEX)]


def lin_key(k: int) -> str:
    return f"lin{k}.model.1.weight"


def random_state_dict(seed: int = 0) -> dict:
    """A seeded state dict in lpips's key names: He-scaled conv weights, small biases, non-negative lin weights (as trained lpips
    lin weights are)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, (wk, bk, _) in enumerate(conv_keys()):
        cin, cout, ks = IN_CHANNELS[k], CHANNELS[k], KERNELS[k]
        sd[wk] = torch.randn(cout, cin, ks, ks, generator=g) * (2.0 / (cin * ks * ks)) ** 0.5
        sd[bk] = torch.randn(cout, generator=g) * 0.02
    for k, c in enumerate(CHANNELS):
        sd[lin_key(k)] = torch.rand(1, c, 1, 1, generator=g) * (2.0 / c)
    return sd


class LpipsOracle(torch.nn.Module):
    """The network on torchvision's AlexNet features; dtype / device follow .to() (fp64 on CPU for the restatement, fp32 on cuDNN
    for timing comparisons)."""

    def __init__(self, state_dict: dict):
        super().__init__()
        feats = torchvision.models.alexnet(weights=None).features
        with torch.no_grad():
            for wk, bk, i in conv_keys():
                feats[i].weight.copy_(state_dict[wk])
                feats[i].bias.copy_(state_dict[bk])
        self.slices = torch.nn.ModuleList([feats[a:b] for a, b in SLICES])
        for k in range(5):
            self.register_buffer(f"lin{k}", state_dict[lin_key(k)].detach().clone().reshape(1, -1, 1, 1))
        self.register_buffer("shift", torch.tensor(SHIFT).reshape(1, 3, 1, 1))
        self.register_buffer("scale", torch.tensor(SCALE).reshape(1, 3, 1, 1))
        for p in self.parameters():
            p.requires_grad_(False)
        self.eval()

    def maps(self, x):
        """relu1..relu5 of images x (lpips's input range)."""
        h = (x - self.shift) / self.scale
        out = []
        for s in self.slices:
            h = s(h)
            out.append(h)
        return out

    def forward(self, in0, in1, normalize: bool = False):
        if normalize:
            in0, in1 = 2 * in0 - 1, 2 * in1 - 1
        f0, f1 = self.maps(in0), self.maps(in1)
        val = 0
        for k in range(5):
            a = f0[k] / (torch.sqrt(torch.sum(f0[k] ** 2, dim=1, keepdim=True)) + EPS)
            b = f1[k] / (torch.sqrt(torch.sum(f1[k] ** 2, dim=1, keepdim=True)) + EPS)
            d = ((a - b) ** 2 * getattr(self, f"lin{k}")).sum(dim=1, keepdim=True)
            val = val + d.mean(dim=[2, 3], keepdim=True)
        return val


def map_shapes(H: int, W: int):
    """(H_k, W_k) of relu1..relu5 for an H x W image."""
    h, w = (H + 4 - 11) // 4 + 1, (W + 4 - 11) // 4 + 1
    out = [(h, w)]
    h, w = (h - 3) // 2 + 1, (w - 3) // 2 + 1
    out.append((h, w))
    h, w = (h - 3) // 2 + 1, (w - 3) // 2 + 1
    out += [(h, w)] * 3
    return out
