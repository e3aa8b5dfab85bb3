"""`POP_no_unet`-compatible feature net over the fused sm_90a decoder (reference: /root/reference model/network.py:9-83).

All trainable tensors live in ONE flat fp32 buffer (`self.flat`, kernel-friendly packing described in
include/gavatar.h) so that the optimizer step and the data-parallel gradient all-reduce are each a single operation;
`state_dict()` / `load_state_dict()` translate to and from the reference's names and shapes
(`geom_proc_layers.conv1.weight`, `decoder.conv6SH.weight`, `decoder.bn7N.running_var`, ...) so reference checkpoints
(`net.pth["net"]`, model/avatar_model.py:163-207) load unchanged.
"""
from __future__ import annotations

import ctypes
import math
import os
from collections import OrderedDict

import torch
import torch.nn as nn

from . import _lib
from .ops import DecoderNet

_HEADS = ("", "N", "SH")          # head order inside the stacked layers: xyz, scale (N), colour (SH)

# Order of the reference's `net.parameters()` (module registration order of POP_no_unet / ShapeDecoder, model/network.py:18-36,
# model/modules.py:477-528): the indices of torch.optim.Adam's state in a reference checkpoint refer to it
# (model/avatar_model.py:148-155,163-176).  Pinned by tests/golden/pop_param_order.json (generated from the reference).
REFERENCE_PARAM_ORDER = tuple(
    [f"geom_proc_layers.conv{k}.weight" for k in (1, 2, 3)]
    + [f"decoder.conv{l}{sfx}.{wb}" for sfx, ls in (("", range(1, 9)), ("SH", (6, 7, 8)), ("N", (6, 7, 8))) for l in ls for wb in ("weight", "bias")]
    + [f"decoder.bn{l}{sfx}.{wb}" for sfx, ls in (("", range(1, 8)), ("N", (6, 7)), ("SH", (6, 7))) for l in ls for wb in ("weight", "bias")])
_BN_LAYERS = ["bn1", "bn2", "bn3", "bn4", "bn5", "bn6", "bn6N", "bn6SH", "bn7", "bn7N", "bn7SH"]


class DecoderState:
    """Device-side state of one decoder instance: descriptor, activation workspace, BatchNorm running statistics."""

    def __init__(self, S: int, feat_res: int, batch: int, device, c_geom=64, hsize=128, eps=1e-5, momentum=0.1, tensor_cores=True, frames=1):
        self.desc = _lib.GaDecoderDesc(int(S), int(feat_res), int(batch), int(c_geom), int(hsize), float(eps), float(momentum),
                                       _lib.GA_DECODER_TENSOR_CORES if tensor_cores else 0, int(frames))
        nbytes = _lib.lib().ga_decoder_workspace_bytes(ctypes.byref(self.desc))
        if nbytes == 0:
            raise RuntimeError("ga_decoder_workspace_bytes failed: " + _lib.lib().ga_last_error().decode())
        self.workspace = torch.empty(nbytes, dtype=torch.uint8, device=device)
        self.bn_running = None          # set by PopNet
        self.track_running = True
        self.num_batches_tracked = 0


def decoder_layout(c_geom=64, hsize=128) -> _lib.GaDecoderLayout:
    desc = _lib.GaDecoderDesc(2, 1, 1, c_geom, hsize, 1e-5, 0.1, 0, 1)
    lay = _lib.GaDecoderLayout()
    _lib.check(_lib.lib().ga_decoder_layout(ctypes.byref(desc), ctypes.byref(lay)), "ga_decoder_layout")
    return lay


class POP_no_unet(nn.Module):
    """Drop-in for model.network.POP_no_unet (stage-1 configuration: geom_layer_type='conv')."""

    def __init__(self, c_geom=64, geom_layer_type="conv", nf=64, hsize=256, up_mode="upconv", use_dropout=False, uv_feat_dim=2):
        super().__init__()
        if geom_layer_type != "conv":
            raise NotImplementedError("only geom_layer_type='conv' (the reference default, arguments/__init__.py:110) is built")
        if c_geom != 64 or hsize != 128 or uv_feat_dim != 2:
            raise NotImplementedError("only c_geom=64, hsize=128, uv_feat_dim=2 (arguments/__init__.py:101-111) are built")
        self.geom_layer_type = geom_layer_type
        self.c_geom, self.hsize = c_geom, hsize
        # MLP math: TF32 tensor cores (mma.sync) (what the reference's cuDNN convs use on Ampere+) or strict FP32 CUDA cores
        self.tensor_cores = os.environ.get("GA_DECODER_FP32", "0") != "1"
        self.layout = decoder_layout(c_geom, hsize)
        self.flat = nn.Parameter(torch.zeros(int(self.layout.total)))
        self.register_buffer("bn_running", torch.cat([torch.zeros(self.layout.bn_channels), torch.ones(self.layout.bn_channels)]).reshape(2, -1))
        self._states = {}
        self.reset_parameters()

    # ---- initialisation: the distributions nn.Conv2d / nn.Conv1d / nn.BatchNorm1d use by default --------------------
    def reset_parameters(self):
        sd = OrderedDict()
        for k in (1, 2, 3):
            bound = 1.0 / math.sqrt(self.c_geom * 25)
            sd[f"geom_proc_layers.conv{k}.weight"] = torch.empty(self.c_geom, self.c_geom, 5, 5).uniform_(-bound, bound)
        in_size = self.c_geom + 2
        h = self.hsize
        shapes = dict(conv1=(h, in_size), conv2=(h, h), conv3=(h, h), conv4=(h, h), conv5=(h, h + in_size), conv6=(h, h), conv7=(h, h),
                      conv8=(3, h), conv6SH=(h, h), conv7SH=(h, h), conv8SH=(3, h), conv6N=(h, h), conv7N=(h, h), conv8N=(1, h))
        for name, (o, i) in shapes.items():
            bound = 1.0 / math.sqrt(i)
            sd[f"decoder.{name}.weight"] = torch.empty(o, i, 1).uniform_(-bound, bound)
            sd[f"decoder.{name}.bias"] = torch.empty(o).uniform_(-bound, bound)
        for bn in _BN_LAYERS:
            sd[f"decoder.{bn}.weight"] = torch.ones(h)
            sd[f"decoder.{bn}.bias"] = torch.zeros(h)
        self.load_state_dict(sd, strict=False)

    # ---- reference-name <-> flat-buffer translation -------------------------------------------------------------------
    def _slots(self, flat=None):
        """name -> (getter, setter) over a flat buffer (default self.flat) / self.bn_running, shapes as in the reference
        state_dict."""
        L, h, cg = self.layout, self.hsize, self.c_geom
        flat = self.flat.data if flat is None else flat
        out = OrderedDict()

        def seg(off, n):
            return flat[int(off):int(off) + n]

        for k in range(3):
            v = seg(L.gconv[k], 25 * cg * cg).view(25, cg, cg)                    # [tap, ci, co]
            out[f"geom_proc_layers.conv{k + 1}.weight"] = (lambda v=v: v.permute(2, 1, 0).reshape(cg, cg, 5, 5),
                                                           lambda t, v=v: v.copy_(t.reshape(cg, cg, 25).permute(2, 1, 0)))
        w1 = seg(L.w[0], h * 72).view(h, 72)
        out["decoder.conv1.weight"] = (lambda: w1[:, :66].unsqueeze(-1), lambda t: w1[:, :66].copy_(t.reshape(h, 66)))
        for l, name in ((1, "conv2"), (2, "conv3"), (3, "conv4")):
            w = seg(L.w[l], h * h).view(h, h)
            out[f"decoder.{name}.weight"] = (lambda w=w: w.unsqueeze(-1), lambda t, w=w: w.copy_(t.reshape(h, h)))
        w5 = seg(L.w[4], h * 200).view(h, 200)
        out["decoder.conv5.weight"] = (lambda: torch.cat([w5[:, :66], w5[:, 72:]], 1).unsqueeze(-1),
                                       lambda t: (w5[:, :66].copy_(t.reshape(h, 194)[:, :66]), w5[:, 72:].copy_(t.reshape(h, 194)[:, 66:])))
        for l, name in enumerate(("conv1", "conv2", "conv3", "conv4", "conv5")):
            b = seg(L.b[l], h)
            out[f"decoder.{name}.bias"] = (lambda b=b: b, lambda t, b=b: b.copy_(t))
        for l, bn in enumerate(("bn1", "bn2", "bn3", "bn4", "bn5")):
            g, be = seg(L.gamma[l], h), seg(L.beta[l], h)
            out[f"decoder.{bn}.weight"] = (lambda g=g: g, lambda t, g=g: g.copy_(t))
            out[f"decoder.{bn}.bias"] = (lambda be=be: be, lambda t, be=be: be.copy_(t))
        for hi, sfx in enumerate(_HEADS):
            w6 = seg(L.w[5], 3 * h * h).view(3, h, h)[hi]
            w7 = seg(L.w[6], 3 * h * h).view(3, h, h)[hi]
            out[f"decoder.conv6{sfx}.weight"] = (lambda w=w6: w.unsqueeze(-1), lambda t, w=w6: w.copy_(t.reshape(h, h)))
            out[f"decoder.conv7{sfx}.weight"] = (lambda w=w7: w.unsqueeze(-1), lambda t, w=w7: w.copy_(t.reshape(h, h)))
            for l, nm in ((5, "6"), (6, "7")):
                b = seg(L.b[l], 3 * h).view(3, h)[hi]
                g = seg(L.gamma[l], 3 * h).view(3, h)[hi]
                be = seg(L.beta[l], 3 * h).view(3, h)[hi]
                out[f"decoder.conv{nm}{sfx}.bias"] = (lambda b=b: b, lambda t, b=b: b.copy_(t))
                out[f"decoder.bn{nm}{sfx}.weight"] = (lambda g=g: g, lambda t, g=g: g.copy_(t))
                out[f"decoder.bn{nm}{sfx}.bias"] = (lambda be=be: be, lambda t, be=be: be.copy_(t))
        w8 = seg(L.w8, 8 * h).view(8, h)
        b8 = seg(L.b8, 8)
        for sfx, r0, n in (("", 0, 3), ("N", 3, 1), ("SH", 4, 3)):
            out[f"decoder.conv8{sfx}.weight"] = (lambda r0=r0, n=n: w8[r0:r0 + n].unsqueeze(-1), lambda t, r0=r0, n=n: w8[r0:r0 + n].copy_(t.reshape(n, h)))
            out[f"decoder.conv8{sfx}.bias"] = (lambda r0=r0, n=n: b8[r0:r0 + n], lambda t, r0=r0, n=n: b8[r0:r0 + n].copy_(t))
        # BatchNorm running statistics
        offs = list(L.bn_offset)
        run = self.bn_running
        bn_pos = {"bn1": offs[0], "bn2": offs[1], "bn3": offs[2], "bn4": offs[3], "bn5": offs[4]}
        for hi, sfx in enumerate(_HEADS):
            bn_pos[f"bn6{sfx}"] = offs[5] + hi * h
            bn_pos[f"bn7{sfx}"] = offs[6] + hi * h
        for bn, o in bn_pos.items():
            out[f"decoder.{bn}.running_mean"] = (lambda o=o: run[0, o:o + h], lambda t, o=o: run[0, o:o + h].copy_(t))
            out[f"decoder.{bn}.running_var"] = (lambda o=o: run[1, o:o + h], lambda t, o=o: run[1, o:o + h].copy_(t))
        return out

    def reference_grads(self) -> "OrderedDict[str, torch.Tensor]":
        """Gradient of the flat buffer re-expressed under the reference's parameter names / shapes."""
        if self.flat.grad is None:
            return OrderedDict()
        return OrderedDict((k, get().detach().clone()) for k, (get, _) in self._slots(self.flat.grad).items() if "running" not in k)

    def flat_from_reference_tensors(self, tensors) -> torch.Tensor:
        """Scatter per-parameter tensors given in REFERENCE_PARAM_ORDER (e.g. the exp_avg / exp_avg_sq of a reference
        checkpoint's Adam state) into a new buffer laid out like `self.flat`; padding elements stay zero."""
        if len(tensors) != len(REFERENCE_PARAM_ORDER):
            raise ValueError(f"expected {len(REFERENCE_PARAM_ORDER)} per-parameter tensors, got {len(tensors)}")
        buf = torch.zeros_like(self.flat.data)
        slots = self._slots(buf)
        for name, t in zip(REFERENCE_PARAM_ORDER, tensors):
            get, put = slots[name]
            t = torch.as_tensor(t).to(device=buf.device, dtype=buf.dtype)
            if tuple(get().shape) != tuple(t.shape):
                raise ValueError(f"{name}: expected shape {tuple(get().shape)}, got {tuple(t.shape)}")
            put(t)
        return buf

    def reference_tensors_from_flat(self, flat) -> "list[torch.Tensor]":
        """Inverse of flat_from_reference_tensors: views/copies of a flat-layout buffer under the reference's parameter order."""
        slots = self._slots(flat)
        return [slots[name][0]().detach().clone() for name in REFERENCE_PARAM_ORDER]

    def state_dict(self, *args, destination=None, prefix="", keep_vars=False, **kw):
        sd = OrderedDict() if destination is None else destination
        nbt = 0
        for st in self._states.values():
            nbt = max(nbt, st.num_batches_tracked)
        for name, (get, _) in self._slots().items():
            sd[prefix + name] = get().detach().clone()
            if name.endswith("running_var"):
                sd[prefix + name.replace("running_var", "num_batches_tracked")] = torch.tensor(nbt, dtype=torch.long)
        return sd

    def load_state_dict(self, state_dict, strict=True, assign=False):
        slots = self._slots()
        missing = [k for k in slots if k not in state_dict]
        unexpected = [k for k in state_dict if k not in slots and not k.endswith("num_batches_tracked")]
        if strict and (missing or unexpected):
            raise RuntimeError(f"Error(s) in loading state_dict for POP_no_unet: missing {missing}, unexpected {unexpected}")
        with torch.no_grad():
            for k, (_, put) in slots.items():
                if k in state_dict:
                    put(state_dict[k].to(self.flat.device, torch.float32))
        return torch.nn.modules.module._IncompatibleKeys(missing, unexpected)

    # ---- execution ------------------------------------------------------------------------------------------------
    def _state(self, S, feat_res, batch, frames=1) -> DecoderState:
        key = (int(S), int(feat_res), int(batch), self.flat.device, bool(self.tensor_cores), int(frames))
        st = self._states.get(key)
        if st is None:
            st = DecoderState(S, feat_res, batch, self.flat.device, self.c_geom, self.hsize, tensor_cores=self.tensor_cores, frames=frames)
            self._states[key] = st
        st.bn_running = self.bn_running
        st.track_running = True     # the reference never calls .eval(): BatchNorm always uses batch statistics (SURVEY §3.2)
        return st

    def forward_packed(self, geo_feature: torch.Tensor, S: int, batch: int = 1) -> torch.Tensor:
        """Fast path: geo_feature [1,c_geom,h,h] -> packed decoder output [S*S, 8] = (res.xyz, scale, rgb, 0), computed
        once for the whole batch (stage-1 inputs are identical across frames)."""
        st = self._state(S, geo_feature.shape[-1], batch)
        return DecoderNet.apply(self.flat, geo_feature, None, st)

    def forward_packed_frames(self, geo_feature: torch.Tensor, pose_featmap: torch.Tensor, S: int) -> torch.Tensor:
        """Stage 2 (model/network.py:55-58): pix_feature = pose_featmap [B,c,h,h] + geom convs(geo_feature), one decoder evaluation
        per frame, BatchNorm statistics over all B*S*S positions -> packed output [B*S*S, 8]."""
        B = int(pose_featmap.shape[0])
        st = self._state(S, geo_feature.shape[-1], B, frames=B)
        return DecoderNet.apply(self.flat, geo_feature, pose_featmap, st)

    def forward(self, pose_featmap, geom_featmap, uv_loc):
        """Reference signature (model/network.py:39): returns residuals [B,3,HW], scales [B,1,HW], shs [B,3,HW]."""
        B = geom_featmap.shape[0]
        S = int(round(uv_loc.shape[1] ** 0.5))
        if pose_featmap is not None:      # stage 2: per-frame inputs (the reference expands ONE geo_feature to the batch, avatar_model.py:398)
            dec = self.forward_packed_frames(geom_featmap[:1], pose_featmap, S).reshape(B, S * S, 8)
            t = dec.permute(0, 2, 1)                                # [B, 8, HW]
            return t[:, 0:3], t[:, 3:4], t[:, 4:7]
        # the reference expands one geo_feature to the batch (avatar_model.py:298); identical rows -> evaluate once
        geo = geom_featmap[:1]
        dec = self.forward_packed(geo, S, B)                       # [HW, 8]
        t = dec.t()                                                # [8, HW]
        return (t[0:3].unsqueeze(0).expand(B, -1, -1), t[3:4].unsqueeze(0).expand(B, -1, -1), t[4:7].unsqueeze(0).expand(B, -1, -1))
