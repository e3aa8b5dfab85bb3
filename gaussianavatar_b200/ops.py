"""torch.autograd bridges over the C ABI for the non-rasterizer stages of the hot path.

Each Function only moves pointers: all device work happens inside libgavatar_sm90.so on the current CUDA stream.
There is no CPU implementation behind these — CPU tensors raise.
"""
from __future__ import annotations

import ctypes

import torch

from . import _lib
from ._lib import ptr


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _need_cuda(t: torch.Tensor, what: str):
    if not t.is_cuda:
        raise RuntimeError(f"{what}: gaussianavatar_b200 needs CUDA tensors (no CPU fallback)")


def _f32c(t: torch.Tensor) -> torch.Tensor:
    return t.float().contiguous() if (t.dtype != torch.float32 or not t.is_contiguous()) else t


def _rows(t, device) -> torch.Tensor:
    return torch.as_tensor(t).to(device=device, dtype=torch.float32).contiguous()


class Cano2Live(torch.autograd.Function):
    """body (`body.SMPL` / `body.SMPLX`), pose [B,72], rest_pose None, transl [B,3] -> cano2live [B,24,12] (3x4 per joint); SMPL-X:
    pose [B,66] (global + 21 body joints), rest_pose [B,99] (jaw, eyes, 2 x 15 finger joints) -> [B,55,12].  Gradients flow to pose
    and transl only: rest_pose is data.  Reference: model/avatar_model.py:279-296 (SMPL.forward(...).A @ inv_mats)."""

    @staticmethod
    def forward(ctx, body, pose, rest_pose, transl, rest_joints, inv_cano):
        _need_cuda(pose, "Cano2Live")
        B = pose.shape[0]
        got = [None if t is None else tuple(t.shape) for t in (pose, rest_pose, transl)]
        want = [(B, body.pose_width), (B, body.rest_width) if body.rest_width else None, (B, 3)]
        if got != want:
            raise ValueError(f"{body.label} cano2live: (pose, rest_pose, transl) {got}; expected {want}")
        dev = pose.device
        poses = [_rows(p, dev) for p in body.pose_args(pose, rest_pose)]
        transl = _rows(transl, dev)
        C = torch.empty(B, body.joints, 12, device=dev, dtype=torch.float32)
        G = torch.empty(B, body.joints, 12, device=dev, dtype=torch.float32)
        _lib.check(getattr(_lib.lib(), body.cano2live)(B, *(ptr(p) for p in poses), ptr(transl), ptr(rest_joints), ptr(inv_cano), ptr(C),
                                                       ptr(G), _stream()), body.cano2live)
        ctx.body = body
        ctx.save_for_backward(*poses, rest_joints, inv_cano, G)
        return C

    @staticmethod
    def backward(ctx, dC):
        *poses, rest_joints, inv_cano, G = ctx.saved_tensors
        body = ctx.body
        B = poses[0].shape[0]
        dC = _f32c(dC)
        d_pose = torch.empty_like(poses[0])
        d_transl = torch.empty(B, 3, device=dC.device, dtype=torch.float32)
        _lib.check(getattr(_lib.lib(), body.cano2live_bwd)(B, *(ptr(p) for p in poses), ptr(rest_joints), ptr(inv_cano), ptr(G), ptr(dC),
                                                           ptr(d_pose), ptr(d_transl), _stream()), body.cano2live_bwd)
        return None, d_pose, None, d_transl, None, None


class LbsAssemble(torch.autograd.Function):
    """dec_out [S*S,8] (stage 1: one output for all frames) or [B*S*S,8] (stage 2: per frame), cano2live [B,J,12] (J = 24 for SMPL,
    55 for SMPL-X), query_lbs [N,ld] (ld = 24, or 56 for SMPL-X: the 55 weights and a zero column)
    -> means3D, scales, colors [B,N,3] (model/avatar_model.py:308-326 / :407-420).

    exposure [F,3,4] (optional, with pose_idx [B]): frame b's colours become A c + t, [A | t] = exposure[pose_idx[b]], inside the
    same kernel; the table gets a gradient, zero in row 0 (the gauge anchor, DESIGN.md §4).  pose_idx is moved to the device as
    int32 and read there only."""

    @staticmethod
    def forward(ctx, dec_out, cano2live, valid_index, query_points, query_lbs, scale_mul, per_frame=False, exposure=None, pose_idx=None):
        _need_cuda(dec_out, "LbsAssemble")
        dec_out, cano2live = _f32c(dec_out), _f32c(cano2live)
        N, B = int(query_points.shape[0]), int(cano2live.shape[0])
        J, ld = int(cano2live.shape[1]), int(query_lbs.shape[1])
        stride = (dec_out.shape[0] // B) * 8 if per_frame else 0
        if per_frame and dec_out.shape[0] % B:
            raise RuntimeError("per-frame decoder output must have B * S*S rows")
        dev = dec_out.device
        means = torch.empty(B, N, 3, device=dev, dtype=torch.float32)
        scales = torch.empty(B, N, 3, device=dev, dtype=torch.float32)
        colors = torch.empty(B, N, 3, device=dev, dtype=torch.float32)
        if exposure is None:
            _lib.check(_lib.lib().ga_lbs_forward_ex(N, B, J, ld, float(scale_mul), stride, ptr(dec_out), ptr(valid_index), ptr(query_points),
                                                    ptr(query_lbs), ptr(cano2live), ptr(means), ptr(scales), ptr(colors), _stream()),
                       "ga_lbs_forward_ex")
            table = idx = None
        else:
            if pose_idx is None:
                raise ValueError("LbsAssemble: an exposure table needs the pose_idx it is indexed by")
            if exposure.dim() != 3 or tuple(exposure.shape[1:]) != (3, 4):
                raise ValueError(f"exposure {tuple(exposure.shape)}: expected [F,3,4]")
            table = _f32c(exposure.detach())
            idx = torch.as_tensor(pose_idx).to(device=dev, dtype=torch.int32).reshape(-1).contiguous()
            if idx.numel() != B:
                raise ValueError(f"pose_idx has {idx.numel()} entries for {B} frames")
            _lib.check(_lib.lib().ga_lbs_forward_exposure(N, B, J, ld, float(scale_mul), stride, ptr(dec_out), ptr(valid_index),
                                                          ptr(query_points), ptr(query_lbs), ptr(cano2live), int(table.shape[0]), ptr(table),
                                                          ptr(idx), ptr(means), ptr(scales), ptr(colors), _stream()),
                       "ga_lbs_forward_exposure")
        ctx.save_for_backward(dec_out, cano2live, valid_index, query_points, query_lbs, table, idx)
        ctx.scale_mul, ctx.stride = float(scale_mul), stride
        return means, scales, colors

    @staticmethod
    def backward(ctx, d_means, d_scales, d_colors):
        dec_out, cano2live, valid_index, query_points, query_lbs, table, idx = ctx.saved_tensors
        N, B = int(query_points.shape[0]), int(cano2live.shape[0])
        dev = dec_out.device
        zeros = None

        def z(t):
            nonlocal zeros
            if t is None:
                if zeros is None:
                    zeros = torch.zeros(B, N, 3, device=dev, dtype=torch.float32)
                return zeros
            return _f32c(t)

        d_means, d_scales, d_colors = z(d_means), z(d_scales), z(d_colors)
        d_dec = torch.empty_like(dec_out)
        dC = torch.empty_like(cano2live)
        J, ld = int(cano2live.shape[1]), int(query_lbs.shape[1])
        if table is None:
            _lib.check(_lib.lib().ga_lbs_backward_ex(N, B, J, ld, int(dec_out.shape[0]), ctx.scale_mul, ctx.stride, ptr(dec_out),
                                                     ptr(valid_index), ptr(query_points), ptr(query_lbs), ptr(cano2live), ptr(d_means),
                                                     ptr(d_scales), ptr(d_colors), ptr(d_dec), ptr(dC), _stream()), "ga_lbs_backward_ex")
            return d_dec, dC, None, None, None, None, None, None, None
        L = _lib.lib()
        nbytes = int(L.ga_lbs_exposure_workspace_bytes(N, J))
        ws = torch.empty(max(nbytes, 4), device=dev, dtype=torch.uint8)
        d_table = torch.empty_like(table)
        _lib.check(L.ga_lbs_backward_exposure(N, B, J, ld, int(dec_out.shape[0]), ctx.scale_mul, ctx.stride, ptr(dec_out), ptr(valid_index),
                                              ptr(query_points), ptr(query_lbs), ptr(cano2live), int(table.shape[0]), ptr(table), ptr(idx),
                                              ptr(d_means), ptr(d_scales), ptr(d_colors), ptr(d_dec), ptr(dC), ptr(d_table), ptr(ws), nbytes,
                                              _stream()), "ga_lbs_backward_exposure")
        return d_dec, dC, None, None, None, None, None, d_table, None


class DecoderNet(torch.autograd.Function):
    """flat params, geo_feature [1,64,h,h] (+ pose_featmap [B,64,h,h] in stage 2) -> dec_out [frames*S*S,8]
    (model/network.py:39-83; frames = 1 with pose_featmap=None: the batch shares one evaluation)."""

    @staticmethod
    def forward(ctx, flat, geo_feature, pose_feat, state):
        _need_cuda(flat, "DecoderNet")
        L = _lib.lib()
        desc = state.desc
        S = desc.S
        frames = max(1, int(desc.frames))
        dec = torch.empty(frames * S * S, 8, device=flat.device, dtype=torch.float32)
        geo = _f32c(geo_feature)
        pf = _f32c(pose_feat) if pose_feat is not None else None
        if pf is not None and (pf.shape[0] != frames or tuple(pf.shape[1:]) != tuple(geo.shape[1:])):
            raise RuntimeError(f"pose_featmap {tuple(pf.shape)} does not match frames={frames} x geo_feature {tuple(geo.shape[1:])}")
        running = state.bn_running if state.track_running else None
        _lib.check(L.ga_decoder_forward(ctypes.byref(desc), ptr(flat), ptr(geo), ptr(pf), ptr(running), ptr(state.workspace), ptr(dec),
                                        _stream()), "ga_decoder_forward")
        if state.track_running:
            state.num_batches_tracked += 1
        # the activations live in ONE workspace per decoder state, not per autograd graph: stamp the forward so that a backward that
        # arrives after a later forward on the same state (a second loss(), a logging render, retain_graph reuse) fails loudly
        # instead of differentiating through the wrong activations
        state.generation = getattr(state, "generation", 0) + 1
        ctx.generation = state.generation
        ctx.state = state
        ctx.geo_shape = geo_feature.shape
        ctx.pose_shape = None if pose_feat is None else pose_feat.shape
        ctx.save_for_backward(flat, dec)
        return dec

    @staticmethod
    def backward(ctx, d_dec):
        flat, dec = ctx.saved_tensors
        state = ctx.state
        if ctx.generation != state.generation:
            raise RuntimeError("DecoderNet.backward: the decoder ran forward again on the same (S, feat_res, batch) state since this graph was "
                               "built; its activation workspace has been overwritten (run backward before the next forward)")
        d_dec = _f32c(d_dec)
        d_flat = torch.empty_like(flat)
        d_geo = torch.empty(ctx.geo_shape, device=flat.device, dtype=torch.float32)
        d_pose = torch.empty(ctx.pose_shape, device=flat.device, dtype=torch.float32) if ctx.pose_shape is not None else None
        _lib.check(_lib.lib().ga_decoder_backward(ctypes.byref(state.desc), ptr(flat), ptr(state.workspace), ptr(dec), ptr(d_dec),
                                                  ptr(d_flat), ptr(d_geo), ptr(d_pose), _stream()), "ga_decoder_backward")
        return d_flat, d_geo, d_pose, None
