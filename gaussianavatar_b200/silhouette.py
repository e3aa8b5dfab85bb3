"""Soft silhouettes of a posed body and SMPL / SMPL-X pose refinement against a capture's masks, on the device.

The reference's "Run on Your Own Video" path refines raw monocular pose estimates (ROMP) by fitting the body's silhouette to the
masks with pytorch3d's soft rasterizer (InstantAvatar's preprocessing, which writes poses_optimized.npz).  `SilhouetteRenderer`
draws the library's own soft silhouette (`ga_silhouette_forward` / `ga_silhouette_backward`, csrc/silhouette.cu; the function is
defined there and in DESIGN.md §2, PARITY UNPINNED) and `PoseRefiner` fits a whole sequence of one camera with it.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import _lib
from ._lib import ptr
from .mesh_render import MeshRenderer, coverage_iou, vertex_face_csr
from .posmap import MAX_FRAMES_PER_CALL, vertices_backward
from .rasterizer import CAM_STRIDE

MAX_SIDE = 16384
BETAS = (0.9, 0.999)
EPS = 1e-8


class SilhouetteRenderer:
    """Soft silhouettes of a fixed triangle mesh, faces [F,3] over V vertices; sigma in pixels^2.

    `render(verts [B,V,3], cams [B,40], H, W)` -> sil [B,H,W]; `loss(verts, cams, masks [B,H,W] uint8)` -> [B] = mean_p (S - M)^2
    with M = (mask >= 128), differentiable with respect to verts; `verts_grad(verts, cams, masks, w [B])` -> d_verts [B,V,3] of
    sum_b w_b loss_b.  Frames go to the kernels at most 8 per call; everything runs on the current CUDA stream and there is no
    CPU fallback."""

    def __init__(self, faces, V: int, sigma: float = 1.0, device="cuda"):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("SilhouetteRenderer runs on CUDA only (no CPU fallback)")
        f = np.asarray(faces.cpu() if torch.is_tensor(faces) else faces)
        if f.ndim != 2 or f.shape[1] != 3 or not np.issubdtype(f.dtype, np.integer):
            raise ValueError(f"faces {f.shape} {f.dtype}: expected an integer [F,3] array")
        self.V, self.F = int(V), f.shape[0]
        if not 1 <= self.V <= 1 << 24 or self.F > 1 << 24:
            raise ValueError(f"{self.V} vertices / {self.F} faces outside the kernel's range (1..2^24 / 0..2^24)")
        if f.size and (f.min() < 0 or f.max() >= self.V):
            raise ValueError(f"a face indexes a vertex outside 0..{self.V - 1}")
        self.sigma = float(np.float32(sigma))
        if not (self.sigma > 0 and math.isfinite(self.sigma)):
            raise ValueError(f"sigma {sigma} is not a positive number")
        off, adj = vertex_face_csr(f, self.V)
        self.faces = torch.from_numpy(f.astype(np.int32)).to(self.device).contiguous()
        self.adj_offsets = torch.from_numpy(off).to(self.device)
        self.adj_faces = torch.from_numpy(adj).to(self.device)
        self._ws = None

    def _workspace(self, B, H, W):
        n = _lib.lib().ga_silhouette_workspace_bytes(B, self.V, self.F, H, W)
        if self._ws is None or self._ws.numel() < n:
            self._ws = torch.empty(n, dtype=torch.uint8, device=self.device)
        return self._ws

    def _check(self, verts, cams, H, W, masks=None):
        H, W = int(H), int(W)
        if not (1 <= H <= MAX_SIDE and 1 <= W <= MAX_SIDE):
            raise ValueError(f"frame {H} x {W} outside [1, {MAX_SIDE}]^2")
        verts = torch.as_tensor(verts).detach().to(device=self.device, dtype=torch.float32).contiguous()
        if verts.dim() != 3 or tuple(verts.shape[1:]) != (self.V, 3):
            raise ValueError(f"vertices {tuple(verts.shape)}: expected [B,{self.V},3]")
        B = verts.shape[0]
        cams = torch.as_tensor(cams).to(device=self.device, dtype=torch.float32).contiguous()
        if tuple(cams.shape) != (B, CAM_STRIDE):
            raise ValueError(f"cameras {tuple(cams.shape)}: expected [{B},{CAM_STRIDE}]")
        if masks is not None:
            masks = torch.as_tensor(masks).to(self.device)
            if masks.dtype == torch.bool:
                masks = masks.to(torch.uint8) * 255
            if masks.dtype != torch.uint8 or tuple(masks.shape) != (B, H, W):
                raise ValueError(f"masks {tuple(masks.shape)} {masks.dtype}: expected uint8 or bool [{B},{H},{W}]")
            masks = masks.contiguous()
        return verts, cams, H, W, masks

    @staticmethod
    def _stream():
        return torch.cuda.current_stream().cuda_stream

    def _forward(self, verts, cams, H, W, masks):
        B = verts.shape[0]
        sil = torch.empty(B, H, W, dtype=torch.float32, device=self.device)
        loss = torch.empty(B, dtype=torch.float32, device=self.device) if masks is not None else None
        L = _lib.lib()
        for s in range(0, B, MAX_FRAMES_PER_CALL):
            e = min(B, s + MAX_FRAMES_PER_CALL)
            ws = self._workspace(e - s, H, W)
            _lib.check(L.ga_silhouette_forward(e - s, self.V, self.F, H, W, self.sigma, ptr(verts[s:e]), ptr(self.faces), ptr(cams[s:e]),
                                               None if masks is None else ptr(masks[s:e]), ptr(ws), ptr(sil[s:e]),
                                               None if loss is None else ptr(loss[s:e]), self._stream()), "ga_silhouette_forward")
        return sil, loss

    @torch.no_grad()
    def render(self, verts, cams, H: int, W: int) -> torch.Tensor:
        verts, cams, H, W, _ = self._check(verts, cams, H, W)
        return self._forward(verts, cams, H, W, None)[0]

    @torch.no_grad()
    def losses(self, verts, cams, masks) -> torch.Tensor:
        """Per-frame losses [B] without a graph (the forward kernel alone)."""
        masks = torch.as_tensor(masks)
        verts, cams, H, W, masks = self._check(verts, cams, masks.shape[-2], masks.shape[-1], masks)
        return self._forward(verts, cams, H, W, masks)[1]

    @torch.no_grad()
    def verts_grad(self, verts, cams, masks, w) -> torch.Tensor:
        masks = torch.as_tensor(masks)
        verts, cams, H, W, masks = self._check(verts, cams, masks.shape[-2], masks.shape[-1], masks)
        B = verts.shape[0]
        w = torch.as_tensor(w).to(device=self.device, dtype=torch.float32).reshape(-1).contiguous()
        if w.numel() != B:
            raise ValueError(f"weights {w.numel()}: expected {B}")
        d_verts = torch.empty(B, self.V, 3, dtype=torch.float32, device=self.device)
        L = _lib.lib()
        for s in range(0, B, MAX_FRAMES_PER_CALL):
            e = min(B, s + MAX_FRAMES_PER_CALL)
            ws = self._workspace(e - s, H, W)
            _lib.check(L.ga_silhouette_backward(e - s, self.V, self.F, H, W, self.sigma, ptr(verts[s:e]), ptr(self.faces),
                                                ptr(self.adj_offsets), ptr(self.adj_faces), ptr(cams[s:e]), ptr(masks[s:e]), ptr(w[s:e]),
                                                ptr(ws), ptr(d_verts[s:e]), self._stream()), "ga_silhouette_backward")
        return d_verts

    def loss(self, verts, cams, masks) -> torch.Tensor:
        """Per-frame losses [B], differentiable with respect to verts."""
        return _SilhouetteLoss.apply(self, verts, cams, masks)


class _SilhouetteLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, renderer, verts, cams, masks):
        ctx.renderer = renderer
        ctx.save_for_backward(verts.detach(), torch.as_tensor(cams), torch.as_tensor(masks))
        return renderer.losses(verts, cams, masks)

    @staticmethod
    def backward(ctx, d_loss):
        verts, cams, masks = ctx.saved_tensors
        d = ctx.renderer.verts_grad(verts, cams, masks, d_loss)
        return None, d.to(verts.dtype), None, None


class PoseRefiner:
    """Refines the SMPL / SMPL-X poses and translations of a whole sequence of one camera against its masks.

    poser: `posmap.BodyPoser` or `SmplxBodyPoser` (betas fixed); renderer: a `SilhouetteRenderer` over the poser's faces.
    `refine(pose, transl, cam, masks)` minimises, with theta = [pose | transl] and frames in the order given,

        sum_f loss_f + lambda_smooth sum_f |theta_{f+1} - theta_f|^2 + lambda_prior sum_f |theta_f - theta_f^0|^2

    by `iters` Adam steps (`ga_adam_step_dev`) on the whole sequence at once: each step runs every chunk of <= 8 frames through the
    vertices, the silhouette loss's backward and the vertex-posing backward into one [F, W+3] gradient.  SMPL-X's rest pose (jaw,
    eyes, hands) is held fixed."""

    def __init__(self, poser, renderer, iters: int = 100, lr: float = 1e-2, lambda_smooth: float = 0.0, lambda_prior: float = 0.0):
        if int(iters) < 0:
            raise ValueError(f"iters {iters} is negative")
        if not (lr > 0 and math.isfinite(lr)):
            raise ValueError(f"lr {lr} is not a positive number")
        if not (lambda_smooth >= 0 and lambda_prior >= 0):
            raise ValueError("lambda_smooth and lambda_prior must be >= 0")
        if renderer.V != poser.V or renderer.F != poser.F:
            raise ValueError(f"the renderer's mesh ({renderer.V} / {renderer.F}) is not the poser's ({poser.V} / {poser.F})")
        self.poser, self.renderer = poser, renderer
        self.iters, self.lr = int(iters), float(lr)
        self.lambda_smooth, self.lambda_prior = float(lambda_smooth), float(lambda_prior)
        self.dev = poser.device
        self._mesh = None
        b1, b2 = BETAS
        k = torch.arange(1, self.iters + 1, dtype=torch.float64)
        hyper = torch.stack([torch.full_like(k, self.lr), torch.full_like(k, b1), torch.full_like(k, b2), torch.full_like(k, EPS),
                             1.0 - b1 ** k, torch.sqrt(1.0 - b2 ** k), torch.ones_like(k)], 1)
        self._hyper = hyper.float().to(self.dev).contiguous()

    def _quadratic(self, theta, theta0):
        """(value, gradient) of the smoothness and prior terms."""
        d = theta[1:] - theta[:-1]
        r = theta - theta0
        val = self.lambda_smooth * (d * d).sum() + self.lambda_prior * (r * r).sum()
        g = 2.0 * self.lambda_prior * r
        g[1:] += 2.0 * self.lambda_smooth * d
        g[:-1] -= 2.0 * self.lambda_smooth * d
        return val, g

    def _chunk(self, theta, rest, s, e):
        """(pose, rest_pose, transl) of frames s..e-1, from theta = [pose | transl] and the rest poses (None for SMPL)."""
        W = self.poser.body.pose_width
        return theta[s:e, :W].contiguous(), None if rest is None else rest[s:e], theta[s:e, W:].contiguous()

    def _losses(self, theta, rest, cams, masks):
        out = []
        for s in range(0, theta.shape[0], MAX_FRAMES_PER_CALL):
            e = min(theta.shape[0], s + MAX_FRAMES_PER_CALL)
            verts = self.poser.posed(*self._chunk(theta, rest, s, e))
            out.append(self.renderer.losses(verts, cams[s:e], masks[s:e]))
        return torch.cat(out)

    def _ious(self, theta, rest, cams, masks):
        """Each frame's hard IoU: ga_mesh_render coverage against mask >= 128 (tools/body_overlay.py --iou's rule)."""
        if self._mesh is None:
            self._mesh = MeshRenderer(self.poser.faces, self.poser.V, device=self.dev)
        H, Wd = masks.shape[-2:]
        ious = []
        for s in range(0, theta.shape[0], MAX_FRAMES_PER_CALL):
            e = min(theta.shape[0], s + MAX_FRAMES_PER_CALL)
            verts = self.poser.posed(*self._chunk(theta, rest, s, e))
            _, face_id, _ = self._mesh.render(verts, cams[s:e], H, Wd)
            ious += [coverage_iou(face_id[i] >= 0, masks[s + i] >= 128) for i in range(e - s)]
        return ious

    def refine(self, pose, transl, cam, masks):
        """pose [F,72] / [F,165], transl [F,3], cam: one camera block [40] (or [F,40]), masks [F,H,W] uint8 (>= 128: subject).
        Returns (pose, transl, report) on the host, pose as wide as given (SMPL-X's rest pose unchanged); report holds the objective
        and each frame's IoU before and after."""
        p, rest = self.poser.body.split(torch.as_tensor(pose).to(device=self.dev, dtype=torch.float32))
        transl = torch.as_tensor(transl).to(device=self.dev, dtype=torch.float32).reshape(-1, 3)
        n = p.shape[0]
        if transl.shape[0] != n:
            raise ValueError(f"pose has {n} frames, transl {transl.shape[0]}")
        masks = torch.as_tensor(masks).to(self.dev)
        if masks.dtype != torch.uint8 or masks.dim() != 3 or masks.shape[0] != n:
            raise ValueError(f"masks {tuple(masks.shape)} {masks.dtype}: expected uint8 [{n},H,W]")
        masks = masks.contiguous()
        cams = torch.as_tensor(cam).to(device=self.dev, dtype=torch.float32)
        cams = (cams.reshape(1, CAM_STRIDE).expand(n, CAM_STRIDE) if cams.numel() == CAM_STRIDE else cams.reshape(n, CAM_STRIDE)).contiguous()
        W = self.poser.body.pose_width
        theta0 = torch.cat([p, transl], 1).contiguous()
        theta = theta0.clone()

        def objective(t):
            return float(self._losses(t, rest, cams, masks).double().sum()) + float(self._quadratic(t, theta0)[0])

        before, iou_before = objective(theta), self._ious(theta, rest, cams, masks)
        if self.iters:
            L = _lib.lib()
            stream = torch.cuda.current_stream().cuda_stream
            grad = torch.empty_like(theta)
            exp_avg, exp_avg_sq = torch.zeros_like(theta), torch.zeros_like(theta)
            ones = torch.ones(MAX_FRAMES_PER_CALL, dtype=torch.float32, device=self.dev)
            for k in range(self.iters):
                for s in range(0, n, MAX_FRAMES_PER_CALL):
                    e = min(n, s + MAX_FRAMES_PER_CALL)
                    tp, r, tt = self._chunk(theta, rest, s, e)
                    verts = self.poser.posed(tp, r, tt)
                    d_verts = self.renderer.verts_grad(verts, cams[s:e], masks[s:e], ones[:e - s])
                    d_pose, d_transl = vertices_backward(self.poser, tp, r, d_verts)
                    grad[s:e, :W] = d_pose
                    grad[s:e, W:] = d_transl
                grad += self._quadratic(theta, theta0)[1]
                _lib.check(L.ga_adam_step_dev(theta.numel(), ptr(theta), ptr(grad), ptr(exp_avg), ptr(exp_avg_sq), ptr(self._hyper[k]),
                                              None, stream), "ga_adam_step_dev")
        after, iou_after = objective(theta), self._ious(theta, rest, cams, masks)
        out_pose = self.poser.body.join(theta[:, :W], rest)
        report = dict(objective_before=before, objective_after=after, iou_before=iou_before, iou_after=iou_after,
                      mean_iou_before=float(np.mean(iou_before)), mean_iou_after=float(np.mean(iou_after)))
        return out_pose.cpu(), theta[:, W:].cpu(), report
