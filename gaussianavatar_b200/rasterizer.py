"""`diff_gaussian_rasterization`-compatible Python surface over the sm_90a rasterizer.

Mirrors the API generation the reference binds at /root/reference gaussian_renderer/__init__.py:6,21-48:
``GaussianRasterizationSettings`` (12-field NamedTuple, plus upstream's later 13th field ``antialiasing`` after ``debug``,
default False, so the 12-field positional form still works), ``GaussianRasterizer(raster_settings)(means3D=, means2D=, shs=,
colors_precomp=, opacities=, scales=, rotations=, cov3D_precomp=) -> (color[3,H,W], radii[P])``, gradients returned in
input order.  Validation behaviour follows [UPSTREAM] (SURVEY.md §8b): exactly one of shs / colors_precomp and exactly
one of (scales+rotations) / cov3D_precomp, else ``Exception``.

All four input combinations run on the device: colours precomputed or evaluated from spherical harmonics (``shs`` [P, M, 3]
with ``raster_settings.sh_degree`` D in 0..3, (D+1)^2 <= M, seen from ``raster_settings.campos``), and 3D covariances built from
``scales`` + ``rotations`` (times ``scale_modifier``) or given as ``cov3D_precomp`` [P, 6] = (xx, xy, xz, yy, yz, zz).
GaussianAvatar itself passes precomputed colours with scales + rotations (shs=None at model/avatar_model.py:350,
cov3D_precomp=None at gaussian_renderer/__init__.py:37); the batched training path supports only that combination.

``antialiasing`` (per call here, ``RasterBatchPlan(antialiasing=)`` for the batched path, ``GaussianScene.antialiasing`` for a
scene) is upstream's screen-space filter: each splat's opacity is scaled by sqrt(det Sigma2 / det(Sigma2 + 0.3 I)) so that its
footprint no longer depends on the 0.3 px^2 dilation (include/gavatar.h, DESIGN.md §4).
"""
from __future__ import annotations

import ctypes
from typing import NamedTuple

import torch
import torch.nn as nn

from . import _lib
from ._lib import GaRasterSettings, ptr


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool
    antialiasing: bool = False


def _c(t: torch.Tensor) -> torch.Tensor:
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _grab(buf, addr, shape, dtype):
    """Typed host copy of a region of an opaque device buffer (parity tests)."""
    n = 1
    for d in shape:
        n *= d
    if addr is None or n == 0:
        return torch.zeros(shape, dtype=dtype)
    off = addr - buf.data_ptr()
    nbytes = n * torch.empty((), dtype=dtype).element_size()
    return buf[off:off + nbytes].view(dtype).reshape(shape).clone().cpu()


def _views(B, P, H, W, capacity, geom, binning, img, radii):
    """Per-frame list of dicts with the rasterizer's per-stage state, in the terms upstream's pipeline is specified in
    (SURVEY.md §8 a-8): `keys_sorted` / `vals_sorted` are the sorted (tile << 32 | depth bits, Gaussian index) list —
    rebuilt here from the per-tile sorted index list, the tile ranges and the depths, because the device pipeline bins by
    tile and never materialises global 64-bit keys — and `ranges` / `offsets` are per-frame, starting at 0."""
    L = _lib.lib()
    v = _lib.GaRasterViews()
    _lib.check(L.ga_raster_views(B, P, H, W, capacity, ptr(geom), ptr(binning), ptr(img), ctypes.byref(v)), "ga_raster_views")
    T = ((W + 15) // 16) * ((H + 15) // 16)
    status = _grab(img, v.status, (16,), torch.int32)
    R_total, overflow = int(status[0]), int(status[1])
    n_list = min(R_total, capacity)
    plist = _grab(binning, v.point_list, (n_list,), torch.int32) if binning is not None else torch.zeros(0, dtype=torch.int32)
    allv = dict(depth=_grab(geom, v.depth, (B, P), torch.float32), xy=_grab(geom, v.xy, (B, P, 2), torch.float32),
                conic_opacity=_grab(geom, v.conic_opacity, (B, P, 4), torch.float32), cov3d=_grab(geom, v.cov3d, (B, P, 6), torch.float32),
                tiles_touched=_grab(geom, v.tiles_touched, (B, P), torch.int32), rect=_grab(geom, v.rect, (B, P, 4), torch.int16),
                ranges=_grab(img, v.ranges, (B, T, 2), torch.int32), tile_count=_grab(img, v.tile_count, (B, T), torch.int32),
                final_T=_grab(img, v.final_T, (B, H, W), torch.float32), n_contrib=_grab(img, v.n_contrib, (B, H, W), torch.int32))
    out = []
    for b in range(B):
        base, end = int(status[4 + b]), int(status[4 + b + 1])
        f = {k: t[b] for k, t in allv.items()}
        f["radii"] = radii.reshape(B, P)[b].clone().cpu()
        f["num_rendered"] = end - base
        f["overflow"] = overflow
        f["offsets"] = torch.cumsum(f["tiles_touched"].to(torch.int64), 0).to(torch.int32)
        rg = f["ranges"].to(torch.int64)
        nonempty = rg[:, 1] > rg[:, 0]
        rg[nonempty] -= base
        f["ranges"] = rg.to(torch.int32)
        if not overflow and end > base:
            vals = plist[base:end]
            lens = (rg[:, 1] - rg[:, 0])
            tile_of = torch.repeat_interleave(torch.arange(T, dtype=torch.int64), lens)
            dbits = f["depth"].view(torch.int32).to(torch.int64)[vals.to(torch.int64)] & 0xffffffff
            f["vals_sorted"] = vals
            f["keys_sorted"] = (tile_of << 32) | dbits
        out.append(f)
    return out


class RasterContext:
    """Buffers one forward leaves behind for its backward (upstream's geomBuffer / binningBuffer / imgBuffer).  With shs or
    cov3D_precomp, `cc` is the GaRasterColorCov of the forward and `keep` holds the tensors it points to (rgb [P,3] is the
    evaluated SH colour, clamped [P] uint8 its per-channel clamp bits)."""
    __slots__ = ("settings", "geom", "binning", "img", "num_rendered", "radii", "cc", "keep", "rgb", "clamped")

    def views(self) -> dict:
        """Typed tensor copies of the internal per-stage state (parity tests)."""
        s = self.settings
        return _views(1, s.P, s.H, s.W, self.num_rendered, self.geom, self.binning, self.img, self.radii)[0]


def _on_device(dev, **tensors):
    for name, t in tensors.items():
        if t is not None and t.device != dev:
            raise RuntimeError(f"gaussianavatar_b200 rasterizer: {name} is on {t.device}, means3D on {dev} (no CPU fallback)")


def _color_cov(P, dev, rs, shs, cov3D_precomp):
    """Checks shs / cov3D_precomp and returns (GaRasterColorCov or None, tensors it points to, rgb, clamped)."""
    if shs is None and cov3D_precomp is None:
        return None, (), None, None
    _on_device(dev, shs=shs, cov3D_precomp=cov3D_precomp)
    cc = _lib.GaRasterColorCov()
    keep, rgb, clamped = [], None, None
    if shs is not None:
        D = int(rs.sh_degree)
        if shs.dim() != 3 or shs.shape[0] != P or shs.shape[2] != 3:
            raise ValueError(f"shs must have shape [P={P}, M, 3], got {tuple(shs.shape)}")
        M = int(shs.shape[1])
        if not 0 <= D <= 3:
            raise ValueError(f"sh_degree must be in 0..3, got {D}")
        if (D + 1) ** 2 > M:
            raise ValueError(f"sh_degree {D} needs (D+1)^2 = {(D + 1) ** 2} coefficients, shs has {M}")
        if rs.campos is None or torch.as_tensor(rs.campos).numel() != 3:
            raise ValueError("shs needs raster_settings.campos (3 values)")
        shs = _c(shs)
        campos = _c(torch.as_tensor(rs.campos)).reshape(3).to(dev)
        rgb = torch.empty(P, 3, dtype=torch.float32, device=dev)
        clamped = torch.empty(P, dtype=torch.uint8, device=dev)
        cc.shs, cc.sh_degree, cc.sh_coeffs, cc.campos = ptr(shs), D, M, ptr(campos)
        cc.rgb, cc.clamped = ptr(rgb), ptr(clamped)
        keep += [shs, campos]
    if cov3D_precomp is not None:
        if tuple(cov3D_precomp.shape) != (P, 6):
            raise ValueError(f"cov3D_precomp must have shape [P={P}, 6], got {tuple(cov3D_precomp.shape)}")
        cov3D_precomp = _c(cov3D_precomp)
        cc.cov3D_precomp = ptr(cov3D_precomp)
        keep.append(cov3D_precomp)
    return cc, tuple(keep), rgb, clamped


def _aa(obj) -> int:
    """The C ABI's antialiasing flag of a settings tuple or scene (objects without the field: off, as upstream's 12-field form)."""
    return int(bool(getattr(obj, "antialiasing", False)))


def rasterize_forward(means3D, colors, opacities, scales, rotations, rs: GaussianRasterizationSettings, *, shs=None,
                      cov3D_precomp=None):
    """K1..K6 on the current CUDA stream.  Returns (color [3,H,W], radii [P] int32, RasterContext).
    shs [P,M,3] (colors None; degree and camera position from rs) and cov3D_precomp [P,6] (scales, rotations None) select
    the other input modes of upstream's API; every check runs before anything is launched."""
    if not means3D.is_cuda:
        raise RuntimeError("gaussianavatar_b200 rasterizer needs CUDA tensors (no CPU fallback)")
    L = _lib.lib()
    dev = means3D.device
    P, H, W = int(means3D.shape[0]), int(rs.image_height), int(rs.image_width)
    s = GaRasterSettings(P, H, W, float(rs.tanfovx), float(rs.tanfovy), float(rs.scale_modifier), _aa(rs))
    cc, keep, rgb, clamped = _color_cov(P, dev, rs, shs, cov3D_precomp)
    opt = lambda t: None if t is None else _c(t)
    means3D, colors, scales, rotations = _c(means3D), opt(colors), opt(scales), opt(rotations)
    _on_device(dev, colors=colors, scales=scales, rotations=rotations, opacities=opacities)
    opacities = _c(opacities).reshape(-1)
    bg, view, proj = _c(rs.bg).to(dev), _c(rs.viewmatrix).to(dev), _c(rs.projmatrix).to(dev)

    ctx = RasterContext()
    ctx.settings = s
    ctx.cc, ctx.keep, ctx.rgb, ctx.clamped = cc, keep, rgb, clamped
    ctx.geom = torch.empty(L.ga_raster_geom_bytes(P), dtype=torch.uint8, device=dev)
    ctx.img = torch.empty(L.ga_raster_img_bytes(H, W), dtype=torch.uint8, device=dev)
    ctx.radii = torch.empty(P, dtype=torch.int32, device=dev)
    n = ctypes.c_int64(0)
    st = _stream()
    _lib.check(L.ga_raster_forward_preprocess_ex(ctypes.byref(s), None if cc is None else ctypes.byref(cc), ptr(means3D), ptr(scales),
                                                 ptr(rotations), ptr(opacities), ptr(view), ptr(proj), ptr(ctx.geom), ptr(ctx.img),
                                                 ptr(ctx.radii), ctypes.byref(n), st), "ga_raster_forward_preprocess_ex")
    ctx.num_rendered = int(n.value)
    nb = L.ga_raster_binning_bytes(ctx.num_rendered, H, W)
    ctx.binning = torch.empty(nb, dtype=torch.uint8, device=dev)
    color = torch.empty(3, H, W, dtype=torch.float32, device=dev)
    _lib.check(L.ga_raster_forward_render(ctypes.byref(s), ptr(colors if rgb is None else rgb), ptr(bg), ptr(ctx.geom), ptr(ctx.binning),
                                          nb, ctx.num_rendered, ptr(ctx.img), ptr(color), st), "ga_raster_forward_render")
    return color, ctx.radii, ctx


def rasterize_backward(ctx: RasterContext, means3D, colors, scales, rotations, rs, grad_color, want_opacity=True,
                       want_rotations=True, want_means2D=True, *, return_sh_cov3D=False):
    """Gradients of the forward that filled ctx: (d_means3D, d_means2D, d_colors, d_opacities, d_scales, d_rotations), and with
    return_sh_cov3D=True also (d_sh, d_cov3D).  Gradients of inputs the forward did not take are None: with shs, d_colors (the
    colour is evaluated); with cov3D_precomp, d_scales and d_rotations."""
    if ctx.cc is not None and not return_sh_cov3D:
        raise ValueError("this forward took shs / cov3D_precomp: call rasterize_backward(..., return_sh_cov3D=True)")
    L = _lib.lib()
    dev = means3D.device
    s = ctx.settings
    P = s.P
    sh = ctx.rgb is not None
    cov = ctx.cc is not None and bool(ctx.cc.cov3D_precomp)
    opt = lambda t: None if t is None else _c(t)
    colors, scales, rotations = opt(colors), opt(scales), opt(rotations)
    grad_color = _c(grad_color)
    bg, view, proj = _c(rs.bg).to(dev), _c(rs.viewmatrix).to(dev), _c(rs.projmatrix).to(dev)
    scratch = torch.empty(L.ga_raster_bwd_scratch_bytes(P), dtype=torch.uint8, device=dev)
    d_means3D = torch.empty(P, 3, dtype=torch.float32, device=dev)
    d_colors = torch.empty(P, 3, dtype=torch.float32, device=dev)
    d_scales = torch.empty(P, 3, dtype=torch.float32, device=dev) if not cov else None
    d_rot = torch.empty(P, 4, dtype=torch.float32, device=dev) if want_rotations and not cov else None
    d_opac = torch.empty(P, 1, dtype=torch.float32, device=dev) if want_opacity else None
    d_m2d = torch.empty(P, 3, dtype=torch.float32, device=dev) if want_means2D else None
    d_sh = torch.empty(ctx.keep[0].shape, dtype=torch.float32, device=dev) if sh else None
    d_cov3D = torch.empty(P, 6, dtype=torch.float32, device=dev) if cov else None
    _lib.check(L.ga_raster_backward_ex(ctypes.byref(s), None if ctx.cc is None else ctypes.byref(ctx.cc), ptr(means3D), ptr(colors),
                                       ptr(scales), ptr(rotations), ptr(bg), ptr(view), ptr(proj), ptr(ctx.radii), ptr(ctx.geom),
                                       ptr(ctx.binning), ptr(ctx.img), ctx.num_rendered, ptr(grad_color), ptr(scratch), ptr(d_means3D),
                                       ptr(d_colors), ptr(d_scales), ptr(d_rot), ptr(d_opac), ptr(d_m2d), ptr(d_sh), ptr(d_cov3D),
                                       _stream()), "ga_raster_backward_ex")
    if return_sh_cov3D:
        return d_means3D, d_m2d, None if sh else d_colors, d_opac, d_scales, d_rot, d_sh, d_cov3D
    return d_means3D, d_m2d, d_colors, d_opac, d_scales, d_rot


# ----------------------------------------------------------------------------------------------------------------------
# Batched path: all frames of a step in one set of launches, no host read-back (model/avatar_model.py:332-365 loops frames)
# ----------------------------------------------------------------------------------------------------------------------
CAM_STRIDE = 40
MAX_FRAMES_PER_CALL = 8          # ga_rasterb_*


def pack_cameras(view, proj, tanfovx, tanfovy, device, campos=None):
    """[B,40] device floats: viewmatrix 0..15, projmatrix 16..31 (the reference's transposed 4x4s), tanfovx 32, tanfovy 33 and,
    when campos [B,3] is given, the camera centre 34..36 (upstream's `campos`, which the composite forward's SH colours need)."""
    B = view.shape[0]
    cams = torch.zeros(B, CAM_STRIDE, dtype=torch.float32, device=device)
    cams[:, 0:16] = view.reshape(B, 16).to(device=device, dtype=torch.float32)
    cams[:, 16:32] = proj.reshape(B, 16).to(device=device, dtype=torch.float32)
    if torch.is_tensor(tanfovx):
        cams[:, 32] = tanfovx.to(device=device, dtype=torch.float32)
        cams[:, 33] = tanfovy.to(device=device, dtype=torch.float32)
    else:
        cams[:, 32:34] = torch.tensor([list(map(float, tanfovx)), list(map(float, tanfovy))], dtype=torch.float32).t().to(device)
    if campos is not None:
        cams[:, 34:37] = torch.as_tensor(campos).reshape(B, 3).to(device=device, dtype=torch.float32)
    return cams


class RasterBatchPlan:
    """Caller-owned buffers of the batched rasterizer for one (B, P, H, W): geom / img / binning (capacity-bounded) / backward
    scratch, reused every step.  `capacity` is the number of (Gaussian, tile) instances the binning buffer holds; the device
    raises status[1] when a step needs more (nothing is overrun) and `check()` then grows the buffer — the caller re-runs
    the step.  The status words of every forward are copied to pinned host memory asynchronously; reading them never
    blocks the enqueueing thread unless asked to.

    static_P: the size of a static scene set the plan's forwards composite with (`rasterize_batch_scene`): geom and radii then
    cover P + static_P Gaussians per frame, and `scene_rgb` [B,static_P,3] receives the scene's per-frame SH colours.

    `rasterize_batch_with_depth` also uses `depth_state` (each pixel's depth sums at its checkpoints, sized from `capacity` and
    re-allocated with the binning buffer) and `depth_scratch`, both allocated on its first call.

    antialiasing: every forward and backward through the plan renders its dynamic set with antialiased opacities (`desc()`
    carries the flag; a scene's static set follows its own `GaussianScene.antialiasing`)."""

    def __init__(self, B, P, H, W, device, capacity=None, static_P=0, antialiasing=False):
        L = _lib.lib()
        self.B, self.P, self.H, self.W, self.device = int(B), int(P), int(H), int(W), device
        self.antialiasing = bool(antialiasing)
        self.static_P = int(static_P)
        Pt = self.P + self.static_P
        self.capacity = int(capacity) if capacity else max(1 << 16, 6 * self.B * Pt)
        self.geom = torch.empty(L.ga_rasterb_geom_bytes(self.B, Pt), dtype=torch.uint8, device=device)
        self.img = torch.empty(L.ga_rasterb_img_bytes(self.B, self.H, self.W), dtype=torch.uint8, device=device)
        self.scratch = torch.empty(L.ga_rasterb_bwd_scratch_bytes(self.B, self.P), dtype=torch.uint8, device=device)
        self.radii = torch.empty(self.B, Pt, dtype=torch.int32, device=device)
        self.scene_rgb = torch.empty(self.B, self.static_P, 3, dtype=torch.float32, device=device) if self.static_P else None
        self.binning = None
        self.depth_state = self.depth_scratch = None
        self._alloc_binning()
        off = L.ga_rasterb_status(self.B, self.H, self.W, ptr(self.img)) - self.img.data_ptr()
        self.status_dev = self.img[off:off + 64].view(torch.int32)
        # the 16 status words of the latest forward (+ its serial number in word 15), copied to pinned memory right behind the
        # forward; the serial tells the host WHICH forward the words belong to, so reading them needs no CUDA event (events
        # recorded inside a captured graph cannot be waited on) and never blocks unless the caller asks for it
        self.serial_dev = torch.zeros(1, dtype=torch.int32, device=device)
        self.status_host = torch.full((16,), -1, dtype=torch.int32).pin_memory()
        self.serial = 0
        self.pending = False

    def _alloc_binning(self):
        nb = _lib.lib().ga_rasterb_binning_bytes(self.B, self.H, self.W, self.capacity)
        self.binning = None
        self.binning = torch.empty(nb, dtype=torch.uint8, device=self.device)
        if self.depth_state is not None:
            self.depth_state = None
            self.alloc_depth()

    def alloc_depth(self):
        """The buffers of `rasterize_batch_with_depth` (kept until the plan is dropped; the state follows `capacity`)."""
        L = _lib.lib()
        if self.depth_state is None:
            nb = L.ga_rasterb_depth_state_bytes(self.B, self.H, self.W, self.capacity)
            self.depth_state = torch.empty(nb, dtype=torch.uint8, device=self.device)
        if self.depth_scratch is None:
            nb = L.ga_rasterb_depth_bwd_scratch_bytes(self.B, self.P)
            self.depth_scratch = torch.empty(nb, dtype=torch.uint8, device=self.device)

    def desc(self, rot_shared=True, opac_shared=True, scale_modifier=1.0):
        return _lib.GaRasterBatchDesc(self.B, self.P, self.H, self.W, self.capacity, 0 if rot_shared else 4 * self.P,
                                      0 if opac_shared else self.P, float(scale_modifier), int(self.antialiasing))

    def bump_serial(self):
        """Number the forward that is about to run (eager code; a captured graph cannot change it, so whoever replays a graph
        holding a forward calls this first)."""
        self.serial += 1
        self.serial_dev.fill_(int(self.serial))

    def record_status(self):
        if not torch.cuda.is_current_stream_capturing():
            self.bump_serial()
        _lib.check(_lib.lib().ga_rasterb_status_to_host(self.B, self.H, self.W, ptr(self.img), ptr(self.serial_dev),
                                                        self.status_host.data_ptr(), _stream()), "ga_rasterb_status_to_host")
        self.pending = True

    def check(self, wait=True) -> bool:
        """True if the last forward fitted the binning buffer.  On overflow the buffer is re-allocated (1.5 x the needed
        count) and False is returned: the caller must run the step again."""
        if not self.pending:
            return True
        import time
        while int(self.status_host[15]) != self.serial:      # the copy behind the latest forward has not landed yet
            if not wait:
                return True          # not known yet; ask again later
            time.sleep(5e-5)         # yield the core: a hot spin starves the driver's own threads on boxes with few CPUs
        self.pending = False
        if int(self.status_host[1]) == 0:
            return True
        self.grow(int(self.status_host[0]))
        return False

    def render_checked(self, render, label: str):
        """Runs render(), a call that renders one forward through this plan, and waits for its status.  If the forward overflowed
        the binning buffer (which `check` has then grown), runs it once more.  Returns (render()'s result, whether it was run
        again); a second overflow raises RuntimeError starting with `label`."""
        out = render()
        if self.check(wait=True):
            return out, False
        out = render()
        if not self.check(wait=True):
            raise RuntimeError(f"{label}: the rasterizer's binning buffer overflowed again after growing")
        return out, True

    def grow(self, needed: int):
        """Re-allocate the binning buffer for a forward that needed `needed` instances (status word 0), with headroom."""
        self.capacity = int(1.5 * int(needed)) + 1024
        self._alloc_binning()

    def views(self):
        return _views(self.B, self.P + self.static_P, self.H, self.W, self.capacity, self.geom, self.binning, self.img, self.radii)


def _batch_inputs(plan, means3D, colors, scales, rotations, opacities):
    """Every batched forward's prelude: (descriptor, means3D, colors, scales, rotations, opacities) as the entry points take them,
    opacities flattened and the rotation / opacity strides read from their shapes."""
    if not means3D.is_cuda:
        raise RuntimeError("gaussianavatar_b200 rasterizer needs CUDA tensors (no CPU fallback)")
    means3D, colors, scales, rotations = _c(means3D), _c(colors), _c(scales), _c(rotations)
    opacities = _c(opacities).reshape(-1)
    d = plan.desc(rot_shared=rotations.dim() == 2, opac_shared=opacities.numel() == plan.P)
    return d, means3D, colors, scales, rotations, opacities


def _batch_forward_tail(plan, cams, bg, means3D, colors, scales, rotations, opacities, out):
    """The arguments every ga_rasterb_forward* entry point ends with."""
    return (ptr(cams), ptr(bg), ptr(means3D), ptr(colors), ptr(scales), ptr(rotations), ptr(opacities), ptr(plan.geom), ptr(plan.img),
            ptr(plan.binning), ptr(plan.radii), ptr(out), _stream())


class _RasterizeBatch(torch.autograd.Function):
    """means3D / colors / scales [B,P,3] -> images [B,3,H,W]; rotations [P,4] and opacities [P,1] shared by the frames.  With
    with_depth, (images, depth pass [B,2,H,W]), differentiable in the images and in plane 0 (the mean)."""

    @staticmethod
    def forward(ctx, means3D, colors, scales, rotations, opacities, cams, bg, plan, with_depth):
        d, means3D, colors, scales, rotations, opacities = _batch_inputs(plan, means3D, colors, scales, rotations, opacities)
        L = _lib.lib()
        dev = means3D.device
        depth = None
        if with_depth:
            if plan.static_P:
                raise ValueError("rasterize_batch_with_depth renders the dynamic set alone: the plan has static_P > 0")
            plan.alloc_depth()
        out = torch.empty(plan.B, 3, plan.H, plan.W, dtype=torch.float32, device=dev)
        tail = _batch_forward_tail(plan, cams, bg, means3D, colors, scales, rotations, opacities, out)
        if with_depth:
            depth = torch.empty(plan.B, 2, plan.H, plan.W, dtype=torch.float32, device=dev)
            _lib.check(L.ga_rasterb_forward_depth_train(ctypes.byref(d), ptr(depth), ptr(plan.depth_state), plan.depth_state.numel(), *tail),
                       "ga_rasterb_forward_depth_train")
        else:
            _lib.check(L.ga_rasterb_forward(ctypes.byref(d), *tail), "ga_rasterb_forward")
        plan.record_status()
        ctx.plan, ctx.desc = plan, d
        ctx.save_for_backward(means3D, colors, scales, rotations, cams, bg, depth)
        return out if depth is None else (out, depth)

    @staticmethod
    def backward(ctx, grad_out, grad_depth=None):
        means3D, colors, scales, rotations, cams, bg, depth = ctx.saved_tensors
        plan, d = ctx.plan, ctx.desc
        if d.capacity != plan.capacity:
            raise RuntimeError("the batched rasterizer's buffers were re-allocated between forward and backward")
        if depth is not None:
            grad_out = torch.zeros_like(depth[:, :3]) if grad_out is None else grad_out
            g_m = torch.zeros_like(depth[:, 0]) if grad_depth is None else _c(grad_depth[:, 0])
        grad_out = _c(grad_out)
        d_means3D, d_colors, d_scales = torch.empty_like(means3D), torch.empty_like(colors), torch.empty_like(scales)
        L = _lib.lib()
        head = (ctypes.byref(d), ptr(cams), ptr(bg), ptr(means3D), ptr(colors), ptr(scales), ptr(rotations), ptr(plan.radii), ptr(plan.geom),
                ptr(plan.img), ptr(plan.binning), ptr(grad_out))
        tail = (ptr(d_means3D), ptr(d_colors), ptr(d_scales), None, None, None, _stream())
        if depth is None:
            _lib.check(L.ga_rasterb_backward(*head, ptr(plan.scratch), *tail), "ga_rasterb_backward")
        else:
            _lib.check(L.ga_rasterb_backward_depth(*head, ptr(g_m), ptr(depth), ptr(plan.depth_state), plan.depth_state.numel(),
                                                   ptr(plan.depth_scratch), plan.depth_scratch.numel(), *tail), "ga_rasterb_backward_depth")
        return d_means3D, d_colors, d_scales, None, None, None, None, None, None


def rasterize_batch(means3D, colors, scales, rotations, opacities, cams, bg, plan: RasterBatchPlan):
    return _RasterizeBatch.apply(means3D, colors, scales, rotations, opacities, cams, bg, plan, False)


def rasterize_batch_with_depth(means3D, colors, scales, rotations, opacities, cams, bg, plan: RasterBatchPlan):
    """`rasterize_batch` that also returns the depth pass of `rasterize_batch_depth`: (images [B,3,H,W], depth [B,2,H,W]), both
    bit for bit that call's.  Differentiable in the images and in plane 0, the mean view-space z D / (1 - T) (plane 1, the median,
    is not differentiated): its gradient reaches means3D through the blending weights and through each Gaussian's own z."""
    return _RasterizeBatch.apply(means3D, colors, scales, rotations, opacities, cams, bg, plan, True)


def rasterize_batch_scene(means3D, colors, scales, rotations, opacities, cams, bg, plan: RasterBatchPlan, scene):
    """`rasterize_batch`'s dynamic set splatted together with a static scene set in one sort per tile (correct occlusion both
    ways); forward only, images [B,3,H,W].  scene: a `scene.GaussianScene` on the device (means3D, scales, rotations, opacities
    [Ps], shs [Ps,M,3], sh_degree), with Ps = plan.static_P; cams rows must carry the camera centre (words 34..36).  Frame b's
    index space is the dynamic P, then the scene's Ps (plan.radii [B,P+Ps]); the scene's colours land in plan.scene_rgb."""
    out, = _forward_passes("rasterize_batch_scene", "ga_rasterb_forward_scene", means3D, colors, scales, rotations, opacities, cams, bg,
                           plan, None, scene)
    return out


MAX_SETS = 8                     # ga_rasterb_forward_mattes


def rasterize_batch_mattes(means3D, colors, scales, rotations, opacities, cams, bg, plan: RasterBatchPlan, first, scene=None):
    """`rasterize_batch` (scene None) or `rasterize_batch_scene` that also returns each set's visibility matte; forward only.
    first: K+1 nondecreasing dynamic indices, first[0] = 0 and first[K] <= plan.P; set k is Gaussians first[k]..first[k+1]-1.
    Returns (images [B,3,H,W], mattes [B,K,H,W]): matte k is the weight set k's Gaussians added to each pixel (sum of alpha T
    over its blended entries), so the mattes sum to 1 - final transmittance where every splatted Gaussian is in a set."""
    return _forward_passes("rasterize_batch_mattes", "ga_rasterb_forward_mattes", means3D, colors, scales, rotations, opacities, cams, bg,
                           plan, first, scene)


def rasterize_batch_depth(means3D, colors, scales, rotations, opacities, cams, bg, plan: RasterBatchPlan, scene=None, first=None):
    """`rasterize_batch` (scene None) or `rasterize_batch_scene` that also returns a depth pass, and with `first` the mattes of
    `rasterize_batch_mattes`, all from the one compositing launch; forward only.  Returns (images [B,3,H,W], depth [B,2,H,W]), or
    (images, mattes [B,K,H,W], depth) with `first`.  Depths are view-space z in world units over the entries each pixel blends,
    with the weights its colour uses: plane 0 the mean sum(w z) / (1 - T) (0 where nothing was blended), plane 1 the median, the z
    of the first blended entry after which T <= 0.5 (0 where the final T > 0.5).  0 means no surface (z <= 0.2 is culled)."""
    return _forward_passes("rasterize_batch_depth", "ga_rasterb_forward_depth", means3D, colors, scales, rotations, opacities, cams, bg,
                           plan, first, scene)


def _forward_passes(name, entry, means3D, colors, scales, rotations, opacities, cams, bg, plan, first, scene):
    """The forward-only batched renders through `entry`: ga_rasterb_forward_scene (images), ga_rasterb_forward_mattes (images and
    the mattes of `first`) or ga_rasterb_forward_depth (images, the mattes when `first` is given, and depth)."""
    given = [means3D, colors, scales, rotations, opacities]
    d, means3D, colors, scales, rotations, opacities = _batch_inputs(plan, means3D, colors, scales, rotations, opacities)
    if scene is not None:
        given += [scene.means3D, scene.shs, scene.scales, scene.rotations, scene.opacities]
    if torch.is_grad_enabled() and any(t.requires_grad for t in given):
        raise RuntimeError(f"{name} is forward only: it has no backward (run it under torch.no_grad())")
    K = 0
    if first is not None:
        first = [int(f) for f in first]
        K = len(first) - 1
        if not 1 <= K <= MAX_SETS:
            raise ValueError(f"first has {len(first)} entries: 2..{MAX_SETS + 1} (1..{MAX_SETS} sets)")
    Ps = 0 if scene is None else int(scene.means3D.shape[0])
    if Ps != plan.static_P:
        raise ValueError(f"the scene has {Ps} Gaussians, the plan was sized for static_P={plan.static_P}")
    L = _lib.lib()
    dev = means3D.device
    sc = None
    if scene is not None:
        _on_device(dev, scene_means3D=scene.means3D, scene_shs=scene.shs, cams=cams)
        sc = _lib.GaRasterScene(Ps, int(scene.sh_degree), int(scene.shs.shape[1]), ptr(scene.means3D), ptr(scene.scales),
                                ptr(scene.rotations), ptr(scene.opacities), ptr(scene.shs), ptr(plan.scene_rgb), _aa(scene))
    out = torch.empty(plan.B, 3, plan.H, plan.W, dtype=torch.float32, device=dev)
    mattes = sets = dmap = None
    if first is not None:
        mattes = torch.empty(plan.B, K, plan.H, plan.W, dtype=torch.float32, device=dev)
        sets = _lib.GaRasterSets(K, (ctypes.c_int32 * 9)(*(first + [0] * (9 - len(first)))), ptr(mattes))
    sc = None if sc is None else ctypes.byref(sc)
    sets = None if sets is None else ctypes.byref(sets)
    passes = ()
    if entry == "ga_rasterb_forward_depth":
        dmap = torch.empty(plan.B, 2, plan.H, plan.W, dtype=torch.float32, device=dev)
        passes = (sets, ptr(dmap))
    elif entry == "ga_rasterb_forward_mattes":
        passes = (sets,)
    tail = _batch_forward_tail(plan, cams, bg, means3D, colors, scales, rotations, opacities, out)
    _lib.check(getattr(L, entry)(ctypes.byref(d), sc, *passes, *tail), entry)
    plan.record_status()
    return tuple(t for t in (out, mattes, dmap) if t is not None)


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings):
        given = lambda t: t is not None and t.numel() != 0
        sh = sh if given(sh) else None
        cov3Ds_precomp = cov3Ds_precomp if given(cov3Ds_precomp) else None
        colors_c = None if sh is not None else _c(colors_precomp)
        scales_c, rot_c = (None, None) if cov3Ds_precomp is not None else (_c(scales), _c(rotations))
        means3D_c = _c(means3D)
        color, radii, rctx = rasterize_forward(means3D_c, colors_c, opacities, scales_c, rot_c, raster_settings, shs=sh,
                                               cov3D_precomp=cov3Ds_precomp)
        ctx.rctx = rctx
        ctx.raster_settings = raster_settings
        ctx.save_for_backward(means3D_c, colors_c, scales_c, rot_c)
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def backward(ctx, grad_color, _grad_radii):
        means3D, colors, scales, rotations = ctx.saved_tensors
        need = ctx.needs_input_grad
        d_means3D, d_m2d, d_colors, d_opac, d_scales, d_rot, d_sh, d_cov3D = rasterize_backward(
            ctx.rctx, means3D, colors, scales, rotations, ctx.raster_settings, grad_color,
            want_opacity=need[4], want_rotations=need[6], want_means2D=need[1], return_sh_cov3D=True)
        keep = lambda g, k: g if need[k] else None
        return (d_means3D, d_m2d, keep(d_sh, 2), d_colors, d_opac, d_scales, d_rot, keep(d_cov3D, 7), None)


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                                     raster_settings)


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings: GaussianRasterizationSettings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions: torch.Tensor) -> torch.Tensor:
        """[UPSTREAM] frustum test (view-space z > 0.2); unused by GaussianAvatar, kept for API compatibility."""
        with torch.no_grad():
            V = self.raster_settings.viewmatrix.to(positions.device).float()   # transposed: p_view = [p,1] @ V
            z = positions.float() @ V[:3, 2] + V[3, 2]
            return z > 0.2

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        empty = torch.Tensor([])
        shs = empty if shs is None else shs
        colors_precomp = empty if colors_precomp is None else colors_precomp
        scales = empty if scales is None else scales
        rotations = empty if rotations is None else rotations
        cov3D_precomp = empty if cov3D_precomp is None else cov3D_precomp
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp,
                                   self.raster_settings)
