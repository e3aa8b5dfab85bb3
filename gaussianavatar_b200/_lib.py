"""ctypes binding of libgavatar_sm90.so (the C ABI declared in include/gavatar.h).

There is no CPU fallback and no alternative backend: if the library is missing or a call fails, a RuntimeError is
raised.  The library is built in-tree by ``gaussianavatar_b200.build.build_library()`` (``__graft_entry__.build()``).
"""
from __future__ import annotations

import ctypes
import os

from .build import LIB_PATH

# developer override: load an experiment build of the same library (same C ABI) instead of the in-tree one
LIB_PATH = os.environ.get("GA_LIB_PATH", LIB_PATH)

c_f32p = ctypes.POINTER(ctypes.c_float)
c_vp = ctypes.c_void_p


class GaRasterSettings(ctypes.Structure):
    _fields_ = [("P", ctypes.c_int32), ("H", ctypes.c_int32), ("W", ctypes.c_int32),
                ("tanfovx", ctypes.c_float), ("tanfovy", ctypes.c_float), ("scale_modifier", ctypes.c_float)]


class GaRasterColorCov(ctypes.Structure):
    _fields_ = [("shs", c_vp), ("sh_degree", ctypes.c_int32), ("sh_coeffs", ctypes.c_int32), ("campos", c_vp),
                ("cov3D_precomp", c_vp), ("rgb", c_vp), ("clamped", c_vp)]


class GaRasterBatchDesc(ctypes.Structure):
    _fields_ = [("B", ctypes.c_int32), ("P", ctypes.c_int32), ("H", ctypes.c_int32), ("W", ctypes.c_int32),
                ("capacity", ctypes.c_int64), ("rot_stride", ctypes.c_int64), ("opac_stride", ctypes.c_int64),
                ("scale_modifier", ctypes.c_float)]


class GaRasterViews(ctypes.Structure):
    _fields_ = [(n, c_vp) for n in ("depth", "xy", "conic_opacity", "cov3d", "tiles_touched", "rect", "point_list", "ranges",
                                    "tile_count", "final_T", "n_contrib", "status")]


class GaDecoderDesc(ctypes.Structure):
    _fields_ = [("S", ctypes.c_int32), ("feat_res", ctypes.c_int32), ("batch", ctypes.c_int32), ("c_geom", ctypes.c_int32),
                ("hsize", ctypes.c_int32), ("bn_eps", ctypes.c_float), ("bn_momentum", ctypes.c_float), ("flags", ctypes.c_int32),
                ("frames", ctypes.c_int32)]


class GaDecoderLayout(ctypes.Structure):
    _fields_ = [("gconv", ctypes.c_int64 * 3), ("w", ctypes.c_int64 * 7), ("b", ctypes.c_int64 * 7), ("gamma", ctypes.c_int64 * 7),
                ("beta", ctypes.c_int64 * 7), ("w8", ctypes.c_int64), ("b8", ctypes.c_int64), ("total", ctypes.c_int64),
                ("bn_channels", ctypes.c_int32), ("bn_offset", ctypes.c_int32 * 7)]


class GaDecoderViews(ctypes.Structure):
    _fields_ = [(n, c_vp) for n in ("conv3_nhwc", "feat", "y1", "y5", "bn_mean", "bn_rstd", "d_feat")]


class GaLpipsViews(ctypes.Structure):
    _fields_ = [("relu", c_vp * 5), ("pool", c_vp * 2), ("pool_arg", c_vp * 2), ("partials", c_vp), ("in_scale", c_vp),
                ("dz", c_vp * 5), ("dnext", c_vp * 4), ("dpool", c_vp * 2)]


# name -> (restype, argtypes); every symbol include/gavatar.h declares must be listed here (tests check both ways)
_SIGNATURES = {
    "ga_version": (ctypes.c_int, []),
    "ga_last_error": (ctypes.c_char_p, []),
    "ga_launch_count": (ctypes.c_longlong, []),
    "ga_profile_enable": (None, [ctypes.c_int]),
    "ga_profile_report": (ctypes.c_int, [ctypes.c_char_p, ctypes.c_size_t]),
    "ga_raster_geom_bytes": (ctypes.c_size_t, [ctypes.c_int32]),
    "ga_raster_img_bytes": (ctypes.c_size_t, [ctypes.c_int32, ctypes.c_int32]),
    "ga_raster_binning_bytes": (ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int32, ctypes.c_int32]),
    "ga_raster_bwd_scratch_bytes": (ctypes.c_size_t, [ctypes.c_int32]),
    "ga_raster_forward_preprocess": (ctypes.c_int, [ctypes.POINTER(GaRasterSettings)] + [c_vp] * 9 + [ctypes.POINTER(ctypes.c_int64), c_vp]),
    "ga_raster_forward_render": (ctypes.c_int, [ctypes.POINTER(GaRasterSettings), c_vp, c_vp, c_vp, c_vp, ctypes.c_size_t, ctypes.c_int64, c_vp, c_vp, c_vp]),
    "ga_raster_backward": (ctypes.c_int, [ctypes.POINTER(GaRasterSettings)] + [c_vp] * 11 + [ctypes.c_int64] + [c_vp] * 9),
    "ga_raster_forward_preprocess_ex": (ctypes.c_int, [ctypes.POINTER(GaRasterSettings), ctypes.POINTER(GaRasterColorCov)] + [c_vp] * 9
                                        + [ctypes.POINTER(ctypes.c_int64), c_vp]),
    "ga_raster_backward_ex": (ctypes.c_int, [ctypes.POINTER(GaRasterSettings), ctypes.POINTER(GaRasterColorCov)] + [c_vp] * 11
                              + [ctypes.c_int64] + [c_vp] * 11),
    "ga_smpl_forward": (ctypes.c_int, [ctypes.c_int32] + [c_vp] * 7),
    "ga_smpl_backward": (ctypes.c_int, [ctypes.c_int32] + [c_vp] * 8),
    "ga_lbs_forward": (ctypes.c_int, [ctypes.c_int32, ctypes.c_int32, ctypes.c_float, ctypes.c_int64] + [c_vp] * 9),
    "ga_lbs_backward": (ctypes.c_int, [ctypes.c_int32, ctypes.c_int32, ctypes.c_int32, ctypes.c_float, ctypes.c_int64] + [c_vp] * 11),
    "ga_smplx_forward": (ctypes.c_int, [ctypes.c_int32] + [c_vp] * 8),
    "ga_smplx_backward": (ctypes.c_int, [ctypes.c_int32] + [c_vp] * 9),
    "ga_lbs_forward_ex": (ctypes.c_int, [ctypes.c_int32] * 4 + [ctypes.c_float, ctypes.c_int64] + [c_vp] * 9),
    "ga_lbs_backward_ex": (ctypes.c_int, [ctypes.c_int32] * 5 + [ctypes.c_float, ctypes.c_int64] + [c_vp] * 11),
    "ga_smpl_vertices": (ctypes.c_int, [ctypes.c_int32] * 2 + [c_vp] * 8),
    "ga_posmap_layout": (ctypes.c_int, [ctypes.c_int32] * 2 + [c_vp] * 4),
    "ga_posmap_fill": (ctypes.c_int, [ctypes.c_int32] * 3 + [c_vp] * 6),
    "ga_decoder_layout":(ctypes.c_int, [ctypes.POINTER(GaDecoderDesc), ctypes.POINTER(GaDecoderLayout)]),
    "ga_decoder_workspace_bytes": (ctypes.c_size_t, [ctypes.POINTER(GaDecoderDesc)]),
    "ga_decoder_forward": (ctypes.c_int, [ctypes.POINTER(GaDecoderDesc)] + [c_vp] * 7),
    "ga_decoder_backward": (ctypes.c_int, [ctypes.POINTER(GaDecoderDesc)] + [c_vp] * 8),
    "ga_decoder_views": (ctypes.c_int, [ctypes.POINTER(GaDecoderDesc), c_vp, ctypes.POINTER(GaDecoderViews)]),
    "ga_loss_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int32] * 3),
    "ga_loss_forward": (ctypes.c_int, [ctypes.c_int32] * 3 + [c_vp, c_vp, ctypes.c_float, ctypes.c_float, c_vp, c_vp, c_vp]),
    "ga_loss_backward": (ctypes.c_int, [ctypes.c_int32] * 3 + [c_vp, c_vp, ctypes.c_float, ctypes.c_float, c_vp, c_vp, c_vp, c_vp]),
    "ga_adam_step": (ctypes.c_int, [ctypes.c_int64, c_vp, c_vp, c_vp, c_vp] + [ctypes.c_float] * 4 + [ctypes.c_int64, ctypes.c_float, c_vp, c_vp]),
    "ga_adam_step_dev": (ctypes.c_int, [ctypes.c_int64] + [c_vp] * 7),
    "ga_tc_linear_forward": (ctypes.c_int, [ctypes.c_int32, ctypes.c_int32, c_vp, ctypes.c_int32, c_vp, c_vp, c_vp, ctypes.c_int32, c_vp, c_vp,
                                            ctypes.c_int32, ctypes.c_int32, c_vp, c_vp, c_vp]),
    "ga_tc_linear_backward": (ctypes.c_int, [ctypes.c_int32, c_vp, c_vp, ctypes.c_int32, c_vp, c_vp, ctypes.c_int32, c_vp, c_vp, ctypes.c_int32, c_vp,
                                             ctypes.c_int32, c_vp, ctypes.c_int32, ctypes.c_int32, c_vp, c_vp, c_vp]),
    "ga_tc_linear_backward_ex": (ctypes.c_int, [ctypes.c_int32, c_vp, c_vp, ctypes.c_int32, c_vp, c_vp, ctypes.c_int32, c_vp, c_vp, ctypes.c_int32,
                                                c_vp, ctypes.c_int32, c_vp, ctypes.c_int32, ctypes.c_int32, c_vp, c_vp, ctypes.c_int32, ctypes.c_int32,
                                                c_vp]),
    "ga_raster_views": (ctypes.c_int, [ctypes.c_int32] * 4 + [ctypes.c_int64, c_vp, c_vp, c_vp, ctypes.POINTER(GaRasterViews)]),
    "ga_rasterb_geom_bytes": (ctypes.c_size_t, [ctypes.c_int32] * 2),
    "ga_rasterb_img_bytes": (ctypes.c_size_t, [ctypes.c_int32] * 3),
    "ga_rasterb_binning_bytes": (ctypes.c_size_t, [ctypes.c_int32] * 3 + [ctypes.c_int64]),
    "ga_rasterb_bwd_scratch_bytes": (ctypes.c_size_t, [ctypes.c_int32] * 2),
    "ga_rasterb_status": (c_vp, [ctypes.c_int32] * 3 + [c_vp]),
    "ga_rasterb_status_to_host": (ctypes.c_int, [ctypes.c_int32] * 3 + [c_vp] * 4),
    "ga_rasterb_forward": (ctypes.c_int, [ctypes.POINTER(GaRasterBatchDesc)] + [c_vp] * 13),
    "ga_rasterb_backward": (ctypes.c_int, [ctypes.POINTER(GaRasterBatchDesc)] + [c_vp] * 19),
    "ga_tc_conv5x5": (ctypes.c_int, [ctypes.c_int32, ctypes.c_int32, c_vp, c_vp, c_vp, ctypes.c_int32, c_vp]),
    "ga_round_tf32": (ctypes.c_int, [c_vp, c_vp, ctypes.c_int64, c_vp]),
    "ga_lpips_weights_floats": (ctypes.c_size_t, []),
    "ga_lpips_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int32] * 3),
    "ga_lpips_forward": (ctypes.c_int, [ctypes.c_int32] * 3 + [c_vp] * 3 + [ctypes.c_float] * 2 + [c_vp] * 3),
    "ga_lpips_backward": (ctypes.c_int, [ctypes.c_int32] * 3 + [c_vp] * 5),
    "ga_lpips_views": (ctypes.c_int, [ctypes.c_int32] * 3 + [c_vp, ctypes.POINTER(GaLpipsViews)]),
}

_lib = None


def lib() -> ctypes.CDLL:
    """Load the shared library (once).  Raises RuntimeError if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: the sm_90a CUDA library has not been built. Run "
                "`python -c 'import __graft_entry__ as g; g.build()'` (needs nvcc). There is no CPU fallback.")
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(L, name)     # AttributeError if the .so is stale -> loud
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib().ga_last_error()
        raise RuntimeError(f"libgavatar {what} failed (status {rc}): {msg.decode() if msg else ''}")


def ptr(t) -> int | None:
    """Device pointer of a torch tensor (None -> NULL)."""
    if t is None:
        return None
    return t.data_ptr()


def profile(on: bool) -> None:
    lib().ga_profile_enable(1 if on else 0)


def profile_report() -> dict:
    """{kernel name: (launches, total_ms)} since the last report; synchronises the device."""
    buf = ctypes.create_string_buffer(1 << 16)
    check(lib().ga_profile_report(buf, len(buf)), "ga_profile_report")
    out = {}
    for line in buf.value.decode().splitlines():
        name, n, ms = line.rsplit(" ", 2)
        out[name] = (int(n), float(ms))
    return out


def launch_count() -> int:
    return int(lib().ga_launch_count())
