"""ORACLE — TEST INFRASTRUCTURE ONLY.

ctypes front-end of ``oracle/build/liboracle_raster_ex.so``: the C restatement of ``raster_oracle.py`` extended with the
other input modes of upstream's rasterizer API (``raster_oracle_ex.inc``): spherical-harmonic colours and precomputed 3D
covariances.  Only tests/ may import this module.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

from .raster_oracle import _HERE, _Q, OracleForward, _f32, _ptr

_SO = os.path.join(_HERE, "build", "liboracle_raster_ex.so")
_SRCS = ("raster_oracle_ex.c", "raster_oracle_ex.inc", "raster_oracle.c", "raster_oracle_impl.inc")
_QX = dict(_Q, rgb=100, clamped=101)


def build(force: bool = False) -> str:
    """Compile the extended restatement with the flags of oracle/Makefile (gcc, OpenMP, no FMA contraction)."""
    src_m = max(os.path.getmtime(os.path.join(_HERE, f)) for f in _SRCS)
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < src_m:
        os.makedirs(os.path.dirname(_SO), exist_ok=True)
        cc = "/usr/bin/gcc" if os.access("/usr/bin/gcc", os.X_OK) else "gcc"
        subprocess.run([cc, "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-Wall",
                        "-Wno-unused-function", "-o", _SO, os.path.join(_HERE, "raster_oracle_ex.c"), "-lm"],
                       check=True, capture_output=True)
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(_SO)
        fp = ctypes.POINTER(ctypes.c_float)
        dp = ctypes.POINTER(ctypes.c_double)
        for pfx in ("oracle32ex", "oracle64ex"):
            f = getattr(L, pfx + "_forward")
            f.restype = ctypes.c_void_p
            f.argtypes = [ctypes.c_int] * 3 + [fp] * 8 + [ctypes.c_float] * 3 + [fp, ctypes.c_int, ctypes.c_int, fp, fp]
            g = getattr(L, pfx + "_get")
            g.restype = ctypes.c_int
            g.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
            n = getattr(L, pfx + "_num_rendered")
            n.restype = ctypes.c_longlong
            n.argtypes = [ctypes.c_void_p]
            fr = getattr(L, pfx + "_free")
            fr.restype = None
            fr.argtypes = [ctypes.c_void_p]
            b = getattr(L, pfx + "_backward")
            b.restype = None
            b.argtypes = [ctypes.c_void_p, fp] + [dp] * 9
        _lib = L
    return _lib


class OracleForwardEx(OracleForward):
    """OracleForward of the extended restatement: get() also knows "rgb" [P,3] and "clamped" [P] (bit c = channel c clamped),
    backward() also returns "d_sh" [P,M,3] when shs were given (d_colors is then dL/drgb before the clamp mask)."""
    M: int = 0

    @property
    def _pfx(self):
        return "oracle32ex" if self.precision == "f32" else "oracle64ex"

    @property
    def num_rendered(self) -> int:
        return int(getattr(lib(), self._pfx + "_num_rendered")(self._h))

    def get(self, name: str) -> np.ndarray:
        if name not in ("rgb", "clamped"):
            return self._get_typed(name)
        arr = np.zeros((self.P, 3), np.float64) if name == "rgb" else np.zeros((self.P,), np.uint8)
        if arr.size:
            assert getattr(lib(), self._pfx + "_get")(self._h, _QX[name], arr.ctypes.data_as(ctypes.c_void_p)) == 0
        return arr

    def _get_typed(self, name):
        # the base class's shapes and dtypes, read through this library
        P, H, W, R = self.P, self.H, self.W, self.num_rendered
        T = self.grid[0] * self.grid[1]
        spec = dict(depth=((P,), np.float64), radii=((P,), np.int32), xy=((P, 2), np.float64), conic_o=((P, 4), np.float64),
                    cov3d=((P, 6), np.float64), tiles=((P,), np.int32), rect=((P, 4), np.int32), offsets=((P,), np.uint32),
                    keys_unsorted=((R,), np.uint64), vals_unsorted=((R,), np.uint32), keys=((R,), np.uint64),
                    vals=((R,), np.uint32), ranges=((T, 2), np.uint32), out=((3, H, W), np.float64),
                    final_T=((H, W), np.float64), n_contrib=((H, W), np.uint32))[name]
        arr = np.zeros(spec[0], dtype=spec[1])
        if arr.size:
            assert getattr(lib(), self._pfx + "_get")(self._h, _QX[name], arr.ctypes.data_as(ctypes.c_void_p)) == 0
        return arr

    def backward(self, dL_dout) -> dict:
        P = self.P
        g = _f32(dL_dout, (3, self.H, self.W))
        order = ["d_mean2D", "d_conic", "d_opacity", "d_colors", "d_means3D", "d_scales", "d_rots", "d_cov3d", "d_sh"]
        outs = dict(d_mean2D=np.zeros((P, 2)), d_conic=np.zeros((P, 3)), d_opacity=np.zeros((P,)), d_colors=np.zeros((P, 3)),
                    d_means3D=np.zeros((P, 3)), d_scales=np.zeros((P, 3)), d_rots=np.zeros((P, 4)), d_cov3d=np.zeros((P, 6)),
                    d_sh=np.zeros((P, max(self.M, 1), 3)))
        getattr(lib(), self._pfx + "_backward")(self._h, _ptr(g, ctypes.c_float), *[_ptr(outs[k], ctypes.c_double) for k in order])
        if not self.M:
            del outs["d_sh"]
        return outs

    def close(self):
        if self._h:
            getattr(lib(), self._pfx + "_free")(self._h)
            self._h = 0


def forward(means3D, colors, opacities, scales, rotations, bg, viewmatrix, projmatrix, tanfovx, tanfovy, H, W,
            scale_modifier=1.0, precision="f32", shs=None, sh_degree=0, campos=None, cov3D_precomp=None) -> OracleForwardEx:
    """raster_oracle.forward with upstream's other inputs: shs [P,M,3] (with sh_degree 0..3 and campos [3]) replaces colors,
    cov3D_precomp [P,6] = (xx, xy, xz, yy, yz, zz) replaces scales / rotations / scale_modifier (those may then be None)."""
    means3D = _f32(means3D).reshape(-1, 3)
    P = means3D.shape[0]
    M = 0 if shs is None else int(np.shape(shs)[1])
    if shs is not None:
        assert 0 <= sh_degree <= 3 and (sh_degree + 1) ** 2 <= M and campos is not None
    opt = lambda a, shape: None if a is None else _f32(a, shape)
    arrs = dict(means3D=means3D, colors=None if shs is not None else _f32(colors, (P, 3)), opacities=_f32(opacities, (P,)),
                scales=None if cov3D_precomp is not None else _f32(scales, (P, 3)),
                rotations=None if cov3D_precomp is not None else _f32(rotations, (P, 4)),
                bg=_f32(bg, (3,)), view=_f32(viewmatrix, (16,)), proj=_f32(projmatrix, (16,)), shs=opt(shs, (P, M, 3)),
                campos=opt(campos, (3,)), cov=opt(cov3D_precomp, (P, 6)))
    p = lambda k: None if arrs[k] is None else _ptr(arrs[k], ctypes.c_float)
    pfx = "oracle32ex" if precision == "f32" else "oracle64ex"
    h = getattr(lib(), pfx + "_forward")(P, int(H), int(W), p("means3D"), p("colors"), p("opacities"), p("scales"), p("rotations"),
                                          p("bg"), p("view"), p("proj"), float(tanfovx), float(tanfovy), float(scale_modifier),
                                          p("shs"), int(sh_degree), M, p("campos"), p("cov"))
    o = OracleForwardEx(P=P, H=int(H), W=int(W), precision=precision, _h=h)
    o.M = M
    return o
