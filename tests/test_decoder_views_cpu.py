"""CPU: ga_decoder_views hands out every decoder workspace buffer, inside the workspace, disjoint and aligned.

ga_decoder_views only computes addresses, so it runs on a fake base pointer. The sizes below restate the workspace's
contents from the descriptor (include/gavatar.h); the views must match them exactly, without gaps that hide a buffer.
"""
import ctypes

import pytest

from gaussianavatar_b200 import _lib

BASE = 1 << 40                      # fake device address, 4 KB aligned


def _desc(S, Hf, frames, batch=1, flags=1):
    return _lib.GaDecoderDesc(S, Hf, batch, 64, 128, 1e-5, 0.1, flags, frames)


def _views(desc):
    L = _lib.lib()
    nbytes = L.ga_decoder_workspace_bytes(ctypes.byref(desc))
    assert nbytes > 0, L.ga_last_error()
    v = _lib.GaDecoderViews()
    _lib.check(L.ga_decoder_views(ctypes.byref(desc), ctypes.c_void_p(BASE), ctypes.byref(v)), "ga_decoder_views")
    return nbytes, v


def _expected(v, S, Hf, frames):
    """name -> (address, bytes, element size) of every view."""
    nf = max(frames, 1)
    M, P = nf * S * S, Hf * Hf
    fp = nf * P * 64 if nf > 1 else 4
    out = {}
    for i in range(4):
        out[f"F[{i}]"] = (v.F[i], P * 64 * 4, 4)
    out["wr"] = (v.wr, 3 * 25 * 64 * 64 * 4, 4)
    for i in range(2):
        out[f"dF[{i}]"] = (v.dF[i], P * 64 * 4, 4)
    out["Fp"], out["dFp"] = (v.Fp, fp * 4, 4), (v.dFp, fp * 4, 4)
    out["feat"], out["d_feat"] = (v.feat, M * 72 * 4, 4), (v.d_feat, M * 72 * 4, 4)
    for i in range(5):
        out[f"Y[{i}]"] = (v.Y[i], M * 128 * 4, 4)
    out["Y6"], out["Y7"] = (v.Y6, M * 384 * 4, 4), (v.Y7, M * 384 * 4, 4)
    out["dZa"], out["dZb"] = (v.dZa, M * 128 * 4, 4), (v.dZb, M * 128 * 4, 4)
    out["dZ6"], out["dZ7"] = (v.dZ6, M * 384 * 4, 4), (v.dZ7, M * 384 * 4, 4)
    out["stat"] = (v.stat, 4 * 1408 * 8, 8)
    out["coef"] = (v.coef, 7 * 1408 * 4, 4)
    return out


@pytest.mark.parametrize("S,Hf,frames,batch", [(2, 1, 0, 1), (46, 5, 1, 1), (92, 40, 8, 1), (128, 128, 1, 4), (512, 128, 0, 2),
                                               (512, 128, 2, 2), (512, 128, 8, 8)])
@pytest.mark.parametrize("flags", [0, 1])
def test_views_inside_disjoint_aligned(S, Hf, frames, batch, flags):
    nbytes, v = _views(_desc(S, Hf, frames, batch, flags))
    views = _expected(v, S, Hf, frames)
    spans = []
    for name, (addr, size, elem) in views.items():
        assert addr is not None, f"{name} is NULL"
        off = addr - BASE
        assert 0 <= off and off + size <= nbytes, f"{name} [{off}, {off + size}) outside the {nbytes}-byte workspace"
        assert addr % (16 if elem == 4 else 8) == 0, f"{name} at offset {off} is misaligned"
        spans.append((off, off + size, name))
    spans.sort()
    for (a0, a1, an), (b0, b1, bn) in zip(spans, spans[1:]):
        assert a1 <= b0, f"{an} [{a0}, {a1}) overlaps {bn} [{b0}, {b1})"
    # the views account for the whole workspace: what is left is alignment padding only
    used = sum(e - s for s, e, _ in spans)
    assert nbytes - used < 256 * len(spans), f"{nbytes - used} bytes of the workspace belong to no view"


def test_views_refuse_bad_descriptors():
    L = _lib.lib()
    v = _lib.GaDecoderViews()
    for desc in (_desc(512, 128, 9), _desc(3, 1, 1), _lib.GaDecoderDesc(64, 16, 1, 32, 128, 1e-5, 0.1, 1, 1)):
        assert L.ga_decoder_views(ctypes.byref(desc), ctypes.c_void_p(BASE), ctypes.byref(v)) != 0
    assert L.ga_decoder_views(ctypes.byref(_desc(64, 16, 1)), None, ctypes.byref(v)) != 0
