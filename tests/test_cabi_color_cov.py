"""CPU: the C ABI rejects malformed GaRasterColorCov descriptors with GA_ERR_INVALID before touching the device."""
import ctypes

import pytest

from gaussianavatar_b200 import _lib

GA_ERR_INVALID = -1
FAKE = 256        # never dereferenced: every case below fails validation first


def _cc(**kw):
    base = dict(shs=FAKE, sh_degree=3, sh_coeffs=16, campos=FAKE, cov3D_precomp=None, rgb=FAKE, clamped=FAKE)
    base.update(kw)
    return _lib.GaRasterColorCov(**base)


@pytest.mark.parametrize("kw,why", [
    (dict(sh_degree=4), "sh_degree"),
    (dict(sh_degree=-1), "sh_degree"),
    (dict(sh_degree=2, sh_coeffs=8), "sh_coeffs"),
    (dict(campos=None), "campos"),
    (dict(rgb=None), "campos"),
    (dict(clamped=None), "campos"),
])
def test_bad_descriptor_is_rejected(kw, why):
    L = _lib.lib()
    s = _lib.GaRasterSettings(10, 32, 32, 0.5, 0.5, 1.0)
    n = ctypes.c_int64(0)
    rc = L.ga_raster_forward_preprocess_ex(ctypes.byref(s), ctypes.byref(_cc(**kw)), *[FAKE] * 9, ctypes.byref(n), None)
    assert rc == GA_ERR_INVALID and why in L.ga_last_error().decode()
    rc = L.ga_raster_backward_ex(ctypes.byref(s), ctypes.byref(_cc(**kw)), *[FAKE] * 11, 1, *[FAKE] * 10, None)
    assert rc == GA_ERR_INVALID and why in L.ga_last_error().decode()


def test_missing_arrays_are_rejected():
    L = _lib.lib()
    s = _lib.GaRasterSettings(10, 32, 32, 0.5, 0.5, 1.0)
    n = ctypes.c_int64(0)
    # scales / rotations NULL without cov3D_precomp
    rc = L.ga_raster_forward_preprocess_ex(ctypes.byref(s), ctypes.byref(_cc()), FAKE, None, None, *[FAKE] * 6, ctypes.byref(n), None)
    assert rc == GA_ERR_INVALID
    # shs without d_sh, cov3D_precomp without d_cov3D
    args = [FAKE] * 11 + [1] + [FAKE] * 8
    assert L.ga_raster_backward_ex(ctypes.byref(s), ctypes.byref(_cc()), *args, None, FAKE, None) == GA_ERR_INVALID
    assert L.ga_raster_backward_ex(ctypes.byref(s), ctypes.byref(_cc(shs=None, cov3D_precomp=FAKE)), *args, FAKE, None,
                                   None) == GA_ERR_INVALID
