"""CPU: training against depth maps.  The new C entries' argument checks (which run before any launch), the datasets' depth maps
(<split>/depths/<name>.npy in float32 metres or .png in uint16 millimetres, zeroed outside the mask, the file named on a missing or
mis-sized map) and the option fields a reference-style namespace lacks."""
import ctypes
import os
import sys
import types

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gaussianavatar_b200 import _lib  # noqa: E402

FAKE = 256         # never dereferenced: every call below must fail its checks before any launch


def _L():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    return _lib.lib()


def _refused(L, rc, message):
    assert rc != 0
    assert message in L.ga_last_error().decode(), L.ga_last_error().decode()


def test_depth_state_and_scratch_sizes():
    L = _L()
    a = L.ga_rasterb_depth_state_bytes(2, 100, 140, 1 << 16)
    assert L.ga_rasterb_depth_state_bytes(2, 100, 140, 1 << 18) > a > 0         # grows with capacity ...
    assert L.ga_rasterb_depth_state_bytes(3, 100, 140, 1 << 16) > a             # ... and with the frames' tiles
    assert L.ga_rasterb_depth_bwd_scratch_bytes(2, 1000) >= L.ga_rasterb_bwd_scratch_bytes(2, 1000) + 4 * 2000


@pytest.mark.parametrize("case,message", [
    ("NULL depth", "NULL pointer"),
    ("NULL state", "NULL pointer"),
    ("small state", "depth state too small"),
    ("B=0", "bad frame count"),
])
def test_forward_depth_train_refuses_before_any_launch(case, message):
    L = _L()
    B = 0 if case == "B=0" else 2
    d = _lib.GaRasterBatchDesc(B, 10, 16, 16, 4096, 0, 0, 1.0)
    nb = L.ga_rasterb_depth_state_bytes(2, 16, 16, 4096)
    depth, state = (None if case == "NULL depth" else FAKE), (None if case == "NULL state" else FAKE)
    nb = nb - 1 if case == "small state" else nb
    before = L.ga_launch_count()
    _refused(L, L.ga_rasterb_forward_depth_train(ctypes.byref(d), depth, state, nb, *[FAKE] * 12, None), message)
    assert L.ga_launch_count() == before


@pytest.mark.parametrize("case,message", [
    ("NULL dL_ddepth", "NULL pointer"),
    ("NULL depth", "NULL pointer"),
    ("NULL state", "NULL pointer"),
    ("small state", "depth state too small"),
    ("small scratch", "scratch too small"),
])
def test_backward_depth_refuses_before_any_launch(case, message):
    L = _L()
    d = _lib.GaRasterBatchDesc(2, 10, 16, 16, 4096, 0, 0, 1.0)
    ns, nc = L.ga_rasterb_depth_state_bytes(2, 16, 16, 4096), L.ga_rasterb_depth_bwd_scratch_bytes(2, 10)
    g = None if case == "NULL dL_ddepth" else FAKE
    dp = None if case == "NULL depth" else FAKE
    st = None if case == "NULL state" else FAKE
    ns -= case == "small state"
    nc -= case == "small scratch"
    before = L.ga_launch_count()
    rc = L.ga_rasterb_backward_depth(ctypes.byref(d), *[FAKE] * 11, g, dp, st, ns, FAKE, nc, *[FAKE] * 3, None, None, None, None)
    _refused(L, rc, message)
    assert L.ga_launch_count() == before


@pytest.mark.parametrize("case,message", [
    ("NULL depth", "NULL pointer"),
    ("NULL target", "NULL pointer"),
    ("small workspace", "workspace too small"),
    ("H=0", "bad depth loss dims"),
])
def test_depth_loss_refuses_before_any_launch(case, message):
    L = _L()
    H = 0 if case == "H=0" else 8
    nb = L.ga_depth_loss_workspace_bytes(2, 8, 8) - (case == "small workspace")
    dp, tg = (None if case == "NULL depth" else FAKE), (None if case == "NULL target" else FAKE)
    before = L.ga_launch_count()
    _refused(L, L.ga_depth_loss_forward(2, H, 8, dp, tg, 1.0, FAKE, nb, FAKE, None), message)
    _refused(L, L.ga_depth_loss_backward(2, H, 8, dp, tg, None, FAKE, nb, FAKE, None), message)
    assert L.ga_launch_count() == before


# ---- datasets ---------------------------------------------------------------------------------------------------------------------
def _dataset(tmp_path, fmt):
    from dataset_fixture import write_synthetic_dataset
    from PIL import Image
    mp = write_synthetic_dataset(str(tmp_path), num_frames=3)
    mp.depth_maps = True
    g = np.random.default_rng(5)
    want = {}
    for split in ("train", "test"):
        folder = os.path.join(mp.source_path, split)
        os.makedirs(os.path.join(folder, "depths"))
        for n in sorted(os.listdir(os.path.join(folder, "images"))):
            name = n.split(".")[0]
            mm = g.integers(0, 4000, size=(64, 64)).astype(np.uint16)
            mm[g.random((64, 64)) < 0.1] = 0                                      # holes: no measurement
            if fmt == "png":
                Image.fromarray(mm).save(os.path.join(folder, "depths", name + ".png"))
                metres = mm.astype(np.float32) * np.float32(1e-3)
            else:
                metres = mm.astype(np.float32) * np.float32(1.1e-3)
                np.save(os.path.join(folder, "depths", name + ".npy"), metres)
            mext = sorted(os.listdir(os.path.join(folder, "masks")))[0].split(".")[-1]
            mask = np.array(Image.open(os.path.join(folder, "masks", name + "." + mext)))
            m = mask if mask.ndim == 2 else mask[..., 0]
            want[(split, name)] = np.where(m >= 128, metres, 0.0).astype(np.float32)
    return mp, want


@pytest.mark.parametrize("fmt", ["npy", "png"])
def test_dataset_reads_depth_maps(tmp_path, fmt):
    import torch
    from gaussianavatar_b200 import dataset as ds
    mp, want = _dataset(tmp_path, fmt)
    for split, cls in (("train", ds.MonoDataset_train), ("test", ds.MonoDataset_test)):
        d = cls(mp)
        for i in range(len(d)):
            item = d[i]
            got = item["depth"]
            assert got.dtype == torch.float32 and tuple(got.shape) == (64, 64)
            assert np.array_equal(got.numpy(), want[(split, d.name_list[i][1])])
            assert (got > 0).any() and (got == 0).any()
    ref_style = types.SimpleNamespace(**{k: v for k, v in vars(mp).items() if k != "depth_maps"})      # no depth_maps field: off
    assert "depth" not in ds.MonoDataset_train(ref_style)[0]


def test_dataset_names_a_missing_or_missized_map(tmp_path):
    from gaussianavatar_b200 import dataset as ds
    mp, _ = _dataset(tmp_path, "npy")
    d = ds.MonoDataset_train(mp)
    name = d.name_list[1][1]
    path = os.path.join(mp.source_path, "train", "depths", name + ".npy")
    np.save(path, np.ones((32, 64), np.float32))
    with pytest.raises(ValueError, match=name + ".npy"):
        d[1]
    os.remove(path)
    with pytest.raises(FileNotFoundError, match=name + ".npy"):
        d[1]
    d[0]                                                                     # the other frames still read


def test_reference_namespace_reads_as_depth_off():
    """An argparse-style namespace without depth_maps / lambda_depth (the reference's own option groups) trains colour only."""
    from gaussianavatar_b200.config import ModelParams, OptimizationParams
    from gaussianavatar_b200.trainer import Stage1Trainer
    mp = types.SimpleNamespace(**{k: v for k, v in vars(ModelParams()).items() if k != "depth_maps"})
    assert not getattr(mp, "depth_maps", False)
    op = types.SimpleNamespace(**{k: v for k, v in vars(OptimizationParams()).items() if k != "lambda_depth"})
    tr = Stage1Trainer.__new__(Stage1Trainer)
    tr.opt = op
    assert not tr._depth_active({"original_image": None})
    assert tr._depth_active({"depth": np.zeros((1, 2, 2))})                  # lambda_depth defaults to 1.0
    tr.opt = types.SimpleNamespace(lambda_depth=0.0)
    assert not tr._depth_active({"depth": np.zeros((1, 2, 2))})
    assert ModelParams().depth_maps is False and OptimizationParams().lambda_depth == 1.0
