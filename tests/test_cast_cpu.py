"""CPU: several avatars rendered together.  ga_rasterb_forward_mattes' argument checks (which run before any launch), the playback
schedule of an ensemble against a numpy restatement, and tools/animate.py's --cast file errors, each naming its entry."""
import ctypes
import importlib.util
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gaussianavatar_b200 import animate as an  # noqa: E402
from gaussianavatar_b200 import _lib  # noqa: E402


def _tool():
    spec = importlib.util.spec_from_file_location("animate_tool", os.path.join(ROOT, "tools", "animate.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("case,message", [
    ("K=0", "set count K=0"),
    ("K=9", "set count K=9"),
    ("decreasing", "must not decrease"),
    ("past P", "> P = 10"),
    ("NULL mattes", "mattes is NULL"),
    ("first[0]", "first[0] = 2"),
])
def test_mattes_cabi_rejects_bad_sets(case, message):
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    L = _lib.lib()
    fake = 256         # never dereferenced: every call below must fail its checks before any launch
    d = _lib.GaRasterBatchDesc(2, 10, 16, 16, 4096, 0, 0, 1.0)
    K, first, mattes = 3, [0, 4, 4, 10], fake
    if case == "K=0":
        K = 0
    elif case == "K=9":
        K, first = 9, list(range(10))[:9] + [9]
    elif case == "decreasing":
        first = [0, 6, 5, 10]
    elif case == "past P":
        first = [0, 4, 8, 11]
    elif case == "NULL mattes":
        mattes = None
    elif case == "first[0]":
        first = [2, 4, 8, 10]
    sets = _lib.GaRasterSets(K, (ctypes.c_int32 * 9)(*(first + [0] * (9 - len(first)))[:9]), mattes)
    before = L.ga_launch_count()
    args = [fake] * 13
    assert L.ga_rasterb_forward_mattes(ctypes.byref(d), None, ctypes.byref(sets), *args) != 0
    assert message in L.ga_last_error().decode()
    assert L.ga_launch_count() == before
    assert L.ga_rasterb_forward_mattes(ctypes.byref(d), None, None, *args) != 0
    assert b"sets descriptor is NULL" in L.ga_last_error()
    assert L.ga_matte_pack(0, fake, fake, None) != 0 and L.ga_matte_pack(4, None, fake, None) != 0
    assert L.ga_launch_count() == before
    assert L.ga_version() >= 109


def _restated_times(keys, fps, speeds, fps_out):
    n = 0
    for T, f, v in zip(keys, fps, speeds):
        step = v * f / fps_out
        n = max(n, int(np.floor((T - 1) / step)) + 1)
    out = np.zeros((len(keys), n))
    for k, (T, f, v) in enumerate(zip(keys, fps, speeds)):
        for j in range(n):
            out[k, j] = min(j * (v * f / fps_out), T - 1)
    return out


@pytest.mark.parametrize("keys,fps,speeds,fps_out", [
    ([6], [30.0], [1.0], 60.0),
    ([6, 3], [30.0, 30.0], [1.0, 1.0], 60.0),
    ([11, 40, 2], [30.0, 120.0, 25.0], [0.5, 1.0, 1.5], 30.0),
    ([1, 5], [30.0, 24.0], [1.0, 2.0], 60.0),
    ([9, 9, 9, 9, 9, 9, 9, 9], [30.0] * 8, [0.25 * (k + 1) for k in range(8)], 45.0),
])
def test_cast_times_match_restatement(keys, fps, speeds, fps_out):
    got = an.cast_times(keys, fps, speeds, fps_out)
    want = _restated_times(keys, fps, speeds, fps_out)
    assert got.shape == want.shape and np.array_equal(got, want)
    longest = max(len(an.sample_times(T, f, fps_out, v)) for T, f, v in zip(keys, fps, speeds))
    assert got.shape[1] == longest
    for k, (T, f, v) in enumerate(zip(keys, fps, speeds)):
        own = an.sample_times(T, f, fps_out, v)
        assert np.array_equal(got[k, :len(own)], own)                  # each actor's own playback, then its last pose held
        assert (got[k, len(own):] == T - 1).all()
    with pytest.raises(ValueError):
        an.cast_times([5, 5], [30.0, 30.0], [1.0, 0.0], 30.0)


def _write_clip(path, width, T=4):
    torch.save({"body_pose": torch.zeros(T, width), "trans": torch.zeros(T, 3)}, path)
    return str(path)


def _entry(tmp_path, **kw):
    e = dict(source_path=str(tmp_path), model_path=str(tmp_path), epoch=1, motion=_write_clip(tmp_path / "smpl.pth", 72), clip_fps=30)
    e.update(kw)
    return e


def _cast(tmp_path, entries):
    p = tmp_path / "cast.json"
    p.write_text(json.dumps(entries))
    return str(p)


def test_cast_file_reads_back(tmp_path):
    tool = _tool()
    smplx = _write_clip(tmp_path / "smplx.pth", 165, T=7)
    got = tool.read_cast(_cast(tmp_path, [_entry(tmp_path), _entry(tmp_path, body="smplx", motion=smplx, speed=2.0, align_to=1)]))
    assert len(got) == 2
    assert got[0]["stage"] == 1 and got[0]["body"] == "smpl" and got[0]["clip"].num_keys == 4 and got[0]["speed"] == 1.0
    assert got[1]["body"] == "smplx" and got[1]["clip"].pose.shape == (7, 165) and got[1]["speed"] == 2.0 and got[1]["align_to"] == 1


@pytest.mark.parametrize("bad,message", [
    ("missing", r"actor 1: missing epoch"),
    ("body", r"actor 1: .*expected \[T,165\] for body='smplx'"),
    ("background", r"actor 2: white_background .*one background"),
    ("unknown", r"actor 0: unknown field colour"),
    ("stage2", r"actor 1: stage 2 needs smpl_model and uv_template"),
    ("empty", r"a list of 1..8 actors"),
])
def test_cast_file_errors_name_the_entry(tmp_path, bad, message):
    tool = _tool()
    entries = [_entry(tmp_path), _entry(tmp_path), _entry(tmp_path)]
    if bad == "missing":
        del entries[1]["epoch"]
    elif bad == "body":
        entries[1]["body"] = "smplx"                 # an SMPL clip for an SMPL-X avatar
    elif bad == "background":
        entries[2]["white_background"] = False
    elif bad == "unknown":
        entries[0]["colour"] = 1
    elif bad == "stage2":
        entries[1]["stage"] = 2
    elif bad == "empty":
        entries = []
    with pytest.raises(ValueError, match=message):
        tool.read_cast(_cast(tmp_path, entries))
    # the tool turns it into a usage error before loading any model
    with pytest.raises(SystemExit) as e:
        tool.main(["--cast", _cast(tmp_path, entries), "--png", str(tmp_path / "out")])
    assert e.value.code == 2


def test_cast_replaces_the_single_avatar_flags(tmp_path, capsys):
    tool = _tool()
    cast = _cast(tmp_path, [_entry(tmp_path)])
    with pytest.raises(SystemExit):
        tool.main(["--cast", cast, "--body", "smpl", "--png", str(tmp_path)])
    assert "--cast replaces --body" in capsys.readouterr().err
    with pytest.raises(SystemExit):
        tool.main(["-s", str(tmp_path), "-m", str(tmp_path), "--epoch", "1", "--png", str(tmp_path)])
    assert "--motion" in capsys.readouterr().err
