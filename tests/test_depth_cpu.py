"""CPU: the depth pass.  ga_rasterb_forward_depth's argument checks (which run before any launch) and tools/animate.py's --depth
argument handling."""
import ctypes
import importlib.util
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gaussianavatar_b200 import _lib  # noqa: E402


def _tool():
    spec = importlib.util.spec_from_file_location("animate_tool", os.path.join(ROOT, "tools", "animate.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("case,message", [
    ("NULL depth", "depth is NULL"),
    ("K=0", "set count K=0"),
    ("K=9", "set count K=9"),
    ("decreasing", "must not decrease"),
    ("past P", "> P = 10"),
    ("NULL mattes", "mattes is NULL"),
    ("first[0]", "first[0] = 2"),
])
def test_depth_cabi_refuses_before_any_launch(case, message):
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    L = _lib.lib()
    fake = 256         # never dereferenced: every call below must fail its checks before any launch
    d = _lib.GaRasterBatchDesc(2, 10, 16, 16, 4096, 0, 0, 1.0)
    K, first, mattes, depth = 3, [0, 4, 4, 10], fake, fake
    if case == "NULL depth":
        depth = None
    elif case == "K=0":
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
    scene = _lib.GaRasterScene(0, 0, 1, None, None, None, None, None, None)
    before = L.ga_launch_count()
    args = [fake] * 13
    assert L.ga_rasterb_forward_depth(ctypes.byref(d), None, ctypes.byref(sets), depth, *args) != 0
    assert message in L.ga_last_error().decode()
    assert L.ga_rasterb_forward_depth(ctypes.byref(d), ctypes.byref(scene), ctypes.byref(sets), depth, *args) != 0
    assert message in L.ga_last_error().decode()
    if case == "NULL depth":                       # without sets too
        assert L.ga_rasterb_forward_depth(ctypes.byref(d), None, None, None, *args) != 0
        assert message in L.ga_last_error().decode()
    assert L.ga_launch_count() == before


def test_version():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    assert _lib.lib().ga_version() == 110


def test_tool_depth_arguments(tmp_path, capsys):
    """--depth counts as an output (no "nothing to write" error), and is accepted next to --cast, --scene and --mattes: each of these
    command lines gets past argument handling and fails only where it first needs the missing dataset."""
    tool = _tool()
    with pytest.raises(SystemExit) as e:
        tool.main(["-s", str(tmp_path), "-m", str(tmp_path), "--epoch", "1", "--motion", "clip.npz"])
    assert e.value.code == 2 and "nothing to write" in capsys.readouterr().err
    with pytest.raises(SystemExit) as e:
        tool.main(["-s", str(tmp_path), "-m", str(tmp_path), "--epoch", "1", "--motion", "clip.npz", "--depth", str(tmp_path / "d"),
                   "--mattes", str(tmp_path / "m"), "--camera", "bogus"])
    err = capsys.readouterr().err
    assert e.value.code == 2 and "nothing to write" not in err and "--camera bogus" in err
    with pytest.raises(SystemExit) as e:
        tool.main(["--cast", str(tmp_path / "missing.json"), "--depth", str(tmp_path / "d"), "--scene", "s.ply"])
    err = capsys.readouterr().err
    assert e.value.code == 2 and "nothing to write" not in err and "missing.json" in err
    with pytest.raises(SystemExit) as e:
        tool.main(["--depth"])
    assert e.value.code == 2 and "--depth: expected one argument" in capsys.readouterr().err
