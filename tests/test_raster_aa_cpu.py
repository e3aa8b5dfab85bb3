"""CPU: the antialiasing setting's plumbing and its fp64 restatement.

Struct and settings defaults (12-field settings still construct, omitted trailing fields are 0), ModelParams and namespaces
without the field, the tools' flags and cast entries, and dr/d(a0, b, c0) of tests/raster_aa_fp64.py against central differences.
"""
import ctypes
import json
import os
import sys
import types

import pytest
import torch

import raster_aa_fp64 as aa
import raster_fp64 as rf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def test_struct_defaults():
    from gaussianavatar_b200 import _lib
    s = _lib.GaRasterSettings(10, 20, 30, 0.5, 0.4, 1.0)
    assert s.antialiasing == 0 and [f[0] for f in _lib.GaRasterSettings._fields_][-1] == "antialiasing"
    d = _lib.GaRasterBatchDesc(2, 10, 20, 30, 1 << 16, 0, 0, 1.0)
    assert d.antialiasing == 0
    sc = _lib.GaRasterScene(5, 1, 4, None, None, None, None, None, None)
    assert sc.antialiasing == 0
    assert _lib.GaRasterSettings(1, 1, 1, 0.1, 0.1, 1.0, 1).antialiasing == 1
    # the batch descriptor's flag fills what was tail padding: its size and every other offset are unchanged
    assert ctypes.sizeof(_lib.GaRasterBatchDesc) == 48 and _lib.GaRasterBatchDesc.scale_modifier.offset == 40


def test_settings_13th_field():
    from gaussianavatar_b200.rasterizer import GaussianRasterizationSettings, _aa
    twelve = GaussianRasterizationSettings(64, 48, 0.5, 0.4, None, 1.0, None, None, 0, None, False, False)
    assert twelve.antialiasing is False and _aa(twelve) == 0
    assert GaussianRasterizationSettings._fields.index("antialiasing") == GaussianRasterizationSettings._fields.index("debug") + 1
    on = GaussianRasterizationSettings(64, 48, 0.5, 0.4, None, 1.0, None, None, 0, None, False, False, True)
    assert _aa(on) == 1
    assert _aa(types.SimpleNamespace(image_height=1)) == 0          # a reference-style 12-field object without the field


def test_model_params():
    from gaussianavatar_b200.config import ModelParams
    assert ModelParams().antialiasing is False and ModelParams(antialiasing=True).antialiasing is True
    ns = types.SimpleNamespace(**{k: v for k, v in vars(ModelParams()).items() if k != "antialiasing"})
    assert bool(getattr(ns, "antialiasing", False)) is False


def test_scene_flag():
    from gaussianavatar_b200.scene import GaussianScene
    z = torch.zeros(2, 3)
    sc = GaussianScene(z, z, torch.zeros(2, 4), torch.zeros(2), torch.zeros(2, 1, 3), 0)
    assert sc.antialiasing is False and sc.to("cpu").antialiasing is False
    assert GaussianScene(z, z, torch.zeros(2, 4), torch.zeros(2), torch.zeros(2, 1, 3), 0, True).to("cpu").antialiasing is True


def _cast(tmp_path, entries):
    p = tmp_path / "cast.json"
    p.write_text(json.dumps(entries))
    return str(p)


def test_cast_mismatch(tmp_path, monkeypatch):
    import animate as tool
    monkeypatch.setattr(tool.MotionClip, "load", staticmethod(lambda *a, **k: None))
    e = dict(source_path="s", model_path="m", epoch=1, motion="x.npz")
    specs = tool.read_cast(_cast(tmp_path, [dict(e, antialiasing=True), dict(e, antialiasing=True)]))
    assert [d["antialiasing"] for d in specs] == [True, True]
    assert tool.read_cast(_cast(tmp_path, [e]))[0]["antialiasing"] is False
    with pytest.raises(ValueError, match="actor 1: antialiasing"):
        tool.read_cast(_cast(tmp_path, [e, dict(e, antialiasing=True)]))


def test_ensemble_refuses_mixed_modes():
    from gaussianavatar_b200.animate import Actor, Ensemble
    bg = torch.ones(3)
    mk = lambda on: types.SimpleNamespace(antialiasing=on, background=bg, device=torch.device("cpu"),
                                          model_parms=types.SimpleNamespace(train_stage=1))
    actors = [Actor(mk(False), None), Actor(mk(True), None)]
    with pytest.raises(ValueError, match="actor 1 renders with antialiasing=True, actor 0 with antialiasing=False"):
        Ensemble(actors, {"height": 64, "width": 64}, 64, 64)


def test_tool_flags(tmp_path):
    import animate as tool_animate
    import extract_mesh as tool_mesh
    import fit_poses as tool_fit
    (tmp_path / "test").mkdir()
    (tmp_path / "test" / "smpl_parms.pth").write_bytes(b"")
    d = str(tmp_path)
    a = tool_fit.parse_args(["-s", d, "-m", "m", "--epoch", "1", "--antialiasing"])
    assert a.antialiasing is True
    assert tool_fit.parse_args(["-s", d, "-m", "m", "--epoch", "1"]).antialiasing is False
    a = tool_mesh.parse(["-s", "d", "-m", "m", "--epoch", "1", "--frame", "0", "--out", "o", "--antialiasing"])
    assert a.antialiasing is True
    with pytest.raises(SystemExit):
        tool_animate.main(["-s", "d", "-m", "m", "--epoch", "1", "--motion", "x", "--png", "o", "--scene_antialiasing"])
    with pytest.raises(SystemExit):
        tool_animate.main(["--cast", "c.json", "--antialiasing", "--png", "o"])


def test_drho_against_central_differences():
    """The backward's expanded dr/d(a0, c0, b) numerators and the chain dL/drho = gO o, drho/dr = 1 / (2 rho) restated by
    raster_aa_fp64 (values) against central differences of o rho(a0, b, c0) in fp64."""
    g = torch.Generator().manual_seed(3)
    n = 200
    a0 = torch.exp(torch.randn(n, generator=g, dtype=torch.float64) * 2)
    c0 = torch.exp(torch.randn(n, generator=g, dtype=torch.float64) * 2)
    b = (torch.rand(n, generator=g, dtype=torch.float64) * 1.8 - 0.9) * torch.sqrt(a0 * c0)
    o = torch.rand(n, generator=g, dtype=torch.float64)
    r, rho, _, det1 = aa.rho_of((a0, 0.0), (b, 0.0), (c0, 0.0))
    rho_v, det1_v = rho[0], det1[0]
    gco = 1.0 / (2 * rho_v * det1_v ** 2)
    da = gco * (0.3 * (c0 * c0 + b * b) + 0.09 * c0)
    dc = gco * (0.3 * (a0 * a0 + b * b) + 0.09 * a0)
    db = -gco * 2 * b * (0.3 * (a0 + c0) + 0.09)
    h = 1e-6
    for x, d in ((a0, da), (c0, dc), (b, db)):
        step = h * (1 + x.abs())
        up = lambda s: aa.rho64(*(t + s if t is x else t for t in (a0, b, c0)))
        fd = (up(step) - up(-step)) / (2 * step)
        act = r[0] > 2.5e-5 * 1.01
        assert torch.allclose(d[act], fd[act], rtol=1e-5, atol=1e-9 * float(fd.abs().max()))
    # and the expanded numerators equal the issue's forms c0 det1 - det0 c etc.
    d0, d1 = a0 * c0 - b * b, (a0 + 0.3) * (c0 + 0.3) - b * b
    assert torch.allclose(0.3 * (c0 * c0 + b * b) + 0.09 * c0, c0 * d1 - d0 * (c0 + 0.3), rtol=1e-9, atol=1e-12 * float((c0 * d1).abs().max()))
    # the clamp: below 2.5e-5 rho is constant
    assert torch.equal(aa.rho64(torch.tensor([1.0]), torch.tensor([0.9999999]), torch.tensor([1.0])), torch.tensor([2.5e-5]).sqrt().double())


def test_restatement_hook_matches_plain_backward_without_terms():
    """With no_drho the antialiased restatement's gradients are raster_fp64's (the hook changes nothing else)."""
    g = torch.Generator().manual_seed(1)
    from scenes import random_scene
    sc = random_scene(P=40, H=32, W=32, seed=2)
    P = 40
    view, proj = sc["cam"].world_view_transform.reshape(16), sc["cam"].full_proj_transform.reshape(16)
    cov = torch.rand(P, 6, generator=g) * 1e-3
    cov[:, [0, 3, 5]] += 1e-3
    inp = dict(means=sc["means3D"], view=view, proj=proj, tanfovx=sc["tanfovx"], tanfovy=sc["tanfovy"], H=32, W=32, mod=1.0,
               radii=torch.ones(P, dtype=torch.int32), cov3d=cov, d_mean2D=torch.randn(P, 2, generator=g),
               d_conic_op=torch.randn(P, 4, generator=g), scales=sc["scales"], rots=sc["rotations"])
    base = rf.preprocess_backward(**inp)
    same = aa.preprocess_backward(co_w=torch.rand(P, generator=g), bug=("no_drho",), **inp)
    for k in ("d_means3D", "d_scales", "d_rotations", "d_cov3D"):
        assert torch.equal(base[k][0], same[k][0]) and torch.equal(base[k][1], same[k][1])
    full = aa.preprocess_backward(co_w=torch.rand(P, generator=g), **inp)
    assert not torch.equal(base["d_cov3D"][0], full["d_cov3D"][0])
