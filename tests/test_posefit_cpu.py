"""CPU: the fp64 restatement behind the pose-fitting gradients (oracle/posefit_oracle.py) against the numpy oracles and their golden
fixtures, its autograd gradients against central differences, the C-ABI argument checks of the new backward entries, and
tools/fit_poses.py's argument handling and output format up to the point where it needs the device."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gaussianavatar_b200 import _lib
from gaussianavatar_b200 import synthetic as syn
from oracle import cano_oracle as co
from oracle import posefit_oracle as pfo
from oracle import posmap_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
FAKE = 16        # a non-NULL address that is never dereferenced: every call below is rejected before a launch


def _smpl_model():
    return syn.smpl_mesh_model(syn.make_body(0), syn.make_uv_template(0))


def _smplx_model():
    return syn.smplx_mesh_model(syn.make_smplx_body(0), syn.make_smplx_uv_template(0), syn.smplx_posedirs(0))


def test_forward_matches_the_numpy_oracles_and_fixtures():
    g = np.load(os.path.join(GOLDEN, "posmap_vertices.npz"))
    model = syn.smpl_mesh_model(syn.make_body(int(g["body_seed"])), syn.make_uv_template(0))
    body = pfo.Body(model, g["betas"])
    v = pfo.vertices(body, torch.from_numpy(np.asarray(g["pose"], np.float64)), torch.from_numpy(np.asarray(g["transl"], np.float64))).numpy()
    assert np.abs(v[:, g["keep"]] - g["verts"]).max() < 1e-5
    assert np.abs(v - po.smpl_vertices(model, g["betas"], g["pose"], g["transl"])).max() < 1e-10
    x = np.load(os.path.join(GOLDEN, "cano_smplx_vertices.npz"))
    bx = pfo.Body(_smplx_model(), x["betas"])
    full = torch.from_numpy(np.concatenate([x["pose66"], x["rest99"]], 1).astype(np.float64))
    vx = pfo.vertices(bx, full, torch.from_numpy(np.asarray(x["transl"], np.float64))).numpy()
    assert np.abs(vx[:, x["keep"]] - x["verts"]).max() < 1e-5
    assert np.abs(vx - co.smplx_vertices(_smplx_model(), x["betas"], x["pose66"], x["rest99"], x["transl"])).max() < 1e-10
    # the fill
    t = syn.make_uv_template(0)
    face_id, bary = po.layout(t[2][t[3]], 16)
    got = pfo.fill(torch.from_numpy(v[:2]), t[1], face_id, bary).numpy()
    assert np.abs(got - po.fill(v[:2], t[1], face_id, bary)).max() < 1e-12


@pytest.mark.parametrize("body", ["smpl", "smplx"])
def test_oracle_gradients_match_central_differences(body):
    """A random linear function of the vertices and of a 12 x 12 map: autograd's gradient with respect to pose and transl against
    central differences in fp64."""
    gen = torch.Generator().manual_seed(1)
    if body == "smpl":
        model, t = _smpl_model(), syn.make_uv_template(0)
        b = pfo.Body(model, syn.make_body(0).betas[0].numpy())
        p, tr = syn.synthetic_poses(1, seed=2)
        full0, rest = p.double(), None
    else:
        model, t = _smplx_model(), syn.make_smplx_uv_template(0)
        b = pfo.Body(model, syn.make_smplx_body(0).betas[0].numpy())
        p, r, tr = syn.synthetic_smplx_poses(1, seed=2)
        full0, rest = p.double(), r.double()
    face_id, bary = po.layout(t[2][t[3]], 12)
    V = b.v_shaped.shape[0]
    wv = torch.randn(1, V, 3, generator=gen, dtype=torch.float64)
    wm = torch.randn(1, 3, 12, 12, generator=gen, dtype=torch.float64)

    def f(x):
        pose, transl = x[:, :-3], x[:, -3:]
        full = pose if rest is None else torch.cat([pose, rest], 1)
        v = pfo.vertices(b, full, transl)
        return (v * wv).sum() + (pfo.fill(v, t[1], face_id, bary) * wm).sum()

    x = torch.cat([full0, tr.double()], 1)
    # only a few coordinates by differences (each costs two evaluations): the root, one body joint, a hand-side joint, transl
    cols = [0, 1, 2, 3 * 4, 3 * 4 + 1, 3 * 18 + 2, x.shape[1] - 3, x.shape[1] - 1]
    xg = x.clone().requires_grad_(True)
    g, = torch.autograd.grad(f(xg), xg)
    for c in cols:
        e = torch.zeros_like(x)
        e[0, c] = 1e-6
        num = (f(x + e) - f(x - e)) / 2e-6
        assert abs(float(num) - float(g[0, c])) <= 1e-5 * max(1.0, abs(float(num))), (c, float(num), float(g[0, c]))


def test_c_abi_rejects_bad_arguments_before_device_work():
    L = _lib.lib()
    assert L.ga_version() >= 107
    ptrs = [FAKE] * 6
    for B in (0, 9):
        assert L.ga_smpl_vertices_backward(B, 6890, *ptrs, FAKE, 1 << 30, FAKE, FAKE, None) != 0
        assert L.ga_smplx_vertices_backward(B, 10475, *ptrs, FAKE, FAKE, 1 << 30, FAKE, FAKE, None) != 0
        assert L.ga_posmap_fill_backward(B, 64, 6890, FAKE, FAKE, FAKE, FAKE, FAKE, None) != 0
    assert L.ga_smpl_vertices_backward(2, 0, *ptrs, FAKE, 1 << 30, FAKE, FAKE, None) != 0
    # NULL pointers
    assert L.ga_smpl_vertices_backward(2, 6890, None, *ptrs[1:], FAKE, 1 << 30, FAKE, FAKE, None) != 0
    assert L.ga_smplx_vertices_backward(2, 10475, FAKE, None, *ptrs[2:], FAKE, FAKE, 1 << 30, FAKE, FAKE, None) != 0
    assert L.ga_smpl_vertices_backward(2, 6890, *ptrs, None, 1 << 30, FAKE, FAKE, None) != 0
    assert L.ga_posmap_fill_backward(1, 64, 6890, FAKE, None, FAKE, FAKE, FAKE, None) != 0
    assert L.ga_posmap_vertex_csr(64, 6890, FAKE, FAKE, None, FAKE, None) != 0
    # map sizes
    for S in (0, 513):
        assert L.ga_posmap_fill_backward(1, S, 6890, FAKE, FAKE, FAKE, FAKE, FAKE, None) != 0
        assert L.ga_posmap_vertex_csr(S, 6890, FAKE, FAKE, FAKE, FAKE, None) != 0
    # the workspace size
    need = L.ga_smpl_vertices_backward_workspace_bytes(3, 6890)
    assert need == -(-6890 // 32) * 3 * (24 * 12 + 207 + 3) * 4
    assert L.ga_smplx_vertices_backward_workspace_bytes(8, 10475) == -(-10475 // 32) * 8 * (55 * 12 + 486 + 3) * 4
    assert L.ga_smpl_vertices_backward_workspace_bytes(9, 6890) == 0
    assert L.ga_smpl_vertices_backward(3, 6890, *ptrs, FAKE, need - 1, FAKE, FAKE, None) != 0
    assert b"workspace" in L.ga_last_error()
    need_x = L.ga_smplx_vertices_backward_workspace_bytes(2, 10475)
    assert L.ga_smplx_vertices_backward(2, 10475, *ptrs, FAKE, FAKE, need_x - 4, FAKE, FAKE, None) != 0


# ---- tools/fit_poses.py -----------------------------------------------------------------------------------------------------------
def _tool(args, cwd=ROOT):
    return subprocess.run([sys.executable, os.path.join(ROOT, "tools", "fit_poses.py"), *args], capture_output=True, text=True, cwd=cwd)


def test_tool_rejects_bad_arguments(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from dataset_fixture import write_synthetic_dataset
    mp = write_synthetic_dataset(str(tmp_path), seed=0)
    base = ["-s", mp.source_path, "-m", mp.model_path, "--epoch", "1"]
    r = _tool(base + ["--stage", "2"])
    assert r.returncode == 2 and "--smpl_model and --uv_template" in r.stderr
    r = _tool(base + ["--split", "nope"])
    assert r.returncode == 2 and "no split folder" in r.stderr
    r = _tool(base + ["--iters", "-1"])
    assert r.returncode == 2 and "negative" in r.stderr
    r = _tool(base + ["--lr", "0"])
    assert r.returncode == 2 and "not positive" in r.stderr
    os.remove(os.path.join(mp.source_path, "test", "smpl_parms_pred.pth"))
    r = _tool(base + ["--stage", "2", "--smpl_model", "x.pkl", "--uv_template", "t.obj"])
    assert r.returncode == 2 and "smpl_parms_pred.pth" in r.stderr


@pytest.mark.parametrize("width,total", [(72, 72), (66, 165)])
def test_tool_output_format(tmp_path, width, total):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import fit_poses
    g = torch.Generator().manual_seed(0)
    d = dict(beta=torch.randn(1, 10, generator=g), body_pose=torch.randn(6, total, generator=g), trans=torch.randn(6, 3, generator=g))
    src, dst = str(tmp_path / "smpl_parms.pth"), str(tmp_path / fit_poses.OUT_NAME)
    torch.save(d, src)
    pose, transl = torch.randn(4, width, generator=g), torch.randn(4, 3, generator=g)
    fit_poses.write_fit(src, dst, pose, transl)
    out = torch.load(dst, weights_only=False)
    assert set(out) == {"beta", "body_pose", "trans"}
    assert torch.equal(out["beta"], d["beta"])
    assert torch.equal(out["body_pose"][:4, :width], pose) and torch.equal(out["trans"][:4], transl)
    assert torch.equal(out["body_pose"][:4, width:], d["body_pose"][:4, width:])      # SMPL-X rest columns unchanged
    assert torch.equal(out["body_pose"][4:], d["body_pose"][4:]) and torch.equal(out["trans"][4:], d["trans"][4:])
    assert torch.equal(torch.load(src, weights_only=False)["body_pose"], d["body_pose"])       # the input is untouched
    with pytest.raises(ValueError):
        fit_poses.write_fit(src, src, pose, transl)
