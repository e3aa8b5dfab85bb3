"""CPU: the SMPL-X vertex and weight-map restatements (oracle/cano_oracle.py) against the reference's own outputs
(oracle/gen_golden_cano.py), the canonical pose and joint matrices, the C-ABI argument checks of ga_smplx_vertices /
ga_posmap_weights, and the canonical-asset tools' handling of missing inputs."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gaussianavatar_b200 import _lib
from gaussianavatar_b200 import synthetic as syn
from gaussianavatar_b200.posmap import CANO_TRANSL, canonical_pose
from oracle import cano_oracle as co
from oracle import posmap_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
FAKE = 16        # a non-NULL address that is never dereferenced: every call below is rejected before a launch


def _smplx_model():
    return syn.smplx_mesh_model(syn.make_smplx_body(0), syn.make_smplx_uv_template(0), syn.smplx_posedirs(0))


def test_smplx_vertex_oracle_matches_the_reference():
    g = np.load(os.path.join(GOLDEN, "cano_smplx_vertices.npz"))
    v = co.smplx_vertices(_smplx_model(), g["betas"], g["pose66"], g["rest99"], g["transl"])
    assert np.abs(v[:, g["keep"]] - g["verts"]).max() < 1e-5
    assert np.abs(v.mean(1) - g["mean"]).max() < 1e-5
    assert np.abs((v ** 2).mean(1) - g["mean_sq"]).max() < 1e-5
    # the pose blend shapes matter at these poses: without them the vertices move by far more than the bound
    model = dict(_smplx_model(), posedirs=np.zeros((syn.SMPLX_NUM_VERTS, 3, 486)))
    v0 = co.smplx_vertices(model, g["betas"], g["pose66"][2:], g["rest99"][2:], g["transl"][2:])
    assert np.abs(v0[:, g["keep"]] - g["verts"][2:]).max() > 1e-3


def test_canonical_pose_and_joint_matrices_match_the_reference():
    x = np.load(os.path.join(GOLDEN, "cano_smplx_vertices.npz"))
    s = np.load(os.path.join(GOLDEN, "cano_smpl.npz"))
    # frame 0 of the SMPL-X fixture is the reference's canonical pose (smplx_cpose_param) at transl (0, 0.30, 0)
    cx = canonical_pose("smplx").numpy()[0]
    assert np.array_equal(np.concatenate([x["pose66"][0], x["rest99"][0]]), cx)
    assert np.array_equal(s["pose"][0], canonical_pose("smpl").numpy()[0])
    assert np.allclose(x["transl"][0], CANO_TRANSL) and np.allclose(s["transl"][0], CANO_TRANSL)
    bx, bs = syn.make_smplx_body(0), syn.make_body(0)
    Ax = syn.joint_transforms_np(bx.rest_joints().double().numpy(), cx, np.asarray(CANO_TRANSL), syn.SMPLX_PARENTS)
    As = syn.joint_transforms_np(bs.rest_joints().double().numpy(), canonical_pose("smpl").numpy()[0].astype(np.float64),
                                 np.asarray(CANO_TRANSL))
    # the rest joints are the fp32 J of the loaders; the fixture's are fp64
    assert np.abs(Ax - x["A"][0]).max() < 1e-5
    assert np.abs(As - s["A"][0]).max() < 1e-5
    # the canonical SMPL vertices of the oracle are the reference's
    v = po.smpl_vertices(syn.smpl_mesh_model(bs, syn.make_uv_template(0)), s["betas"], s["pose"], s["transl"])
    assert np.abs(v[:, s["keep"]] - s["verts"]).max() < 1e-5
    assert np.abs(v.mean(1) - s["mean"]).max() < 1e-5


@pytest.mark.parametrize("body", ["smpl", "smplx"])
def test_weight_map_oracle_matches_the_reference(body):
    g = np.load(os.path.join(GOLDEN, "cano_lbs_weights.npz"))
    b, t = (syn.make_body(0), syn.make_uv_template(0)) if body == "smpl" else (syn.make_smplx_body(0), syn.make_smplx_uv_template(0))
    fid, bary = g[f"{body}/face_id"], g[f"{body}/bary"]
    # the fixture's layout is the library's layout of the same template
    fid_ref, bary_ref = po.layout(t[2].astype(np.float32)[t[3]], int(g["S"]))
    assert np.array_equal(fid, fid_ref) and np.array_equal(bary, bary_ref)
    w = co.weight_map(b.lbs_weights.numpy(), t[1], fid, bary)
    cov = fid >= 0
    assert cov.mean() > 0.5
    assert np.abs(w[cov] - g[f"{body}/lbs_map"][cov]).max() < 1e-6
    assert (w[~cov] == 0).all()


def test_new_entry_points_reject_bad_arguments():
    L = _lib.lib()

    def err(rc, text):
        assert rc != 0
        assert text in L.ga_last_error().decode()

    ok = [FAKE] * 8
    err(L.ga_smplx_vertices(9, 10475, *ok, None), "batch")
    err(L.ga_smplx_vertices(-1, 10475, *ok, None), "batch")
    err(L.ga_smplx_vertices(2, 0, *ok, None), "vertex count")
    for i in range(8):
        args = list(ok)
        args[i] = None
        err(L.ga_smplx_vertices(2, 10475, *args, None), "NULL")
    ok = [FAKE] * 5
    err(L.ga_posmap_weights(0, 24, *ok, None), "map size")
    err(L.ga_posmap_weights(513, 55, *ok, None), "map size")
    for J in (0, 23, 25, 54, 56):
        err(L.ga_posmap_weights(16, J, *ok, None), "joint count")
    for i in range(5):
        args = list(ok)
        args[i] = None
        err(L.ga_posmap_weights(16, 24, *args, None), "NULL")


def _run(tool, *args):
    return subprocess.run([sys.executable, os.path.join(ROOT, "tools", tool), *args], capture_output=True, text=True)


def test_tools_name_missing_input_files(tmp_path):
    folder = tmp_path / "subject"
    folder.mkdir()
    model, obj = str(tmp_path / "SMPLX_NEUTRAL.npz"), str(tmp_path / "template.obj")
    r = _run("cano_assets.py", str(folder), "--body", "smplx", "--model", model, "--uv_template", obj, "--size", "16")
    assert r.returncode != 0 and "smpl_parms.pth" in r.stderr
    torch.save(dict(beta=torch.zeros(1, 10), body_pose=torch.zeros(2, 165), trans=torch.zeros(2, 3)), str(folder / "smpl_parms.pth"))
    r = _run("cano_assets.py", str(folder), "--body", "smplx", "--model", model, "--uv_template", obj, "--size", "16")
    assert r.returncode != 0 and "SMPLX_NEUTRAL.npz" in r.stderr
    syn.write_smplx_model_npz(model, syn.make_smplx_body(0))
    r = _run("cano_assets.py", str(folder), "--body", "smplx", "--model", model, "--uv_template", obj, "--size", "16")
    assert r.returncode != 0 and "template.obj" in r.stderr
    r = _run("pose_maps.py", str(folder), "--body", "smplx", "--smpl_model", str(tmp_path / "nope.npz"), "--uv_template", obj)
    assert r.returncode != 0 and "nope.npz" in r.stderr
    r = _run("pose_maps.py", str(tmp_path / "empty"), "--body", "smplx", "--smpl_model", model, "--uv_template", obj)
    assert r.returncode != 0 and "smpl_parms.pth" in r.stderr
