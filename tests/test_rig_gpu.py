"""GPU: ga_skin_weights against oracle/skin_oracle.py at ragged sizes, the glTF skeleton chain against the device's own posed
Gaussians, rigged canonical meshes of synthetic SMPL / SMPL-X / stage-2 avatars (closed, model state unchanged, silhouette IoU of the
posed rig against extract_mesh at the same pose), and tools/extract_mesh.py --format glb on a saved checkpoint."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from gaussianavatar_b200 import mesh_extract as me  # noqa: E402
from gaussianavatar_b200 import rig as rg  # noqa: E402
from oracle import skin_oracle as so  # noqa: E402
from test_mesh_extract_cpu import closed_manifold  # noqa: E402
from test_mesh_extract_gpu import _avatar, _state  # noqa: E402
from test_rig_cpu import accessor, read_glb  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
# the posed rig's silhouette IoU may fall this far below extract_mesh's at the same pose (DESIGN.md §2)
IOU_GAP = 0.01


@pytest.mark.parametrize("J,ld", [(24, 24), (55, 56)])
@pytest.mark.parametrize("k,K", [(1, 1), (8, 4), (16, 8), (8, 8), (16, 1)])
def test_skin_weights_match_oracle(J, ld, k, K):
    rng = np.random.default_rng(100 * k + K + J)
    V, N = 1000 + 37, 3 * 512 + 211                       # neither a multiple of the block (128) nor of the tile (512)
    means = rng.normal(size=(N, 3)).astype(np.float32) * 0.3
    means[N - 5:] = means[:5]                             # duplicated means: equal distances, ties by index
    verts = np.concatenate([rng.normal(size=(V - 20, 3)).astype(np.float32) * 0.3, means[:20]])
    lbs = np.zeros((N, ld), np.float32)
    lbs[:, :J] = rng.random((N, J)).astype(np.float32) ** 8
    lbs[::7, :J] = 0.0                                    # some all-zero rows
    lbs[::5, J // 2] = lbs[::5, J // 3]                   # some equal weights
    if ld > J:
        lbs[:, J:] = 1.0                                  # padding columns never count
    dj, dw = (t.cpu().numpy() for t in rg.skin_weights(*(torch.from_numpy(a).to(DEV) for a in (verts, means, lbs)), J, k, K))
    oj, ow = so.skin_weights(verts, means, lbs, J, k, K)
    assert np.array_equal(dj, oj)
    assert np.abs(dw - ow).max() <= 1e-6
    nbits = int((dw.view(np.int32) != ow.view(np.int32)).sum())
    dj2, dw2 = (t.cpu().numpy() for t in rg.skin_weights(*(torch.from_numpy(a).to(DEV) for a in (verts, means, lbs)), J, k, K))
    assert np.array_equal(dj, dj2) and np.array_equal(dw.view(np.int32), dw2.view(np.int32))
    print(f"J {J} k {k} K {K}: joints equal, weights differing in any bit {nbits}")


@pytest.mark.parametrize("body", ["smpl", "smplx"])
def test_skeleton_chain_reproduces_posed_gaussians(body):
    m, mapper, pose, transl, rest = _avatar(body, 1)
    with torch.no_grad(), me.kept_state(m):
        cano = rg.canonical_gaussians(m)[0][0].double().cpu().numpy()
        posed = me.posed_gaussians(m, pose, transl, rest)[0][0].double().cpu().numpy()
    sk = rg.skeleton(m._rest_joints, m._inv_cano, m.body.parents)
    full = m.body.join(pose[None], rest.reshape(1, -1)) if m.body.rest_width else pose[None]
    mo = rg.bake_poses(m._rest_joints, full, transl[None], 30.0, "y")
    loc = sk["translations"].copy()
    loc[0] = mo.root_translation[0]
    A = rg.node_globals(m.body.parents, loc, mo.rotations[0]) @ sk["ibm"]
    w = m._query_lbs[:, :m.body.joints].double().cpu().numpy()
    M = np.einsum("nj,jab->nab", w, A)
    got = np.einsum("nab,nb->na", M[:, :3, :3], cano) + M[:, :3, 3]
    extent = float((posed.max(0) - posed.min(0)).max())
    err = np.abs(got - posed).max()
    print(f"{body}: max |rig - posed_gaussians| {err:.3g} of extent {extent:.3g}")
    assert err <= 1e-5 * extent


@pytest.mark.parametrize("body,stage", [("smpl", 1), ("smplx", 1), ("smpl", 2)])
def test_rigged_mesh_closed_state_kept_and_iou(body, stage):
    m, mapper, pose, transl, rest = _avatar(body, stage)
    before = _state(m)
    rig = rg.extract_rigged_mesh(m, res=256, views=64, size=512, influences=4, pose_mapper=mapper)
    after = _state(m)
    assert before.keys() == after.keys() and all(torch.equal(before[k], after[k]) for k in before)
    F = rig.faces.cpu().numpy()
    assert closed_manifold(F) and len(F) > 1000
    w = rig.weights.double()
    assert (rig.joints.long() < m.body.joints).all() and (w.sum(1) - 1).abs().max() < 1e-6
    V, Fd, _ = me.extract_mesh(m, pose, transl, rest, res=256, views=64, size=512, pose_mapper=mapper)
    with torch.no_grad():
        means, scales, _ = me.posed_gaussians(m, pose, transl, rest, mapper)
    origin, voxel, dims, _ = me.fusion_grid(means, scales, 256, 4)
    center = np.asarray(origin) + 0.5 * voxel * (np.asarray(dims) - 1)
    held_out = me.fusion_cameras(center, 0.5 * voxel * float(np.linalg.norm(np.asarray(dims) - 1)), 8, 512)
    full = m.body.join(pose[None], rest.reshape(1, -1)) if m.body.rest_width else pose[None]
    mo = rg.bake_poses(m._rest_joints, full, transl[None], 30.0, "y")
    Vr = torch.from_numpy(rg.pose_rig(rig, mo, 0)).float().to(DEV)
    iou_rig = me.silhouette_iou(m, pose, transl, Vr, rig.faces, held_out, 512, 512, rest, mapper)
    iou_dir = me.silhouette_iou(m, pose, transl, V, Fd, held_out, 512, 512, rest, mapper)
    print(f"{body} stage {stage}: rig IoU min {min(iou_rig):.4f} mean {np.mean(iou_rig):.4f}; extract_mesh IoU min {min(iou_dir):.4f} "
          f"mean {np.mean(iou_dir):.4f}; V {rig.verts.shape[0]} F {len(F)}")
    assert min(iou_rig) >= min(iou_dir) - IOU_GAP


def test_tool_end_to_end(tmp_path):
    from dataset_fixture import write_synthetic_dataset
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams, OptimizationParams
    mp = write_synthetic_dataset(str(tmp_path), seed=0)
    torch.manual_seed(0)
    m = AvatarModel(mp, NetworkParams(nf=8), OptimizationParams(), train=True)
    m.training_setup()
    with torch.no_grad():
        sd = m.net.state_dict()
        sd["decoder.conv8N.bias"] = torch.tensor([-5.3])
        m.net.load_state_dict(sd, strict=False)
    m.save(7)
    base = [sys.executable, os.path.join(ROOT, "tools", "extract_mesh.py"), "-s", mp.source_path, "-m", mp.model_path, "--project_path",
            mp.project_path, "--smpl_model", os.path.join(mp.smpl_model_path, "SMPL_NEUTRAL.pkl"), "--query_posmap_size",
            str(mp.query_posmap_size), "--inp_posmap_size", str(mp.inp_posmap_size), "--epoch", "7", "--res", "64", "--views", "16",
            "--size", "128", "--format", "glb"]
    out = tmp_path / "still"
    r = subprocess.run(base + ["--frame", "0", "--frame", "2", "--iou", "--out", str(out)], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    rec = json.loads([x for x in r.stdout.splitlines() if x.startswith("{")][-1])
    print("tool (frames)", rec)
    assert rec["frames"] == 0 and rec["joints"] == 24 and len(rec["iou"]) == 2 and all(0.0 <= x <= 1.0 for x in rec["iou"])
    g, binc = read_glb(rec["mesh"])
    assert "animations" not in g and accessor(g, binc, g["meshes"][0]["primitives"][0]["indices"]).size == 3 * rec["faces"]
    clip = os.path.join(mp.test_folder, "smpl_parms.pth")
    out2 = tmp_path / "clip"
    r = subprocess.run(base + ["--motion", clip, "--clip_fps", "30", "--fps", "15", "--align_to", "1", "--influences", "8", "--iou",
                               "--out", str(out2)], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    rec = json.loads([x for x in r.stdout.splitlines() if x.startswith("{")][-1])
    print("tool (motion)", rec)
    assert rec["frames"] >= 1 and len(rec["iou"]) == rec["frames"]
    g, binc = read_glb(os.path.join(out2, "avatar.glb"))
    assert "JOINTS_1" in g["meshes"][0]["primitives"][0]["attributes"] and len(g["animations"][0]["channels"]) == 25
