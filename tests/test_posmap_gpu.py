"""GPU: device position maps (csrc/posmap.cu) against the oracle and the reference's LBS fixture, and stage 2 with
ModelParams.inp_posmap_from_pose against the same step reading maps from files."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gaussianavatar_b200 import _lib
from gaussianavatar_b200 import synthetic as syn
from gaussianavatar_b200._lib import ptr
from gaussianavatar_b200.posmap import PoseMapper
from oracle import posmap_oracle as po

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

# fp32 bounds: vertices are ~1 m, posed through 24 affine products and 207 pose blend shapes; a map texel is a convex combination of
# three fp32 vertices
VERT_TOL = 3e-5
MAP_TOL = 3e-5


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _mapper(S):
    t = syn.make_uv_template(0)
    body = syn.make_body(0)
    return PoseMapper(syn.smpl_mesh_model(body, t), body.betas[0], t, S, device=DEV), t


def _layout(corners, S):
    corners = torch.from_numpy(np.ascontiguousarray(corners, np.float32)).to(DEV)
    fid = torch.full((S, S), 12345, dtype=torch.int32, device=DEV)
    bary = torch.full((S, S, 3), float("nan"), device=DEV)
    _lib.check(_lib.lib().ga_posmap_layout(corners.shape[0], S, ptr(corners), ptr(fid), ptr(bary), _stream()), "ga_posmap_layout")
    return fid.cpu().numpy(), bary.cpu().numpy()


@pytest.mark.parametrize("S", [16, 100, 128, 512])
def test_layout_of_the_template_is_bit_identical_to_the_oracle(S):
    m, t = _mapper(S)
    corners = t[2].astype(np.float32)[t[3]]
    fid_ref, bary_ref = po.layout(corners, S)
    fid = m.face_id.cpu().numpy()
    assert np.array_equal(fid, fid_ref), int((fid != fid_ref).sum())
    assert (fid >= 0).mean() > 0.5
    assert np.abs(m.bary.cpu().numpy() - bary_ref).max() <= 1e-7        # both fp64 quotients of the same integers, rounded once


def test_layout_ties_overlaps_and_degenerate_faces_match_the_oracle():
    """Corners on texel centres (ties on edges and vertices), a seam, overlapping faces, zero-area and out-of-range faces."""
    from test_posmap_cpu import _square_triangulation
    extra = np.array([[[0.2, 0.2], [0.7, 0.2], [0.2, 0.7]],               # overlaps the square faces, which come after it
                      [[0.1, 0.1], [0.9, 0.9], [0.5, 0.5]],               # collinear
                      [[0.0, 0.0], [5000.0, 0.0], [0.0, 1.0]]], np.float32)
    for S, n, jitter in ((16, 32, 0.0), (100, 200, 0.0), (100, 24, 0.3)):
        sq = _square_triangulation(n, S + n, jitter)
        for corners in (sq, np.concatenate([extra, sq])):
            fid, bary = _layout(corners, S)
            fid_ref, bary_ref = po.layout(corners, S)
            assert np.array_equal(fid, fid_ref), (S, n, int((fid != fid_ref).sum()))
            assert np.abs(bary - bary_ref).max() <= 1e-7
        assert (fid >= 0).all()


@pytest.mark.parametrize("B", [1, 2, 8])
def test_vertices_match_the_reference_lbs_fixture(B):
    g = np.load(os.path.join(GOLDEN, "posmap_vertices.npz"))
    m, _ = _mapper(16)
    pose, transl = torch.from_numpy(g["pose"][:B]), torch.from_numpy(g["transl"][:B])
    v = m.vertices(pose, transl).cpu().numpy().astype(np.float64)
    assert np.abs(v[:, g["keep"]] - g["verts"][:B]).max() < VERT_TOL
    assert np.abs(v.mean(1) - g["mean"][:B]).max() < VERT_TOL
    # a frame's vertices do not depend on the batch it is posed in (so maps are reproducible bit for bit)
    one = m.vertices(pose[B - 1:B], transl[B - 1:B])
    assert torch.equal(one[0], torch.from_numpy(v[B - 1]).float().to(DEV))


def test_maps_match_the_oracle_and_every_element_is_written():
    S, B = 128, 3
    m, t = _mapper(S)
    pose, transl = syn.synthetic_poses(B, seed=4)
    verts = m.vertices(pose, transl)
    out = torch.full((B, 3, S, S), float("nan"), device=DEV)
    _lib.check(_lib.lib().ga_posmap_fill(B, S, m.V, ptr(verts), ptr(m.faces), ptr(m.face_id), ptr(m.bary), ptr(out), _stream()),
               "ga_posmap_fill")
    assert torch.isfinite(out).all()
    ref = po.fill(verts.cpu().numpy(), t[1], m.face_id.cpu().numpy(), m.bary.cpu().numpy())
    assert np.abs(out.cpu().numpy() - ref).max() < MAP_TOL
    assert torch.equal(out, m(pose, transl))
    assert (out[:, :, m.face_id < 0] == 0).all()
    # vertices: sentinel-filled output, fully written, and close to the fp64 oracle
    vs = torch.full((B, m.V, 3), float("nan"), device=DEV)
    p32, t32 = pose.float().contiguous().to(DEV), transl.float().contiguous().to(DEV)
    _lib.check(_lib.lib().ga_smpl_vertices(B, m.V, ptr(p32), ptr(t32), ptr(m.rest_joints), ptr(m.v_shaped), ptr(m.posedirs),
                                           ptr(m.weights), ptr(vs), _stream()), "ga_smpl_vertices")
    assert torch.equal(vs, verts)
    ref_v = po.smpl_vertices(syn.smpl_mesh_model(syn.make_body(0), t), syn.make_body(0).betas[0].numpy(), pose.numpy(), transl.numpy())
    assert np.abs(verts.cpu().numpy() - ref_v).max() < VERT_TOL


# ---- stage 2 through AvatarModel -------------------------------------------------------------------------------------------------
def _batch(items):
    from gaussianavatar_b200.workload import to_cuda
    batch = {k: (torch.stack([torch.as_tensor(it[k]) for it in items]) if not isinstance(items[0][k], (int, float)) else [it[k] for it in items])
             for k in items[0]}
    batch["pose_idx"] = torch.tensor([it["pose_idx"] for it in items])
    return to_cuda(batch, DEV)[0]


def _rel(a, b):
    return float((a - b).norm() / (b.norm() + 1e-30))


def test_stage2_step_with_device_maps_matches_the_step_with_file_maps(tmp_path):
    from posmap_fixture import write_posmap_dataset
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams, OptimizationParams
    from gaussianavatar_b200.trainer import AvatarTrainer
    inp = 32
    mp_on = write_posmap_dataset(str(tmp_path), N=700, S=48, num_frames=4, side=64, inp=inp)
    pk = os.path.join(mp_on.smpl_model_path, "SMPL_NEUTRAL.pkl")
    obj = os.path.join(mp_on.project_path, "assets", "template_mesh_smpl_uv.obj")
    train_dir = os.path.join(mp_on.source_path, "train")
    tool = [sys.executable, os.path.join(ROOT, "tools", "pose_maps.py"), train_dir, "--smpl_model", pk, "--uv_template", obj, "--size", str(inp)]
    subprocess.run(tool, check=True, capture_output=True, text=True)
    # --check against the files just written and against the oracle's face ids
    t = syn.make_uv_template(0)
    mask = os.path.join(str(tmp_path), "uv_mask.npy")
    np.save(mask, po.layout(t[2].astype(np.float32)[t[3]], inp)[0])
    chk = json.loads(subprocess.run(tool + ["--check", "--uv_mask", mask], check=True, capture_output=True, text=True).stdout.strip().splitlines()[-1])
    assert chk["max_abs_map_error"] == 0.0 and chk["face_id_mismatches"] == 0 and chk["missing_files"] == 0, chk

    mp_off = type(mp_on)(**{**vars(mp_on), "inp_posmap_from_pose": False})
    results = {}
    for name, mp in (("files", mp_off), ("device", mp_on)):
        torch.manual_seed(0)
        m = AvatarModel(mp, NetworkParams(nf=8), OptimizationParams(), train=True)
        seen = []
        m.pose_encoder.register_forward_pre_hook(lambda mod, args: seen.append(args[0].detach().clone()))
        tr = AvatarTrainer(m, use_graph=False)
        ds = m.train_dataset
        batch = _batch([ds[1], ds[2]])
        assert ("inp_pos_map" in batch) == (name == "files")
        with torch.backends.cudnn.flags(allow_tf32=False, deterministic=True):
            loss, image = tr.loss(batch, 3000, epoch=1)
            m.zero_grad(1)
            loss.backward()
        results[name] = dict(inp=seen[0], loss=loss.item(), image=image.detach(), net=m.net.flat.grad.detach().clone(),
                             pe=torch.cat([p.grad.reshape(-1) for p in m.pose_encoder.parameters()]))
    f, d = results["files"], results["device"]
    assert torch.equal(f["inp"], d["inp"])
    assert abs(f["loss"] - d["loss"]) <= 1e-6 * max(1.0, abs(f["loss"]))
    assert (f["image"] - d["image"]).abs().max().item() <= 1e-5
    assert _rel(d["net"], f["net"]) < 1e-3 and _rel(d["pe"], f["pe"]) < 1e-3

    # a novel-pose folder without inp_map/ renders from its poses
    assert not os.path.exists(os.path.join(mp_on.test_folder, "inp_map"))
    nds = m.getNovelposeDataset()
    nb = _batch([nds[0]])
    assert "inp_pos_map" not in nb
    with torch.no_grad():
        out = m.render_free_stage2(nb, 3000)
        ref_map = m.pose_mapper(nb["pose_data"], nb["transl_data"])
    assert out.shape == (1, 3, 1024, 1024) and torch.isfinite(out).all()
    assert torch.equal(m._pose_map(nb), ref_map)


def test_from_assets_builds_device_maps():
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams
    a = syn.make_avatar_assets(500, 32, seed=0)
    t = syn.make_uv_template(0)
    assets = dict(valid_idx=a.valid_idx, query_points=a.query_points, query_lbs=a.query_lbs, cano_joint_mats=a.cano_joint_mats,
                  rest_joints=a.rest_joints, betas=a.body.betas[0], S=a.S, smpl_mesh=syn.smpl_mesh_model(a.body, t), uv_template=t)
    pose, transl = syn.synthetic_poses(3, seed=2)
    m = AvatarModel.from_assets(assets, [], pose, transl, batch_size=2, net_parms=NetworkParams(nf=8), train_stage=2, inp_posmap_size=32,
                                inp_posmap_from_pose=True)
    got = m._pose_map({"pose_idx": torch.tensor([2, 0])})
    assert torch.equal(got, m.pose_mapper(pose[[2, 0]], transl[[2, 0]]))
    assert got.shape == (2, 3, 32, 32) and (got[:, :, m.pose_mapper.face_id < 0] == 0).all()
