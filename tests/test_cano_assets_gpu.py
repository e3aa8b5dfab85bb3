"""GPU: SMPL-X mesh posing (ga_smplx_vertices) and the texel skinning-weight map (ga_posmap_weights) against the reference's
fixtures and the oracle, the canonical assets of both bodies, and subject folders whose canonical files are rebuilt by
tools/cano_assets.py (and, for SMPL-X, whose stage-2 input maps are written by tools/pose_maps.py --body smplx)."""
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from gaussianavatar_b200 import _lib
from gaussianavatar_b200 import synthetic as syn
from gaussianavatar_b200._lib import ptr
from gaussianavatar_b200.posmap import PoseMapper, SmplxPoseMapper, canonical_assets
from oracle import cano_oracle as co
from oracle import posmap_oracle as po

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

# fp32 bounds.  Vertices are ~1 m from the origin and posed through up to 11 chained affine products (a fingertip) and 486 pose
# blend-shape terms; each fp32 step rounds at ~6e-8 relative, so the accumulated error stays a few 1e-6 m.  The SMPL bound (3e-5)
# holds here too.  A map texel is a convex combination of three such vertices, a weight-map texel of three fp32 weight rows.
VERT_TOL = 3e-5
MAP_TOL = 3e-5
A_TOL = 1e-5
W_TOL = 1e-6


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _smplx_inputs():
    body, t = syn.make_smplx_body(0), syn.make_smplx_uv_template(0)
    return syn.smplx_mesh_model(body, t, syn.smplx_posedirs(0)), body, t


def _smplx_mapper(S):
    model, body, t = _smplx_inputs()
    return SmplxPoseMapper(model, body.betas[0], t, S, device=DEV), model, t


@pytest.mark.parametrize("B", [1, 2, 8])
def test_smplx_vertices_match_the_reference_fixture(B):
    g = np.load(os.path.join(GOLDEN, "cano_smplx_vertices.npz"))
    m, _, _ = _smplx_mapper(16)
    pose, rest, transl = (torch.from_numpy(g[k][:B]) for k in ("pose66", "rest99", "transl"))
    v = m.vertices(pose, rest, transl).cpu().numpy().astype(np.float64)
    assert np.abs(v[:, g["keep"]] - g["verts"][:B]).max() < VERT_TOL
    assert np.abs(v.mean(1) - g["mean"][:B]).max() < VERT_TOL
    # a frame's vertices do not depend on the batch it is posed in, nor on its position in that batch
    for b in range(B):
        one = m.vertices(pose[b:b + 1], rest[b:b + 1], transl[b:b + 1])
        assert torch.equal(one[0], torch.from_numpy(v[b]).float().to(DEV)), b


def test_both_kernels_write_every_element_and_match_the_oracle():
    S, B = 64, 3
    m, model, t = _smplx_mapper(S)
    pose, rest, transl = syn.synthetic_smplx_poses(B, seed=7)
    vs = torch.full((B, m.V, 3), float("nan"), device=DEV)
    p, r, tr = (x.float().contiguous().to(DEV) for x in (pose, rest, transl))
    _lib.check(_lib.lib().ga_smplx_vertices(B, m.V, ptr(p), ptr(r), ptr(tr), ptr(m.rest_joints), ptr(m.v_shaped), ptr(m.posedirs),
                                            ptr(m.weights), ptr(vs), _stream()), "ga_smplx_vertices")
    assert torch.isfinite(vs).all()
    assert torch.equal(vs, m.vertices(pose, rest, transl))
    ref_v = co.smplx_vertices(model, syn.make_smplx_body(0).betas[0].numpy(), pose.numpy(), rest.numpy(), transl.numpy())
    assert np.abs(vs.cpu().numpy() - ref_v).max() < VERT_TOL
    maps = m(pose, rest, transl)
    ref_map = po.fill(vs.cpu().numpy(), t[1], m.face_id.cpu().numpy(), m.bary.cpu().numpy())
    assert np.abs(maps.cpu().numpy() - ref_map).max() < MAP_TOL
    for mapper in (m, PoseMapper(syn.smpl_mesh_model(syn.make_body(0), syn.make_uv_template(0)), syn.make_body(0).betas[0],
                                 syn.make_uv_template(0), S, device=DEV)):
        J = mapper.JOINTS
        out = torch.full((S, S, J), float("nan"), device=DEV)
        _lib.check(_lib.lib().ga_posmap_weights(S, J, ptr(mapper.weights), ptr(mapper.faces), ptr(mapper.face_id), ptr(mapper.bary),
                                                ptr(out), _stream()), "ga_posmap_weights")
        assert torch.isfinite(out).all()
        assert torch.equal(out, mapper.weight_map())
        fid = mapper.face_id.cpu().numpy()
        ref = co.weight_map(mapper.weights.cpu().numpy(), mapper.faces.cpu().numpy(), fid, mapper.bary.cpu().numpy())
        assert np.abs(out.cpu().numpy() - ref).max() < W_TOL
        assert (out[mapper.face_id < 0] == 0).all()
        # rows sum to 1 at covered texels wherever the vertex rows do (the synthetic weights are softmax rows: all of them)
        vsum = mapper.weights.double().sum(1)
        assert (vsum - 1).abs().max() < 1e-6
        cov = mapper.face_id >= 0
        assert cov.float().mean() > 0.5
        assert (out[cov].double().sum(1) - 1).abs().max() < 1e-5


@pytest.mark.parametrize("body", ["smpl", "smplx"])
def test_weight_map_matches_the_reference_fixture(body):
    g = np.load(os.path.join(GOLDEN, "cano_lbs_weights.npz"))
    S = int(g["S"])
    if body == "smplx":
        m, _, _ = _smplx_mapper(S)
    else:
        t = syn.make_uv_template(0)
        m = PoseMapper(syn.smpl_mesh_model(syn.make_body(0), t), syn.make_body(0).betas[0], t, S, device=DEV)
    fid = m.face_id.cpu().numpy()
    assert np.array_equal(fid, g[f"{body}/face_id"])
    w = m.weight_map().cpu().numpy()
    cov = fid >= 0
    assert np.abs(w[cov] - g[f"{body}/lbs_map"][cov]).max() < W_TOL


@pytest.mark.parametrize("body", ["smpl", "smplx"])
def test_canonical_assets_match_the_fixtures(body):
    S = 128
    if body == "smplx":
        g = np.load(os.path.join(GOLDEN, "cano_smplx_vertices.npz"))
        model, b, t = _smplx_inputs()
        i = 0                                  # frame 0 of the fixture is the canonical pose
        ref_v = co.smplx_vertices(model, b.betas[0].numpy(), g["pose66"][:1], g["rest99"][:1], g["transl"][:1])
    else:
        g = np.load(os.path.join(GOLDEN, "cano_smpl.npz"))
        b, t = syn.make_body(0), syn.make_uv_template(0)
        model = syn.smpl_mesh_model(b, t)
        i = 0
        ref_v = po.smpl_vertices(model, b.betas[0].numpy(), g["pose"], g["transl"])
    assert np.abs(ref_v[0][g["keep"]] - g["verts"][i]).max() < 1e-5          # the oracle's canonical mesh is the reference's
    res = canonical_assets(model, b.betas[0], t, S, body=body, device=DEV)
    J = 55 if body == "smplx" else 24
    assert res.posmap.shape == (S, S, 3) and res.joint_mats.shape == (J, 4, 4) and res.face_id.shape == (S, S)
    assert res.lbs_map.shape == (S, S, J) and res.bary.shape == (S, S, 3)
    assert np.abs(res.joint_mats.cpu().numpy() - g["A"][i]).max() < A_TOL
    fid, bary = po.layout(t[2].astype(np.float32)[t[3]], S)
    assert np.array_equal(res.face_id.cpu().numpy(), fid)
    ref_map = po.fill(ref_v, t[1], fid, bary)[0].transpose(1, 2, 0)
    assert np.abs(res.posmap.cpu().numpy() - ref_map).max() < MAP_TOL
    assert (res.posmap[res.face_id < 0] == 0).all()


# ---- subject folders rebuilt by the tools --------------------------------------------------------------------------------------
def _tool(name, *args):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", name), *args], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return json.loads(r.stdout.strip().splitlines()[-1])


def _batch(items):
    from gaussianavatar_b200.workload import to_cuda
    batch = {k: (torch.stack([torch.as_tensor(it[k]) for it in items]) if not isinstance(items[0][k], (int, float)) else [it[k] for it in items])
             for k in items[0]}
    batch["pose_idx"] = torch.tensor([it["pose_idx"] for it in items])
    return to_cuda(batch, DEV)[0]


def _step(mp):
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams, OptimizationParams
    from gaussianavatar_b200.trainer import AvatarTrainer
    torch.manual_seed(0)
    m = AvatarModel(mp, NetworkParams(nf=8), OptimizationParams(), train=True)
    tr = AvatarTrainer(m, use_graph=False)
    batch = _batch([m.train_dataset[0], m.train_dataset[1]])
    with torch.backends.cudnn.flags(allow_tf32=False):
        loss, image = tr.loss(batch, 3000, epoch=1)
        m.zero_grad(1)
        loss.backward()
    assert np.isfinite(loss.item()) and torch.isfinite(image).all()
    assert torch.isfinite(m.net.flat.grad).all()
    return m, batch


def _rebuild(mp, body, model, template, S):
    """Delete the folder's canonical files, rebuild them with the tool, check them against themselves, and check AvatarModel."""
    train = os.path.join(mp.source_path, "train")
    assets = os.path.join(mp.project_path, "assets")
    for f in (os.path.join(train, f"query_posemap_{S}_cano_{body}.npz"), os.path.join(train, f"{body}_cano_joint_mat.pth"),
              os.path.join(assets, "uv_masks", f"uv_mask{S}_with_faceid_{body}.npy"), os.path.join(assets, f"lbs_map_{body}_{S}.npy")):
        os.remove(f)
    args = [train, "--body", body, "--model", model, "--uv_template", template, "--size", str(S), "--assets", assets]
    _tool("cano_assets.py", *args)
    chk = _tool("cano_assets.py", *args, "--check")
    assert chk["missing_files"] == [] and chk["face_id_mismatches"] == 0 and chk["max_abs_error_all"] == 0.0, chk
    qmap = np.load(os.path.join(train, f"query_posemap_{S}_cano_{body}.npz"))[f"posmap{S}"].reshape(-1, 3)
    fid = np.load(os.path.join(assets, "uv_masks", f"uv_mask{S}_with_faceid_{body}.npy")).reshape(-1)
    stage1 = type(mp)(**{**vars(mp), "train_stage": 1})
    m, _ = _step(stage1)
    cov = fid >= 0
    assert m._query_points.shape[0] == int(cov.sum()) > 0
    assert torch.equal(m._query_points.cpu(), torch.from_numpy(qmap[cov]))


def test_smpl_folder_rebuilt_by_the_tool_trains(tmp_path):
    from dataset_fixture import write_synthetic_dataset
    import pickle
    S = 32
    mp = write_synthetic_dataset(str(tmp_path), S=S, num_frames=4, side=64)
    t = syn.make_uv_template(0)
    model = os.path.join(mp.smpl_model_path, "SMPL_NEUTRAL.pkl")
    with open(model, "wb") as fh:
        pickle.dump(syn.smpl_mesh_model(syn.make_body(0), t), fh)
    obj = os.path.join(mp.project_path, "assets", "template_mesh_smpl_uv.obj")
    syn.write_uv_template_obj(obj, t)
    _rebuild(mp, "smpl", model, obj, S)


def test_smplx_folder_rebuilt_by_the_tools_trains_both_stages(tmp_path):
    from dataset_fixture_smplx import write_synthetic_smplx_dataset
    S, inp = 32, 32          # the pose encoder's five stride-2 levels need input maps of at least 32^2
    mp = write_synthetic_smplx_dataset(str(tmp_path), S=S, num_frames=4, side=64, inp=inp, stage2=True)
    body, t = syn.make_smplx_body(0), syn.make_smplx_uv_template(0)
    model = os.path.join(mp.smplx_model_path, "SMPLX_NEUTRAL.npz")
    syn.write_smplx_model_npz(model, body, seed=0, posedirs=syn.smplx_posedirs(0), faces=t[1])
    obj = os.path.join(mp.project_path, "assets", "template_mesh_smplx_uv.obj")
    syn.write_uv_template_obj(obj, t)
    _rebuild(mp, "smplx", model, obj, S)

    # stage 2 from the input maps the tool writes
    train = os.path.join(mp.source_path, "train")
    shutil.rmtree(os.path.join(train, "inp_map"))
    _tool("pose_maps.py", train, "--body", "smplx", "--smpl_model", model, "--uv_template", obj, "--size", str(inp))
    prm = torch.load(os.path.join(train, "smpl_parms_pred.pth"), weights_only=False)
    bp = torch.as_tensor(prm["body_pose"]).float()
    mapper = SmplxPoseMapper(syn.smplx_mesh_model(body, t, syn.smplx_posedirs(0)), torch.as_tensor(prm["beta"]).reshape(-1, 10)[0], t,
                             inp, device=DEV)
    ref = mapper(bp[:, :66], bp[:, 66:], torch.as_tensor(prm["trans"]).float()).permute(0, 2, 3, 1).cpu().numpy()
    for i in range(bp.shape[0]):
        got = np.load(os.path.join(train, "inp_map", "inp_posemap_%s_%s.npz" % (inp, str(i).zfill(8))))[f"posmap{inp}"]
        assert np.array_equal(got, ref[i]), i
    chk = _tool("pose_maps.py", train, "--body", "smplx", "--smpl_model", model, "--uv_template", obj, "--size", str(inp), "--check")
    assert chk["max_abs_map_error"] == 0.0 and chk["missing_files"] == 0, chk
    m, batch = _step(mp)
    for k in range(2):
        got = batch["inp_pos_map"][k].cpu()
        assert torch.equal(got, torch.from_numpy(ref[int(batch["pose_idx"][k])]).permute(2, 0, 1)), k
