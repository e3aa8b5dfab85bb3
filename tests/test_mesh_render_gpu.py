"""GPU: the mesh renderer (ga_mesh_render, MeshRenderer) against the oracle, bit for bit in face_id and depth, on the synthetic SMPL
and SMPL-X bodies, the known-answer meshes and full-frame faces, at 64^2, 1024^2 and 540 x 960 for B = 1, 2 and 8; and
tools/body_overlay.py and tools/export_stage1_poses.py end to end."""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch
from PIL import Image

from gaussianavatar_b200 import _lib
from gaussianavatar_b200 import synthetic as syn
from gaussianavatar_b200._lib import ptr
from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, make_camera
from gaussianavatar_b200.mesh_render import MeshRenderer, cameras
from gaussianavatar_b200.posmap import BodyPoser, SmplxBodyPoser
from oracle import mesh_oracle as mo
from test_mesh_render_cpu import octahedron, sphere

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RGB_TOL = 1e-5
SIZES = [(64, 64), (1024, 1024), (540, 960)]


def _K(H, W, f=1100.0):
    s = min(H, W) / 1024.0
    return np.array([[f * s, 0, W / 2], [0, f * s, H / 2], [0, 0, 1]], np.float32)


def _cams(H, W, B, extr):
    return cameras([make_camera(_K(H, W), extr, H, W) for _ in range(B)])


def _known():
    """A sphere, an octahedron and two pairs of overlapping triangles (one pair at equal depth), in front of an identity camera."""
    Xs, Fs = sphere()
    Xo, Fo = octahedron()
    near = [[-0.3, -0.3, 2.0], [0.3, -0.3, 2.0], [0.0, 0.3, 2.0]]
    far = [[-0.3, -0.2, 2.5], [0.3, -0.2, 2.5], [0.0, 0.4, 2.5]]
    tri = np.array(far + near + near, np.float64) + [0.2, 0.1, 0.0]
    parts = [(Xs * 0.3 + [-0.25, 0.0, 3.0], Fs), (Xo * 0.25 + [0.3, -0.2, 2.8], Fo), (tri, np.arange(9).reshape(3, 3))]
    X, F, off = [], [], 0
    for x, f in parts:
        X.append(x); F.append(f + off); off += len(x)
    return np.concatenate(X).astype(np.float32), np.concatenate(F)


def _full_frame():
    """Faces that cover the whole frame: a wall of two triangles, tilted, and a large triangle in front of part of it."""
    X = np.array([[-50, -50, 4.0], [50, -50, 6.0], [50, 50, 6.0], [-50, 50, 4.0], [-40, -40, 3.0], [40, -30, 3.5], [0, 40, 3.2]], np.float32)
    return X, np.array([[0, 1, 2], [0, 2, 3], [4, 5, 6]])


def _mesh(name, B):
    """verts [B,V,3] (device), faces [F,3], extrinsic."""
    if name == "smpl":
        body, t = syn.make_body(0), syn.make_uv_template(0)
        poser = BodyPoser(syn.smpl_mesh_model(body, t), body.betas[0], device=DEV)
        pose, transl = syn.synthetic_poses(B, seed=5)
        return poser.vertices(pose, transl), t[1], TEST_POSE_EXTRINSIC
    if name == "smplx":
        body, t = syn.make_smplx_body(0), syn.make_smplx_uv_template(0)
        poser = SmplxBodyPoser(syn.smplx_mesh_model(body, t, syn.smplx_posedirs(0)), body.betas[0], device=DEV)
        pose, rest, transl = syn.synthetic_smplx_poses(B, seed=5)
        return poser.vertices(pose, rest, transl), t[1], TEST_POSE_EXTRINSIC
    X, F = _known() if name == "known" else _full_frame()
    shift = torch.tensor([[0.01 * b, -0.007 * b, 0.05 * b] for b in range(B)], dtype=torch.float32)
    return (torch.from_numpy(X)[None] + shift[:, None]).to(DEV), F, np.eye(4)


@pytest.fixture(scope="module")
def renders():
    """name -> size -> (verts, faces, cams, background, (rgb, face_id, depth) of all 8 frames in one call)."""
    out = {}
    for name in ("smpl", "smplx", "known", "full"):
        verts, F, extr = _mesh(name, 8)
        r = MeshRenderer(F, verts.shape[1], device=DEV)
        out[name] = {}
        for H, W in SIZES:
            cams = _cams(H, W, 8, extr)
            bg = torch.rand(8, 3, H, W, generator=torch.Generator().manual_seed(H)).to(DEV) if name == "known" else None
            out[name][(H, W)] = (r, verts, F, cams, bg, r.render(verts, cams, H, W, background=bg))
    return out


@pytest.mark.parametrize("name", ["smpl", "smplx", "known", "full"])
@pytest.mark.parametrize("size", SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_matches_the_oracle_bit_for_bit(renders, name, size):
    H, W = size
    r, verts, F, cams, bg, (rgb, fid, depth) = renders[name][size]
    off, adj = r.adj_offsets.cpu().numpy(), r.adj_faces.cpu().numpy()
    small, body = H * W <= 64 * 64, name in ("smpl", "smplx")
    frames = range(8) if small else (3,) if body else (0, 3, 7)
    # the synthetic bodies' faces join random points of the body (bounding boxes of ~2e4 pixels each at 1024^2): the oracle
    # restates every 16th row of their large frames
    o, k = (0, 1) if small or not body else (5, 16)
    rows = np.arange(o, H, k)
    X = verts.cpu().numpy()
    for b in frames:
        o_rgb, o_fid, o_depth = mo.render_frame(X[b], F, off, adj, cams[b].numpy(), H, W,
                                                None if bg is None else bg[b].cpu().numpy(), rows=(o, k))
        o_rgb, o_fid, o_depth = o_rgb[:, rows], o_fid[rows], o_depth[rows]
        g_fid, g_depth = fid[b].cpu().numpy()[rows], depth[b].cpu().numpy()[rows]
        assert np.array_equal(g_fid, o_fid), (b, int((g_fid != o_fid).sum()))
        assert np.array_equal(g_depth.view(np.uint32), o_depth.view(np.uint32)), b
        assert np.abs(rgb[b].cpu().numpy()[:, rows] - o_rgb).max() <= RGB_TOL, b
        drawn = o_fid >= 0
        assert drawn.mean() > (0.99 if name == "full" else 0.005), (b, drawn.mean())
    if body and small:                     # many overlapping faces: the depth test decides a good share of the drawn pixels
        s = mo.setup_faces(F, *mo.project(X[0], cams[0].numpy(), H, W), H, W)
        assert (mo.coverage(s, H, W) > 1).sum() > 0.2 * (fid[0] >= 0).sum().item()


@pytest.mark.parametrize("name", ["smpl", "smplx", "known", "full"])
@pytest.mark.parametrize("size", SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_a_frame_does_not_depend_on_its_batch(renders, name, size):
    H, W = size
    r, verts, F, cams, bg, full = renders[name][size]
    for sel in ([5], [3, 4], [7, 0]):
        part = r.render(verts[sel], cams[sel], H, W, background=None if bg is None else bg[sel])
        for a, b in zip(part, full):
            assert torch.equal(a, b[sel])
    again = r.render(verts, cams, H, W, background=bg)
    for a, b in zip(again, full):
        assert torch.equal(a, b)


def test_every_output_element_is_written():
    verts, F, extr = _mesh("known", 3)
    r = MeshRenderer(F, verts.shape[1], device=DEV)
    H, W = 37, 53
    cams = _cams(H, W, 3, extr).to(DEV)
    ref = r.render(verts, cams, H, W)
    L = _lib.lib()
    for fill in (float("nan"), 7.0):
        rgb = torch.full((3, 3, H, W), fill, device=DEV)
        depth = torch.full((3, H, W), fill, device=DEV)
        fid = torch.full((3, H, W), 0x7f7f7f7f, dtype=torch.int32, device=DEV)
        ws = torch.full((L.ga_mesh_render_workspace_bytes(3, r.V, r.F, H, W),), 0x5a, dtype=torch.uint8, device=DEV)
        _lib.check(L.ga_mesh_render(3, r.V, r.F, H, W, ptr(verts), ptr(r.faces), ptr(r.adj_offsets), ptr(r.adj_faces), ptr(cams),
                                    *r.color, None, ptr(ws), ptr(fid), ptr(depth), ptr(rgb), torch.cuda.current_stream().cuda_stream),
                   "ga_mesh_render")
        assert torch.equal(rgb, ref[0]) and torch.equal(fid, ref[1]) and torch.equal(depth, ref[2])
    assert (ref[1] >= 0).any() and (ref[1] == -1).any()


def test_rejects_bad_arguments():
    verts, F, extr = _mesh("known", 1)
    with pytest.raises(ValueError, match="outside"):
        MeshRenderer(np.array([[0, 1, verts.shape[1]]]), verts.shape[1], device=DEV)
    r = MeshRenderer(F, verts.shape[1], device=DEV)
    cams = _cams(16, 16, 1, extr)
    with pytest.raises(ValueError, match="vertices"):
        r.render(verts[:, :-1], cams, 16, 16)
    with pytest.raises(ValueError, match="cameras"):
        r.render(verts, cams[:, :32], 16, 16)
    with pytest.raises(ValueError, match="background"):
        r.render(verts, cams, 16, 16, background=torch.zeros(1, 3, 16, 15))
    with pytest.raises(RuntimeError, match="CUDA only"):
        MeshRenderer(F, verts.shape[1], device="cpu")
    L = _lib.lib()
    assert L.ga_mesh_render(9, r.V, r.F, 16, 16, *([None] * 5), 1.0, 1.0, 1.0, *([None] * 6)) != 0
    assert "batch" in L.ga_last_error().decode()


def _tool(name, *args):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", name), *map(str, args)], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout


def _folder(root):
    """The dataset fixture's folder with the full synthetic SMPL mesh model."""
    from dataset_fixture import write_synthetic_dataset
    mp = write_synthetic_dataset(root, seed=0)
    model = os.path.join(mp.smpl_model_path, "SMPL_NEUTRAL.pkl")
    with open(model, "wb") as f:
        pickle.dump(syn.smpl_mesh_model(syn.make_body(0), syn.make_uv_template(0)), f)
    return mp, os.path.join(mp.source_path, "train"), model


def _expected(folder, model, params):
    """face_id of each frame, drawn in-process, and the IoU the tool should print."""
    from gaussianavatar_b200.posmap import load_body_model
    prm = torch.load(os.path.join(folder, params), weights_only=False)
    poser = BodyPoser(load_body_model(model), torch.as_tensor(prm["beta"]).reshape(-1, 10)[0], device=DEV)
    names = sorted(os.listdir(os.path.join(folder, "images")))
    verts = poser.vertices(prm["body_pose"][:len(names)], prm["trans"][:len(names)])
    cam = np.load(os.path.join(folder, "cam_parms.npz"))
    H, W = np.array(Image.open(os.path.join(folder, "images", names[0]))).shape[:2]
    cams = cameras([make_camera(cam["intrinsic"], cam["extrinsic"], H, W)] * len(names))
    rgb, fid, _ = MeshRenderer(poser.faces, poser.V, device=DEV).render(verts, cams, H, W)
    ious = []
    for i, n in enumerate(names):
        m = np.array(Image.open(os.path.join(folder, "masks", n))) >= 128
        d = fid[i].cpu().numpy() >= 0
        ious.append((m & d).sum() / (m | d).sum())
    return names, rgb.cpu().numpy(), fid.cpu().numpy(), ious


def test_body_overlay_end_to_end(tmp_path):
    _, folder, model = _folder(str(tmp_path))
    out = tmp_path / "overlay"
    res = json.loads(_tool("body_overlay.py", folder, "--body", "smpl", "--smpl_model", model, "--params", "smpl_parms.pth",
                           "--out", out, "--iou").strip().splitlines()[-1])
    names, rgb, fid, ious = _expected(folder, model, "smpl_parms.pth")
    assert res["frames"] == len(names) and np.allclose(res["iou"], ious, rtol=0, atol=1e-12)
    assert abs(res["mean_iou"] - np.mean(ious)) < 1e-12
    assert any((f >= 0).any() for f in fid) and all((f < 0).any() for f in fid)
    for i, n in enumerate(names):
        got = np.array(Image.open(out / "pred_smpl_render" / n))
        src = np.array(Image.open(os.path.join(folder, "images", n)).convert("RGB"))
        drawn = fid[i] >= 0
        assert np.array_equal(got[~drawn], src[~drawn])
        want = np.floor(rgb[i].transpose(1, 2, 0) * 255.0 + 0.5).clip(0, 255).astype(np.uint8)
        assert np.array_equal(got[drawn], want[drawn])


def test_export_then_overlay_on_a_saved_checkpoint(tmp_path):
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams, OptimizationParams
    mp, folder, model = _folder(str(tmp_path))
    torch.manual_seed(0)
    m = AvatarModel(mp, NetworkParams(nf=8), OptimizationParams(), train=True)
    m.training_setup()
    with torch.no_grad():
        m.pose.weight[:, 3:] += 0.2 * torch.randn_like(m.pose.weight[:, 3:])
        m.transl.weight += 0.01
    m.save(7)
    ckpt = os.path.join(mp.model_path, "net", "iteration_7")
    _tool("export_stage1_poses.py", ckpt, folder)
    pred = torch.load(os.path.join(folder, "smpl_parms_pred.pth"), weights_only=False)
    F = m.pose.weight.shape[0]
    assert torch.equal(pred["body_pose"][:F], m.pose.weight.detach().cpu()) and torch.equal(pred["trans"][:F], m.transl.weight.detach().cpu())
    out = tmp_path / "overlay"
    res = json.loads(_tool("body_overlay.py", folder, "--smpl_model", model, "--out", out, "--iou").strip().splitlines()[-1])
    assert res["params"] == "smpl_parms_pred.pth"
    _, _, _, ious = _expected(folder, model, "smpl_parms_pred.pth")
    assert np.allclose(res["iou"], ious, rtol=0, atol=1e-12)
