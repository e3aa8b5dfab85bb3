"""GPU: the soft silhouette (ga_silhouette_forward / ga_silhouette_backward, SilhouetteRenderer) against the fp64 oracle, its output
contract, the pose refiner on the synthetic SMPL and SMPL-X bodies, and tools/refine_poses.py end to end."""
import json
import os
import pickle
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch
from PIL import Image

from gaussianavatar_b200 import _lib
from gaussianavatar_b200 import synthetic as syn
from gaussianavatar_b200._lib import ptr
from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, TEST_POSE_K, make_camera, scaled_intrinsics
from gaussianavatar_b200.mesh_render import MeshRenderer, cameras
from gaussianavatar_b200.posmap import BodyPoser, SmplxBodyPoser
from gaussianavatar_b200.silhouette import PoseRefiner, SilhouetteRenderer
from oracle import silhouette_oracle as so

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIGMA = 1.0
# S tolerance.  The kernel projects in fp32: a corner lands within ~1e-4 pixel of the fp64 position at 1080 pixels (a few ulp of
# coordinates up to 2^11), and dS/d(corner) <= 2 d D (1 - D) / sigma <= ~0.7 per pixel per face within the truncation radius, so
# a face moves S by ~1e-4; a pixel sees a handful of faces.  2e-3 leaves room for that and for the fp32 sums; a corruption of
# 5e-3 must fail it.
SIL_TOL = 2e-3
# marginal pixels: an outside distance^2 within 2 d |delta d| (d <= 3.04, |delta d| <= 1e-3) of the truncation radius^2
TOL_D2 = 6e-3
GRAD_REL_L2 = 1e-2          # d_verts per frame, relative L2 against fp64 autograd
GRAD_ELEM = 2e-2            # element-wise, relative to the frame's largest gradient, on vertices away from marginal pixels


def _K(H, W, f=1100.0):
    s = min(H, W) / 1024.0
    return np.array([[f * s, 0, W / 2], [0, f * s, H / 2], [0, 0, 1]], np.float32)


def _body(name, B, seed=5):
    """(poser, pose [B,72|165], transl [B,3])."""
    if name == "smpl":
        body, t = syn.make_body(0), syn.make_uv_template(0)
        poser = BodyPoser(syn.smpl_mesh_model(body, t), body.betas[0], device=DEV)
        pose, transl = syn.synthetic_poses(B, seed=seed)
        return poser, pose, transl
    body, t = syn.make_smplx_body(0), syn.make_smplx_uv_template(0)
    poser = SmplxBodyPoser(syn.smplx_mesh_model(body, t, syn.smplx_posedirs(0)), body.betas[0], device=DEV)
    pose, rest, transl = syn.synthetic_smplx_poses(B, seed=seed)
    return poser, torch.cat([pose, rest], 1), transl


def _verts(poser, pose, transl):
    if isinstance(poser, SmplxBodyPoser):
        return poser.vertices(pose[:, :66], pose[:, 66:], transl)
    return poser.vertices(pose, transl)


def _mesh(name, B, H, W):
    """verts [B,V,3], faces [F,3] int64, cams [B,40]."""
    if name in ("smpl", "smplx"):
        poser, pose, transl = _body(name, B)
        cams = cameras([make_camera(_K(H, W), TEST_POSE_EXTRINSIC, H, W) for _ in range(B)])
        return _verts(poser, pose, transl), poser.faces.long().cpu().numpy(), cams.to(DEV)
    if name == "full":        # a wall covering the frame, tilted, and a triangle in front
        X = np.array([[-50, -50, 4.0], [50, -50, 6.0], [50, 50, 6.0], [-50, 50, 4.0], [-0.02, -0.02, 3.0], [0.02, -0.015, 3.5],
                      [0.0, 0.02, 3.2]], np.float32)
        F = np.array([[0, 1, 2], [0, 2, 3], [4, 5, 6]])
    else:                     # small triangles at pixel scale, a coincident pair, one crossing the near plane, a degenerate one
        g = np.random.default_rng(3)
        X = np.concatenate([g.uniform([-0.1, -0.1, 1.5], [0.1, 0.1, 2.5], (30, 3)), [[0, 0, 0.005], [0.01, 0.01, 2.0]]]).astype(np.float32)
        F = np.concatenate([g.integers(0, 30, (20, 3)), [[0, 1, 2], [0, 1, 2], [3, 4, 30], [5, 5, 6], [31, 31, 31]]])
    shift = torch.tensor([[0.004 * b, -0.003 * b, 0.02 * b] for b in range(B)], dtype=torch.float32)
    verts = (torch.from_numpy(X)[None] + shift[:, None]).to(DEV)
    cams = cameras([make_camera(_K(H, W, 300.0), np.eye(4), H, W) for _ in range(B)]).to(DEV)
    return verts, F, cams


def _masks(B, H, W, seed=0):
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    m = np.stack([(((yy - H * 0.5) ** 2 + (xx - W * (0.45 + 0.02 * b)) ** 2) < (0.3 * min(H, W)) ** 2) * 255 for b in range(B)])
    m[:, ::7, ::5] = g.integers(100, 160, m[:, ::7, ::5].shape)       # bytes around the 128 threshold
    return torch.from_numpy(m.astype(np.uint8)).to(DEV)


def _check_sil(got, want, marg):
    """max |got - want| over non-marginal pixels, asserting the marginal share is small."""
    assert float(marg.float().mean()) < 0.05, float(marg.float().mean())        # SMPL-X: ~3 % of the sampled rows
    err = (got.double() - want).abs()[~marg]
    return float(err.max()) if err.numel() else 0.0


CASES = [("known", 1, 1, [1]), ("known", 37, 53, [1, 2]), ("full", 64, 80, [1, 2]), ("smpl", 540, 540, [1, 2, 8]),
         ("smpl", 1080, 1080, [2]), ("smplx", 540, 540, [2])]


@pytest.mark.parametrize("name,H,W,Bs", CASES)
def test_forward_matches_fp64_oracle(name, H, W, Bs):
    for B in Bs:
        verts, F, cams = _mesh(name, B, H, W)
        masks = _masks(B, H, W)
        r = SilhouetteRenderer(F, verts.shape[1], sigma=SIGMA, device=DEV)
        sil = r.render(verts, cams, H, W)
        loss = r.losses(verts, cams, masks)
        rows = None if H * W * len(F) <= 3e8 else np.linspace(0, H - 1, 12).round().astype(int)
        want, marg = so.silhouette(verts.double(), F, cams.double(), H, W, SIGMA, rows=rows, tol_d2=TOL_D2)
        got = sil if rows is None else sil[:, torch.as_tensor(rows, device=DEV)]
        assert _check_sil(got, want, marg) <= SIL_TOL, (name, H, W, B)
        bad = got.clone()
        i = int(torch.nonzero(~marg.reshape(-1))[0])
        bad.view(-1)[i] += 5e-3
        assert _check_sil(bad, want, marg) > SIL_TOL                         # the bound rejects a corrupted value
        if rows is not None:
            assert float((want > 0.5).double().mean()) > 0.001 or name == "known"
        M = (masks >= 128).double()
        ref = ((sil.double() - M) ** 2).mean((1, 2))
        assert torch.allclose(loss.double(), ref, rtol=1e-5, atol=1e-7), (loss, ref)
        if rows is None:
            assert torch.allclose(loss.double(), so.loss_and_grad(verts, F, cams, masks, H, W, SIGMA)[0], rtol=0, atol=SIL_TOL ** 2 + 2 * SIL_TOL)


@pytest.mark.parametrize("name,H,W", [("known", 37, 53), ("full", 32, 40), ("smpl", 96, 128), ("smplx", 96, 128)])
def test_backward_matches_fp64_autograd(name, H, W):
    B = 2
    verts, F, cams = _mesh(name, B, H, W)
    masks = _masks(B, H, W)
    r = SilhouetteRenderer(F, verts.shape[1], sigma=SIGMA, device=DEV)
    w = torch.tensor([1.0, 0.5], device=DEV)
    got = r.verts_grad(verts, cams, masks, w).double()
    _, want = so.loss_and_grad(verts, F, cams, masks, H, W, SIGMA, w=w)
    c, ok = so.face_corners(verts.double(), F, cams.double(), H, W)
    for b in range(B):
        n = float(want[b].norm())
        assert n > 0
        assert float((got[b] - want[b]).norm()) <= GRAD_REL_L2 * n, (name, b, float((got[b] - want[b]).norm()) / n)
        # vertices none of whose faces has a pixel at an outside distance^2 within TOL_D2 of its truncation radius^2
        p = torch.stack(torch.meshgrid(torch.arange(W, device=DEV), torch.arange(H, device=DEV), indexing="xy"), -1).reshape(-1, 2).double()
        fm = torch.zeros(len(F), dtype=torch.bool, device=DEV)
        for s0 in range(0, len(F), 512):
            d2, inside = so.signed_d2(c[b, s0:s0 + 512], p)
            fm[s0:s0 + 512] = (~inside & ((d2 - SIGMA * so.LN_INV_EPS).abs() <= TOL_D2)).any(0) & ok[b, s0:s0 + 512]
        clean = torch.ones(verts.shape[1], dtype=torch.bool, device=DEV)
        clean[torch.as_tensor(F, device=DEV)[fm].reshape(-1)] = False
        assert int(clean.sum()) > 0.4 * verts.shape[1]                    # SMPL-X at 96 x 128: 49 % (small hand and face faces)
        scale = float(want[b].abs().max())
        assert float((got[b] - want[b])[clean].abs().max()) <= GRAD_ELEM * scale
    # the loss's autograd Function gives the same gradient
    v = verts.clone().requires_grad_(True)
    (r.loss(v, cams, masks) * w).sum().backward()
    assert torch.equal(v.grad.double(), got)


def test_contract_sentinels_determinism_batch_and_bad_arguments():
    H, W = 45, 70
    verts, F, cams = _mesh("smpl", 8, H, W)
    masks = _masks(8, H, W)
    r = SilhouetteRenderer(F, verts.shape[1], device=DEV)
    L = _lib.lib()
    ws = torch.empty(L.ga_silhouette_workspace_bytes(8, r.V, r.F, H, W), dtype=torch.uint8, device=DEV)
    w = torch.ones(8, device=DEV)
    s = torch.cuda.current_stream().cuda_stream

    def run(b0, b1):
        sil = torch.full((b1 - b0, H, W), float("nan"), device=DEV)
        loss = torch.full((b1 - b0,), float("nan"), device=DEV)
        d = torch.full((b1 - b0, r.V, 3), float("nan"), device=DEV)
        ws.fill_(0xAB)
        _lib.check(L.ga_silhouette_forward(b1 - b0, r.V, r.F, H, W, 1.0, ptr(verts[b0:b1]), ptr(r.faces), ptr(cams[b0:b1]), ptr(masks[b0:b1]),
                                           ptr(ws), ptr(sil), ptr(loss), s))
        _lib.check(L.ga_silhouette_backward(b1 - b0, r.V, r.F, H, W, 1.0, ptr(verts[b0:b1]), ptr(r.faces), ptr(r.adj_offsets), ptr(r.adj_faces),
                                            ptr(cams[b0:b1]), ptr(masks[b0:b1]), ptr(w[b0:b1]), ptr(ws), ptr(d), s))
        return sil, loss, d

    a, b = run(0, 8), run(0, 8)
    for x, y in zip(a, b):
        assert torch.isfinite(x).all() and torch.equal(x, y)
    for b0, b1 in ((3, 4), (2, 7)):
        for x, y in zip(run(b0, b1), a):
            assert torch.equal(x, y[b0:b1])
    assert float(a[2].abs().max()) > 0
    nul = [None] * 9
    assert L.ga_silhouette_forward(9, r.V, r.F, H, W, 1.0, ptr(verts), ptr(r.faces), ptr(cams), None, ptr(ws), ptr(a[0]), None, s) != 0
    assert "batch" in L.ga_last_error().decode()
    assert L.ga_silhouette_forward(1, r.V, r.F, 0, W, 1.0, ptr(verts), ptr(r.faces), ptr(cams), None, ptr(ws), ptr(a[0]), None, s) != 0
    assert L.ga_silhouette_forward(1, r.V, r.F, H, W, 0.0, ptr(verts), ptr(r.faces), ptr(cams), None, ptr(ws), ptr(a[0]), None, s) != 0
    assert L.ga_silhouette_forward(1, r.V, r.F, H, W, 1.0, *nul[:7], s) != 0
    assert L.ga_silhouette_backward(1, r.V, r.F, H, W, 1.0, ptr(verts), ptr(r.faces), ptr(r.adj_offsets), ptr(r.adj_faces), ptr(cams), None,
                                    ptr(w), ptr(ws), ptr(a[2]), s) != 0
    with pytest.raises(ValueError):
        r.render(verts, cams, 0, W)
    with pytest.raises(ValueError):
        SilhouetteRenderer(F, verts.shape[1], sigma=0.0, device=DEV)
    with pytest.raises(RuntimeError, match="CUDA only"):
        SilhouetteRenderer(F, verts.shape[1], device="cpu")


def _hard_masks(poser, pose, transl, cam, H, W):
    mr = MeshRenderer(poser.faces, poser.V, device=DEV)
    verts = _verts(poser, pose, transl)
    out = []
    for s in range(0, verts.shape[0], 8):
        _, fid, _ = mr.render(verts[s:s + 8], cam[None].expand(min(8, verts.shape[0] - s), -1).contiguous(), H, W)
        out.append((fid >= 0).to(torch.uint8) * 255)
    return torch.cat(out)


# The refinement starts from poses displaced from the ones the masks were drawn at; its mean hard IoU must rise from below
# IOU_BEFORE_MAX to above IOU_AFTER_MIN.
IOU_BEFORE_MAX, IOU_AFTER_MIN = 0.85, 0.85


@pytest.mark.parametrize("name", ["smpl", "smplx"])
def test_refiner_recovers_displaced_poses(name):
    H = W = 256
    n = 10
    poser, pose, transl = _body(name, n, seed=11)
    cam = cameras([make_camera(_K(H, W), TEST_POSE_EXTRINSIC, H, W)])[0].to(DEV)
    masks = _hard_masks(poser, pose, transl, cam, H, W)
    g = torch.Generator().manual_seed(1)
    width = 66 if name == "smplx" else 72
    p0 = pose.clone()
    p0[:, :width] += 0.08 * torch.randn(n, width, generator=g)
    t0 = transl + 0.04 * torch.randn(n, 3, generator=g)
    r = SilhouetteRenderer(poser.faces, poser.V, sigma=SIGMA, device=DEV)
    ref = PoseRefiner(poser, r, iters=60, lr=1e-2, lambda_smooth=0.0, lambda_prior=1e-3)
    out_pose, out_t, rep = ref.refine(p0, t0, cam, masks)
    print(name, json.dumps({k: rep[k] for k in ("objective_before", "objective_after", "mean_iou_before", "mean_iou_after")}))
    assert rep["objective_after"] < rep["objective_before"]
    assert rep["mean_iou_before"] < IOU_BEFORE_MAX and rep["mean_iou_after"] > IOU_AFTER_MIN
    assert rep["mean_iou_after"] > rep["mean_iou_before"]
    assert out_pose.shape == p0.shape and out_t.shape == t0.shape
    if name == "smplx":
        assert torch.equal(out_pose[:, 66:], p0[:, 66:])


def test_tool_end_to_end(tmp_path):
    from dataset_fixture import write_synthetic_dataset
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams, OptimizationParams
    mp = write_synthetic_dataset(str(tmp_path / "ds"), seed=0)
    model = os.path.join(mp.smpl_model_path, "SMPL_NEUTRAL.pkl")
    body = syn.make_body(0)
    with open(model, "wb") as f:
        pickle.dump(syn.smpl_mesh_model(body, syn.make_uv_template(0)), f)
    # the capture: masks drawn at known poses, raw poses displaced from them
    H = W = 128
    n = 10
    poser, pose, transl = _body("smpl", n, seed=11)
    K = scaled_intrinsics(TEST_POSE_K, W)
    cam = cameras([make_camera(K, TEST_POSE_EXTRINSIC, H, W)])[0].to(DEV)
    masks = _hard_masks(poser, pose, transl, cam, H, W).cpu().numpy()
    cap = tmp_path / "capture"
    for sub in ("images", "masks"):
        os.makedirs(cap / sub)
    g = np.random.default_rng(0)
    for i in range(n):
        Image.fromarray(g.integers(0, 256, (H, W, 3), dtype=np.uint8)).save(cap / "images" / f"image_{i:04d}.png")
        Image.fromarray(masks[i]).save(cap / "masks" / f"image_{i:04d}.png")
    np.savez(cap / "cameras.npz", intrinsic=K, extrinsic=TEST_POSE_EXTRINSIC)
    gt = torch.Generator().manual_seed(2)
    raw = pose + 0.08 * torch.randn(n, 72, generator=gt)
    np.savez(cap / "poses.npz", betas=body.betas[0].numpy().reshape(1, 10).astype(np.float32), global_orient=raw[:, :3].numpy(),
             body_pose=raw[:, 3:].numpy(), transl=(transl + 0.03 * torch.randn(n, 3, generator=gt)).numpy())

    def tool(*args):
        r = subprocess.run([sys.executable, *map(str, args)], capture_output=True, text=True, cwd=ROOT)
        assert r.returncode == 0, r.stdout + r.stderr
        return json.loads(r.stdout.strip().splitlines()[-1])

    out0, out = tmp_path / "data0", tmp_path / "data"
    tool(os.path.join(ROOT, "tools", "refine_poses.py"), cap, "--out", out0, "--iters", "0")
    res = tool(os.path.join(ROOT, "tools", "refine_poses.py"), cap, "--smpl_model", model, "--out", out, "--iters", "60")
    assert res["mean_iou_after"] > res["mean_iou_before"] and res["objective_after"] < res["objective_before"]
    assert set(np.load(cap / "poses_optimized.npz").files) == {"betas", "global_orient", "body_pose", "transl"}
    ious = [tool(os.path.join(ROOT, "tools", "body_overlay.py"), d / "train", "--smpl_model", model, "--params", "smpl_parms.pth",
                 "--out", tmp_path / f"ov_{d.name}", "--iou")["mean_iou"] for d in (out0, out)]
    print("overlay mean IoU --iters 0 / 60:", ious)
    assert ious[1] > ious[0]
    # AvatarModel builds from the folder the tool wrote (with the fixture's per-subject assets beside it)
    train = os.path.join(mp.source_path, "train")
    for x in ("images", "masks"):
        shutil.rmtree(os.path.join(train, x))
        shutil.copytree(out / "train" / x, os.path.join(train, x))
    for x in ("smpl_parms.pth", "cam_parms.npz"):
        shutil.copy(out / "train" / x, os.path.join(train, x))
    os.remove(os.path.join(train, "smpl_parms_pred.pth"))
    m = AvatarModel(mp, NetworkParams(nf=8), OptimizationParams(), train=True)
    assert m.pose.weight.shape[0] == len(os.listdir(out / "train" / "images")) == res["train"]
