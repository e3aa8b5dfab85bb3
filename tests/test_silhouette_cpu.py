"""CPU: the fp64 soft-silhouette oracle (oracle/silhouette_oracle.py) against central differences and known answers, and
tools/refine_poses.py's capture-to-folder conversion (--iters 0) against tests/golden/romp_split.npz, which pins the split and the
parameter format by the reference's own code."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from PIL import Image

from gaussianavatar_b200.camera import make_camera
from gaussianavatar_b200.mesh_render import cameras
from oracle import silhouette_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "romp_split.npz")


def _S(corners, p, sigma=1.0):
    c = torch.tensor(corners, dtype=torch.float64).reshape(-1, 3, 2)
    ok = torch.ones(c.shape[0], dtype=torch.bool)
    return -torch.expm1(so.log_one_minus(c, ok, torch.tensor(p, dtype=torch.float64).reshape(-1, 2), sigma))


def _sig(x):
    return 1.0 / (1.0 + math.exp(-x))


TRI = [[0.0, 0.0], [10.0, 0.0], [0.0, 10.0]]


def test_outside_an_edge():
    for d in (0.0, 0.3, 1.0, 2.0):            # d^2 / sigma <= 8, inside the truncation radius
        for sigma in (0.5, 1.0, 2.0):
            got = float(_S(TRI, [4.0, -d], sigma)[0])
            assert abs(got - _sig(-d * d / sigma)) < 1e-15, (d, sigma)
    # nearest feature a vertex: distance to the corner
    got = float(_S(TRI, [-1.0, -1.0])[0])
    assert abs(got - _sig(-2.0)) < 1e-15


def test_truncation_boundary():
    sigma = 1.5
    r = math.sqrt(sigma * so.LN_INV_EPS)
    inside = float(_S(TRI, [4.0, -(r - 1e-9)], sigma)[0])
    assert abs(inside - 1e-4) < 1e-11
    assert float(_S(TRI, [4.0, -(r + 1e-9)], sigma)[0]) == 0.0


def test_deep_inside_and_coincident_and_winding():
    big = [[-1000.0, -1000.0], [3000.0, -1000.0], [-1000.0, 3000.0]]
    assert abs(float(_S(big, [5.0, 5.0])[0]) - 1.0) < 1e-15
    # two coincident triangles: 1 - (1 - D)^2
    for p in ([4.0, -0.7], [2.0, 2.0], [4.0, 0.5]):
        one = float(_S(TRI, p)[0])
        two = float(_S(TRI + TRI, p)[0])
        assert abs(two - (1 - (1 - one) ** 2)) < 1e-15
        # winding does not matter
        assert float(_S([TRI[0], TRI[2], TRI[1]], p)[0]) == one
    assert abs(float(_S(TRI, [2.0, 2.0])[0]) - _sig(4.0)) < 1e-15    # inside, 2 from the nearest edges: sigmoid(+4)


def _camera(H, W):
    K = np.array([[2.0 * W, 0, W / 2], [0, 2.0 * W, H / 2], [0, 0, 1]], np.float32)
    return cameras([make_camera(K, np.eye(4), H, W)])


def test_near_plane_faces_are_ignored():
    H = W = 16
    cams = _camera(H, W).double()
    X = torch.tensor([[[-0.5, -0.5, 2.0], [0.5, -0.5, 2.0], [0.0, 0.5, 2.0], [0.0, 0.0, 0.005]]], dtype=torch.float64)
    c, ok = so.face_corners(X, np.array([[0, 1, 2], [0, 1, 3]]), cams, H, W)
    assert ok[0].tolist() == [True, False]
    S = so.silhouette(X, np.array([[0, 1, 2], [0, 1, 3]]), cams, H, W, 1.0)
    S1 = so.silhouette(X, np.array([[0, 1, 2]]), cams, H, W, 1.0)
    assert torch.equal(S, S1) and S.max() > 0.99


def test_oracle_gradient_matches_central_differences():
    H, W, sigma = 20, 24, 2.0
    cams = _camera(H, W).double()
    X = torch.tensor([[[-0.08, -0.07, 2.0], [0.09, -0.05, 2.1], [0.0, 0.1, 1.9], [0.11, 0.09, 2.05]]], dtype=torch.float64)
    faces = np.array([[0, 1, 2], [1, 3, 2]])
    masks = np.zeros((1, H, W), np.uint8)
    masks[0, 6:15, 7:16] = 255
    tol_d2 = 1e-3                                    # a step of h moves a corner by about 2.4e-5 pixel
    _, marg = so.silhouette(X, faces, cams, H, W, sigma, tol_d2=tol_d2)
    assert int(marg.sum()) == 0                      # no pixel near the truncation radius, where the function jumps by 1e-4
    loss, g = so.loss_and_grad(X, faces, cams, masks, H, W, sigma)
    h = 1e-6
    for v in range(4):
        for k in range(3):
            Xp, Xm = X.clone(), X.clone()
            Xp[0, v, k] += h
            Xm[0, v, k] -= h
            fd = (so.loss_and_grad(Xp, faces, cams, masks, H, W, sigma)[0] - so.loss_and_grad(Xm, faces, cams, masks, H, W, sigma)[0]) / (2 * h)
            assert abs(float(fd[0]) - float(g[0, v, k])) <= 1e-6 * max(1.0, abs(float(fd[0]))), (v, k, float(fd[0]), float(g[0, v, k]))
    assert float(g.abs().max()) > 1e-3


def _write_capture(root, z, case):
    names = list(z[f"{case}/names"])
    for sub in ("images", "masks"):
        os.makedirs(os.path.join(root, sub), exist_ok=True)
    for i, n in enumerate(names):
        Image.fromarray(np.full((4, 5, 3), i % 256, np.uint8)).save(os.path.join(root, "images", n))
        Image.fromarray(np.full((4, 5), 255 * (i % 2), np.uint8)).save(os.path.join(root, "masks", n))
    np.savez(os.path.join(root, "cameras.npz"), intrinsic=np.eye(3, dtype=np.float32), extrinsic=np.eye(4, dtype=np.float32))
    poses = {k.split("/")[-1]: z[k] for k in z.files if k.startswith(f"{case}/poses/")}
    np.savez(os.path.join(root, "poses.npz"), **poses)
    return poses


@pytest.mark.parametrize("case", ["n7_split", "n10_thetas", "n23_split", "n23_thetas", "n100_thetas"])
def test_tool_conversion_matches_the_reference(tmp_path, case):
    z = np.load(GOLDEN)
    cap, out = tmp_path / "capture", tmp_path / "data"
    poses = _write_capture(str(cap), z, case)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "refine_poses.py"), str(cap), "--out", str(out), "--iters", "0"],
                       capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    with np.load(cap / "poses_optimized.npz") as opt:
        assert sorted(opt.files) == sorted(poses)
        for k, v in poses.items():
            assert opt[k].dtype == v.dtype and np.array_equal(opt[k], v)
    for part in ("train", "test"):
        d = out / part
        assert sorted(os.listdir(d / "images")) == list(z[f"{case}/{part}_names"])
        assert sorted(os.listdir(d / "masks")) == list(z[f"{case}/{part}_names"])
        prm = torch.load(d / "smpl_parms.pth", weights_only=False)
        for k in ("beta", "body_pose", "trans"):
            want = z[f"{case}/{part}/{k}"]
            assert prm[k].dtype == torch.float32 and tuple(prm[k].shape) == want.shape and np.array_equal(prm[k].numpy(), want), (part, k)
        cam = np.load(d / "cam_parms.npz")
        assert np.array_equal(cam["intrinsic"], np.eye(3)) and np.array_equal(cam["extrinsic"], np.eye(4))
