"""CPU: the mesh-render oracle on known answers (coverage, depth order, closed meshes, the near plane, the flat-square shade) and
tools/export_stage1_poses.py on synthetic checkpoints."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gaussianavatar_b200.camera import make_camera
from gaussianavatar_b200.mesh_render import COLORS, vertex_face_csr
from oracle import mesh_oracle as mo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H = W = 64


def cam_block(K, extr=None, H=H, W=W):
    c = make_camera(K, np.eye(4) if extr is None else extr, H, W)
    cam = np.zeros(40, np.float32)
    cam[:16] = c.world_view_transform.numpy().reshape(-1)
    cam[16:32] = c.full_proj_transform.numpy().reshape(-1)
    return cam


K0 = np.array([[100.0, 0, 32.0], [0, 100.0, 32.0], [0, 0, 1]], np.float32)


def frame(X, faces, cam, H=H, W=W):
    faces = np.asarray(faces, np.int64)
    off, adj = vertex_face_csr(faces, len(X))
    return mo.render_frame(np.asarray(X, np.float32), faces, off, adj, cam, H, W)


def setup(X, faces, cam, H=H, W=W):
    x, y, z, ok = mo.project(np.asarray(X, np.float32), cam, H, W)
    return mo.setup_faces(np.asarray(faces, np.int64), x, y, z, ok, H, W)


def test_fma32_is_correctly_rounded():
    g = np.random.default_rng(0)
    a, b, c = (g.standard_normal(20000).astype(np.float32) for _ in range(3))
    got = mo.fma32(a, b, c)
    # exact reference: the fp64 sum of an exact product and c is exact here when it fits 53 bits; compare where it does
    from fractions import Fraction
    for i in range(0, 20000, 97):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo = np.float32(float(exact))
        cands = [lo, np.nextafter(lo, np.float32(-np.inf)), np.nextafter(lo, np.float32(np.inf))]
        best = min(cands, key=lambda v: (abs(Fraction(float(v)) - exact), int(np.float32(v).view(np.uint32)) & 1))
        assert got[i] == best, i
    # a a = 1 + 2^-11 + 2^-24 lies halfway between two float32 values; a tiny c decides which way the fused result rounds, where
    # rounding the fp64 sum to float32 would tie to even
    a, tiny = np.float32(1 + 2 ** -12), np.float32(2 ** -60)
    assert mo.fma32(a, a, np.float32(0)) == np.float32(1 + 2 ** -11)
    assert mo.fma32(a, a, tiny) == np.float32(1 + 2 ** -11 + 2 ** -23)
    assert mo.fma32(a, a, -tiny) == np.float32(1 + 2 ** -11)


def test_camera_facing_square_covers_exactly_the_centres_inside():
    z = 2.0
    x0, x1, y0, y1 = -0.3, 0.235, -0.2, 0.3          # pixel x 16.5 .. 43.25, y 21.5 .. 46.5: no centre on an edge
    X = [[x0, y0, z], [x1, y0, z], [x1, y1, z], [x0, y1, z]]
    _, fid, depth = frame(X, [[0, 1, 2], [0, 2, 3]], cam_block(K0))
    want = np.zeros((H, W), bool)
    want[22:47, 17:44] = True
    assert np.array_equal(fid >= 0, want)
    assert np.array_equal(mo.coverage(setup(X, [[0, 1, 2], [0, 2, 3]], cam_block(K0)), H, W), want.astype(np.int64))
    assert np.all(np.abs(depth[want] - z) < 1e-6) and np.all(depth[~want] == 0)


@pytest.mark.parametrize("order", [(0, 1), (1, 0)])
def test_overlapping_faces_resolve_by_depth_then_index(order):
    near = [[-0.5, -0.5, 2.0], [0.5, -0.5, 2.0], [0.0, 0.5, 2.0]]
    far = [[-0.5, -0.4, 3.0], [0.5, -0.4, 3.0], [0.0, 0.6, 3.0]]
    tris = [near, far]
    X = np.array(tris[order[0]] + tris[order[1]], np.float32)
    F = [[0, 1, 2], [3, 4, 5]]
    _, fid, depth = frame(X, F, cam_block(K0))
    near_idx = order.index(0)
    both = mo.coverage(setup(X, F, cam_block(K0)), H, W) == 2
    assert both.sum() > 100
    assert (fid[both] == near_idx).all() and (depth[both] == np.float32(2.0)).all()
    # equal depth: the lower index wins wherever both cover
    X2 = np.array(near + near, np.float32)
    _, fid2, _ = frame(X2, F, cam_block(K0))
    assert ((fid2 >= 0) == (fid2 == 0)).all() and (fid2 == 0).sum() > 100


def _rotation(seed):
    q, _ = np.linalg.qr(np.random.default_rng(seed).standard_normal((3, 3)))
    return q * np.sign(np.linalg.det(q))


def octahedron():
    X = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float64)
    F = [[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]]
    return X, np.array(F)


def sphere(levels=2):
    X, F = octahedron()
    X, F = list(map(tuple, X)), F.tolist()
    for _ in range(levels):
        mid, nf = {}, []

        def m(a, b):
            k = (min(a, b), max(a, b))
            if k not in mid:
                p = (np.array(X[a]) + np.array(X[b])) / 2
                X.append(tuple(p / np.linalg.norm(p)))
                mid[k] = len(X) - 1
            return mid[k]
        for a, b, c in F:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [[a, ab, ca], [ab, b, bc], [ca, bc, c], [ab, bc, ca]]
        F = nf
    return np.array(X), np.array(F)


@pytest.mark.parametrize("mesh", ["octahedron", "sphere"])
def test_closed_mesh_covers_each_interior_centre_once_per_side(mesh):
    X, F = octahedron() if mesh == "octahedron" else sphere()
    X = (X @ _rotation(3).T) * 0.5 + np.array([0.013, -0.021, 3.0])
    X = X.astype(np.float32)
    s = setup(X, F, cam_block(K0))
    total = mo.coverage(s, H, W)
    front = mo.coverage(s, H, W, s["front"])
    inside = total > 0
    assert inside.sum() > 200
    assert (total[inside] == 2).all() and (front[inside] == 1).all()
    _, fid, depth = frame(X, F, cam_block(K0))
    assert np.array_equal(fid >= 0, inside)
    assert s["front"][fid[inside]].all()                     # the nearer face of a convex mesh is the one facing the camera
    assert (depth[inside] >= 2.5 - 1e-6).all() and (depth[inside] <= 3.5).all()


def test_faces_behind_the_near_plane_or_off_screen_draw_nothing():
    tris = [
        [[-0.5, -0.5, 0.005], [0.5, -0.5, 2.0], [0.0, 0.5, 2.0]],       # one corner in front of znear = 0.01
        [[-0.5, -0.5, -2.0], [0.5, -0.5, -2.0], [0.0, 0.5, -2.0]],      # behind the camera
        [[5.0, 5.0, 2.0], [6.0, 5.0, 2.0], [5.5, 6.0, 2.0]],            # off-screen
        [[-1e5, -0.5, 2.0], [0.5, -0.5, 2.0], [0.0, 0.5, 2.0]],         # a corner beyond the 2^20-pixel guard band
    ]
    for t in tris:
        rgb, fid, depth = frame(np.array(t, np.float32), [[0, 1, 2]], cam_block(K0))
        assert (fid == -1).all() and (depth == 0).all() and (rgb == 0).all(), t


def test_flat_square_shade_is_the_closed_form_on_the_axis():
    K = np.array([[100.0, 0, 32.5], [0, 100.0, 32.5], [0, 0, 1]], np.float32)     # the optical axis through the centre of pixel (32, 32)
    X = [[-1, -1, 2.0], [1, -1, 2.0], [1, 1, 2.0], [-1, 1, 2.0]]
    rgb, fid, _ = frame(X, [[0, 1, 2], [0, 2, 3]], cam_block(K))
    assert fid[32, 32] >= 0
    m, r, I = 0.2, 0.6, 3.0
    a2 = (r * r) ** 2
    base = np.array(COLORS["white"])
    F0 = 0.04 * (1 - m) + base * m
    cdiff = base * 0.96 * (1 - m)
    # n = l = v: F = F0, V = 0.5 / (1 + 1), D = a2 / (pi a2^2)
    want = I * ((1 - F0) * cdiff / np.pi + F0 * 0.25 / (np.pi * a2))
    assert np.abs(rgb[:, 32, 32] - np.clip(want, 0, 1)).max() < 1e-5


def test_vertex_face_csr_lists_each_corner_in_face_order():
    F = np.array([[0, 1, 2], [2, 1, 3], [3, 1, 0]])
    off, adj = vertex_face_csr(F, 5)
    assert off.tolist() == [0, 2, 5, 7, 9, 9]
    assert adj.tolist() == [0, 2, 0, 1, 2, 0, 1, 1, 2]


def _export(ckpt, folder, body):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "export_stage1_poses.py"), ckpt, folder, "--body", body],
                       capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("body", ["smpl", "smplx"])
def test_export_replaces_the_refined_rows_only(tmp_path, body):
    g = torch.Generator().manual_seed(1)
    N, F = 7, 5
    width, full = (72, 72) if body == "smpl" else (66, 165)
    smpl = dict(beta=torch.randn(1, 10, generator=g), body_pose=torch.randn(N, full, generator=g), trans=torch.randn(N, 3, generator=g),
                extra=torch.arange(3))
    folder, ckpt = tmp_path / "data", tmp_path / "ckpt"
    folder.mkdir(); ckpt.mkdir()
    torch.save(smpl, folder / "smpl_parms.pth")
    pose, transl = torch.randn(F, width, generator=g), torch.randn(F, 3, generator=g)
    torch.save({"net": {}, "pose": {"weight": pose}, "transl": {"weight": transl}}, ckpt / "net.pth")
    res = _export(str(ckpt), str(folder), body)
    assert res["frames"] == F
    out = torch.load(folder / "smpl_parms_pred.pth", weights_only=False)
    assert torch.equal(out["body_pose"][:F, :width], pose) and torch.equal(out["trans"][:F], transl)
    assert torch.equal(out["body_pose"][F:], smpl["body_pose"][F:]) and torch.equal(out["trans"][F:], smpl["trans"][F:])
    assert torch.equal(out["body_pose"][:, width:], smpl["body_pose"][:, width:])       # SMPL-X: jaw, eyes and hands kept
    assert torch.equal(out["beta"], smpl["beta"]) and torch.equal(out["extra"], smpl["extra"])
    assert torch.equal(torch.load(folder / "smpl_parms.pth", weights_only=False)["body_pose"], smpl["body_pose"])
