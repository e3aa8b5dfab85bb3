"""CPU: reading 3DGS's point_cloud.ply and cameras.json, and the placement's camera mapping."""
import numpy as np
import pytest
import torch

from gaussianavatar_b200.scene import GaussianScene, Placement, load_scene_cameras, scene_cameras_path
from scene_fixture import activated, random_static, write_cameras_json, write_ply

Rotation = pytest.importorskip("scipy.spatial.transform").Rotation


@pytest.mark.parametrize("degree", [0, 1, 2, 3])
@pytest.mark.parametrize("shuffle", [None, 5])
def test_ply_reads_back_activated(tmp_path, degree, shuffle):
    raw = random_static(37, degree, seed=degree)
    path = tmp_path / "point_cloud.ply"
    write_ply(path, raw, shuffle_seed=shuffle, extra=True)
    sc = GaussianScene.load_ply(path)
    want = activated(raw)
    assert sc.sh_degree == degree and len(sc) == 37
    assert sc.shs.shape == (37, (degree + 1) ** 2, 3)
    for k in ("means3D", "scales", "rotations", "opacities", "shs"):
        got = getattr(sc, k)
        assert got.dtype == torch.float32 and got.is_contiguous(), k
        np.testing.assert_allclose(got.numpy(), want[k].numpy(), rtol=1e-6, atol=0, err_msg=k)
    # the layout, spelled out: shs[:, 0] is f_dc, shs[:, 1 + k, c] is f_rest_{c (M-1) + k}
    M = (degree + 1) ** 2
    np.testing.assert_array_equal(sc.shs[:, 0].numpy(), raw["f_dc"])
    flat = raw["f_rest"].reshape(37, -1)
    for c in range(3):
        for k in range(M - 1):
            np.testing.assert_array_equal(sc.shs[:, 1 + k, c].numpy(), flat[:, c * (M - 1) + k])
    np.testing.assert_allclose(sc.rotations.norm(dim=1).numpy(), 1.0, rtol=1e-6)
    assert (sc.opacities > 0).all() and (sc.opacities < 1).all()


@pytest.mark.parametrize("kind,kw,message", [
    ("ascii", dict(fmt="ascii"), "ascii"),
    ("big-endian", dict(fmt="binary_big_endian"), "binary_big_endian"),
    ("missing opacity", dict(drop="opacity"), "opacity"),
    ("missing rot_3", dict(drop="rot_3"), "rot_3"),
    ("f_rest count", dict(n_rest=12), "12 f_rest"),
])
def test_malformed_ply_rejected_with_its_message(tmp_path, kind, kw, message):
    path = tmp_path / "bad.ply"
    write_ply(path, random_static(8, 1, seed=1), **kw)
    with pytest.raises(ValueError, match=message):
        GaussianScene.load_ply(path)


def test_truncated_ply_rejected(tmp_path):
    path = tmp_path / "cut.ply"
    write_ply(path, random_static(8, 1, seed=2))
    data = path.read_bytes()
    path.write_bytes(data[:-10])
    with pytest.raises(ValueError, match="truncated"):
        GaussianScene.load_ply(path)


def test_placement_camera_scales_camera_coordinates():
    """A placed point's camera coordinates through Placement.extrinsic are s x the unplaced ones (fp64)."""
    g = np.random.default_rng(3)
    for trial in range(5):
        s = float(g.uniform(0.3, 3.0))
        R = Rotation.random(random_state=trial).as_matrix()
        t = g.normal(size=3) * 4
        place = Placement(s, R, t)
        E = np.eye(4)
        E[:3, :3] = Rotation.random(random_state=100 + trial).as_matrix()
        E[:3, 3] = g.normal(size=3)
        En = place.extrinsic(E)
        x = g.normal(size=(50, 3))
        xs = s * x @ R.T + t
        cam = x @ E[:3, :3].T + E[:3, 3]
        cam_n = xs @ En[:3, :3].T + En[:3, 3]
        np.testing.assert_allclose(cam_n, s * cam, rtol=0, atol=1e-12 * max(1.0, np.abs(cam_n).max()))
        np.testing.assert_allclose(En[:3, :3] @ En[:3, :3].T, np.eye(3), atol=1e-12)
    # from_axis_angle and the 3x4 form
    p = Placement.from_axis_angle(2.0, [0, 0, np.pi / 2], [1, 2, 3])
    np.testing.assert_allclose(p.matrix() @ np.array([1.0, 0, 0, 1]), [1, 4, 3], atol=1e-12)
    with pytest.raises(ValueError):
        Placement(-1.0)
    with pytest.raises(ValueError):
        Placement(1.0, np.diag([1.0, 1.0, -1.0]))


def test_placement_fold_matches_the_point_map():
    """fold: [s R | t] composed with every joint's 3x4 row gives the placed point of the joint's posed point."""
    g = torch.Generator().manual_seed(0)
    p = Placement.from_axis_angle(1.7, [0.3, -0.2, 0.9], [0.5, -1.0, 2.0])
    c2l = torch.randn(2, 24, 12, generator=g)
    out = p.fold(c2l)
    x = torch.randn(5, 3, generator=g)
    A = c2l.double().reshape(2, 24, 3, 4)
    posed = torch.einsum("bjrc,nc->bjnr", A[..., :3], x.double()) + A[..., 3][:, :, None]
    M = torch.from_numpy(p.matrix())
    want = posed @ M[:, :3].T + M[:, 3]
    B = out.double().reshape(2, 24, 3, 4)
    got = torch.einsum("bjrc,nc->bjnr", B[..., :3], x.double()) + B[..., 3][:, :, None]
    assert (got - want).abs().max() < 1e-5


def test_cameras_json(tmp_path):
    """Each camera's centre maps to the origin of its camera coordinates, and a point on its optical axis lands at the image
    centre; the file is found next to point_cloud/iteration_*/."""
    from gaussianavatar_b200.camera import make_camera
    g = np.random.default_rng(4)
    cams = []
    for i in range(3):
        E = np.eye(4)
        E[:3, :3] = Rotation.random(random_state=i).as_matrix()
        E[:3, 3] = g.normal(size=3)
        w, h = 160 + 16 * i, 90 + 8 * i
        cams.append((np.array([[200.0 + i, 0, w / 2], [0, 190.0, h / 2], [0, 0, 1]]), E, w, h))
    model = tmp_path / "room"
    (model / "point_cloud" / "iteration_7000").mkdir(parents=True)
    write_cameras_json(model / "cameras.json", cams)
    ply = model / "point_cloud" / "iteration_7000" / "point_cloud.ply"
    assert scene_cameras_path(ply) == str(model / "cameras.json")
    got = load_scene_cameras(scene_cameras_path(ply))
    assert len(got) == 3
    for sc, (K, E, w, h) in zip(got, cams):
        assert (sc.width, sc.height) == (w, h)
        C = -E[:3, :3].T @ E[:3, 3]
        np.testing.assert_allclose(sc.E[:3, :3] @ C + sc.E[:3, 3], 0, atol=1e-12)
        np.testing.assert_allclose(sc.E, E, atol=1e-12)
        np.testing.assert_allclose(sc.K, K, atol=1e-12)
        axis = C + 3.0 * E[2, :3]                              # 3 units along the optical axis (camera +z)
        cam = make_camera(sc.K, sc.E, h, w)
        clip = torch.cat([torch.from_numpy(axis).float(), torch.ones(1)]) @ cam.full_proj_transform
        ndc = clip[:2] / clip[3]
        pix = ((ndc.double() + 1) * torch.tensor([w, h]) - 1) * 0.5                # the rasterizer's ndc -> pixel map
        np.testing.assert_allclose(pix.numpy(), [(w - 1) / 2, (h - 1) / 2], atol=1e-3)
        c = sc.camera()
        np.testing.assert_allclose(c.camera_center.numpy(), C, atol=1e-5)
    with pytest.raises(ValueError, match="fx"):
        bad = tmp_path / "bad.json"
        bad.write_text('[{"width": 4, "height": 4, "position": [0, 0, 0], "rotation": [[1, 0, 0], [0, 1, 0], [0, 0, 1]], "fy": 1}]')
        load_scene_cameras(bad)
