"""CPU: the position-map oracle against the reference's own LBS and OBJ parser (fixtures), its coverage rules on known answers, the
UV template parser, and the stage-2 plumbing of ModelParams.inp_posmap_from_pose that runs before any device work."""
import os
import pickle

import numpy as np
import pytest
import torch

from gaussianavatar_b200 import synthetic as syn
from gaussianavatar_b200.posmap import load_uv_template_obj
from oracle import posmap_oracle as po

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_oracle_vertices_match_reference_lbs_fixture():
    g = np.load(os.path.join(GOLDEN, "posmap_vertices.npz"))
    body = syn.make_body(int(g["body_seed"]))
    model = syn.smpl_mesh_model(body, syn.make_uv_template(0))
    v = po.smpl_vertices(model, g["betas"], g["pose"], g["transl"])
    assert np.abs(v[:, g["keep"]] - g["verts"]).max() < 1e-5
    assert np.abs(v.mean(1) - g["mean"]).max() < 1e-5
    assert np.abs((v ** 2).mean(1) - g["mean_sq"]).max() < 1e-5
    assert np.abs(g["pose"][0]).max() == 0.0          # the T-pose is one of the cases


def test_obj_parser_matches_reference_parser_fixture():
    g = np.load(os.path.join(GOLDEN, "posmap_obj_parser.npz"))
    verts, faces, uvs, faces_uv = load_uv_template_obj(os.path.join(GOLDEN, "posmap_obj_parser.obj"))
    for got, key in ((verts, "verts"), (faces, "faces"), (uvs, "uvs"), (faces_uv, "faces_uv")):
        assert got.shape == g[key].shape, key
        assert np.array_equal(got, g[key]), key
    assert not np.array_equal(faces, faces_uv)        # the case has a seam


def test_obj_parser_rejects_faces_without_texture(tmp_path):
    p = tmp_path / "t.obj"
    p.write_text("v 0 0 0\nv 1 0 0\nv 0 1 0\nvt 0 0\nf 1 2 3\n")
    with pytest.raises(ValueError, match="texture coordinate"):
        load_uv_template_obj(str(p))


def test_synthetic_template_round_trips_through_obj(tmp_path):
    t = syn.make_uv_template(0)
    syn.write_uv_template_obj(str(tmp_path / "t.obj"), t)
    back = load_uv_template_obj(str(tmp_path / "t.obj"))
    assert np.array_equal(back[1], t[1]) and np.array_equal(back[3], t[3]) and np.array_equal(back[2], t[2])
    assert t[1].shape == (13416, 3) and t[1].max() == syn.NUM_VERTS - 1
    assert not np.array_equal(t[1], t[3])


def _square_triangulation(n, seed, jitter):
    """A watertight triangulation of the unit square on an (n+1)^2 grid (boundary points on the boundary, random diagonals), with a
    seam: the middle column of points is duplicated, faces left of it use one copy and faces right of it the other."""
    g = np.random.default_rng(seed)
    x = np.linspace(0, 1, n + 1)
    P = np.stack(np.meshgrid(x, x, indexing="xy"), -1)
    P[1:-1, 1:-1] += g.uniform(-jitter, jitter, (n - 1, n - 1, 2)) / n
    pts = np.concatenate([P.reshape(-1, 2), P[:, n // 2]])                 # copies of the seam column at the end
    idx = np.arange((n + 1) ** 2).reshape(n + 1, n + 1)
    seam = (n + 1) ** 2 + np.arange(n + 1)
    faces = []
    for r in range(n):
        for c in range(n):
            def vid(rr, cc):
                return seam[rr] if (cc == n // 2 and c >= n // 2) else idx[rr, cc]
            a, b, cc_, d = vid(r, c), vid(r, c + 1), vid(r + 1, c + 1), vid(r + 1, c)
            faces += [[a, b, cc_], [a, cc_, d]] if g.random() < 0.5 else [[a, b, d], [b, cc_, d]]
    faces = np.asarray(faces)
    g.shuffle(faces)
    return pts.astype(np.float32)[faces]


@pytest.mark.parametrize("S,n,jitter", [(16, 32, 0.0), (16, 7, 0.35), (33, 11, 0.4), (100, 24, 0.3)])
def test_watertight_square_covers_every_texel_centre_once(S, n, jitter):
    corners = _square_triangulation(n, S + n, jitter)
    assert np.array_equal(po.coverage_count(corners, S), np.ones((S, S), np.int64))
    fid, bary = po.layout(corners, S)
    assert (fid >= 0).all()
    assert np.abs(bary.sum(-1) - 1).max() < 1e-6 and bary.min() >= -1e-7


def test_overlap_lowest_index_wins_and_orientation():
    S = 8
    big = [[0.0, 0.0], [1.0, 0.0], [0.0, 1.0]]
    top = [[0.0, 0.55], [0.4, 0.55], [0.0, 0.95]]                         # inside `big`, only v > 0.5
    fid, _ = po.layout(np.array([top, big], np.float32), S)
    fid2, _ = po.layout(np.array([big, top], np.float32), S)
    assert (fid2[fid2 >= 0] == 0).all()                                   # face 0 covers everything face 1 does
    assert (fid == 0).sum() > 0 and (fid == 1).sum() > 0
    rows = np.nonzero((fid == 0).any(1))[0]
    assert rows.max() < S // 2                                            # v > 0.5 lands in the top rows
    assert fid[1, 0] == 0 and fid[S - 1, 0] == 1 and fid[0, S - 1] == -1


def test_degenerate_and_out_of_range_faces_cover_nothing():
    S = 16
    corners = np.array([[[0.1, 0.1], [0.9, 0.9], [0.5, 0.5]],            # collinear
                        [[0.3, 0.3], [0.3, 0.3], [0.8, 0.1]],            # repeated corner
                        [[0.0, 0.0], [1.0, 0.0], [np.nan, 1.0]],         # non-finite corner
                        [[0.0, 0.0], [5000.0, 0.0], [0.0, 1.0]]],        # beyond the coordinate range
                       np.float32)
    fid, bary = po.layout(corners, S)
    assert (fid == -1).all() and (bary == 0).all()
    assert (po.coverage_count(corners, S) == 0).all()


def test_uncovered_texels_are_zero_and_minus_one():
    S = 12
    corners = np.array([[[0.0, 0.0], [0.5, 0.0], [0.0, 0.5]]], np.float32)
    fid, bary = po.layout(corners, S)
    verts = np.random.default_rng(0).normal(size=(2, 3, 3))
    out = po.fill(verts, np.array([[0, 1, 2]]), fid, bary)
    assert (fid == -1).any() and (fid == 0).any()
    assert (out[:, :, fid == -1] == 0).all() and (bary[fid == -1] == 0).all()
    # the corner texel nearest uv (0,0) interpolates close to vertex 0
    assert np.abs(out[:, :, S - 1, 0] - verts[:, 0]).max() < 0.2 * np.abs(verts).max()


def test_c_abi_rejects_bad_arguments_before_device_work():
    from gaussianavatar_b200 import _lib
    L = _lib.lib()
    assert L.ga_posmap_layout(10, 513, None, None, None, None) != 0
    assert L.ga_smpl_vertices(9, 6890, *([None] * 8)) != 0
    assert L.ga_posmap_fill(1, 0, 6890, *([None] * 6)) != 0


# ---- stage-2 plumbing ------------------------------------------------------------------------------------------------------------
def test_datasets_build_without_inp_map_when_maps_come_from_the_pose(tmp_path):
    from posmap_fixture import write_posmap_dataset
    from gaussianavatar_b200.dataset import MonoDataset_novel_pose, MonoDataset_novel_view, MonoDataset_test, MonoDataset_train
    mp = write_posmap_dataset(str(tmp_path))
    assert not os.path.exists(os.path.join(mp.source_path, "train", "inp_map"))
    for cls in (MonoDataset_train, MonoDataset_test, MonoDataset_novel_pose, MonoDataset_novel_view):
        ds = cls(mp)
        item = ds[0]
        assert "inp_pos_map" not in item and "pose_idx" in item, cls.__name__
    mp.inp_posmap_from_pose = False                                     # the reference's behaviour: stage 2 reads the files
    with pytest.raises(FileNotFoundError):
        MonoDataset_train(mp)[0]


def test_model_parms_without_the_field_read_the_files(tmp_path):
    """A namespace without inp_posmap_from_pose (the reference's own ModelParams) keeps reading inp_map/."""
    import types
    from dataset_fixture import write_synthetic_dataset
    from gaussianavatar_b200.dataset import MonoDataset_train
    mp = write_synthetic_dataset(str(tmp_path), stage2=True)
    ns = types.SimpleNamespace(**{k: v for k, v in vars(mp).items() if k != "inp_posmap_from_pose"})
    assert "inp_pos_map" in MonoDataset_train(ns)[0]


def _model(mp):
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams, OptimizationParams
    return AvatarModel(mp, NetworkParams(nf=8), OptimizationParams(), train=True)


def test_smplx_with_pose_maps_is_not_implemented(tmp_path):
    from posmap_fixture import write_posmap_dataset
    mp = write_posmap_dataset(str(tmp_path))
    mp.smpl_type = "smplx"
    with pytest.raises(NotImplementedError, match="SMPL mesh only"):
        _model(mp)


def test_missing_uv_template_names_the_path(tmp_path):
    from posmap_fixture import write_posmap_dataset
    mp = write_posmap_dataset(str(tmp_path))
    path = os.path.join(mp.project_path, "assets", "template_mesh_smpl_uv.obj")
    os.remove(path)
    with pytest.raises(FileNotFoundError, match="template_mesh_smpl_uv.obj"):
        _model(mp)


@pytest.mark.parametrize("field", ["posedirs", "weights", "f"])
def test_pickle_without_mesh_fields_raises(tmp_path, field):
    from posmap_fixture import write_posmap_dataset
    mp = write_posmap_dataset(str(tmp_path))
    pk = os.path.join(mp.smpl_model_path, "SMPL_NEUTRAL.pkl")
    with open(pk, "rb") as f:
        sm = pickle.load(f)
    del sm[field]
    with open(pk, "wb") as f:
        pickle.dump(sm, f)
    with pytest.raises(ValueError, match=field):
        _model(mp)


def test_pose_mapper_rejects_incomplete_model_before_device_work():
    from gaussianavatar_b200.posmap import PoseMapper
    t = syn.make_uv_template(0)
    model = syn.smpl_mesh_model(syn.make_body(0), t)
    del model["posedirs"]
    with pytest.raises(ValueError, match="posedirs"):
        PoseMapper(model, torch.zeros(10), t, 16)
