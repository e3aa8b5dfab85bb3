"""CPU: the SMPL-X (55-joint) contract pinned against the reference's own `smplx.SMPLX` and dataset classes through
tests/golden/smplx_A.npz and tests/golden/dataset_items_smplx.npz (oracle/gen_golden_smplx.py), the asset loader's checks, and the C ABI's
validation of the SMPL-X joint-transform and 55-joint LBS entry points."""
import ctypes
import os

import numpy as np
import pytest
import torch

from dataset_fixture_smplx import write_synthetic_smplx_dataset
from gaussianavatar_b200 import _lib
from gaussianavatar_b200 import synthetic as syn
from oracle import avatar_oracle_smplx as aox

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GA_ERR_INVALID = -1
FAKE = 256        # never dereferenced: every case below fails validation first


def test_parent_tables_agree_with_the_reference_model():
    d = np.load(os.path.join(GOLD, "smplx_A.npz"))
    assert d["parents"].tolist() == syn.SMPLX_PARENTS == aox.SMPLX_PARENTS
    assert all(p < j for j, p in enumerate(syn.SMPLX_PARENTS))          # index order is a valid walk of the chain


def test_loader_rest_joints_match_the_reference(tmp_path):
    from gaussianavatar_b200.avatar_model import smplx_rest_joints
    d = np.load(os.path.join(GOLD, "smplx_A.npz"))
    body = syn.make_smplx_body(int(d["body_seed"]))
    assert np.array_equal(body.betas[0].numpy(), d["betas"])
    path = str(tmp_path / "SMPLX_NEUTRAL.npz")
    syn.write_smplx_model_npz(path, body, seed=0)
    J = smplx_rest_joints(path, torch.tensor(d["betas"]), syn.SMPLX_PARENTS)
    assert J.shape == (55, 3)
    np.testing.assert_allclose(J.numpy(), d["rest_joints"], rtol=0, atol=2e-6)
    np.testing.assert_allclose(body.rest_joints().numpy(), d["rest_joints"], rtol=0, atol=2e-6)


def test_wrong_kintree_table_raises(tmp_path):
    from gaussianavatar_b200.avatar_model import smplx_rest_joints
    body = syn.make_smplx_body(0)
    path = str(tmp_path / "SMPLX_NEUTRAL.npz")
    syn.write_smplx_model_npz(path, body, seed=0)
    m = dict(np.load(path))
    m["kintree_table"] = m["kintree_table"].copy()
    m["kintree_table"][0, 30] = 21          # a left-hand joint hung from the right wrist
    bad = str(tmp_path / "bad.npz")
    np.savez(bad, **m)
    with pytest.raises(ValueError, match="kintree_table"):
        smplx_rest_joints(bad, body.betas[0], syn.SMPLX_PARENTS)


def test_oracle_with_smplx_parents_reproduces_the_reference_A():
    d = np.load(os.path.join(GOLD, "smplx_A.npz"))
    A = aox.smplx_joint_transforms(torch.tensor(d["rest_joints"]).double(), torch.tensor(d["pose66"]).double(),
                                   torch.tensor(d["rest99"]).double(), torch.tensor(d["transl"]).double())
    assert A.shape == (d["pose66"].shape[0], 55, 4, 4)
    ref = torch.tensor(d["A"]).double()
    err = (A - ref).abs().max().item()
    assert err < 2e-5, err
    # the fixture really exercises the hands: finger joints move away from the wrists' frames
    assert (ref[8:, 25:, :3, :3] - ref[8:, 20:21, :3, :3]).abs().max() > 0.5


def test_synthetic_assets_and_host_transforms_agree_with_the_oracle():
    a = syn.make_avatar_assets(500, 32, seed=0, body="smplx")
    assert a.query_lbs.shape == (500, 55) and torch.allclose(a.query_lbs.sum(1), torch.ones(500), atol=1e-5)
    J = a.rest_joints.double()
    cano = torch.cat([torch.tensor(syn.star_pose()[:66]), torch.zeros(99)])[None]
    A = aox.joint_transforms(J, cano, torch.tensor(syn.CANO_TRANSL)[None])[0]
    assert (A.float() - a.cano_joint_mats).abs().max() < 1e-5


def test_dataset_items_match_the_reference_classes(tmp_path):
    from gaussianavatar_b200 import dataset as ds
    mp = write_synthetic_smplx_dataset(str(tmp_path))
    mp.no_mask = 1
    gold = np.load(os.path.join(GOLD, "dataset_items_smplx.npz"))
    sets = dict(train=ds.MonoDataset_train(mp), test=ds.MonoDataset_test(mp), novel_pose=ds.MonoDataset_novel_pose(mp))
    fields = ("original_image", "world_view_transform", "projection_matrix", "full_proj_transform", "camera_center", "pose_data",
              "transl_data", "rest_pose")
    for name, dset in sets.items():
        assert len(dset) == int(gold[f"{name}/len"])
        for i in range(len(dset)):
            item = dset[i]
            a = {k: np.asarray(item[k], dtype=np.float64) for k in fields if k in item}
            if "original_image" in a:
                img = a["original_image"].reshape(-1)
                a["original_image"] = img[np.random.default_rng(i).choice(img.size, 64, replace=False)]
            a["scalars"] = np.array([item["FovX"], item["FovY"], item["width"], item["height"], item["pose_idx"]], dtype=np.float64)
            b = {k.split("/", 2)[2]: gold[k] for k in gold.files if k.startswith(f"{name}/{i}/")}
            assert a.keys() == b.keys() and "rest_pose" in a
            assert a["rest_pose"].shape == (99,)
            if "pose_data" in a:
                assert a["pose_data"].shape == (66,)
            for k in a:
                np.testing.assert_allclose(a[k], b[k], rtol=0, atol=1e-7, err_msg=f"{name}[{i}].{k}")


# ---------------------------------------------------------------------------------------------------------------- C ABI
def _err(rc, what):
    assert rc == GA_ERR_INVALID, rc
    assert what in _lib.lib().ga_last_error().decode()


def test_smplx_entry_points_reject_null_rest_pose():
    L = _lib.lib()
    _err(L.ga_smplx_forward(2, FAKE, None, FAKE, FAKE, FAKE, FAKE, FAKE, None), "NULL")
    _err(L.ga_smplx_backward(2, FAKE, None, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, None), "NULL")


@pytest.mark.parametrize("J,ld,B,what", [
    (23, 24, 2, "num_joints"), (56, 56, 2, "num_joints"), (0, 24, 2, "num_joints"),
    (55, 52, 2, "lbs_ld"), (55, 55, 2, "lbs_ld"), (24, 22, 2, "lbs_ld"), (55, 58, 2, "lbs_ld"),
    (55, 56, 9, "B=9"), (24, 24, 9, "B=9"),
])
def test_lbs_ex_rejects_bad_layouts_before_any_launch(J, ld, B, what):
    L = _lib.lib()
    _err(L.ga_lbs_forward_ex(100, B, J, ld, 1.0, 0, *[FAKE] * 8, None), what)
    _err(L.ga_lbs_backward_ex(100, B, J, ld, 100, 1.0, 0, *[FAKE] * 10, None), what)


def test_lbs_ex_names_the_built_row_strides():
    """A stride that is legal (a multiple of 4, >= num_joints) but not one of the built layouts is refused with the built ones named."""
    L = _lib.lib()
    _err(L.ga_lbs_forward_ex(100, 2, 55, 60, 1.0, 0, *[FAKE] * 8, None), "not built")
    _err(L.ga_lbs_forward_ex(100, 2, 24, 28, 1.0, 0, *[FAKE] * 8, None), "not built")
