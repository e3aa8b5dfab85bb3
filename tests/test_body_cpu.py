"""CPU: the body records (gaussianavatar_b200/body.py): a full pose splits into (pose, rest_pose) and joins back unchanged, and
the rest joints are bit for bit what the three formulas they replaced computed."""
import os

import numpy as np
import pytest
import torch

from gaussianavatar_b200 import synthetic as syn
from gaussianavatar_b200.body import SMPL, SMPLX, body_of, load_model

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("name", ["smpl", "smplx"])
def test_split_join_round_trip(name):
    b = body_of(name)
    full = torch.randn(5, b.full_width, generator=torch.Generator().manual_seed(1))
    pose, rest = b.split(full)
    assert pose.shape == (5, b.pose_width) and pose.is_contiguous()
    assert rest is None if b is SMPL else (rest.shape == (5, 99) and rest.is_contiguous())
    assert len(b.pose_args(pose, rest)) == (1 if b is SMPL else 2)
    assert torch.equal(b.join(pose, rest), full)
    with pytest.raises(ValueError, match="pose"):
        b.split(full[:, 1:])


def _dense(x):
    return np.asarray(x.todense() if hasattr(x, "todense") else x)


def _avatar_model_smpl(sm, beta):
    """AvatarModel._load_reference_assets' SMPL formula (torch, shapedirs[..., :10])."""
    v_t = torch.as_tensor(np.asarray(sm["v_template"])).double()
    sd = torch.as_tensor(np.asarray(sm["shapedirs"])[:, :, :10]).double()
    Jr = torch.as_tensor(_dense(sm["J_regressor"])).double()
    return (Jr @ (v_t + torch.einsum("l,mkl->mk", torch.as_tensor(beta).float().double(), sd))).float()


def _smplx_loader(sm, beta):
    """The SMPL-X asset loader's formula (torch, shapedirs[..., :len(betas)])."""
    beta = torch.as_tensor(beta).double().reshape(-1)
    v_t = torch.as_tensor(np.asarray(sm["v_template"])).double()
    sd = torch.as_tensor(np.asarray(sm["shapedirs"])[:, :, :beta.numel()]).double()
    Jr = torch.as_tensor(_dense(sm["J_regressor"])).double()
    return (Jr @ (v_t + torch.einsum("l,mkl->mk", beta, sd))).float()


def _poser(sm, beta):
    """The vertex poser's formula (numpy)."""
    beta = np.asarray(torch.as_tensor(beta).double().reshape(-1))
    v_shaped = np.asarray(sm["v_template"], np.float64) + np.einsum("l,mkl->mk", beta,
                                                                      np.asarray(sm["shapedirs"])[:, :, :beta.size].astype(np.float64))
    return torch.from_numpy(_dense(sm["J_regressor"]).astype(np.float64) @ v_shaped).float()


def _models(tmp_path):
    b = syn.make_body(0)
    yield SMPL, syn.smpl_mesh_model(b, syn.make_uv_template(0)), b.betas[0]
    bx = syn.make_smplx_body(0)
    yield SMPLX, syn.smplx_mesh_model(bx, syn.make_smplx_uv_template(0), syn.smplx_posedirs(0)), bx.betas[0]
    d = np.load(os.path.join(GOLD, "smplx_A.npz"))
    path = str(tmp_path / "SMPLX_NEUTRAL.npz")
    syn.write_smplx_model_npz(path, syn.make_smplx_body(int(d["body_seed"])), seed=0)
    yield SMPLX, load_model(path), torch.tensor(d["betas"])


def test_rest_joints_equal_the_formulas_they_replace(tmp_path):
    for body, sm, beta in _models(tmp_path):
        J = body.rest_joints(sm, beta)
        assert J.shape == (body.joints, 3) and J.dtype == torch.float32
        for old in (_avatar_model_smpl, _smplx_loader, _poser):
            assert torch.equal(J, old(sm, beta)), (body.name, old.__name__)
