"""CPU: the C oracle's SH-colour and precomputed-covariance modes against the fp64 autograd twin and analytic known answers."""
import math

import numpy as np
import pytest
import torch

from oracle import raster_oracle_ex as ro
from oracle.raster_twin_ex import SH_C0, SH_C1, sh_to_rgb, twin_forward_ex
from scenes import oracle_args, random_scene
from sh_scenes import random_shs, sigma_of

DEG_M = [(0, 1), (0, 16), (1, 4), (1, 16), (2, 9), (2, 16), (3, 16)]
MODES = [(False, False, 0, 0)] + [(True, False, d, m) for d, m in DEG_M] + [(False, True, 0, 0)] + [(True, True, d, m) for d, m in DEG_M]


def _inputs(sc, sh, cov, D, M, seed=3):
    kw = {}
    if sh:
        kw.update(shs=random_shs(sc, D, M, seed=seed), sh_degree=D, campos=sc["cam"].camera_center.numpy())
    if cov:
        kw.update(cov3D_precomp=sigma_of(sc["scales"], sc["rotations"]))
    return kw


@pytest.mark.parametrize("sh,cov,D,M", MODES, ids=lambda v: str(int(v)))
def test_c_oracle_backward_matches_autograd_twin(sh, cov, D, M):
    sc = random_scene(P=150, H=48, W=64, seed=12, scale_mean=0.04)
    kw = _inputs(sc, sh, cov, D, M)
    args = oracle_args(sc)
    if sh:
        args["colors"] = None
    if cov:
        args["scales"] = args["rotations"] = None
    o64 = ro.forward(**args, precision="f64", **{k: (v.numpy() if torch.is_tensor(v) else v) for k, v in kw.items()})

    leaf = {k: sc[k].clone().double().requires_grad_(True) for k in ("means3D", "opacities")}
    tw = dict(colors=None if sh else sc["colors"], scales=None if cov else sc["scales"], rotations=None if cov else sc["rotations"])
    for k in ("shs", "cov3D_precomp"):
        if k in kw:
            leaf[k] = kw[k].clone().double().requires_grad_(True)
    out = twin_forward_ex(leaf["means3D"], tw["colors"], leaf["opacities"], tw["scales"], tw["rotations"], sc["bg"],
                       sc["cam"].world_view_transform, sc["cam"].full_proj_transform, sc["tanfovx"], sc["tanfovy"], sc["H"], sc["W"],
                       shs=leaf.get("shs"), sh_degree=D, campos=kw.get("campos"), cov3D_precomp=leaf.get("cov3D_precomp"))
    assert np.abs(out.detach().numpy() - o64.image).max() < 1e-6
    gw = torch.randn(3, sc["H"], sc["W"], generator=torch.Generator().manual_seed(5)).double()
    (out * gw).sum().backward()
    gb = o64.backward(gw.numpy())
    checks = [("d_means3D", "means3D"), ("d_opacity", "opacities")]
    if sh:
        checks.append(("d_sh", "shs"))
        if D >= 1:   # the scene exercises the direction term of d_means3D
            assert np.abs(o64.get("rgb")).max() > 0
    if cov:
        checks.append(("d_cov3d", "cov3D_precomp"))
    # the whole pipeline agrees to the bar of the existing oracle-vs-twin test: the oracle's constants are fp32 literals (0.3f, 1.3f,
    # 0.2f) widened to fp64, the twin's are exact decimals, which moves the gradients by a few 1e-8 relative
    for k, tk in checks:
        ref = leaf[tk].grad.numpy().reshape(gb[k].shape)
        assert np.abs(ref - gb[k]).max() <= 1e-6 * max(1.0, np.abs(ref).max()), k
    if sh:
        assert o64.get("clamped").any()            # the deliberately clamped subset reached the image path
        nk = (D + 1) ** 2
        assert not gb["d_sh"][:, nk:].any()
        # the SH chain alone, from the same dL/drgb (the oracle's d_colors): autograd of the twin's colour function
        m = sc["means3D"].clone().double().requires_grad_(True)
        shs = kw["shs"].clone().double().requires_grad_(True)
        rgb = sh_to_rgb(m, shs, D, kw["campos"])
        vis = torch.from_numpy(o64.get("radii") > 0)[:, None].double()
        (rgb * torch.from_numpy(gb["d_colors"]) * vis).sum().backward()
        assert np.abs(shs.grad.numpy() - gb["d_sh"]).max() <= 1e-10 * max(1.0, np.abs(gb["d_sh"]).max())


def _single(mean, H=64, W=64, bg=(1, 1, 1)):
    from gaussianavatar_b200.camera import make_camera
    K = np.array([[80.0, 0, W / 2], [0, 80.0, H / 2], [0, 0, 1]], dtype=np.float32)
    cam = make_camera(K, np.eye(4), H, W)
    P = np.asarray(mean, dtype=np.float32).reshape(-1, 3)
    n = P.shape[0]
    return dict(means3D=P, colors=None, opacities=np.full((n,), 0.8, np.float32), scales=np.full((n, 3), 0.05, np.float32),
                rotations=np.tile(np.array([1, 0, 0, 0], np.float32), (n, 1)), bg=np.asarray(bg, np.float32),
                viewmatrix=cam.world_view_transform.numpy(), projmatrix=cam.full_proj_transform.numpy(),
                tanfovx=math.tan(cam.FovX / 2), tanfovy=math.tan(cam.FovY / 2), H=H, W=W)


def test_known_answer_degree0_is_constant_colour():
    sc = random_scene(P=200, H=48, W=64, seed=4)
    shs = random_shs(sc, 0, 1, seed=1, clamp_frac=0.0)
    args = oracle_args(sc)
    args["colors"] = None
    o = ro.forward(**args, precision="f64", shs=shs.numpy(), sh_degree=0, campos=sc["cam"].camera_center.numpy())
    vis = o.get("radii") > 0
    expect = SH_C0 * shs[:, 0].double().numpy() + 0.5
    assert vis.sum() > 50
    np.testing.assert_allclose(o.get("rgb")[vis], expect[vis], rtol=0, atol=1e-12)


@pytest.mark.parametrize("axis", range(6), ids=["+x", "-x", "+y", "-y", "+z", "-z"])
def test_known_answer_degree1_from_axis_cameras(axis):
    """Only degree-1 coefficients: seen along the unit direction d, c = -C1 d_y sh1 + C1 d_z sh2 - C1 d_x sh3."""
    args = _single([0.0, 0.0, 2.0])
    d = np.zeros(3)
    d[axis // 2] = 1.0 if axis % 2 == 0 else -1.0
    shs = np.zeros((1, 4, 3), np.float32)
    shs[0, 1:4] = [[0.3, -0.2, 0.1], [0.25, 0.4, -0.3], [-0.35, 0.15, 0.2]]
    campos = (np.array([0.0, 0.0, 2.0]) - 3.0 * d).astype(np.float32)      # dir = (mean - campos) / |.| = d
    o = ro.forward(**args, precision="f64", shs=shs, sh_degree=1, campos=campos)
    assert o.get("radii")[0] > 0
    c = -SH_C1 * d[1] * shs[0, 1] + SH_C1 * d[2] * shs[0, 2] - SH_C1 * d[0] * shs[0, 3]
    np.testing.assert_allclose(o.get("rgb")[0], np.maximum(c + 0.5, 0.0), rtol=0, atol=1e-12)


def test_known_answer_clamped_channel_is_black_and_gets_no_gradient():
    args = _single([0.0, 0.0, 2.0], bg=(0, 0, 0))
    shs = np.zeros((1, 4, 3), np.float32)
    shs[0, 0] = [-1.0 / SH_C0, 0.5, 0.2]            # channel 0: c + 0.5 = -0.5 + (degree-1 part) < 0
    shs[0, 1:4] = [[0.1, 0.2, -0.1], [0.2, -0.1, 0.1], [-0.1, 0.1, 0.2]]
    for prec in ("f32", "f64"):
        o = ro.forward(**args, precision=prec, shs=shs, sh_degree=1, campos=np.array([0.3, -0.2, -1.0], np.float32))
        assert o.get("clamped")[0] == 1 and o.get("rgb")[0, 0] == 0.0
        assert np.all(o.image[0] == 0.0) and o.image[1].max() > 0.1
        gb = o.backward(np.random.default_rng(1).standard_normal((3, 64, 64)).astype(np.float32))
        assert np.all(gb["d_sh"][0, :, 0] == 0.0) and np.abs(gb["d_sh"][0, :, 1:]).max() > 0


def test_known_answer_precomputed_sigma_matches_scale_rotation():
    """cov3D_precomp = the Sigma the fp32 oracle builds from scales / rotations: every output is identical."""
    sc = random_scene(P=600, H=80, W=96, seed=6, scale_mean=0.03)
    from oracle import raster_oracle
    base = raster_oracle.forward(**oracle_args(sc), precision="f32")          # the original restatement
    args = oracle_args(sc)
    cov = base.get("cov3d").astype(np.float32)
    args["scales"] = args["rotations"] = None
    o = ro.forward(**args, precision="f32", cov3D_precomp=cov)
    assert o.num_rendered == base.num_rendered > 0
    for k in ("radii", "xy", "conic_o", "depth", "rect", "keys", "vals", "ranges", "out", "final_T", "n_contrib", "cov3d"):
        np.testing.assert_array_equal(o.get(k), base.get(k), err_msg=k)
    gw = np.random.default_rng(2).standard_normal((3, 80, 96)).astype(np.float32)
    g0, g1 = base.backward(gw), o.backward(gw)
    for k in ("d_means3D", "d_opacity", "d_colors", "d_cov3d"):
        np.testing.assert_array_equal(g1[k], g0[k], err_msg=k)
    assert not g1["d_scales"].any() and not g1["d_rots"].any()
