"""GPU: the per-frame rasterizer's SH-colour and precomputed-covariance modes (through the C ABI) against the CPU oracle, against
the scale / rotation and precomputed-colour modes on the device, and through the module surface upstream's callers use."""
import numpy as np
import pytest
import torch

from oracle.raster_twin import quat_to_rot
from oracle.raster_twin_ex import SH_C0
from scenes import oracle_args, random_scene
from sh_scenes import random_shs

pytestmark = pytest.mark.gpu

CASES = [
    dict(P=300, H=64, W=80, seed=1, scale_mean=0.03),
    dict(P=2000, H=200, W=136, seed=2, scale_mean=0.02),                       # H, W not multiples of 16
    dict(P=1500, H=128, W=128, seed=4, scale_mean=0.05, spread=2.5),           # guard band / off-screen / clipped rects
    dict(P=800, H=96, W=96, seed=5, scale_mean=0.02, z_extra=2.4),            # many behind the near plane (z <= 0.2)
]
CASE_IDS = [f"P{c['P']}_{c['H']}x{c['W']}" for c in CASES]
# (shs, cov3D_precomp, degree, coefficients): M % 4 == 0 takes the float4 path, the others the scalar one
FWD_MODES = [(False, True, 0, 0)] + [(True, cov, d, m) for cov in (False, True) for d, m in ((0, 1), (1, 4), (2, 9), (3, 16), (2, 16))]
BWD_MODES = [(False, True, 0, 0), (True, False, 3, 16), (True, False, 1, 4), (True, True, 2, 9), (True, True, 0, 1)]
mode_id = lambda m: ("sh%d_M%d" % (m[2], m[3]) if m[0] else "rgb") + ("_cov" if m[1] else "_sr")


def _settings(sc, dev, degree=0, campos=True):
    from gaussianavatar_b200.rasterizer import GaussianRasterizationSettings
    cam = sc["cam"]
    return GaussianRasterizationSettings(sc["H"], sc["W"], sc["tanfovx"], sc["tanfovy"], sc["bg"].to(dev), 1.0,
                                         cam.world_view_transform.to(dev), cam.full_proj_transform.to(dev), degree,
                                         cam.camera_center.to(dev) if campos else None, False, False)


def _inputs(sc, sh, cov, D, M, seed=3):
    """Device inputs and oracle keywords of one mode; cov3D_precomp is the fp32 Sigma of the scene's scales / rotations."""
    shs = random_shs(sc, D, M, seed=seed) if sh else None
    cov3D = None
    if cov:
        from sh_scenes import sigma_of
        cov3D = sigma_of(sc["scales"], sc["rotations"])
    okw = {}
    args = oracle_args(sc)
    if sh:
        args["colors"] = None
        okw.update(shs=shs.numpy(), sh_degree=D, campos=sc["cam"].camera_center.numpy())
    if cov:
        args["scales"] = args["rotations"] = None
        okw.update(cov3D_precomp=cov3D.numpy())
    return shs, cov3D, args, okw


def _run(sc, shs=None, D=0, cov3D=None):
    from gaussianavatar_b200.rasterizer import rasterize_forward
    dev = torch.device("cuda:0")
    rs = _settings(sc, dev, D)
    t = {k: sc[k].to(dev) for k in ("means3D", "colors", "opacities", "scales", "rotations")}
    color, radii, ctx = rasterize_forward(t["means3D"], None if shs is not None else t["colors"], t["opacities"],
                                          None if cov3D is not None else t["scales"], None if cov3D is not None else t["rotations"], rs,
                                          shs=None if shs is None else shs.to(dev), cov3D_precomp=None if cov3D is None else cov3D.to(dev))
    torch.cuda.synchronize()
    return color, radii, ctx, rs, t


def _rel(a, b):
    a = a.detach().cpu().numpy().astype(np.float64).reshape(b.shape)
    return np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30)


@pytest.mark.parametrize("mode", FWD_MODES, ids=mode_id)
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_forward_parity(case, mode):
    from oracle import raster_oracle_ex as ro
    sh, cov, D, M = mode
    sc = random_scene(**case)
    shs, cov3D, args, okw = _inputs(sc, sh, cov, D, M)
    color, radii, ctx, rs, _ = _run(sc, shs, D, cov3D)
    v = ctx.views()
    o = ro.forward(**args, precision="f32", **okw)
    assert v["num_rendered"] == o.num_rendered
    np.testing.assert_array_equal(v["radii"].numpy(), o.get("radii"))
    np.testing.assert_array_equal(v["tiles_touched"].numpy(), o.get("tiles"))
    np.testing.assert_array_equal(v["offsets"].numpy().view(np.uint32), o.get("offsets"))
    vis = o.get("radii") > 0
    assert vis.sum() > 20
    np.testing.assert_array_equal(v["rect"].numpy().astype(np.int32)[vis], o.get("rect")[vis])
    np.testing.assert_array_equal(v["depth"].numpy().view(np.uint32)[vis], o.get("depth").astype(np.float32).view(np.uint32)[vis])
    np.testing.assert_array_equal(v["xy"].numpy()[vis], o.get("xy").astype(np.float32)[vis])
    np.testing.assert_array_equal(v["conic_opacity"].numpy()[vis], o.get("conic_o").astype(np.float32)[vis])
    if cov:
        np.testing.assert_array_equal(v["cov3d"].numpy()[vis], cov3D.numpy()[vis])
    if o.num_rendered:
        np.testing.assert_array_equal(v["keys_sorted"].numpy().view(np.uint64), o.get("keys"))
        np.testing.assert_array_equal(v["vals_sorted"].numpy().view(np.uint32), o.get("vals"))
    np.testing.assert_array_equal(v["ranges"].numpy().view(np.uint32), o.get("ranges"))
    if sh:
        rgb = ctx.rgb.cpu().numpy().astype(np.float64)
        assert np.abs(rgb[vis] - o.get("rgb")[vis]).max() <= 1e-6
        assert not rgb[~vis].any()
        np.testing.assert_array_equal(ctx.clamped.cpu().numpy()[vis], o.get("clamped")[vis])
        assert (o.get("clamped")[vis] != 0).any()
    img = color.cpu().numpy().astype(np.float64)
    assert np.abs(img - o.image).mean() <= 1e-4, np.abs(img - o.image).mean()
    nc_mismatch = int((v["n_contrib"].numpy().view(np.uint32) != o.get("n_contrib")).sum())
    assert nc_mismatch <= max(2, sc["H"] * sc["W"] // 2000), nc_mismatch


@pytest.mark.parametrize("mode", BWD_MODES, ids=mode_id)
@pytest.mark.parametrize("case", CASES[:3], ids=CASE_IDS[:3])
def test_backward_parity(case, mode):
    from gaussianavatar_b200.rasterizer import rasterize_backward
    from oracle import raster_oracle_ex as ro
    sh, cov, D, M = mode
    sc = random_scene(**case)
    shs, cov3D, args, okw = _inputs(sc, sh, cov, D, M)
    color, radii, ctx, rs, t = _run(sc, shs, D, cov3D)
    gw = torch.randn(3, sc["H"], sc["W"], generator=torch.Generator().manual_seed(11))
    d_means3D, d_m2d, d_colors, d_opac, d_scales, d_rot, d_sh, d_cov3D = rasterize_backward(
        ctx, t["means3D"], None if sh else t["colors"], None if cov else t["scales"], None if cov else t["rotations"], rs, gw.cuda(),
        return_sh_cov3D=True)
    torch.cuda.synchronize()
    o = ro.forward(**args, precision="f32", **okw)
    gb = o.backward(gw.numpy())
    assert _rel(d_means3D, gb["d_means3D"]) < 5e-4
    assert _rel(d_opac, gb["d_opacity"]) < 2e-4
    culled = o.get("radii") <= 0                   # none in the first two cases
    assert not d_means3D.cpu().numpy()[culled].any()
    if sh:
        assert d_colors is None
        assert _rel(d_sh, gb["d_sh"]) < 2e-4
        dsh = d_sh.cpu().numpy()
        assert not dsh[:, (D + 1) ** 2:].any() and not dsh[culled].any()
        cl = ctx.clamped.cpu().numpy()
        mask = ((cl[:, None] >> np.arange(3)) & 1).astype(bool)           # [P, 3]
        assert mask.any() and not dsh.transpose(0, 2, 1)[mask].any()
    else:
        assert _rel(d_colors, gb["d_colors"]) < 1e-4
    if cov:
        assert d_scales is None and d_rot is None
        assert _rel(d_cov3D, gb["d_cov3d"]) < 5e-4
        assert not d_cov3D.cpu().numpy()[culled].any()
    else:
        assert _rel(d_scales, gb["d_scales"]) < 5e-4


def _sigma6(scales, rots):
    """Sigma(s, q) = M^T M, M = S R^T, as (xx, xy, xz, yy, yz, zz) — differentiable fp64."""
    R = quat_to_rot(rots)
    M = torch.diag_embed(scales) @ R.transpose(1, 2)
    S = M.transpose(1, 2) @ M
    return torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], -1)


def test_precomputed_sigma_reproduces_scale_rotation_run():
    """cov3D_precomp = the Sigma K1 built from scales / rotations: bit-identical radii, lists, ranges and image; the chain rule of
    d_cov3D through Sigma(s, q) reproduces that run's d_scales / d_rotations."""
    from gaussianavatar_b200.rasterizer import rasterize_backward
    sc = random_scene(**CASES[1])
    color0, radii0, ctx0, rs, t = _run(sc)
    v0 = ctx0.views()
    color1, radii1, ctx1, _, _ = _run(sc, cov3D=v0["cov3d"].contiguous())
    v1 = ctx1.views()
    assert torch.equal(radii0, radii1) and torch.equal(color0, color1)
    for k in ("keys_sorted", "vals_sorted", "ranges", "n_contrib", "final_T", "conic_opacity", "xy"):
        assert torch.equal(v0[k], v1[k]), k
    gw = torch.randn(3, sc["H"], sc["W"], generator=torch.Generator().manual_seed(12)).cuda()
    d0 = rasterize_backward(ctx0, t["means3D"], t["colors"], t["scales"], t["rotations"], rs, gw)
    d1 = rasterize_backward(ctx1, t["means3D"], t["colors"], None, None, rs, gw, return_sh_cov3D=True)
    torch.cuda.synchronize()
    s = t["scales"].double().cpu().requires_grad_(True)
    q = t["rotations"].double().cpu().requires_grad_(True)
    (_sigma6(s, q) * d1[7].double().cpu()).sum().backward()
    assert _rel(s.grad, d0[4].double().cpu().numpy()) < 1e-5
    assert _rel(q.grad, d0[5].double().cpu().numpy()) < 1e-5
    assert _rel(d1[0], d0[0].double().cpu().numpy()) < 1e-5


def test_degree0_sh_equals_precomputed_colours():
    """sh_0 = (c - 0.5) / C0 at degree 0 renders the colors_precomp = c image, and d_sh[:, 0] = C0 d_colors."""
    from gaussianavatar_b200.rasterizer import rasterize_backward
    sc = random_scene(**CASES[0])
    sc["colors"] = 0.05 + 0.9 * sc["colors"]                    # no colour near the clamp
    shs = ((sc["colors"].double() - 0.5) / SH_C0).float()[:, None, :].contiguous()
    color0, _, ctx0, rs, t = _run(sc)
    color1, _, ctx1, _, _ = _run(sc, shs=shs, D=0)
    assert (color0 - color1).abs().max().item() <= 1e-6
    gw = torch.randn(3, sc["H"], sc["W"], generator=torch.Generator().manual_seed(13)).cuda()
    d0 = rasterize_backward(ctx0, t["means3D"], t["colors"], t["scales"], t["rotations"], rs, gw)
    d1 = rasterize_backward(ctx1, t["means3D"], None, t["scales"], t["rotations"], rs, gw, return_sh_cov3D=True)
    assert d1[2] is None and d1[6].shape == (sc["means3D"].shape[0], 1, 3)
    assert _rel(d1[6][:, 0], (SH_C0 * d0[2].double()).cpu().numpy()) < 1e-5


def test_module_surface_gradients_in_input_order():
    from gaussianavatar_b200.rasterizer import GaussianRasterizer
    from gaussianavatar_b200.renderer import render_batch
    from oracle import raster_oracle_ex as ro
    dev = torch.device("cuda:0")
    sc = random_scene(P=1000, H=128, W=128, seed=7, aniso=False, opacity_one=True)
    D, M = 3, 16
    shs, cov3D, args, okw = _inputs(sc, True, True, D, M)
    gw = torch.randn(3, 128, 128, generator=torch.Generator().manual_seed(3))
    o = ro.forward(**args, precision="f32", **okw)
    gb = o.backward(gw.numpy())

    pts = sc["means3D"].to(dev).requires_grad_(True)
    op = sc["opacities"].to(dev).requires_grad_(True)
    sh_d = shs.to(dev).requires_grad_(True)
    cov_d = cov3D.to(dev).requires_grad_(True)
    m2d = torch.zeros_like(pts, requires_grad=True)
    r = GaussianRasterizer(_settings(sc, dev, D))
    img, radii = r(means3D=pts, means2D=m2d, opacities=op, shs=sh_d, cov3D_precomp=cov_d)
    (img * gw.to(dev)).sum().backward()
    assert np.abs(img.detach().cpu().numpy() - o.image).mean() <= 1e-4
    assert _rel(pts.grad, gb["d_means3D"]) < 5e-4 and _rel(op.grad, gb["d_opacity"]) < 2e-4
    assert _rel(sh_d.grad, gb["d_sh"]) < 2e-4 and _rel(cov_d.grad, gb["d_cov3d"]) < 5e-4
    assert _rel(m2d.grad[:, :2], gb["d_mean2D"]) < 2e-4

    # the autograd Function's backward: one gradient per input of upstream's order, None for inputs that were not given
    from gaussianavatar_b200.rasterizer import _RasterizeGaussians
    empty = torch.empty(0, device=dev)
    for given_sh, given_cov in ((True, False), (False, True)):
        leaves = dict(means3D=sc["means3D"].to(dev), means2D=torch.zeros(1000, 3, device=dev), sh=sh_d.detach() if given_sh else empty,
                      colors=empty if given_sh else sc["colors"].to(dev), opac=sc["opacities"].to(dev),
                      scales=empty if given_cov else sc["scales"].to(dev), rots=empty if given_cov else sc["rotations"].to(dev),
                      cov=cov_d.detach() if given_cov else empty)
        for k in leaves:
            if leaves[k].numel():
                leaves[k].requires_grad_(True)
        img, _ = _RasterizeGaussians.apply(*leaves.values(), _settings(sc, dev, D))
        (img * gw.to(dev)).sum().backward()
        for k, x in leaves.items():
            assert (x.grad is not None) == bool(x.numel()), k
            if x.grad is not None:
                assert x.grad.shape == x.shape, k

    # render_batch (the reference's gaussian_renderer entry point) with shs and active_sh_degree
    cam = sc["cam"].to(dev)
    pts2 = sc["means3D"].to(dev).requires_grad_(True)
    sh2 = shs.to(dev).requires_grad_(True)
    _, _, args2, okw2 = _inputs(sc, True, False, D, M)
    img2 = render_batch(points=pts2, shs=sh2, colors_precomp=None, rotations=sc["rotations"].to(dev), scales=sc["scales"].to(dev),
                        opacity=sc["opacities"].to(dev), FovX=cam.FovX, FovY=cam.FovY, height=cam.height, width=cam.width,
                        bg_color=sc["bg"].to(dev), world_view_transform=cam.world_view_transform,
                        full_proj_transform=cam.full_proj_transform, active_sh_degree=D, camera_center=cam.camera_center)
    (img2 * gw.to(dev)).sum().backward()
    o2 = ro.forward(**args2, precision="f32", **okw2)
    gb2 = o2.backward(gw.numpy())
    assert np.abs(img2.detach().cpu().numpy() - o2.image).mean() <= 1e-4
    assert _rel(pts2.grad, gb2["d_means3D"]) < 5e-4 and _rel(sh2.grad, gb2["d_sh"]) < 2e-4


def test_bad_inputs_raise_before_any_launch():
    from gaussianavatar_b200 import _lib
    from gaussianavatar_b200.rasterizer import GaussianRasterizer
    dev = torch.device("cuda:0")
    sc = random_scene(P=64, H=32, W=32, seed=0)
    m, op = sc["means3D"].to(dev), sc["opacities"].to(dev)
    sr = dict(scales=sc["scales"].to(dev), rotations=sc["rotations"].to(dev))
    shs16 = torch.zeros(64, 16, 3, device=dev)
    bad = [
        (3, dict(shs=torch.zeros(64, 16, device=dev), **sr)),                    # not [P, M, 3]
        (3, dict(shs=torch.zeros(63, 16, 3, device=dev), **sr)),                 # wrong P
        (3, dict(shs=torch.zeros(64, 16, 4, device=dev), **sr)),
        (4, dict(shs=shs16, **sr)),                                              # degree outside 0..3
        (-1, dict(shs=shs16, **sr)),
        (2, dict(shs=torch.zeros(64, 4, 3, device=dev), **sr)),                  # (D+1)^2 > M
        (3, dict(shs=shs16.cpu(), **sr)),                                        # CPU tensors
        (0, dict(colors_precomp=sc["colors"].to(dev), cov3D_precomp=torch.zeros(64, 6))),
        (0, dict(colors_precomp=sc["colors"].to(dev), cov3D_precomp=torch.zeros(64, 5, device=dev))),
        (0, dict(shs=shs16, cov3D_precomp=torch.zeros(64, 6, device=dev), **sr)),  # both covariance sources
    ]
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    for degree, kw in bad:
        r = GaussianRasterizer(_settings(sc, dev, degree))
        with pytest.raises(Exception):
            r(means3D=m, means2D=m, opacities=op, **kw)
    with pytest.raises(Exception):                                               # shs without campos
        GaussianRasterizer(_settings(sc, dev, 1, campos=False))(means3D=m, means2D=m, opacities=op, shs=shs16, **sr)
    assert _lib.launch_count() == n0
