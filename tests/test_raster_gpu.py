"""GPU parity: sm_90a rasterizer (through the C ABI) vs the CPU oracle on the same seeded inputs.

Bars (SURVEY.md Appendix C): radii / tiles / rect / offsets / sort keys / sorted values / ranges bit-exact; depth bits
exact; image mean-L1 <= 1e-4 per pixel; gradients rel-L2 <= 1e-4 vs the fp32 oracle... (float atomics order noise).
"""
import math

import numpy as np
import pytest
import torch

from scenes import oracle_args, random_scene

pytestmark = pytest.mark.gpu


def _run_cuda(sc, need_grad=False):
    from gaussianavatar_b200.rasterizer import GaussianRasterizationSettings, rasterize_backward, rasterize_forward
    dev = torch.device("cuda:0")
    cam = sc["cam"]
    rs = GaussianRasterizationSettings(sc["H"], sc["W"], sc["tanfovx"], sc["tanfovy"], sc["bg"].to(dev), 1.0,
                                       cam.world_view_transform.to(dev), cam.full_proj_transform.to(dev), 0,
                                       cam.camera_center.to(dev), False, False)
    t = {k: sc[k].to(dev) for k in ("means3D", "colors", "opacities", "scales", "rotations")}
    color, radii, ctx = rasterize_forward(t["means3D"], t["colors"], t["opacities"], t["scales"], t["rotations"], rs)
    torch.cuda.synchronize()
    return color, radii, ctx, rs, t


CASES = [
    dict(P=300, H=64, W=80, seed=1, scale_mean=0.03),
    dict(P=2000, H=200, W=136, seed=2, scale_mean=0.02),                       # H, W not multiples of 16
    dict(P=5000, H=256, W=256, seed=3, scale_mean=0.01, aniso=False, opacity_one=True),   # the avatar's regime
    dict(P=1500, H=128, W=128, seed=4, scale_mean=0.05, spread=2.5),           # guard band / off-screen / clipped rects
    dict(P=800, H=96, W=96, seed=5, scale_mean=0.02, z_extra=2.4),            # many behind the near plane (z <= 0.2)
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"P{c['P']}_{c['H']}x{c['W']}")
def test_forward_parity(case):
    from oracle import raster_oracle as ro
    sc = random_scene(**case)
    color, radii, ctx, rs, _ = _run_cuda(sc)
    v = ctx.views()
    o = ro.forward(**oracle_args(sc), precision="f32")
    assert v["num_rendered"] == o.num_rendered
    np.testing.assert_array_equal(v["radii"].numpy(), o.get("radii"))
    np.testing.assert_array_equal(v["tiles_touched"].numpy(), o.get("tiles"))
    np.testing.assert_array_equal(v["offsets"].numpy().view(np.uint32), o.get("offsets"))
    vis = o.get("radii") > 0
    np.testing.assert_array_equal(v["rect"].numpy().astype(np.int32)[vis], o.get("rect")[vis])
    d_o = o.get("depth").astype(np.float32)
    np.testing.assert_array_equal(v["depth"].numpy().view(np.uint32)[vis], d_o.view(np.uint32)[vis])
    # same op order => xy / conic bit-identical too
    np.testing.assert_array_equal(v["xy"].numpy()[vis], o.get("xy").astype(np.float32)[vis])
    np.testing.assert_array_equal(v["conic_opacity"].numpy()[vis], o.get("conic_o").astype(np.float32)[vis])
    if o.num_rendered:
        # the device bins by tile and sorts each tile's bucket; upstream's unsorted duplicate list has no counterpart, its
        # SORTED (tile | depth, index) list and the tile ranges are the contract
        np.testing.assert_array_equal(v["keys_sorted"].numpy().view(np.uint64), o.get("keys"))
        np.testing.assert_array_equal(v["vals_sorted"].numpy().view(np.uint32), o.get("vals"))
    np.testing.assert_array_equal(v["ranges"].numpy().view(np.uint32), o.get("ranges"))
    img = color.cpu().numpy().astype(np.float64)
    ref = o.image
    assert np.abs(img - ref).mean() <= 1e-4, np.abs(img - ref).mean()
    # expf ulp differences may flip a 1/255 or 1e-4 threshold on isolated pixels: count, don't hide
    nc_mismatch = int((v["n_contrib"].numpy().view(np.uint32) != o.get("n_contrib")).sum())
    assert nc_mismatch <= max(2, sc["H"] * sc["W"] // 2000), nc_mismatch
    assert np.abs(img - ref).max() < 2e-2
    assert np.abs(v["final_T"].numpy() - o.get("final_T")).mean() <= 1e-4


@pytest.mark.parametrize("case", CASES[:4], ids=lambda c: f"P{c['P']}_{c['H']}x{c['W']}")
def test_backward_parity(case):
    from gaussianavatar_b200.rasterizer import rasterize_backward
    from oracle import raster_oracle as ro
    sc = random_scene(**case)
    color, radii, ctx, rs, t = _run_cuda(sc)
    g = torch.Generator().manual_seed(11)
    gw = torch.randn(3, sc["H"], sc["W"], generator=g)
    d_means3D, d_m2d, d_colors, d_opac, d_scales, d_rot = rasterize_backward(
        ctx, t["means3D"], t["colors"], t["scales"], t["rotations"], rs, gw.cuda())
    torch.cuda.synchronize()
    o = ro.forward(**oracle_args(sc), precision="f32")
    gb = o.backward(gw.numpy())

    def rel(a, b):
        a = a.cpu().numpy().astype(np.float64).reshape(b.shape)
        return np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30)

    assert rel(d_colors, gb["d_colors"]) < 1e-4
    assert rel(d_m2d[:, :2], gb["d_mean2D"]) < 2e-4
    assert rel(d_opac, gb["d_opacity"]) < 2e-4
    assert rel(d_means3D, gb["d_means3D"]) < 5e-4
    assert rel(d_scales, gb["d_scales"]) < 5e-4
    assert rel(d_rot, gb["d_rots"]) < 5e-4


def test_autograd_module_surface():
    """The nn.Module / autograd.Function surface the reference calls (gaussian_renderer/__init__.py:36-48)."""
    from gaussianavatar_b200.renderer import render_batch
    from oracle import raster_oracle as ro
    sc = random_scene(P=1000, H=128, W=128, seed=7, aniso=False, opacity_one=True)
    dev = torch.device("cuda:0")
    cam = sc["cam"].to(dev)
    pts = sc["means3D"].to(dev).requires_grad_(True)
    cols = sc["colors"].to(dev).requires_grad_(True)
    scl = sc["scales"].to(dev).requires_grad_(True)
    img = render_batch(points=pts, shs=None, colors_precomp=cols, rotations=sc["rotations"].to(dev), scales=scl,
                       opacity=sc["opacities"].to(dev), FovX=cam.FovX, FovY=cam.FovY, height=cam.height, width=cam.width,
                       bg_color=sc["bg"].to(dev), world_view_transform=cam.world_view_transform,
                       full_proj_transform=cam.full_proj_transform, active_sh_degree=0, camera_center=cam.camera_center)
    assert img.shape == (3, 128, 128)
    gw = torch.randn(3, 128, 128, generator=torch.Generator().manual_seed(3))
    (img * gw.to(dev)).sum().backward()
    o = ro.forward(**oracle_args(sc), precision="f32")
    gb = o.backward(gw.numpy())
    for got, ref in ((pts.grad, gb["d_means3D"]), (cols.grad, gb["d_colors"]), (scl.grad, gb["d_scales"])):
        a = got.cpu().numpy().astype(np.float64)
        assert np.linalg.norm(a - ref) / (np.linalg.norm(ref) + 1e-30) < 5e-4


def test_validation_errors():
    from gaussianavatar_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer
    dev = torch.device("cuda:0")
    sc = random_scene(P=10, H=32, W=32, seed=0)
    cam = sc["cam"].to(dev)
    rs = GaussianRasterizationSettings(32, 32, sc["tanfovx"], sc["tanfovy"], sc["bg"].to(dev), 1.0, cam.world_view_transform,
                                       cam.full_proj_transform, 0, cam.camera_center, False, False)
    r = GaussianRasterizer(rs)
    m = sc["means3D"].to(dev)
    with pytest.raises(Exception):
        r(means3D=m, means2D=m, opacities=sc["opacities"].to(dev), shs=None, colors_precomp=None, scales=sc["scales"].to(dev),
          rotations=sc["rotations"].to(dev))
    with pytest.raises(Exception):
        r(means3D=m, means2D=m, opacities=sc["opacities"].to(dev), colors_precomp=sc["colors"].to(dev), scales=None, rotations=None)


def test_empty_and_all_culled():
    """P=0 and an all-culled frame render the background (SURVEY.md Appendix C known-answer list)."""
    from gaussianavatar_b200.rasterizer import GaussianRasterizationSettings, rasterize_forward
    dev = torch.device("cuda:0")
    sc = random_scene(P=50, H=48, W=40, seed=0, z_extra=50.0)   # everything behind the camera (it looks down -z)
    cam = sc["cam"].to(dev)
    rs = GaussianRasterizationSettings(48, 40, sc["tanfovx"], sc["tanfovy"], torch.tensor([0.25, 0.5, 0.75], device=dev), 1.0,
                                       cam.world_view_transform, cam.full_proj_transform, 0, cam.camera_center, False, False)
    t = {k: sc[k].to(dev) for k in ("means3D", "colors", "opacities", "scales", "rotations")}
    color, radii, ctx = rasterize_forward(t["means3D"], t["colors"], t["opacities"], t["scales"], t["rotations"], rs)
    assert ctx.num_rendered == 0 and int(radii.abs().sum()) == 0
    expect = torch.tensor([0.25, 0.5, 0.75], device=dev)[:, None, None].expand(3, 48, 40)
    assert torch.equal(color, expect)
    e = {k: v[:0] for k, v in t.items()}
    color0, radii0, ctx0 = rasterize_forward(e["means3D"], e["colors"], e["opacities"], e["scales"], e["rotations"], rs)
    assert torch.equal(color0, expect) and radii0.numel() == 0


def _batched(scs, capacity=None):
    """Render same-size scenes (different Gaussians / cameras) through the batched, read-back-free path."""
    from gaussianavatar_b200.rasterizer import RasterBatchPlan, pack_cameras, rasterize_batch
    dev = torch.device("cuda:0")
    B, P, H, W = len(scs), scs[0]["means3D"].shape[0], scs[0]["H"], scs[0]["W"]
    plan = RasterBatchPlan(B, P, H, W, dev, capacity=capacity)
    cams = pack_cameras(torch.stack([s["cam"].world_view_transform for s in scs]), torch.stack([s["cam"].full_proj_transform for s in scs]),
                        [s["tanfovx"] for s in scs], [s["tanfovy"] for s in scs], dev)
    t = {k: torch.stack([s[k] for s in scs]).to(dev).requires_grad_(k != "opacities") for k in ("means3D", "colors", "scales")}
    rot, opac = scs[0]["rotations"].to(dev), scs[0]["opacities"].to(dev)
    img = rasterize_batch(t["means3D"], t["colors"], t["scales"], rot, opac, cams, scs[0]["bg"].to(dev), plan)
    return img, t, plan


def test_batched_path_matches_oracle_per_frame():
    """Two frames with different Gaussians in one set of launches: every frame's stages, image and gradients vs the oracle."""
    from oracle import raster_oracle as ro
    scs = [random_scene(P=3000, H=200, W=136, seed=21 + i, scale_mean=0.02, aniso=False, opacity_one=True) for i in range(3)]
    for s in scs[1:]:
        s["rotations"], s["opacities"] = scs[0]["rotations"], scs[0]["opacities"]
    img, t, plan = _batched(scs)
    gw = torch.randn(3, 3, 200, 136, generator=torch.Generator().manual_seed(2))
    (img * gw.cuda()).sum().backward()
    torch.cuda.synchronize()
    assert plan.check(wait=True)
    views = plan.views()
    for b, sc in enumerate(scs):
        o = ro.forward(**oracle_args(sc), precision="f32")
        v = views[b]
        assert v["num_rendered"] == o.num_rendered and v["overflow"] == 0
        np.testing.assert_array_equal(v["radii"].numpy(), o.get("radii"))
        np.testing.assert_array_equal(v["keys_sorted"].numpy().view(np.uint64), o.get("keys"))
        np.testing.assert_array_equal(v["vals_sorted"].numpy().view(np.uint32), o.get("vals"))
        np.testing.assert_array_equal(v["ranges"].numpy().view(np.uint32), o.get("ranges"))
        assert np.abs(img[b].detach().cpu().numpy().astype(np.float64) - o.image).mean() <= 1e-4
        gb = o.backward(gw[b].numpy())
        for got, ref in ((t["means3D"].grad[b], gb["d_means3D"]), (t["colors"].grad[b], gb["d_colors"]), (t["scales"].grad[b], gb["d_scales"])):
            a = got.cpu().numpy().astype(np.float64)
            assert np.linalg.norm(a - ref) / (np.linalg.norm(ref) + 1e-30) < 5e-4


def test_long_tile_lists_sorted_in_runs_and_many_segments():
    """Everything piled into a few tiles: tile lists far beyond the 8192 keys one CTA sorts at once (run-merge path) and
    beyond one 256-entry backward segment; opacity < 1 so that pixels blend deep into the list."""
    from gaussianavatar_b200.rasterizer import rasterize_backward
    from oracle import raster_oracle as ro
    sc = random_scene(P=30000, H=48, W=48, seed=31, scale_mean=0.004, aniso=False, spread=0.15)
    sc["opacities"] = torch.full_like(sc["opacities"], 0.02)
    color, radii, ctx, rs, t = _run_cuda(sc)
    v = ctx.views()
    o = ro.forward(**oracle_args(sc), precision="f32")
    rg = o.get("ranges").astype(np.int64)
    assert (rg[:, 1] - rg[:, 0]).max() > 8192
    np.testing.assert_array_equal(v["keys_sorted"].numpy().view(np.uint64), o.get("keys"))
    np.testing.assert_array_equal(v["vals_sorted"].numpy().view(np.uint32), o.get("vals"))
    np.testing.assert_array_equal(v["ranges"].numpy().view(np.uint32), o.get("ranges"))
    assert np.abs(color.cpu().numpy().astype(np.float64) - o.image).mean() <= 1e-4
    assert o.get("n_contrib").max() > 1000
    gw = torch.randn(3, 48, 48, generator=torch.Generator().manual_seed(4))
    d_means3D, d_m2d, d_colors, d_opac, d_scales, d_rot = rasterize_backward(ctx, t["means3D"], t["colors"], t["scales"], t["rotations"], rs, gw.cuda())
    gb = o.backward(gw.numpy())

    def rel(a, b):
        a = a.cpu().numpy().astype(np.float64).reshape(b.shape)
        return np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30)

    assert rel(d_colors, gb["d_colors"]) < 2e-4
    assert rel(d_opac, gb["d_opacity"]) < 5e-4
    assert rel(d_means3D, gb["d_means3D"]) < 5e-4
    assert rel(d_scales, gb["d_scales"]) < 5e-4


def test_batched_overflow_is_flagged_not_overrun_and_recovers():
    """A binning buffer that is too small: the device raises the flag, skips what does not fit (no out-of-bounds write: the
    guard words behind the buffer stay intact), plan.check() grows the buffer and the re-run is exact."""
    from oracle import raster_oracle as ro
    from gaussianavatar_b200.rasterizer import pack_cameras, rasterize_batch
    scs = [random_scene(P=2000, H=128, W=128, seed=41 + i, scale_mean=0.02, aniso=False, opacity_one=True) for i in range(2)]
    for s in scs[1:]:
        s["rotations"], s["opacities"] = scs[0]["rotations"], scs[0]["opacities"]
    with torch.no_grad():
        img, t, plan = _batched(scs, capacity=1000)
        torch.cuda.synchronize()
        assert int(plan.status_host[1]) == 1 and int(plan.status_host[0]) > 1000 and int(plan.status_host[15]) == plan.serial
        assert not plan.check(wait=True)                       # grows the buffer
        assert plan.capacity > int(plan.status_host[0])
        dev = torch.device("cuda:0")
        cams = pack_cameras(torch.stack([s["cam"].world_view_transform for s in scs]), torch.stack([s["cam"].full_proj_transform for s in scs]),
                            [s["tanfovx"] for s in scs], [s["tanfovy"] for s in scs], dev)
        img = rasterize_batch(t["means3D"], t["colors"], t["scales"], scs[0]["rotations"].to(dev), scs[0]["opacities"].to(dev), cams,
                              scs[0]["bg"].to(dev), plan)
        assert plan.check(wait=True)
    for b, sc in enumerate(scs):
        o = ro.forward(**oracle_args(sc), precision="f32")
        assert np.abs(img[b].cpu().numpy().astype(np.float64) - o.image).mean() <= 1e-4


@pytest.mark.parametrize("kind", ["pairs", "pile"])
def test_equal_depths_keep_upstream_tie_order(kind):
    """Equal depth bits inside a tile: upstream's stable key sort leaves them in Gaussian-index order.  'pairs': every Gaussian has an
    exact duplicate; 'pile': hundreds share one position (one depth bin overflows -> the sort kernel's bitonic fallback)."""
    from oracle import raster_oracle as ro
    sc = random_scene(P=2400, H=96, W=96, seed=51, scale_mean=0.02, aniso=False)
    if kind == "pairs":
        for k in ("means3D", "scales"):
            sc[k][1200:] = sc[k][:1200]
    else:
        sc["means3D"][300:1000] = sc["means3D"][299]
        sc["scales"][300:1000] = sc["scales"][299]
    color, radii, ctx, rs, _ = _run_cuda(sc)
    v = ctx.views()
    o = ro.forward(**oracle_args(sc), precision="f32")
    k = o.get("keys")
    assert (k[1:] == k[:-1]).sum() > (500 if kind == "pairs" else 300)          # the case really has ties
    np.testing.assert_array_equal(v["keys_sorted"].numpy().view(np.uint64), k)
    np.testing.assert_array_equal(v["vals_sorted"].numpy().view(np.uint32), o.get("vals"))
    assert np.abs(color.cpu().numpy().astype(np.float64) - o.image).mean() <= 1e-4
