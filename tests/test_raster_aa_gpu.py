"""GPU: the rasterizer's antialiasing setting (upstream's `antialiasing`, Mip-Splatting's screen-space filter) through every layer.

Preprocess forward: with the filter, K1's stored opacity conic_opacity.w matches o rho restated in fp64 from the kernel's own
inputs under the bound of tests/raster_aa_fp64.py, and every other geom field, the radii, the point list and the tile ranges are the
call without it's, bit for bit.  Preprocess backward: every output element against raster_aa_fp64.preprocess_backward, with
d_opacities = gO rho under its bound; Gaussians on both sides of the 2.5e-5 clamp; each bound rejects the bugs named there.
Both APIs, the four per-frame colour / covariance modes, B = 1..8, ragged P and the step's 200k / 1024^2 size.

Then a known answer (an isolated Gaussian's footprint at two sampling rates), the drop-in against the fp64 autograd twin, training,
scenes with each set's own flag, and mattes / depth with the filter.
"""
import contextlib
import math

import numpy as np
import pytest
import torch

import gaussianavatar_b200.rasterizer  # noqa: F401  (binds the unpatched structs before `antialiased` swaps _lib's)
import raster_aa_fp64 as aa
import test_raster_preprocess_gpu as tp
from scenes import random_scene
from test_raster_gpu import CASES as RASTER_CASES

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key, (r, where) in sorted(WORST.items()):
        print(f"\nraster antialiasing: largest error/bound, {key}: {r:.3g} ({where})")


def _L():
    from gaussianavatar_b200 import _lib
    return _lib


@contextlib.contextmanager
def antialiased(on=True):
    """The per-frame settings and batch descriptors the launch helpers of test_raster_preprocess_gpu build (through _lib's names)
    carry the flag."""
    L = _L()
    S0, D0 = L.GaRasterSettings, L.GaRasterBatchDesc

    class S(S0):
        def __init__(self, *a):
            super().__init__(*a)
            self.antialiasing = int(on)

    class D(D0):
        def __init__(self, *a):
            super().__init__(*a)
            self.antialiasing = int(on)
    L.GaRasterSettings, L.GaRasterBatchDesc = S, D
    try:
        yield
    finally:
        L.GaRasterSettings, L.GaRasterBatchDesc = S0, D0


def check(key, where, got, ref, bound, mask):
    r = tp.ratio(got, ref, bound, mask)
    if r > WORST.get(key, (-1.0, ""))[0]:
        WORST[key] = (r, where)
    assert r <= 1.0, f"{key}, {where}: error/bound {r:.4g}"


def rejects(what, bad, ref, bound, mask):
    assert tp.ratio(bad, ref, bound, mask) > 1.0, f"self-check: the bound accepts {what}"


def same_bits(a, b):
    a, b = torch.as_tensor(a), torch.as_tensor(b)
    if a.dtype == torch.float32:
        a, b = a.view(torch.int32), b.view(torch.int32)
    return torch.equal(a.cpu(), b.cpu())


def check_forward(where, v_on, v_off, opacities, inp, bug=()):
    """K1 with the filter against the same call without it (bit for bit except conic_opacity.w) and against fp64."""
    for k in ("radii", "depth", "xy", "cov3d", "tiles_touched", "rect", "ranges", "tile_count", "num_rendered"):
        assert same_bits(v_on[k], v_off[k]) if k != "num_rendered" else v_on[k] == v_off[k], f"{where}: {k} differs with the filter"
    co_on, co_off = v_on["conic_opacity"], v_off["conic_opacity"]
    assert same_bits(co_on[:, :3].contiguous(), co_off[:, :3].contiguous()), f"{where}: conic differs with the filter"
    if "vals_sorted" in v_off:
        assert same_bits(v_on["vals_sorted"], v_off["vals_sorted"]), f"{where}: point list differs with the filter"
    vis = (v_on["radii"] > 0).to(DEV)
    (wv, we), parts = aa.forward_opacity(inp["cov3d"], inp["means"], inp["view"], inp["tanfovx"], inp["tanfovy"], inp["H"], inp["W"],
                                         opacities, bug=bug)
    got = co_on[:, 3].to(DEV)
    if bug:
        return got, wv, we, vis
    check("K1 o rho", where, got, wv, we, vis)
    assert bool((co_on[~vis.cpu(), 3] == 0).all())
    return parts


def check_backward(where, inp, got, exact, co_w):
    ref = aa.preprocess_backward(co_w=co_w, **inp)
    vis = ref["vis"]
    ok = vis & ~ref["marg_clamp"]
    # a needle's det0 = a0 c0 - b^2 cancels, so its r can lie within the bound of 2.5e-5: such Gaussians are left out, and must
    # stay a minority
    assert int(ref["marg_clamp"].sum()) <= max(8, int(vis.sum()) // 2), f"{where}: clamp decisions within the bound"
    assert not bool(ref["marg_overflow"].any())
    for k, t in got.items():
        if t is None:
            continue
        v, e = ref[k]
        check(k, where, t, v, e, tp._row(ok, t))
        assert bool((t[~vis] == 0).all()), f"{where}: {k} of a culled Gaussian is not zero"
    if exact.get("d_opacities") is not None:
        d = exact["d_opacities"].reshape(-1)
        check("d_opacities", where, d, *ref["d_opacities"], ok)
        assert bool((d[~vis] == 0).all())
    if exact.get("d_means2D") is not None:
        m2 = exact["d_means2D"]
        assert same_bits(m2[:, :2].contiguous(), inp["d_mean2D"].contiguous()), where
    return ref


def run_pair(run, *args, **kw):
    """run(*args) with and without the filter: (on, off)."""
    with antialiased(True):
        on = run(*args, **kw)
    with antialiased(False):
        off = run(*args, **kw)
    return on, off


# --------------------------------------------------------------------------------------------- per-frame, the four modes
def _thin(sc, frac=0.5, seed=5):
    """About frac of the Gaussians become needles (two scales of 1e-7): their projected covariance is all but singular, r < 2.5e-5."""
    g = torch.Generator().manual_seed(seed)
    P = sc["scales"].shape[0]
    pick = torch.rand(P, generator=g) < frac
    s = sc["scales"].clone()
    s[pick, 1:] = 1e-7
    sc["scales"] = s.contiguous()
    return sc


MODES = {"rgb": (None, False), "sh3_M16": ((3, 16), False), "rgb_cov": (None, True), "sh3_M16_cov": ((3, 16), True)}


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("case,mod", [(0, 0.37), (3, 2.5), (1, 1.0)], ids=["case0", "case3", "case1"])
def test_perframe_modes(case, mod, mode):
    sh, cov = MODES[mode]
    sc = _thin(random_scene(**RASTER_CASES[case]), seed=case)
    where = f"per-frame {mode} case{case} mod={mod}"
    (inp, got, exact, v), (_, _, _, v_off) = run_pair(tp.run_perframe, sc, mod=mod, sh=sh, cov=cov, seed=case)
    check_forward(where, v, v_off, sc["opacities"].reshape(-1), inp)
    ref = check_backward(where, inp, got, exact, v["conic_opacity"][:, 3])
    vis = ref["vis"]
    act, ok = ref["active"], vis & ~ref["marg_clamp"]
    assert int((ok & act).sum()) >= 10 and int((ok & ~act).sum()) >= 5, f"{where}: both sides of the clamp"
    if case == 0 and mode == "rgb":
        # each bound rejects a plausible bug
        bad = aa.preprocess_backward(co_w=v["conic_opacity"][:, 3], bug=("no_rho_dopac",), **inp)
        rejects("dL/do without rho", bad["d_opacities"][0], *ref["d_opacities"], vis & ~ref["marg_clamp"])
        for bug in ("no_drho", "dilated_num", "clamp_grad"):
            bad = aa.preprocess_backward(co_w=v["conic_opacity"][:, 3], bug=(bug,), **inp)
            k = "d_scales"
            rejects(bug, bad[k][0], *ref[k], tp._row(vis & ~ref["marg_clamp"], got[k]))
        got_w, wv, we, visd = check_forward(where, v, v_off, sc["opacities"].reshape(-1), inp, bug=("dilated_num",))
        rejects("K1 with det1 as r's numerator", got_w, wv, we, visd)


# ------------------------------------------------------------------------------------------------------------ batched
@pytest.mark.parametrize("B,per_frame,mod", [(1, False, 1.0), (3, True, 0.37), (8, True, 2.5)])
def test_batched(B, per_frame, mod):
    P, H, W = 1500 + 37 * B, 96, 128                 # ragged P
    scs = tp._cams_scenes(B, P, H, W, seed=160 + B)
    for s in scs:
        _thin(s, frac=0.3, seed=B)
    g = torch.Generator().manual_seed(161 + B)
    rot = opac = None
    if per_frame:
        rot = scs[0]["rotations"][None] * (0.7 + 0.6 * torch.rand(B, P, 1, generator=g)) + 0.05 * torch.randn(B, P, 4, generator=g)
        opac = 0.1 + 0.9 * torch.rand(B, P, generator=g)
    on, off = run_pair(tp.run_batched, scs, mod=mod, rot_pf=rot, opac_pf=opac, seed=B)
    for b in range(B):
        where = f"batched B={B} frame {b}"
        inp, got, exact, v = on[b]
        o = (opac[b] if opac is not None else scs[0]["opacities"].reshape(-1))
        check_forward(where, v, off[b][3], o, inp)
        check_backward(where, inp, got, exact, v["conic_opacity"][:, 3])


def test_batched_config3_two_frames():
    """The Gaussians the workload poses at config 3 (200k, 1024^2), B = 2, with the filter."""
    from gaussianavatar_b200.workload import Stage1Workload
    wl = Stage1Workload(3, 1, device=DEV)
    m = wl.model
    with torch.no_grad():
        means, scales, colors, _ = m._posed_gaussians(torch.tensor([3, 9], device=DEV), 5000)
    c = wl.cam
    scs = [dict(means3D=means[b].float(), scales=scales[b].float(), colors=colors[b].float(), cam=c, H=wl.side, W=wl.side,
                tanfovx=math.tan(c.FovX / 2), tanfovy=math.tan(c.FovY / 2), rotations=m.fix_rotation.float(),
                opacities=m.fix_opacity.float(), bg=m.background.float()) for b in range(2)]
    on, off = run_pair(tp.run_batched, scs, capacity=8 * means.shape[1], seed=91)
    for b in range(2):
        inp, got, exact, v = on[b]
        where = f"config 3 frame {b}"
        check_forward(where, v, off[b][3], scs[b]["opacities"].reshape(-1), inp)
        ref = check_backward(where, inp, got, exact, v["conic_opacity"][:, 3])
        assert int(ref["vis"].sum()) > 100000


# ------------------------------------------------------------------------------------------------------------ depth backward
def test_depth_train_backward():
    """ga_rasterb_backward_depth with the filter: its preprocess backward (the kZ variant) adds the same terms.  The depth term's
    own contribution to d_means3D is the kernel's d_z times the view z row, checked through the colour-only difference."""
    from gaussianavatar_b200.rasterizer import (RasterBatchPlan, pack_cameras, rasterize_batch, rasterize_batch_with_depth)
    B, P, H, W = 2, 1300, 80, 96
    scs = tp._cams_scenes(B, P, H, W, seed=300)
    cams = pack_cameras(torch.stack([s["cam"].world_view_transform for s in scs]), torch.stack([s["cam"].full_proj_transform for s in scs]),
                        [s["tanfovx"] for s in scs], [s["tanfovy"] for s in scs], DEV)
    st = lambda k: torch.stack([s[k] for s in scs]).to(DEV).float().contiguous()
    rot, opac, bg = scs[0]["rotations"].to(DEV).float(), scs[0]["opacities"].reshape(-1).to(DEV), scs[0]["bg"].to(DEV).float()
    g = torch.Generator().manual_seed(301)
    gw = torch.randn(B, 3, H, W, generator=g).to(DEV)
    grads = {}
    for depth in (False, True):
        plan = RasterBatchPlan(B, P, H, W, DEV, antialiasing=True)
        means, scales, colors = st("means3D").requires_grad_(True), st("scales").requires_grad_(True), st("colors").requires_grad_(True)
        for _ in range(3):
            out = (rasterize_batch_with_depth if depth else rasterize_batch)(means, colors, scales, rot, opac, cams, bg, plan)
            if plan.check():
                break
        img = out[0] if depth else out
        (img * gw).sum().backward()
        torch.cuda.synchronize()
        grads[depth] = (means.grad.clone(), scales.grad.clone(), plan)
    # with a zero depth gradient the depth backward is the colour backward: same kernels' sums, so equal up to the atomics' order
    for a, b in zip(grads[False][:2], grads[True][:2]):
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-6 * float(a.abs().max()))
    # and against the restatement from the depth plan's own state
    plan = grads[True][2]
    vs = plan.views()
    off = tp.align_up(8 * B * P) // 4
    sc = plan.depth_scratch.view(torch.float32)
    for b in range(B):
        inp = dict(means=st("means3D")[b], view=cams[b, 0:16], proj=cams[b, 16:32], tanfovx=float(cams[b, 32]), tanfovy=float(cams[b, 33]),
                   H=H, W=W, mod=1.0, radii=plan.radii[b], cov3d=vs[b]["cov3d"].to(DEV), d_mean2D=sc[:2 * B * P].view(B, P, 2)[b],
                   d_conic_op=sc[off:off + 4 * B * P].view(B, P, 4)[b], depth=vs[b]["depth"].to(DEV), scales=st("scales")[b], rots=rot)
        ref = aa.preprocess_backward(co_w=vs[b]["conic_opacity"][:, 3], **inp)
        ok = ref["vis"] & ~ref["marg_clamp"]
        check("depth-train d_scales", f"depth backward frame {b}", grads[True][1][b], *ref["d_scales"], tp._row(ok, grads[True][1][b]))


# ------------------------------------------------------------------------------------------------------------ known answer
def _isolated(side, sigma_px, o=0.9):
    """One isotropic Gaussian in front of a camera of side x side pixels whose 2D standard deviation is sigma_px."""
    from gaussianavatar_b200.camera import make_camera
    f = float(side)                                       # focal length in pixels (90 degree field of view... about 53)
    K = np.array([[f, 0, side / 2.0], [0, f, side / 2.0], [0, 0, 1.0]])
    E = np.eye(4)
    cam = make_camera(K, E, side, side)
    z = 4.0
    s = sigma_px * z / f                                  # world standard deviation
    sc = dict(means3D=torch.tensor([[0.0, 0.0, z]]), scales=torch.full((1, 3), s), rotations=torch.tensor([[1.0, 0, 0, 0]]),
              opacities=torch.tensor([[o]]), colors=torch.ones(1, 3), bg=torch.zeros(3), cam=cam, H=side, W=side,
              tanfovx=math.tan(cam.FovX * 0.5), tanfovy=math.tan(cam.FovY * 0.5))
    return sc


def _mass(sc, antialiasing):
    """Sum of alpha over the image x pixel area (in units of the 256^2 image's pixel), through the drop-in."""
    from gaussianavatar_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer
    c = sc["cam"]
    rs = GaussianRasterizationSettings(sc["H"], sc["W"], sc["tanfovx"], sc["tanfovy"], sc["bg"].to(DEV), 1.0,
                                       c.world_view_transform.to(DEV), c.full_proj_transform.to(DEV), 0, c.camera_center.to(DEV),
                                       False, False, antialiasing)
    img, _ = GaussianRasterizer(rs)(means3D=sc["means3D"].to(DEV), means2D=torch.zeros(0, device=DEV), opacities=sc["opacities"].to(DEV),
                                    colors_precomp=sc["colors"].to(DEV), scales=sc["scales"].to(DEV), rotations=sc["rotations"].to(DEV))
    return float(img[0].double().sum()) * (256.0 / sc["H"]) ** 2


def test_known_answer_footprint():
    """sigma 0.25 px at 256^2 and the same Gaussian at 1024^2 (sigma 1 px): with the filter both footprints integrate to
    2 pi o sqrt(det Sigma2) (in 256^2 pixels); without it they differ by the dilation's factor, derived below."""
    o, thr = 0.9, 1.0 / 255.0
    small, big = _isolated(256, 0.25, o), _isolated(1024, 1.0, o)
    want = 2.0 * math.pi * o * 0.25 ** 2                   # 2 pi o sqrt(det Sigma2), Sigma2 = 0.0625 I in 256^2 pixels
    got, tol = {}, {}
    for sc, s in ((small, 0.25), (big, 1.0)):
        # the filtered splat: variance s^2 + 0.3, opacity o rho with rho = s^2 / (s^2 + 0.3); the mass of that Gaussian inside the
        # 1/255 cut-off, in 256^2 pixels, differs from `want` by the cut-off alone
        var = s * s + 0.3
        area = (256.0 / sc["H"]) ** 2
        m = aa.truncated_gaussian_mass(o * s * s / var, math.sqrt(var), math.sqrt(var), thr) * area
        assert 0 < want - m <= 2 * math.pi * var * thr * area + 1e-12
        # the pixel sum of a Gaussian of variance var on the unit grid is its integral times 1 + O(exp(-2 pi^2 var)) per axis
        # (Poisson summation); the cut-off's edge adds less than the mass of a one-pixel ring at alpha = 1/255
        tol[s] = 4 * math.exp(-2 * math.pi ** 2 * var) * m + 2 * math.pi * math.sqrt(var) * 3.5 * thr * area
        got[s] = _mass(sc, True)
        assert abs(got[s] - m) <= tol[s], (sc["H"], got[s], m, tol[s])
        assert abs(got[s] - want) <= (want - m) + tol[s], (sc["H"], got[s], want)
    assert abs(got[0.25] - got[1.0]) <= 2 * math.pi * 1.3 * thr + tol[0.25] + tol[1.0]
    # without the filter each splat is the dilated Gaussian at opacity o: in 256^2 pixels variance 0.0625 + 0.3 against
    # (1 + 0.3) / 16, a ratio of 0.3625 / 0.08125 = 4.46 (4.5 x, less the cut-off's share)
    m_small = aa.truncated_gaussian_mass(o, math.sqrt(0.3625), math.sqrt(0.3625), thr)
    m_big = aa.truncated_gaussian_mass(o, math.sqrt(1.3), math.sqrt(1.3), thr) / 16.0
    ratio = m_small / m_big
    assert 4.4 < ratio < 4.5
    got_ratio = _mass(small, False) / _mass(big, False)
    assert abs(got_ratio - ratio) <= 0.02 * ratio, (got_ratio, ratio, got)


# ------------------------------------------------------------------------------------------------------------ drop-in
@pytest.mark.parametrize("sh", [False, True])
@pytest.mark.parametrize("cov", [False, True])
def test_dropin_vs_twin(sh, cov):
    """GaussianRasterizer(antialiasing=True) against the fp64 autograd twin fed opacities o rho(Sigma2), rho differentiable."""
    from oracle.raster_twin_ex import sigma_matrix, twin_forward_ex
    from gaussianavatar_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer
    from sh_scenes import random_shs, sigma_of
    sc = random_scene(**RASTER_CASES[0])
    P = sc["means3D"].shape[0]
    c = sc["cam"]
    rs = GaussianRasterizationSettings(sc["H"], sc["W"], sc["tanfovx"], sc["tanfovy"], sc["bg"].to(DEV), 1.0,
                                       c.world_view_transform.to(DEV), c.full_proj_transform.to(DEV), 3, c.camera_center.to(DEV),
                                       False, False, True)
    leaves = dict(means3D=sc["means3D"], opacities=sc["opacities"])
    if sh:
        leaves["shs"] = random_shs(sc, 3, 16, seed=2)
    else:
        leaves["colors_precomp"] = sc["colors"]
    if cov:
        leaves["cov3D_precomp"] = sigma_of(sc["scales"], sc["rotations"], 1.0)
    else:
        leaves.update(scales=sc["scales"], rotations=sc["rotations"])
    dev_leaves = {k: v.to(DEV).float().contiguous().requires_grad_(True) for k, v in leaves.items()}
    img, radii = GaussianRasterizer(rs)(means2D=torch.zeros(0, device=DEV), **dev_leaves)
    gw = torch.randn(3, sc["H"], sc["W"], generator=torch.Generator().manual_seed(4)).to(DEV)
    (img * gw).sum().backward()
    # the twin in float64 on the CPU
    t = {k: v.detach().double().cpu().requires_grad_(True) for k, v in dev_leaves.items()}
    if cov:
        S3 = sigma_matrix(t["cov3D_precomp"])
    else:
        from oracle.raster_twin import quat_to_rot
        R = quat_to_rot(t["rotations"])
        S3 = R @ torch.diag_embed(t["scales"] * t["scales"]) @ R.transpose(1, 2)
    a0, b, c0 = aa.sigma2_64(t["means3D"], S3, c.world_view_transform.double(), sc["tanfovx"], sc["tanfovy"], sc["H"], sc["W"])
    op = t["opacities"].reshape(-1) * aa.rho64(a0, b, c0)
    img_ref = twin_forward_ex(t["means3D"], t.get("colors_precomp"), op[:, None], t.get("scales"), t.get("rotations"),
                              sc["bg"].double(), c.world_view_transform.double(), c.full_proj_transform.double(), sc["tanfovx"],
                              sc["tanfovy"], sc["H"], sc["W"], shs=t.get("shs"), sh_degree=3, campos=c.camera_center.double(),
                              cov3D_precomp=t.get("cov3D_precomp"))
    (img_ref * gw.double().cpu()).sum().backward()
    assert float((img.detach().double().cpu() - img_ref.detach()).abs().mean()) <= 1e-4
    for k in dev_leaves:
        gk, rk = dev_leaves[k].grad.double().cpu(), t[k].grad
        rel = float((gk - rk).norm() / (rk.norm() + 1e-30))
        assert rel < 5e-3, f"{k}: rel-L2 {rel:.3g}"


# ------------------------------------------------------------------------------------------------------------ scenes, mattes, depth
def _scene_of(sc, aa_on):
    from gaussianavatar_b200.scene import GaussianScene
    from sh_scenes import random_shs
    P = sc["means3D"].shape[0]
    q = sc["rotations"] / sc["rotations"].norm(dim=1, keepdim=True)
    return GaussianScene(sc["means3D"].float(), sc["scales"].float(), q.float().contiguous(), sc["opacities"].reshape(-1).float(),
                         random_shs(sc, 1, 4, seed=8).float(), 1, aa_on).to(DEV)


def test_scene_only_matches_dropin():
    """A scene-only composite with GaRasterScene.antialiasing equals the per-frame drop-in with antialiasing=True on the same
    Gaussians (the existing scene tests' bound), and with the flag off differs."""
    from gaussianavatar_b200.rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, RasterBatchPlan, pack_cameras,
                                                rasterize_batch_scene)
    sc = random_scene(P=3000, H=96, W=128, seed=12, scale_mean=0.02)
    c = sc["cam"]
    imgs = {}
    for on in (True, False):
        scene = _scene_of(sc, on)
        cams = pack_cameras(c.world_view_transform[None], c.full_proj_transform[None], [sc["tanfovx"]], [sc["tanfovy"]], DEV,
                            campos=c.camera_center[None])
        plan = RasterBatchPlan(1, 0, sc["H"], sc["W"], DEV, static_P=len(scene))
        z = torch.zeros(1, 0, 3, device=DEV)
        with torch.no_grad():
            for _ in range(3):
                out = rasterize_batch_scene(z, z, z, torch.zeros(0, 4, device=DEV), torch.zeros(0, device=DEV), cams, sc["bg"].to(DEV), plan,
                                            scene)
                if plan.check():
                    break
        rs = GaussianRasterizationSettings(sc["H"], sc["W"], sc["tanfovx"], sc["tanfovy"], sc["bg"].to(DEV), 1.0,
                                           c.world_view_transform.to(DEV), c.full_proj_transform.to(DEV), 1, c.camera_center.to(DEV),
                                           False, False, on)
        with torch.no_grad():
            ref, _ = GaussianRasterizer(rs)(means3D=scene.means3D, means2D=torch.zeros(0, device=DEV), opacities=scene.opacities[:, None],
                                            shs=scene.shs, scales=scene.scales, rotations=scene.rotations)
        assert float((out[0] - ref).abs().max()) <= 2e-5, on
        imgs[on] = out[0]
    assert float((imgs[True] - imgs[False]).abs().max()) > 1e-2


def test_mixed_flags_each_set_its_own():
    """Avatar (dynamic set) off, scene on and the other way round: each set's conic_opacity.w is that set's own, bit for bit what
    the set gets rendered alone with its flag; everything else is unchanged."""
    from gaussianavatar_b200.rasterizer import RasterBatchPlan, pack_cameras, rasterize_batch_scene
    dyn = random_scene(P=900, H=96, W=128, seed=31, scale_mean=0.02)
    stat = random_scene(P=1100, H=96, W=128, seed=32, scale_mean=0.02)
    c = dyn["cam"]
    cams = pack_cameras(c.world_view_transform[None], c.full_proj_transform[None], [dyn["tanfovx"]], [dyn["tanfovy"]], DEV,
                        campos=c.camera_center[None])
    m = dyn["means3D"][None].to(DEV).float().contiguous()
    s = dyn["scales"][None].to(DEV).float().contiguous()
    col = dyn["colors"][None].to(DEV).float().contiguous()
    rot, opac = dyn["rotations"].to(DEV).float().contiguous(), dyn["opacities"].reshape(-1).to(DEV).float()
    views = {}
    for f_dyn in (False, True):
        for f_stat in (False, True):
            plan = RasterBatchPlan(1, 900, 96, 128, DEV, static_P=1100, antialiasing=f_dyn)
            with torch.no_grad():
                for _ in range(3):
                    rasterize_batch_scene(m, col, s, rot, opac, cams, dyn["bg"].to(DEV), plan, _scene_of(stat, f_stat))
                    if plan.check():
                        break
            views[f_dyn, f_stat] = plan.views()[0]
    for fd in (False, True):
        for fs in (False, True):
            v = views[fd, fs]
            for k in ("radii", "xy", "depth", "rect"):
                assert same_bits(v[k], views[False, False][k]), k
            w = v["conic_opacity"][:, 3]
            assert same_bits(w[:900], views[fd, not fs]["conic_opacity"][:900, 3]), "the dynamic set's opacity follows the scene's flag"
            assert same_bits(w[900:], views[not fd, fs]["conic_opacity"][900:, 3]), "the scene's opacity follows the avatar's flag"
    vis = views[True, True]["radii"] > 0
    assert bool((views[True, True]["conic_opacity"][vis, 3] < views[False, False]["conic_opacity"][vis, 3]).all())


def test_mattes_and_depth_with_filter():
    """With the filter on, the mattes / depth pass leave the image, radii and buffers of the colour-only call bit for bit, and the
    mattes sum to the colour call's 1 - final T (the same weights)."""
    from gaussianavatar_b200.rasterizer import (RasterBatchPlan, pack_cameras, rasterize_batch, rasterize_batch_depth,
                                                rasterize_batch_mattes)
    B, P, H, W = 2, 1500, 96, 128
    scs = tp._cams_scenes(B, P, H, W, seed=410)
    cams = pack_cameras(torch.stack([s["cam"].world_view_transform for s in scs]), torch.stack([s["cam"].full_proj_transform for s in scs]),
                        [s["tanfovx"] for s in scs], [s["tanfovy"] for s in scs], DEV)
    st = lambda k: torch.stack([s[k] for s in scs]).to(DEV).float().contiguous()
    args = (st("means3D"), st("colors"), st("scales"), scs[0]["rotations"].to(DEV).float(), scs[0]["opacities"].reshape(-1).to(DEV),
            cams, scs[0]["bg"].to(DEV).float())
    plan = RasterBatchPlan(B, P, H, W, DEV, capacity=1 << 18, antialiasing=True)
    with torch.no_grad():
        img = rasterize_batch(*args, plan)
        assert plan.check()
        T = plan.views()
        img_m, mattes = rasterize_batch_mattes(*args, plan, [0, 700, P])
        img_d, mattes_d, depth = rasterize_batch_depth(*args, plan, first=[0, 700, P])
    assert same_bits(img, img_m) and same_bits(img, img_d) and same_bits(mattes, mattes_d)
    for b in range(B):
        one_minus_T = 1.0 - T[b]["final_T"].to(DEV)
        assert float((mattes[b].sum(0) - one_minus_T).abs().max()) <= 1e-5
    assert float(depth[:, 0].max()) > 0


# ------------------------------------------------------------------------------------------------------------ training
@pytest.mark.tf32
def test_training_with_filter():
    """ModelParams.antialiasing: graphed and eager stage-1 steps agree and the loss falls over a short run (the depth term's backward
    with the filter is test_depth_train_backward's)."""
    from gaussianavatar_b200.trainer import Stage1Trainer
    from gaussianavatar_b200.workload import Stage1Workload
    losses = {}
    for graphs in (True, False):
        torch.manual_seed(0)
        wl = Stage1Workload(1, 2, device=DEV, N=4000, S=64, side=128, inp_posmap_size=32)
        wl.model.antialiasing = True
        wl.make_ground_truth()
        tr = Stage1Trainer(wl.model, use_graph=graphs)
        ls = [float(tr.step(wl.device_batch(wl.frame_ids(i)), 5000 + i, epoch=1)) for i in range(30)]
        tr.finish()
        losses[graphs] = ls
        assert all(math.isfinite(x) for x in ls)
        assert np.mean(ls[-5:]) < np.mean(ls[:5]), ls
        assert bool(tr._graphs) == graphs
        assert all(k[4] for k in tr._graphs), "the graph key carries the antialiasing flag"
    np.testing.assert_allclose(losses[True][:3], losses[False][:3], rtol=2e-3)
