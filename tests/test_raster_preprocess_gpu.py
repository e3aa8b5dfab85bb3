"""GPU: the rasterizer's fused K8/K9 (preprocess_bwd_kernel) element by element against the fp64 restatement of
tests/raster_fp64.py (`preprocess_backward`, bound derived in its docstring), and K1's floats (preprocess_fwd_kernel) bit for bit
against the fp32 C oracle and, for SH colours, against fp64 under a derived bound.

K1 -> K7 run through the C ABI: ga_raster_forward_preprocess_ex / _render / ga_raster_backward_ex (per frame, all four kernel
instantiations) and ga_rasterb_forward / _backward (batched).  The restatement starts from the launch's own inputs: means3D,
scales, rotations, scale_modifier, the frame's camera, the radii and STAGED cov3d of the geom buffer, the d_mean2D / d_conic_op
K7 left in the scratch buffer (d_conic_op at align_up(8 B P, 256)), and with SH the coefficients, campos, K1's clamp bits and
K7's dL/drgb.  Every output lies inside finite sentinels that must stay bit-identical.  Inputs the kernel must not use are NaN:
the scales, rotations and SH rows of culled Gaussians (written after the forward, which reads them up to its area cull), scales and
rotations entirely with cov3D_precomp, and every SH coefficient at and beyond (D+1)^2.

Tiers, |got - ref| <= bound on every element of every visible Gaussian: d_means3D, d_scales, d_rotations, d_cov3D, d_sh.  Bit for
bit: d_opacities == d_conic_op.w, d_means2D == (d_mean2D, 0), and zeros in every output of a culled Gaussian.  Each bound must
reject a corrupted reference a plausible bug would produce.  Run with -s for the largest error / bound per tier.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import raster_fp64 as rf
from scenes import oracle_args, random_scene
from sh_scenes import random_shs, sigma_of
from test_raster_gpu import CASES as RASTER_CASES
from test_raster_kernels_gpu import PAD, Sent, align_up, ptr, ratio, stream

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WORST = {}
CLAMP_MARG = [0, 0]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key, (r, where) in sorted(WORST.items()):
        print(f"\nraster preprocess: largest error/bound, {key}: {r:.3g} ({where})")
    print(f"raster preprocess: SH clamp decisions within the bound of 0: {CLAMP_MARG[0]} of {CLAMP_MARG[1]}")


def _lib():
    from gaussianavatar_b200 import _lib
    return _lib


def check(key, where, got, ref, bound, mask):
    r = ratio(got, ref, bound, mask)
    if r > WORST.get(key, (-1.0, ""))[0]:
        WORST[key] = (r, where)
    assert r <= 1.0, f"{key}, {where}: error/bound {r:.4g}"


def rejects(what, bad, ref, bound, mask):
    assert ratio(bad, ref, bound, mask) > 1.0, f"self-check: the bound accepts {what}"


def _row(mask, t):
    return mask.reshape(-1, *([1] * (t.dim() - 1))).expand_as(t)


def check_outputs(where, ref, got, radii):
    """Every visible element within the bound, every culled element exactly 0."""
    vis = radii > 0
    assert torch.equal(ref["vis"], vis)
    assert not bool(ref["marg_overflow"].any()), f"{where}: denom^2 + 1e-7 within the bound of overflow"
    for k, t in got.items():
        if t is None:
            continue
        v, e = ref[k]
        check(k, where, t, v, e, _row(vis, t))
        assert bool((t[~vis] == 0).all()), f"{where}: {k} of a culled Gaussian is not zero"


def check_exact(where, got, d_mean2D, d_conic_op, radii):
    if got.get("d_opacities") is not None:
        assert torch.equal(got["d_opacities"].reshape(-1).view(torch.int32), d_conic_op[:, 3].contiguous().view(torch.int32)), where
    if got.get("d_means2D") is not None:
        m2 = got["d_means2D"]
        assert torch.equal(m2[:, :2].contiguous().view(torch.int32), d_mean2D.contiguous().view(torch.int32)), where
        assert bool((m2[:, 2].view(torch.int32) == 0).all()), where


# ------------------------------------------------------------------------------------------------------------ launches
def run_perframe(sc, mod=1.0, sh=None, cov=False, optional=True, shs_off=0, dsh_off=0, seed=0):
    """One frame through the per-frame ABI.  sh = (D, M) selects SH colours, cov the precomputed covariances; shs_off / dsh_off
    shift shs / d_sh by that many floats (4 bytes: the scalar path).  Returns (reference inputs, outputs, views)."""
    from gaussianavatar_b200.rasterizer import _views
    L = _lib()
    lib = L.lib()
    P, H, W = sc["means3D"].shape[0], sc["H"], sc["W"]
    s = L.GaRasterSettings(P, H, W, float(sc["tanfovx"]), float(sc["tanfovy"]), float(mod))
    t = {k: sc[k].to(DEV).float().contiguous().clone() for k in ("means3D", "scales", "rotations", "opacities", "colors")}
    view = sc["cam"].world_view_transform.to(DEV).float().contiguous()
    proj = sc["cam"].full_proj_transform.to(DEV).float().contiguous()
    campos = sc["cam"].camera_center.to(DEV).float().contiguous()
    cc = L.GaRasterColorCov()
    shs = shs_buf = rgb = clamped = cov3D = None
    if sh is not None:
        D, M = sh
        shs = random_shs(sc, D, M, seed=seed + 3).to(DEV)
        shs_buf = torch.zeros(P * M * 3 + 4, device=DEV)
        dev_shs = shs_buf[shs_off:shs_off + P * M * 3].view(P, M, 3)
        dev_shs.copy_(shs)
        dev_shs[:, (D + 1) ** 2:] = float("nan")                    # the float4 loads read some of these: they must be discarded
        rgb = torch.empty(P, 3, device=DEV)
        clamped = torch.empty(P, dtype=torch.uint8, device=DEV)
        cc.shs, cc.sh_degree, cc.sh_coeffs, cc.campos = ptr(dev_shs), D, M, ptr(campos)
        cc.rgb, cc.clamped = ptr(rgb), ptr(clamped)
    if cov:
        cov3D = sigma_of(sc["scales"], sc["rotations"], mod).to(DEV)
        cc.cov3D_precomp = ptr(cov3D)
        t["scales"].fill_(float("nan"))
        t["rotations"].fill_(float("nan"))
    ccp = ctypes.byref(cc) if (sh is not None or cov) else None
    geom = torch.empty(lib.ga_raster_geom_bytes(P), dtype=torch.uint8, device=DEV)
    img = torch.empty(lib.ga_raster_img_bytes(H, W), dtype=torch.uint8, device=DEV)
    radii = torch.empty(max(P, 1), dtype=torch.int32, device=DEV)
    n = ctypes.c_int64(0)
    L.check(lib.ga_raster_forward_preprocess_ex(ctypes.byref(s), ccp, ptr(t["means3D"]), ptr(t["scales"]), ptr(t["rotations"]),
                                                ptr(t["opacities"]), ptr(view), ptr(proj), ptr(geom), ptr(img), ptr(radii),
                                                ctypes.byref(n), stream()), "preprocess")
    R = int(n.value)
    nb = lib.ga_raster_binning_bytes(R, H, W)
    binning = torch.empty(nb, dtype=torch.uint8, device=DEV)
    bg = sc["bg"].to(DEV).float().contiguous()
    out = torch.empty(3, H, W, device=DEV)
    L.check(lib.ga_raster_forward_render(ctypes.byref(s), ptr(t["colors"] if sh is None else rgb), ptr(bg), ptr(geom), ptr(binning), nb,
                                         R, ptr(img), ptr(out), stream()), "render")
    torch.cuda.synchronize()
    culled = radii[:P] <= 0
    t["colors"][culled] = float("nan")
    t["scales"][culled] = float("nan")
    t["rotations"][culled] = float("nan")
    if sh is not None:
        dev_shs[culled] = float("nan")
    v = _views(1, P, H, W, R, geom, binning, img, radii[:P])[0]
    scratch = torch.full((lib.ga_raster_bwd_scratch_bytes(P) // 4,), float("nan"), device=DEV)
    sizes = dict(d_means3D=3, d_colors=3, d_scales=3, d_rotations=4, d_opacities=1, d_means2D=3, d_cov3D=6)
    o = {k: Sent(c * P, seed + i + 1) for i, (k, c) in enumerate(sizes.items())}
    if cov:
        del o["d_scales"], o["d_rotations"]
    else:
        del o["d_cov3D"]
    if not optional:
        for k in ("d_rotations", "d_opacities", "d_means2D"):
            o.pop(k, None)
    dsh = None
    if sh is not None:
        dsh = Sent(P * M * 3 + dsh_off, seed + 20)
        o["d_sh"] = dsh
    dsh_t = dsh.t[dsh_off:] if dsh is not None else None
    g = torch.Generator().manual_seed(seed + 30)
    dL = torch.randn(3, H, W, generator=g).to(DEV)
    L.check(lib.ga_raster_backward_ex(ctypes.byref(s), ccp, ptr(t["means3D"]), ptr(t["colors"]), ptr(t["scales"]), ptr(t["rotations"]),
                                      ptr(bg), ptr(view), ptr(proj), ptr(radii), ptr(geom), ptr(binning), ptr(img), R, ptr(dL),
                                      ptr(scratch), *[ptr(o[k].t) if k in o else None for k in sizes if k != "d_cov3D"],
                                      ptr(dsh_t), ptr(o["d_cov3D"].t) if "d_cov3D" in o else None, stream()), "backward")
    torch.cuda.synchronize()
    for k, b in o.items():
        b.ok(k)
    if dsh_off:
        assert torch.equal(dsh.t[:dsh_off].view(torch.int32), dsh.before[PAD:PAD + dsh_off].view(torch.int32))
    off = align_up(8 * P) // 4
    d_mean2D, d_conic_op = scratch[:2 * P].view(P, 2), scratch[off:off + 4 * P].view(P, 4)
    got = {k: o[k].t.view(P, -1) for k in ("d_means3D", "d_scales", "d_rotations", "d_cov3D") if k in o}
    if dsh is not None:
        got["d_sh"] = dsh_t.view(P, M, 3)
    exact = {k: o[k].t.view(P, -1) for k in ("d_opacities", "d_means2D") if k in o}
    inp = dict(means=sc["means3D"].to(DEV), view=view, proj=proj, tanfovx=sc["tanfovx"], tanfovy=sc["tanfovy"], H=H, W=W, mod=mod,
               radii=radii[:P], cov3d=v["cov3d"].to(DEV), d_mean2D=d_mean2D, d_conic_op=d_conic_op, depth=v["depth"].to(DEV))
    if not cov:
        inp.update(scales=sc["scales"].to(DEV), rots=sc["rotations"].to(DEV))
    if sh is not None:
        inp.update(shs=shs, D=sh[0], campos=campos, clamped=clamped, d_rgb=o["d_colors"].t.view(P, 3))
    v["rgb"], v["clamped"] = rgb, clamped
    return inp, got, exact, v


def check_frame(where, inp, got, exact, v):
    ref = rf.preprocess_backward(**inp)
    check_outputs(where, ref, got, inp["radii"])
    check_exact(where, exact, inp["d_mean2D"], inp["d_conic_op"], inp["radii"])
    if "shs" in inp:
        check_sh_colour(where, inp, v)
    return ref


def check_sh_colour(where, inp, v):
    """K1's rgb against fp64 under the bound; clamp bits exact except within the bound of 0 (counted, must be rare)."""
    vis = inp["radii"] > 0
    (pv, pe), rgb_ref = rf.sh_forward(inp["means"], inp["shs"], inp["D"], inp["campos"])
    cl = torch.stack([(v["clamped"].long() >> ch) & 1 for ch in range(3)], 1).bool()
    marg = (pv.abs() <= pe) & vis[:, None]
    CLAMP_MARG[0] += int(marg.sum())
    CLAMP_MARG[1] += int(vis.sum()) * 3
    assert int(marg.sum()) <= max(1, int(vis.sum()) // 1000), f"{where}: {int(marg.sum())} clamp decisions within the bound"
    clear = vis[:, None] & ~marg
    assert torch.equal(cl[clear], (pv < 0)[clear]), f"{where}: clamp bits"
    assert bool((v["rgb"][cl & vis[:, None]] == 0).all())
    check("K1 rgb", where, v["rgb"], pv, pe, clear & ~cl)
    assert bool((v["rgb"][~vis] == 0).all()) and bool((v["clamped"][~vis] == 0).all())


def k1_exact_vs_oracle(where, sc, v, radii, mod, rotations=None, opacities=None):
    """K1's staged xy / conic_opacity / depth / cov3d bit for bit against the fp32 C oracle on this frame alone."""
    from oracle import raster_oracle as ro
    a = oracle_args(sc)
    if rotations is not None:
        a["rotations"] = rotations.cpu().numpy()
    if opacities is not None:
        a["opacities"] = opacities.cpu().numpy()
    o = ro.forward(**a, scale_modifier=mod, precision="f32")
    rad = radii.cpu().numpy()
    np.testing.assert_array_equal(rad, o.get("radii"), err_msg=where)
    vis = rad > 0
    for k, ok in (("xy", "xy"), ("conic_opacity", "conic_o"), ("depth", "depth"), ("cov3d", "cov3d")):
        got = v[k].cpu().numpy()[vis].view(np.uint32)
        want = o.get(ok).astype(np.float32)[vis].view(np.uint32)
        assert np.array_equal(got, want), f"{where}: K1 {k} differs from the fp32 oracle on {int((got != want).any(-1).sum()) if got.ndim > 1 else int((got != want).sum())} Gaussians"


# ------------------------------------------------------------------------------------------------------------- scenes
def _eccentric(seed=71):
    P = 3000
    sc = random_scene(P=P, H=128, W=128, seed=seed, scale_mean=0.01)
    g = torch.Generator().manual_seed(seed + 1)
    ecc = torch.exp(torch.rand(P, generator=g) * math.log(100.0))
    sc["scales"] = (0.004 * torch.stack([ecc, torch.ones(P), torch.ones(P)], 1)).contiguous()
    return sc


def _unnormalised(sc, seed=17):
    g = torch.Generator().manual_seed(seed)
    sc["rotations"] = (sc["rotations"] * (0.5 + 1.5 * torch.rand(sc["rotations"].shape[0], 1, generator=g))).float().contiguous()
    return sc


def _near_plane(sc, n=40, seed=19):
    """sc plus n small Gaussians at view depth 0.2005 .. 0.202 (within 1 % of the 0.2 near plane) across the middle of the image."""
    g = torch.Generator().manual_seed(seed)
    V = sc["cam"].world_view_transform.double()                  # p_view = [p, 1] @ V
    pv = torch.stack([(torch.rand(n, generator=g) - 0.5) * 0.12, (torch.rand(n, generator=g) - 0.5) * 0.12,
                      0.2005 + 0.0015 * torch.rand(n, generator=g)], 1).double()
    pw = (pv - V[3, :3]) @ torch.linalg.inv(V[:3, :3])
    add = dict(means3D=pw, scales=0.001 * (1 + torch.rand(n, 3, generator=g)), rotations=torch.randn(n, 4, generator=g),
               opacities=0.1 + 0.9 * torch.rand(n, 1, generator=g), colors=torch.rand(n, 3, generator=g))
    for k, t in add.items():
        sc[k] = torch.cat([sc[k], t.float()]).contiguous()
    return sc


SCENES = {f"case{i}": (lambda c=c: random_scene(**c)) for i, c in enumerate(RASTER_CASES)}
SCENES["case4"] = lambda: _near_plane(random_scene(**RASTER_CASES[4]))
SCENES.update({
    "eccentric": _eccentric,
    "unnormalised": lambda: _unnormalised(random_scene(P=2000, H=160, W=120, seed=16, scale_mean=0.02)),
    "avatar": lambda: random_scene(P=4000, H=192, W=192, seed=18, scale_mean=0.01, aniso=False, opacity_one=True),
})
SCENES.update({f"P{p}": (lambda p=p: random_scene(P=p, H=48, W=64, seed=40 + p, scale_mean=0.03, spread=0.3)) for p in (1, 255, 256, 257)})
MODS = [1.0, 0.37, 2.5]


@pytest.mark.parametrize("mod", MODS)
@pytest.mark.parametrize("name", list(SCENES))
def test_perframe_scenes(name, mod):
    sc = SCENES[name]()
    where = f"per-frame {name} mod={mod}"
    inp, got, exact, v = run_perframe(sc, mod=mod, seed=list(SCENES).index(name))
    ref = check_frame(where, inp, got, exact, v)
    vis = ref["vis"]
    if sc["means3D"].shape[0] > 1:
        assert int(vis.sum()) >= 1
    if mod != 1.0:
        k1_exact_vs_oracle(where, sc, v, inp["radii"], mod)
    dm = got["d_means3D"]
    if name == "case3" and mod >= 1.0:
        # the guard band: visible Gaussians with x_grad_mul = 0 and with y_grad_mul = 0 (at mod 0.37 they are all culled)
        assert bool((vis & ~ref["xgm"]).any()) and bool((vis & ~ref["ygm"]).any()), where
    if name == "case3" and mod == 2.5:
        for bug in ("gate", "tz_unclamped"):
            bad = rf.preprocess_backward(**inp, bug=(bug,))
            rejects(bug, bad["d_means3D"][0], *ref["d_means3D"], _row(vis, dm))
    if name == "case4":
        tvz = ref["tvz"][vis]
        assert int((tvz < 0.2 * 1.01).sum()) >= 10, f"{where}: too few visible Gaussians within 1 % of the near plane"
    if name == "case0":
        for bug, key in (("full_offdiag", "d_scales"), ("no_proj_w", "d_means3D")):
            bad = rf.preprocess_backward(**inp, bug=(bug,))
            rejects(bug, bad[key][0], *ref[key], _row(vis, got[key]))
        if mod != 1.0:
            bad = rf.preprocess_backward(**inp, bug=("scale_mod",))
            rejects("d_scales with one factor of scale_modifier", bad["d_scales"][0], *ref["d_scales"], _row(vis, got["d_scales"]))
    if name == "unnormalised":
        n = inp["rots"].norm(dim=1)
        assert float(n.min()) < 0.6 and float(n.max()) > 1.9
        bad = rf.preprocess_backward(**inp, bug=("norm_quat",))
        rejects("d_rotations of the normalised quaternion", bad["d_rotations"][0], *ref["d_rotations"], _row(vis, got["d_rotations"]))


# (sh (D, M) or None, cov, optional outputs, shs offset, d_sh offset)
MODES = {
    "rgb": (None, False, True, 0, 0),
    "rgb_no_optional": (None, False, False, 0, 0),
    "sh0_M1": ((0, 1), False, True, 0, 0),
    "sh1_M4": ((1, 4), False, True, 0, 0),
    "sh2_M9": ((2, 9), False, True, 0, 0),
    "sh3_M16": ((3, 16), False, True, 0, 0),
    "sh2_M16": ((2, 16), False, True, 0, 0),
    "sh3_M20": ((3, 20), False, True, 0, 0),
    "sh3_M16_shs_off4": ((3, 16), False, True, 1, 0),
    "sh3_M16_dsh_off4": ((3, 16), False, True, 0, 1),
    "rgb_cov": (None, True, True, 0, 0),
    "sh3_M16_cov": ((3, 16), True, True, 0, 0),
}


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("case,mod", [(0, 0.37), (3, 2.5)], ids=["case0", "case3"])
def test_perframe_modes(case, mod, mode):
    sh, cov, optional, shs_off, dsh_off = MODES[mode]
    sc = random_scene(**RASTER_CASES[case])
    where = f"per-frame {mode} case{case} mod={mod}"
    inp, got, exact, v = run_perframe(sc, mod=mod, sh=sh, cov=cov, optional=optional, shs_off=shs_off, dsh_off=dsh_off, seed=case)
    ref = check_frame(where, inp, got, exact, v)
    vis = ref["vis"]
    if cov:
        np.testing.assert_array_equal(v["cov3d"].numpy()[vis.cpu().numpy()],
                                      sigma_of(sc["scales"], sc["rotations"], mod).numpy()[vis.cpu().numpy()])
    if sh is not None and case == 0:
        D, M = sh
        if mode == "sh3_M16":
            for bug, key in (("no_sh_dir", "d_means3D"), ("no_clamp_mask", "d_sh")):
                bad = rf.preprocess_backward(**inp, bug=(bug,))
                rejects(bug, bad[key][0], *ref[key], _row(vis, got[key]))
            assert bool((v["clamped"][vis] != 0).any())
        if M > (D + 1) ** 2 and D < 3:             # at D = 3, coefficient 16 has no basis function to write
            bad = rf.preprocess_backward(**inp, bug=("sh_extra",))
            rejects("coefficient (D+1)^2 not zeroed", bad["d_sh"][0], *ref["d_sh"], _row(vis, got["d_sh"]))


# ------------------------------------------------------------------------------------------------------------- batched
def _cams_scenes(B, P, H, W, seed, mod_scene=None):
    """B frames of one Gaussian set seen from B different cameras (the shipped pose, turned and shifted per frame), with per-frame
    means / scales (small jitters)."""
    from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, TEST_POSE_K, make_camera, scaled_intrinsics
    base = random_scene(P=P, H=H, W=W, seed=seed, scale_mean=0.02, spread=0.9)
    g = torch.Generator().manual_seed(seed + 1)
    scs = []
    for b in range(B):
        K = scaled_intrinsics(TEST_POSE_K, max(H, W))
        K[0, 2], K[1, 2] = W / 2.0, H / 2.0
        ang = 0.08 * (b - B / 2)
        Ry = np.array([[math.cos(ang), 0, math.sin(ang), 0], [0, 1, 0, 0], [-math.sin(ang), 0, math.cos(ang), 0], [0, 0, 0, 1]])
        E = TEST_POSE_EXTRINSIC @ Ry
        E[:3, 3] += np.array([0.05 * b, -0.03 * b, 0.1 * (b % 3)])
        cam = make_camera(K, E, H, W)
        sc = dict(base)
        sc["cam"], sc["tanfovx"], sc["tanfovy"] = cam, math.tan(cam.FovX * 0.5), math.tan(cam.FovY * 0.5)
        sc["means3D"] = (base["means3D"] + 0.01 * torch.randn(P, 3, generator=g)).contiguous()
        sc["scales"] = (base["scales"] * (1 + 0.05 * torch.rand(P, 3, generator=g))).contiguous()
        scs.append(sc)
    return scs


def run_batched(scs, mod=1.0, rot_pf=None, opac_pf=None, capacity=1 << 16, seed=0, nan_culled=True):
    """B frames through ga_rasterb_* with every optional output given; rot_pf [B,P,4] / opac_pf [B,P] per-frame."""
    from gaussianavatar_b200.rasterizer import _views, pack_cameras
    L = _lib()
    lib = L.lib()
    B, P, H, W = len(scs), scs[0]["means3D"].shape[0], scs[0]["H"], scs[0]["W"]
    cams = pack_cameras(torch.stack([s["cam"].world_view_transform for s in scs]), torch.stack([s["cam"].full_proj_transform for s in scs]),
                        [s["tanfovx"] for s in scs], [s["tanfovy"] for s in scs], DEV)
    st = lambda k: torch.stack([s[k] for s in scs]).to(DEV).float().contiguous()
    means, scales, colors = st("means3D"), st("scales"), st("colors")
    rots = (rot_pf if rot_pf is not None else scs[0]["rotations"]).to(DEV).float().contiguous().clone()
    opac = (opac_pf if opac_pf is not None else scs[0]["opacities"].reshape(-1)).to(DEV).float().contiguous()
    bg = scs[0]["bg"].to(DEV).float().contiguous()
    geom = torch.empty(lib.ga_rasterb_geom_bytes(B, P), dtype=torch.uint8, device=DEV)
    img = torch.empty(lib.ga_rasterb_img_bytes(B, H, W), dtype=torch.uint8, device=DEV)
    radii = torch.empty(B, P, dtype=torch.int32, device=DEV)
    out = torch.empty(B, 3, H, W, device=DEV)
    for attempt in range(3):
        d = L.GaRasterBatchDesc(B, P, H, W, capacity, 0 if rot_pf is None else 4 * P, 0 if opac_pf is None else P, float(mod))
        binning = torch.empty(lib.ga_rasterb_binning_bytes(B, H, W, capacity), dtype=torch.uint8, device=DEV)
        L.check(lib.ga_rasterb_forward(ctypes.byref(d), ptr(cams), ptr(bg), ptr(means), ptr(colors), ptr(scales), ptr(rots), ptr(opac),
                                       ptr(geom), ptr(img), ptr(binning), ptr(radii), ptr(out), stream()), "rasterb_forward")
        torch.cuda.synchronize()
        off = lib.ga_rasterb_status(B, H, W, ptr(img)) - img.data_ptr()
        words = img[off:off + 64].view(torch.int32).cpu()
        if int(words[1]) == 0:
            break
        capacity = int(1.5 * int(words[0])) + 1024
    scales_in = scales.clone()
    if nan_culled:
        culled = radii <= 0
        colors[culled] = float("nan")
        scales[culled] = float("nan")
        if rot_pf is not None:
            rots[culled] = float("nan")
    scratch = torch.full((lib.ga_rasterb_bwd_scratch_bytes(B, P) // 4,), float("nan"), device=DEV)
    sizes = dict(d_means3D=3, d_colors=3, d_scales=3, d_rotations=4, d_opacities=1, d_means2D=3)
    o = {k: Sent(c * B * P, seed + i + 1) for i, (k, c) in enumerate(sizes.items())}
    g = torch.Generator().manual_seed(seed + 30)
    dL = torch.randn(B, 3, H, W, generator=g).to(DEV)
    L.check(lib.ga_rasterb_backward(ctypes.byref(d), ptr(cams), ptr(bg), ptr(means), ptr(colors), ptr(scales), ptr(rots), ptr(radii),
                                    ptr(geom), ptr(img), ptr(binning), ptr(dL), ptr(scratch), *[ptr(o[k].t) for k in sizes], stream()),
            "rasterb_backward")
    torch.cuda.synchronize()
    for k, b in o.items():
        b.ok(k)
    vs = _views(B, P, H, W, capacity, geom, binning, img, radii)
    off = align_up(8 * B * P) // 4
    frames = []
    rots_ref = (rot_pf if rot_pf is not None else scs[0]["rotations"][None].expand(B, P, 4)).to(DEV).float()
    for b in range(B):
        d_mean2D = scratch[:2 * B * P].view(B, P, 2)[b]
        d_conic_op = scratch[off:off + 4 * B * P].view(B, P, 4)[b]
        sc = scs[b]
        inp = dict(means=means[b], view=cams[b, 0:16], proj=cams[b, 16:32], tanfovx=float(cams[b, 32]), tanfovy=float(cams[b, 33]),
                   H=H, W=W, mod=mod, radii=radii[b], cov3d=vs[b]["cov3d"].to(DEV), d_mean2D=d_mean2D, d_conic_op=d_conic_op,
                   depth=vs[b]["depth"].to(DEV), scales=scales_in[b], rots=rots_ref[b])
        got = {k: o[k].t.view(B, P, -1)[b] for k in ("d_means3D", "d_scales", "d_rotations")}
        exact = {k: o[k].t.view(B, P, -1)[b] for k in ("d_opacities", "d_means2D")}
        frames.append((inp, got, exact, vs[b]))
    return frames


@pytest.mark.parametrize("B,per_frame,mod", [(1, False, 1.0), (3, True, 0.37), (3, False, 2.5), (8, True, 2.5)])
def test_batched(B, per_frame, mod):
    P, H, W = 1500, 96, 128
    scs = _cams_scenes(B, P, H, W, seed=60 + B)
    g = torch.Generator().manual_seed(61 + B)
    rot = opac = None
    if per_frame:
        rot = scs[0]["rotations"][None] * (0.7 + 0.6 * torch.rand(B, P, 1, generator=g)) + 0.05 * torch.randn(B, P, 4, generator=g)
        opac = 0.1 + 0.9 * torch.rand(B, P, generator=g)
    frames = run_batched(scs, mod=mod, rot_pf=rot, opac_pf=opac, seed=B)
    refs = []
    for b, (inp, got, exact, v) in enumerate(frames):
        where = f"batched B={B} frame {b} per_frame={per_frame} mod={mod}"
        ref = rf.preprocess_backward(**inp)
        check_outputs(where, ref, got, inp["radii"])
        check_exact(where, exact, inp["d_mean2D"], inp["d_conic_op"], inp["radii"])
        refs.append(ref)
        if B > 1:
            sc = dict(scs[b])
            k1_exact_vs_oracle(where, sc, v, inp["radii"], mod, rotations=None if rot is None else rot[b],
                               opacities=None if opac is None else opac[b])
    if B == 3:
        # self-check: two frames' d_means3D swapped
        vis = frames[0][0]["radii"] > 0
        rejects("frames 0 and 1 of d_means3D swapped", frames[1][1]["d_means3D"], *refs[0]["d_means3D"], _row(vis, frames[0][1]["d_means3D"]))
    if per_frame:
        # self-check: frame 0's rotations read for every frame
        b = B - 1
        inp = dict(frames[b][0], rots=frames[0][0]["rots"])
        bad = rf.preprocess_backward(**inp)
        vis = inp["radii"] > 0
        rejects("frame 0's rotations used for every frame", bad["d_rotations"][0], *refs[b]["d_rotations"], _row(vis, frames[b][1]["d_rotations"]))


def test_batched_config3_two_frames():
    """The Gaussians the workload poses at config 3 (200k, 1024^2), B = 2, opacity 1, every optional output given."""
    from gaussianavatar_b200.workload import Stage1Workload
    wl = Stage1Workload(3, 1, device=DEV)
    m = wl.model
    with torch.no_grad():
        means, scales, colors, _ = m._posed_gaussians(torch.tensor([3, 9], device=DEV), 5000)
    c = wl.cam
    scs = [dict(means3D=means[b].float(), scales=scales[b].float(), colors=colors[b].float(), cam=c, H=wl.side, W=wl.side,
                tanfovx=math.tan(c.FovX / 2), tanfovy=math.tan(c.FovY / 2), rotations=m.fix_rotation.float(),
                opacities=m.fix_opacity.float(), bg=m.background.float()) for b in range(2)]
    assert scs[0]["means3D"].shape[0] == 200000
    frames = run_batched(scs, capacity=8 * means.shape[1], seed=91)
    for b, (inp, got, exact, v) in enumerate(frames):
        where = f"config 3 frame {b}"
        ref = rf.preprocess_backward(**inp)
        assert int(ref["vis"].sum()) > 100000
        check_outputs(where, ref, got, inp["radii"])
        check_exact(where, exact, inp["d_mean2D"], inp["d_conic_op"], inp["radii"])


def test_rasterize_batch_autograd():
    """rasterize_batch's autograd: d_means3D / d_scales of the wrapper are the kernel's, against the restatement fed the plan's
    own staged state and scratch (catches an argument mix-up in the wrapper)."""
    from gaussianavatar_b200.rasterizer import RasterBatchPlan, pack_cameras, rasterize_batch
    B, P, H, W, mod = 3, 1200, 80, 112, 1.0
    scs = _cams_scenes(B, P, H, W, seed=77)
    cams = pack_cameras(torch.stack([s["cam"].world_view_transform for s in scs]), torch.stack([s["cam"].full_proj_transform for s in scs]),
                        [s["tanfovx"] for s in scs], [s["tanfovy"] for s in scs], DEV)
    st = lambda k: torch.stack([s[k] for s in scs]).to(DEV).float().contiguous()
    means = st("means3D").requires_grad_(True)
    scales = st("scales").requires_grad_(True)
    colors = st("colors").requires_grad_(True)
    g = torch.Generator().manual_seed(78)
    rot = (scs[0]["rotations"][None] + 0.05 * torch.randn(B, P, 4, generator=g)).to(DEV).contiguous()
    opac = scs[0]["opacities"].reshape(-1).to(DEV)
    bg = scs[0]["bg"].to(DEV).float()
    plan = RasterBatchPlan(B, P, H, W, DEV)
    for _ in range(3):
        img = rasterize_batch(means, colors, scales, rot, opac, cams, bg, plan)
        if plan.check():
            break
    gw = torch.randn(B, 3, H, W, generator=g).to(DEV)
    (img * gw).sum().backward()
    torch.cuda.synchronize()
    vs = plan.views()
    off = align_up(8 * B * P) // 4
    sc = plan.scratch.view(torch.float32)
    for b in range(B):
        inp = dict(means=means.detach()[b], view=cams[b, 0:16], proj=cams[b, 16:32], tanfovx=float(cams[b, 32]), tanfovy=float(cams[b, 33]),
                   H=H, W=W, mod=mod, radii=plan.radii[b], cov3d=vs[b]["cov3d"].to(DEV), d_mean2D=sc[:2 * B * P].view(B, P, 2)[b],
                   d_conic_op=sc[off:off + 4 * B * P].view(B, P, 4)[b], depth=vs[b]["depth"].to(DEV), scales=scales.detach()[b], rots=rot[b])
        ref = rf.preprocess_backward(**inp)
        got = dict(d_means3D=means.grad[b], d_scales=scales.grad[b])
        assert int(ref["vis"].sum()) > 100
        check_outputs(f"rasterize_batch frame {b}", ref, got, inp["radii"])
