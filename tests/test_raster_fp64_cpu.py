"""CPU: check the fp64 compositing reference (tests/raster_fp64.py) itself, before any GPU run holds a kernel to it.

1. Fed the fp64 autograd twin's (oracle/raster_twin.py) pixel centres, conics, opacities and depth order, it reproduces the
   twin's image, final_T and n_contrib (n_contrib exactly), and its d_mean2D / d_conic / d_opacity / d_colors, chained through
   the twin's preprocess by autograd, reproduce the twin's full autograd gradients to 1e-10 relative.
2. Fed the fp32 C oracle's xy / conic_o / sorted list, every clear pixel's n_contrib equals the oracle's and the oracle's fp32
   image lies within the reference's error bound: the bound is not too tight for an fp32 composite of the same lists.
3. The K8/K9 restatement (preprocess_backward): fed the fp64 oracle's staged state and K7 gradients it reproduces the oracle's
   d_means3D / d_scales / d_rotations / d_cov3D / d_sh to 1e-12 relative in all four modes and at scale_modifier 1, 0.37, 2.5; the
   fp32 oracle's K8/K9 lies within its bound; and every corrupted copy the GPU file's self-checks use leaves that bound.
"""
import math

import numpy as np
import pytest
import torch

import raster_fp64 as rf
from oracle import raster_oracle as ro
from oracle.raster_twin import twin_forward
from scenes import oracle_args, random_scene

SCENES = {
    "plain": dict(P=250, H=64, W=80, seed=1, scale_mean=0.03),
    "alpha_cap": dict(P=200, H=50, W=70, seed=2, scale_mean=0.02, aniso=False, opacity_one=True),
    "guard_band": dict(P=200, H=64, W=64, seed=3, scale_mean=0.06, spread=2.5),
    # edges: lists past one 256-entry segment (checkpoint restarts), and partial tiles
    "long_lists": dict(P=1500, H=32, W=32, seed=31, scale_mean=0.006, aniso=False, spread=0.12, opacity=0.03),
    "partial_tiles": dict(P=300, H=17, W=33, seed=6, scale_mean=0.03),
}


def _scene(name):
    c = dict(SCENES[name])
    op = c.pop("opacity", None)
    sc = random_scene(**c)
    if op is not None:
        sc["opacities"] = torch.full_like(sc["opacities"], op)
    return sc


def _tile_lists(rect, order, gx, gy):
    """Per-tile lists in depth order from the twin's rects: ranges [T,2] into one flat point list."""
    lists = [[] for _ in range(gx * gy)]
    for g in order.tolist():
        x0, y0, x1, y1 = rect[g].tolist()
        for ty in range(y0, y1):
            for tx in range(x0, x1):
                lists[ty * gx + tx].append(g)
    ranges, flat = [], []
    for l in lists:
        ranges.append((len(flat), len(flat) + len(l)))
        flat += l
    return torch.tensor(ranges, dtype=torch.int64), torch.tensor(flat, dtype=torch.int64)


def _twin(sc):
    a = {k: sc[k].clone().double().requires_grad_(True) for k in ("means3D", "colors", "opacities", "scales", "rotations")}
    out, aux = twin_forward(a["means3D"], a["colors"], a["opacities"], a["scales"], a["rotations"], sc["bg"],
                            sc["cam"].world_view_transform, sc["cam"].full_proj_transform, sc["tanfovx"], sc["tanfovy"],
                            sc["H"], sc["W"], return_aux=True)
    return out, aux, a


@pytest.mark.parametrize("name", list(SCENES))
def test_reference_reproduces_autograd_twin(name):
    sc = _scene(name)
    H, W = sc["H"], sc["W"]
    out, aux, a = _twin(sc)
    ranges, plist = _tile_lists(aux["rect"], aux["order"], (W + 15) // 16, (H + 15) // 16)
    co = torch.cat([aux["conic"].detach(), a["opacities"].detach().reshape(-1, 1)], 1)
    fr = rf.Frame(aux["pix"].detach(), co, a["colors"].detach(), sc["bg"], ranges, plist, H, W,
                  thresholds=(0.99, 1.0 / 255.0, 1e-4))
    fw = rf.forward(fr)
    if name == "long_lists":
        lens = ranges[:, 1] - ranges[:, 0]
        assert lens.max() > 512 and int(fw["n_contrib"].max()) > 300       # restarts from checkpoints 1 and 2 happen
    assert (fw["image"][0] - out.detach()).abs().max() < 1e-12
    assert (fw["final_T"][0] - aux["final_T"]).abs().max() < 1e-12
    assert torch.equal(fw["n_contrib"], aux["n_contrib"])
    assert not fw["marginal"].any()

    gw = torch.randn(3, H, W, generator=torch.Generator().manual_seed(5)).double()
    bw = rf.backward(fr, fw, gw)
    # chain the reference's per-Gaussian gradients through the twin's preprocess
    surrogate = ((bw["d_mean2D"][0][:, 0] / (0.5 * W)) * aux["pix"][:, 0] + (bw["d_mean2D"][0][:, 1] / (0.5 * H)) * aux["pix"][:, 1]).sum()
    dcon = bw["d_conic"][0]
    surrogate = surrogate + (dcon[:, 0] * aux["conic"][:, 0] + 2 * dcon[:, 1] * aux["conic"][:, 1] + dcon[:, 2] * aux["conic"][:, 2]).sum()
    surrogate = surrogate + (bw["d_opacity"][0][:, 0] * a["opacities"].reshape(-1)).sum() + (bw["d_colors"][0] * a["colors"]).sum()
    keys = ("means3D", "colors", "opacities", "scales", "rotations")
    chained = torch.autograd.grad(surrogate, [a[k] for k in keys], retain_graph=True, allow_unused=True)
    full = torch.autograd.grad((out * gw).sum(), [a[k] for k in keys], allow_unused=True)
    for k, c, f in zip(keys, chained, full):
        c = torch.zeros_like(a[k]) if c is None else c
        assert (c - f).abs().max() <= 1e-10 * f.abs().max().clamp_min(1e-300), k


@pytest.mark.parametrize("name", list(SCENES))
def test_fp32_oracle_within_reference_bound(name):
    sc = _scene(name)
    H, W = sc["H"], sc["W"]
    o = ro.forward(**oracle_args(sc), precision="f32")
    rg = o.get("ranges").astype(np.int64)
    fr = rf.Frame(o.get("xy"), o.get("conic_o"), sc["colors"], sc["bg"], rg, o.get("vals").astype(np.int64), H, W)
    fw = rf.forward(fr)
    clear = ~fw["marginal"]
    assert int(clear.sum()) >= H * W - 2
    assert torch.equal(fw["n_contrib"][clear], torch.from_numpy(o.get("n_contrib").astype(np.int64))[clear])
    img, bound = fw["image"]
    err = (torch.from_numpy(o.image) - img).abs()
    assert bool((err <= bound)[:, clear].all()), float((err / bound.clamp_min(1e-300))[:, clear].max())
    terr = (torch.from_numpy(o.get("final_T")) - fw["final_T"][0]).abs()
    assert bool((terr <= fw["final_T"][1])[clear].all())
    # the bound is a bound, not a blanket: well below the image bar of the aggregate tests
    assert float(bound.max()) < 1e-4


# ------------------------------------------------------------------------------------- K8/K9: preprocess_bwd_kernel
# (shs, cov3D_precomp, degree, coefficients) as in test_raster_sh_gpu.py
PRE_MODES = [(False, False, 0, 0), (True, False, 3, 16), (False, True, 0, 0), (True, True, 1, 4)]
pre_mode_id = lambda m: ("sh%d_M%d" % (m[2], m[3]) if m[0] else "rgb") + ("_cov" if m[1] else "_sr")
PRE_SCENES = {"plain": dict(P=300, H=64, W=80, seed=1, scale_mean=0.03),
              "guard_band": dict(P=1500, H=128, W=128, seed=4, scale_mean=0.05, spread=2.5)}


def _unnormalised(sc, seed):
    g = torch.Generator().manual_seed(seed)
    sc["rotations"] = (sc["rotations"] * (0.5 + 1.5 * torch.rand(sc["rotations"].shape[0], 1, generator=g))).float().contiguous()
    return sc


def _pre_case(name, mode, mod, precision, unnormalised=False):
    """Oracle forward + backward of one scene / mode, and the restatement fed with the oracle's staged state."""
    from oracle import raster_oracle_ex as rox
    from sh_scenes import random_shs, sigma_of
    sh, cov, D, M = mode
    sc = random_scene(**PRE_SCENES[name])
    if unnormalised:
        sc = _unnormalised(sc, 17)
    args, okw = oracle_args(sc), {}
    shs = None
    if sh:
        shs = random_shs(sc, D, M, seed=3)
        args["colors"] = None
        okw.update(shs=shs.numpy(), sh_degree=D, campos=sc["cam"].camera_center.numpy())
    if cov:
        args["scales"] = args["rotations"] = None
        okw.update(cov3D_precomp=sigma_of(sc["scales"], sc["rotations"], mod).numpy())
    o = rox.forward(**args, scale_modifier=mod, precision=precision, **okw)
    gw = torch.randn(3, sc["H"], sc["W"], generator=torch.Generator().manual_seed(5)).numpy()
    gb = o.backward(gw)
    x32 = precision == "f32"
    rd = (lambda a: np.asarray(a, np.float32)) if x32 else (lambda a: a)     # the kernel reads K7's sums as fp32
    dco = rd(np.concatenate([gb["d_conic"], gb["d_opacity"][:, None]], 1))
    kw = dict(scales=None if cov else sc["scales"], rots=None if cov else sc["rotations"], shs=shs, D=D,
              campos=sc["cam"].camera_center if sh else None, clamped=o.get("clamped") if sh else None,
              d_rgb=rd(gb["d_colors"]) if sh else None, exact32=x32, depth=o.get("depth") if x32 else None)
    call = lambda bug=(): rf.preprocess_backward(sc["means3D"], sc["cam"].world_view_transform, sc["cam"].full_proj_transform,
                                                 sc["tanfovx"], sc["tanfovy"], sc["H"], sc["W"], mod, o.get("radii"), o.get("cov3d"),
                                                 rd(gb["d_mean2D"]), dco, bug=bug, **kw)
    return call, gb


PRE_OUT = (("d_means3D", "d_means3D"), ("d_scales", "d_scales"), ("d_rotations", "d_rots"), ("d_cov3D", "d_cov3d"), ("d_sh", "d_sh"))


@pytest.mark.parametrize("mod", [1.0, 0.37, 2.5])
@pytest.mark.parametrize("mode", PRE_MODES, ids=pre_mode_id)
@pytest.mark.parametrize("name", list(PRE_SCENES))
def test_preprocess_reference_reproduces_fp64_oracle(name, mode, mod):
    """Fed the fp64 oracle's staged cov3d / radii and its K7 d_mean2D / d_conic (/ dL/drgb and clamp bits), the restatement in
    plain fp64 reproduces the oracle's K8/K9 outputs."""
    call, gb = _pre_case(name, mode, mod, "f64")
    ref = call()
    assert int(ref["vis"].sum()) > 100
    n = 0
    for k, ok in PRE_OUT:
        if k not in ref:
            continue
        v = ref[k][0]
        want = torch.from_numpy(gb[ok]).reshape(v.shape)
        assert float((v - want).abs().max()) <= 1e-12 * float(want.abs().max()), k
        n += 1
    assert n == 2 + 2 * (not mode[1]) + int(mode[0])


@pytest.mark.parametrize("mod", [1.0, 2.5])
@pytest.mark.parametrize("name", list(PRE_SCENES))
def test_fp32_oracle_within_preprocess_bound(name, mod):
    """The fp32 oracle's K8/K9 (the kernel's expression tree without contraction) lies within the restatement's bound, fed the
    oracle's own fp32 staged state: the bound is not too tight.  SH is left out: the oracle's direction term is another tree."""
    for mode in (PRE_MODES[0], PRE_MODES[2]):
        call, gb = _pre_case(name, mode, mod, "f32")
        ref = call()
        for k, ok in PRE_OUT:
            if k in ref:
                v, e = ref[k]
                err = (torch.from_numpy(gb[ok]).reshape(v.shape) - v).abs()
                assert bool((err <= e).all()), (k, float((err / e.clamp_min(1e-300)).max()))
        if name == "guard_band":
            assert bool((ref["vis"] & ~ref["xgm"]).any()) and bool((ref["vis"] & ~ref["ygm"]).any())
        assert not bool(ref["marg_overflow"].any())


# corruption -> (scene, mode, scale_modifier, unnormalised quaternions, output it shows in)
PRE_BUGS = {
    "gate": ("guard_band", PRE_MODES[0], 2.5, False, "d_means3D"),
    "tz_unclamped": ("guard_band", PRE_MODES[0], 2.5, False, "d_means3D"),
    "scale_mod": ("plain", PRE_MODES[0], 0.37, False, "d_scales"),
    "full_offdiag": ("plain", PRE_MODES[0], 1.0, False, "d_cov3D"),
    "no_proj_w": ("plain", PRE_MODES[0], 1.0, False, "d_means3D"),
    "norm_quat": ("plain", PRE_MODES[0], 1.0, True, "d_rotations"),
    "no_sh_dir": ("plain", PRE_MODES[1], 1.0, False, "d_means3D"),
    "no_clamp_mask": ("plain", PRE_MODES[1], 1.0, False, "d_sh"),
    "sh_extra": ("plain", (True, False, 2, 16), 1.0, False, "d_sh"),
}


@pytest.mark.parametrize("bug", list(PRE_BUGS))
def test_preprocess_bound_rejects_corruption(bug):
    """Each corrupted restatement a plausible kernel bug would match leaves the bound of the true one on some element."""
    name, mode, mod, unnorm, key = PRE_BUGS[bug]
    call, gb = _pre_case(name, mode, mod, "f32", unnormalised=unnorm)
    v, e = call()[key]
    bad = call(bug=(bug,))[key][0]
    r = (bad - v).abs() / e.clamp_min(1e-300)
    r = torch.where(e == 0, torch.where(bad == v, 0.0, math.inf), r)
    assert float(r.max()) > 1.0, bug
