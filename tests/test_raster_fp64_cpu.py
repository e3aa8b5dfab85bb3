"""CPU: check the fp64 compositing reference (tests/raster_fp64.py) itself, before any GPU run holds a kernel to it.

1. Fed the fp64 autograd twin's (oracle/raster_twin.py) pixel centres, conics, opacities and depth order, it reproduces the
   twin's image, final_T and n_contrib (n_contrib exactly), and its d_mean2D / d_conic / d_opacity / d_colors, chained through
   the twin's preprocess by autograd, reproduce the twin's full autograd gradients to 1e-10 relative.
2. Fed the fp32 C oracle's xy / conic_o / sorted list, every clear pixel's n_contrib equals the oracle's and the oracle's fp32
   image lies within the reference's error bound: the bound is not too tight for an fp32 composite of the same lists.
"""
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
