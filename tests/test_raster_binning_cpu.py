"""CPU: pin tests/raster_binning.py, the exact restatement of the rasterizer's tile binning, to the upstream contract.

1. Run on the C oracle's own xy / radii / depth, it reproduces the oracle's rects, tiles touched, sorted keys, sorted values
   and tile ranges bit for bit, on scenes with guard-band rects, Gaussians behind the near plane and equal depths.
2. Its scan gives the stated ranges and status words on a hand-built count array cut at a tile end, one entry before it,
   at a 4096-tile round boundary of the device scan, inside the first frame and not at all.
"""
import numpy as np
import pytest

import raster_binning as rb
from oracle import raster_oracle as ro
from scenes import oracle_args, random_scene

CASES = [
    dict(P=300, H=64, W=80, seed=1, scale_mean=0.03),
    dict(P=2000, H=200, W=136, seed=2, scale_mean=0.02),                       # H, W not multiples of 16
    dict(P=1500, H=128, W=128, seed=4, scale_mean=0.05, spread=2.5),           # guard band / off-screen / clipped rects
    dict(P=800, H=96, W=96, seed=5, scale_mean=0.02, z_extra=2.4),             # many behind the near plane (z <= 0.2)
    dict(P=2400, H=96, W=96, seed=51, scale_mean=0.02, aniso=False, ties="pairs"),   # every Gaussian has an exact duplicate
    dict(P=2400, H=96, W=96, seed=51, scale_mean=0.02, aniso=False, ties="pile"),    # 700 Gaussians share one position
]


def _scene(case):
    case = dict(case)
    ties = case.pop("ties", None)
    sc = random_scene(**case)
    if ties == "pairs":
        for k in ("means3D", "scales"):
            sc[k][1200:] = sc[k][:1200]
    elif ties == "pile":
        sc["means3D"][300:1000] = sc["means3D"][299]
        sc["scales"][300:1000] = sc["scales"][299]
    return sc


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"P{c['P']}_{c['H']}x{c['W']}_s{c['seed']}{c.get('ties', '')}")
def test_restatement_matches_oracle(case):
    sc = _scene(case)
    o = ro.forward(**oracle_args(sc), precision="f32")
    P, H, W = sc["means3D"].shape[0], sc["H"], sc["W"]
    radii = o.get("radii")
    R = o.num_rendered
    r = rb.restate(1, P, H, W, R, o.get("xy").astype(np.float32)[None], radii[None], o.get("depth").astype(np.float32)[None])
    np.testing.assert_array_equal(r["rect"][0], o.get("rect"))
    np.testing.assert_array_equal(r["tiles_touched"][0], o.get("tiles"))
    np.testing.assert_array_equal(r["tiles_touched"][0] == 0, radii == 0)
    assert r["instances"] == R and r["words"][0] == R and r["words"][1] == 0
    np.testing.assert_array_equal(r["keys"], o.get("keys"))
    np.testing.assert_array_equal(r["point_list"], o.get("vals"))
    np.testing.assert_array_equal(r["ranges"], o.get("ranges").astype(np.int64))
    np.testing.assert_array_equal(r["tile_count"][0], (o.get("ranges")[:, 1] - o.get("ranges")[:, 0]).astype(np.int64))
    # what the case is there for
    keys = o.get("keys")
    if case.get("ties"):
        assert (keys[1:] == keys[:-1]).sum() > 300
    if case.get("z_extra"):
        assert (radii == 0).sum() > 100 and (radii > 0).sum() > 50
    if case.get("spread", 0) > 2:
        rc = o.get("rect")[radii > 0]
        gx, gy, _ = rb.grid(H, W)
        assert (rc[:, 0] == 0).any() and (rc[:, 1] == 0).any() and (rc[:, 2] == gx).any() and (rc[:, 3] == gy).any()


def test_restatement_rect_rounds_in_float32():
    """pixx + r rounded to float32 before the + 15: a centre half an ulp of pixx + r below 16 with r = 1 rounds up to 17, so
    the rect ends one tile later than exact arithmetic would put it."""
    x = np.float32(16.0) - np.float32(2.0 ** -20)                          # x + 1 = 17 - 2^-20: a tie, rounded to even (17)
    r = rb.rects(np.array([[x, 40.0]], np.float32), np.array([1]), 64, 64)
    assert r[0, 2] == 2 and int((float(x) + 1.0 + 15.0) // 16) == 1
    r = rb.rects(np.array([[-100.0, 2000.0]], np.float32), np.array([50]), 64, 64)
    np.testing.assert_array_equal(r[0], [0, 4, 0, 4])                        # clamped to [0, gx] / [0, gy]: no area


def _cut_counts():
    """B = 2 frames of T = 2100 tiles (one scan round of 4096 tiles and part of a second); global tile -> count."""
    nz = {0: 300, 7: 2048, 100: 5, 2099: 1, 2100: 4000, 3000: 1, 4095: 10, 4096: 2, 4199: 7}
    c = np.zeros(2 * 2100, np.int64)
    for k, v in nz.items():
        c[k] = v
    return c


# total 6374; ends: t0 300, t7 2348, t100 2353, t2099 2354, t2100 6354, t3000 6355, t4095 6365, t4096 6367, t4199 6374
CUT_CASES = {
    # capacity: (fitting tiles, words 2 (segments), 3 (tiles), 13 (long tiles))
    6374: ([0, 7, 100, 2099, 2100, 3000, 4095, 4096, 4199], 2 + 8 + 1 + 1 + 16 + 1 + 1 + 1 + 1, 9, 2),   # exactly the total
    6373: ([0, 7, 100, 2099, 2100, 3000, 4095, 4096], 2 + 8 + 1 + 1 + 16 + 1 + 1 + 1, 8, 2),              # total - 1
    6365: ([0, 7, 100, 2099, 2100, 3000, 4095], 2 + 8 + 1 + 1 + 16 + 1 + 1, 7, 2),                        # end of tile 4095
    6364: ([0, 7, 100, 2099, 2100, 3000], 2 + 8 + 1 + 1 + 16 + 1, 6, 2),                                  # one entry before
    2348: ([0, 7], 2 + 8, 2, 1),                                                                          # end of tile 7
    2347: ([0], 2, 1, 0),                                                                                 # inside frame 0
    0: ([], 0, 0, 0),
}


@pytest.mark.parametrize("capacity", sorted(CUT_CASES))
def test_scan_capacity_cuts(capacity):
    c = _cut_counts()
    ranges, words = rb.scan(c, 2100, capacity)
    fit, segs, tiles, long_ = CUT_CASES[capacity]
    ends = np.cumsum(c)
    want = np.zeros((c.size, 2), np.int64)
    for t in fit:
        want[t] = (ends[t] - c[t], ends[t])
    np.testing.assert_array_equal(ranges, want)
    assert words[0] == 6374 and words[1] == int(capacity < 6374)
    assert (words[2], words[3], words[13]) == (segs, tiles, long_)
    assert (words[4], words[5], words[6]) == (0, 2354, 6374)              # frame bases: not clamped by the capacity


def test_scan_frame_bases_and_empty_frames():
    c = np.zeros(3 * 10, np.int64)
    c[3], c[25] = 4, 2049                                                   # frame 1 empty
    ranges, words = rb.scan(c, 10, 1 << 20)
    assert words == {0: 2053, 1: 0, 2: 1 + 9, 3: 2, 13: 1, 4: 0, 5: 4, 6: 4, 7: 2053}
    assert ranges[3].tolist() == [0, 4] and ranges[25].tolist() == [4, 2053] and int(ranges.sum()) == 4 + 4 + 2053
