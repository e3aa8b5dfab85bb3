"""GPU: the rasterizer's tile binning (K1's per-tile counts, the K2 scan, the K3 scatter and the K4 per-tile sort) exactly against
tests/raster_binning.py, restated from each forward's own K1 state (xy, radii, depth bits).

Every case compares rect, tiles_touched, tile_count, the global tile ranges, the point list and status words 0-3, 4..4+B and 13
with the restatement bit for bit (under overflow, only what is documented: ranges and status words), and keeps every output it
writes (images, depth maps, the binning buffer) inside finite sentinel words that must stay unchanged.  Each case also asserts
from host-side counts that it reaches the paths it exists for; run with -s to see them.

  A. Sort ladder: one tile per (list length, depth pattern), through every sort instance (plain, depth, scene, scene + depth)
     and the per-frame API; the plain variant's compositing and backward under check_frame's fp64 bounds.
  B. The shared-memory tile table's fallback at 1920x1080: CTAs whose rects touch more than 4096 distinct tiles, and 3000-4096.
  C. The scan across 16 rounds of 4096 tiles (B = 8 at 1920x1080) and capacity cuts at the total, one below it, a round
     boundary and inside frame 0; plan.check() grows the buffer and the re-run matches.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import raster_binning as rb
import raster_fp64 as rf
from gaussianavatar_b200 import _lib as GL
from gaussianavatar_b200.camera import make_camera
from gaussianavatar_b200.rasterizer import RasterBatchPlan, _grab, pack_cameras, rasterize_batch
from gaussianavatar_b200.scene import GaussianScene
from test_depth_gpu import _mean_from
from test_raster_kernels_gpu import _unproject, check, check_frame, run_batched

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
PAD = 1024                       # sentinel floats on each side of a guarded buffer (4 KB: the inner buffer keeps its alignment)
REACHED = []


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for line in REACHED:
        print(f"\nraster binning: {line}")


def ptr(t):
    return None if t is None else t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


class Guard:
    """An output of nbytes (whole floats) inside PAD finite sentinel floats on each side; `ok()` checks the sentinels."""

    def __init__(self, nbytes, seed):
        self.n = -(-int(nbytes) // 4)
        g = torch.Generator(device=DEV).manual_seed(seed)
        self.buf = torch.randn(self.n + 2 * PAD, device=DEV, generator=g) * 1000.0
        self.before = self.buf.clone()
        self.f = self.buf[PAD:PAD + self.n]
        self.u8 = self.f.view(torch.uint8)[:int(nbytes)]

    def ok(self, where):
        d = self.buf.view(torch.int32) != self.before.view(torch.int32)
        d[PAD:PAD + self.n] = False
        assert int(d.sum()) == 0, f"{where}: sentinel words changed"


# ------------------------------------------------------------------------------------------------ device state vs restatement
def device_state(B, P, H, W, capacity, geom, binning, img):
    v = GL.GaRasterViews()
    GL.check(GL.lib().ga_raster_views(B, P, H, W, capacity, ptr(geom), ptr(binning), ptr(img), ctypes.byref(v)), "ga_raster_views")
    _, _, T = rb.grid(H, W)
    st = _grab(img, v.status, (16,), torch.int32).numpy().astype(np.int64)
    u32 = lambda t: t.numpy().astype(np.int64) & 0xFFFFFFFF
    n = min(int(st[0]), int(capacity))
    return dict(status=st, xy=_grab(geom, v.xy, (B, P, 2), torch.float32).numpy(), depth=_grab(geom, v.depth, (B, P), torch.float32).numpy(),
                rect=_grab(geom, v.rect, (B, P, 4), torch.int16).numpy().astype(np.int64) & 0xFFFF,
                tiles_touched=u32(_grab(geom, v.tiles_touched, (B, P), torch.int32)), tile_count=u32(_grab(img, v.tile_count, (B, T), torch.int32)),
                ranges=u32(_grab(img, v.ranges, (B * T, 2), torch.int32)), point_list=u32(_grab(binning, v.point_list, (n,), torch.int32)))


def compare(where, B, P, H, W, capacity, geom, binning, img, radii):
    """Everything the binning produced against the restatement of the forward's own K1 state; returns the restatement."""
    s = device_state(B, P, H, W, capacity, geom, binning, img)
    rad = radii.reshape(B, P).cpu().numpy()
    r = rb.restate(B, P, H, W, capacity, s["xy"], rad, s["depth"])
    eq = np.testing.assert_array_equal
    eq(s["rect"], r["rect"], err_msg=f"{where}: rect")
    eq(s["tiles_touched"], r["tiles_touched"], err_msg=f"{where}: tiles_touched")
    eq(r["tiles_touched"] == 0, rad == 0, err_msg=f"{where}: radii == 0 exactly where the rect is empty")
    eq(s["tile_count"], r["tile_count"], err_msg=f"{where}: tile_count")
    eq(s["ranges"], r["ranges"], err_msg=f"{where}: ranges")
    words = [0, 1, 2, 3, 13] + list(range(4, 5 + B))
    assert {k: int(s["status"][k]) for k in words} == {k: r["words"][k] for k in words}, f"{where}: status words"
    if not r["words"][1]:
        eq(s["point_list"], r["point_list"], err_msg=f"{where}: point_list")
    return r


# ------------------------------------------------------------------------------------------------------------------ launches
def forward(plan, dyn, cams, bg, depth=False, scene=None, seed=0):
    """One batched forward through the C ABI with the images, the depth map and the plan's binning buffer guarded:
    ga_rasterb_forward, ga_rasterb_forward_depth (depth) or ga_rasterb_forward_scene (scene).  Returns (images, depth or None)."""
    lib = GL.lib()
    B, H, W = plan.B, plan.H, plan.W
    out = Guard(4 * B * 3 * H * W, seed + 1)
    gb = Guard(plan.binning.numel(), seed + 2)
    plan.binning = gb.u8
    means, colors, scales, rots, opac = dyn
    d = plan.desc()
    tail = (ptr(cams), ptr(bg), ptr(means), ptr(colors), ptr(scales), ptr(rots), ptr(opac), ptr(plan.geom), ptr(plan.img), ptr(plan.binning),
            ptr(plan.radii), ptr(out.f), stream())
    sc = None
    if scene is not None:
        sc = GL.GaRasterScene(len(scene), int(scene.sh_degree), int(scene.shs.shape[1]), ptr(scene.means3D), ptr(scene.scales),
                              ptr(scene.rotations), ptr(scene.opacities), ptr(scene.shs), ptr(plan.scene_rgb), 0)
    dm = None
    if depth:
        dm = Guard(4 * B * 2 * H * W, seed + 3)
        GL.check(lib.ga_rasterb_forward_depth(ctypes.byref(d), None if sc is None else ctypes.byref(sc), None, ptr(dm.f), *tail), "depth")
    elif sc is not None:
        GL.check(lib.ga_rasterb_forward_scene(ctypes.byref(d), ctypes.byref(sc), *tail), "scene")
    else:
        GL.check(lib.ga_rasterb_forward(ctypes.byref(d), *tail), "forward")
    plan.record_status()
    torch.cuda.synchronize()
    out.ok("images")
    gb.ok("binning buffer")
    if dm is not None:
        dm.ok("depth map")
    return out.f.view(B, 3, H, W), None if dm is None else dm.f.view(B, 2, H, W)


def compare_plan(where, plan):
    return compare(where, plan.B, plan.P + plan.static_P, plan.H, plan.W, plan.capacity, plan.geom, plan.binning, plan.img, plan.radii)


def perframe(where, means, scales, rots, opac, colors, cam, H, W, bg, seed):
    """The per-frame API (ga_raster_forward_preprocess + _render, B = 1) with the image and the binning buffer guarded."""
    lib = GL.lib()
    P = means.shape[0]
    s = GL.GaRasterSettings(P, H, W, math.tan(cam.FovX / 2), math.tan(cam.FovY / 2), 1.0)
    view, proj = cam.world_view_transform.to(DEV).contiguous(), cam.full_proj_transform.to(DEV).contiguous()
    geom = torch.empty(lib.ga_raster_geom_bytes(P), dtype=torch.uint8, device=DEV)
    img = torch.empty(lib.ga_raster_img_bytes(H, W), dtype=torch.uint8, device=DEV)
    radii = torch.empty(P, dtype=torch.int32, device=DEV)
    n = ctypes.c_int64(0)
    GL.check(lib.ga_raster_forward_preprocess(ctypes.byref(s), ptr(means), ptr(scales), ptr(rots), ptr(opac), ptr(view), ptr(proj), ptr(geom),
                                              ptr(img), ptr(radii), ctypes.byref(n), stream()), "preprocess")
    R = int(n.value)
    nb = lib.ga_raster_binning_bytes(R, H, W)
    gb, out = Guard(nb, seed), Guard(4 * 3 * H * W, seed + 1)
    GL.check(lib.ga_raster_forward_render(ctypes.byref(s), ptr(colors), ptr(bg), ptr(geom), ptr(gb.u8), nb, R, ptr(img), ptr(out.f), stream()),
             "render")
    torch.cuda.synchronize()
    gb.ok(f"{where}: binning buffer")
    out.ok(f"{where}: image")
    return compare(where, 1, P, H, W, R, geom, gb.u8, img, radii)


def _camera(H, W, f, extrinsic=None):
    K = np.array([[f, 0, W / 2.0], [0, f, H / 2.0], [0, 0, 1]], dtype=np.float32)
    return make_camera(K, np.eye(4) if extrinsic is None else extrinsic, H, W)


AWAY = np.diag([-1.0, 1.0, -1.0, 1.0])          # looks down -z: every Gaussian in front of the other cameras is behind this one


def _means(cam, pix, z, H, W):
    """World points at view depth z [n] (identity extrinsics) projecting to pixel positions pix [n, 2]: the ray through each pixel at
    depth 1, scaled."""
    xy1 = _unproject(cam, torch.as_tensor(pix, dtype=torch.float64), 1.0, W, H)[:, :2].numpy()
    z = np.asarray(z, np.float64)
    return np.concatenate([xy1 * z[:, None], z[:, None]], 1).astype(np.float32)


def _cams(cam_list):
    return pack_cameras(torch.stack([c.world_view_transform for c in cam_list]), torch.stack([c.full_proj_transform for c in cam_list]),
                        [math.tan(c.FovX / 2) for c in cam_list], [math.tan(c.FovY / 2) for c in cam_list], DEV,
                        campos=torch.stack([c.camera_center for c in cam_list]))


def _t(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32).to(DEV)


# ------------------------------------------------------------------------------------------------------------- A. sort ladder
LADDER = ([("uniform", n) for n in (1, 63, 64, 65, 2047, 2048, 2049, 8192, 8193, 16385)] + [("equal", n) for n in (64, 1000, 2048, 5000)]
          + [("crowded", n) for n in (300, 3000)] + [("last_bit", n) for n in (100, 2049)] + [("log_spread", n) for n in (500, 8000)])
LH, LW = 77, 126                 # 5 x 8 tiles, the last row 13 pixels high and the last column 14 wide


def _ladder_depths(kind, n, g):
    if kind == "uniform":              # about two keys per depth value: ties inside the bins of the insertion path
        lv = max(n // 2, 1)
        return (0.5 + 4.0 * np.floor(g.random(n) * lv) / lv).astype(np.float32)
    if kind == "equal":
        return np.full(n, 2.0, np.float32)
    if kind == "crowded":              # 60 distinct depths within 6e-5 of each other: one bin holds more than 48 keys
        z = (1.0 + 4.0 * g.random(n)).astype(np.float32)
        z[g.choice(n, 60, replace=False)] = (3.0 + 1e-6 * np.arange(60)).astype(np.float32)
        return z
    if kind == "last_bit":
        a = np.float32(1.5)
        return np.where(g.random(n) < 0.5, a, np.nextafter(a, np.float32(2.0))).astype(np.float32)
    return np.exp(g.uniform(np.log(0.21), np.log(1e4), n)).astype(np.float32)      # log_spread: the first bin crowds


def _sort_path(n, z):
    """The tile_sort_kernel path a list of n keys with depths z (float32) takes: instance and branch."""
    long_ = n >= rb.LONG
    threads, kmax = (512, 8192) if long_ else (128, 2048)
    inst = "long" if long_ else "short"
    if n > kmax:
        return inst, "runs merged by rank"
    if n < 64:
        return inst, "bitonic (n < 64)"
    lo, hi = z.min(), z.max()
    if not hi > lo:
        return inst, "bitonic (all depths equal)"
    nb = min(2 * threads, max(32, n >> 3))
    scale = np.float32(nb) / (hi - lo)
    b = np.minimum(nb - 1, ((z - lo) * scale).astype(np.int64))
    return inst, "bitonic (a bin above 48)" if np.bincount(b).max() > 48 else "bins + insertion"


def _ladder(seed):
    """Frames 0 and 1 hold the ladder on the same tiles (a random half of the Gaussians, the static half, is shared with the same
    depths; the other half is re-drawn per frame and indexed in a per-frame order); frame 2 looks away, so everything is culled.
    Returns the per-frame means [3, P, 3], the split Pd, the cameras and, per ladder entry, (tile, index array of frame 0)."""
    cam = _camera(LH, LW, 100.0)
    gx, gy, T = rb.grid(LH, LW)
    g = np.random.default_rng(seed)
    tiles = g.choice(T, len(LADDER), replace=False)
    pix, z0, z1, owner = [], [], [], []
    for e, ((kind, n), t) in enumerate(zip(LADDER, tiles)):
        # near pixel centres 4..11 of the tile (radius 3 stays inside it), 0.2-0.8 px off them: a Gaussian exactly on a pixel centre
        # has power 0 there, a decision (power > 0) the fp64 reference can only call marginal
        off = g.integers(4, 12, size=(n, 2)) + g.uniform(0.2, 0.8, size=(n, 2))
        pix.append(np.stack([(t % gx) * 16 + off[:, 0], (t // gx) * 16 + off[:, 1]], 1))
        z0.append(_ladder_depths(kind, n, g))
        z1.append(_ladder_depths(kind, n, g))
        owner.append(np.full(n, e))
    pix, z0, z1, owner = map(np.concatenate, (pix, z0, z1, owner))
    N = pix.shape[0]
    static = g.permutation(N)[:N // 2]
    dyn = np.setdiff1d(np.arange(N), static)
    Pd = dyn.size
    frames, owners = [], []
    for b, z in enumerate((z0, z0, z0)):
        zb = z.copy()
        if b == 1:
            zb[dyn] = z1[dyn]
        order = np.concatenate([g.permutation(dyn), static])          # frame b's index space: dynamic (own order), then static
        frames.append(_means(cam, pix[order], zb[order], LH, LW))
        owners.append(owner[order])
    cams = [cam, cam, _camera(LH, LW, 100.0, AWAY)]
    return np.stack(frames), Pd, cams, tiles, owners


def test_sort_ladder_every_instance_and_api():
    means, Pd, cam_list, tiles, owners = _ladder(7)
    B, N = 3, means.shape[1]
    Ps = N - Pd
    g = np.random.default_rng(8)
    opac = (0.02 + 0.28 * g.random(N)).astype(np.float32)
    colors = g.random((B, N, 3)).astype(np.float32)
    scales = np.full((B, N, 3), 1e-5, np.float32)
    rots = np.tile(np.array([1, 0, 0, 0], np.float32), (N, 1))
    shs = (0.5 * g.standard_normal((Ps, 1, 3))).astype(np.float32)
    cams, bg = _cams(cam_list), _t(g.random(3))
    full = (_t(means), _t(colors), _t(scales), _t(rots), _t(opac))
    with torch.no_grad():
        # plain
        plan = RasterBatchPlan(B, N, LH, LW, DEV)
        img, _ = forward(plan, full, cams, bg, seed=10)
        r = compare_plan("ladder, plain", plan)
        # what the ladder reaches: one tile per entry, each Gaussian on one tile, every sort path in both instances
        assert (r["tiles_touched"][:2] == 1).all() and (r["tiles_touched"][2] == 0).all()
        paths = {}
        dep = device_state(B, N, LH, LW, plan.capacity, plan.geom, plan.binning, plan.img)["depth"]
        for b in range(2):
            for e, ((kind, n), t) in enumerate(zip(LADDER, tiles)):
                assert r["tile_count"][b, t] == n, (b, kind, n)
                paths.setdefault(_sort_path(n, dep[b][owners[b] == e]), set()).add(n)
        want = {(i, p) for i in ("short", "long") for p in ("bins + insertion", "bitonic (all depths equal)", "bitonic (a bin above 48)")}
        want |= {("short", "bitonic (n < 64)"), ("long", "runs merged by rank")}
        assert want <= set(paths), sorted(set(want) - set(paths))
        assert r["words"][13] == 2 * sum(n >= rb.LONG for _, n in LADDER)
        assert max(n for (i, p), ns in paths.items() for n in ns if p == "runs merged by rank") > 2 * 8192       # three runs
        for (inst, p), ns in sorted(paths.items()):
            REACHED.append(f"ladder: {inst} instance, {p}: list lengths {sorted(ns)}")
        REACHED.append(f"ladder: status[13] = {r['words'][13]}, frame bases {[r['words'][4 + b] for b in range(B + 1)]}")

        # depth pass (kZ): images bit-identical, plane 0 the indicator render's mean
        plan_d = RasterBatchPlan(B, N, LH, LW, DEV)
        img_d, depth = forward(plan_d, full, cams, bg, depth=True, seed=20)
        rd = compare_plan("ladder, depth", plan_d)
        np.testing.assert_array_equal(rd["point_list"], r["point_list"])
        assert torch.equal(img_d, img)
        vd = plan_d.views()
        ind = torch.zeros(B, N, 3, device=DEV)
        ind[..., 0] = torch.stack([v["depth"] for v in vd]).to(DEV)
        plan_i = RasterBatchPlan(B, N, LH, LW, DEV)
        red = rasterize_batch(full[0], ind, full[2], full[3], full[4], cams, torch.zeros(3, device=DEV), plan_i)[:, 0]
        assert plan_i.check(wait=True)
        for b in range(B):
            want_m = _mean_from(red[b], vd[b]["final_T"].to(DEV), vd[b]["n_contrib"].to(DEV))
            assert torch.equal(depth[b, 0], want_m), f"ladder depth plane 0, frame {b}"

        # scene (kScene) and scene + depth: the static half as a scene set
        sc = GaussianScene(_t(means[0, Pd:]), _t(scales[0, Pd:]), _t(rots[Pd:]), _t(opac[Pd:]), _t(shs), 0)
        dyn = (_t(means[:, :Pd]), _t(colors[:, :Pd]), _t(scales[:, :Pd]), _t(rots[:Pd]), _t(opac[:Pd]))
        plan_s = RasterBatchPlan(B, Pd, LH, LW, DEV, static_P=Ps)
        img_s, _ = forward(plan_s, dyn, cams, bg, scene=sc, seed=30)
        rs = compare_plan("ladder, scene", plan_s)
        np.testing.assert_array_equal(rs["point_list"], r["point_list"])
        both = torch.cat([dyn[1], plan_s.scene_rgb], 1).contiguous()
        plan_c = RasterBatchPlan(B, N, LH, LW, DEV)
        img_c = rasterize_batch(full[0], both, full[2], full[3], full[4], cams, bg, plan_c)
        assert plan_c.check(wait=True)
        assert torch.equal(img_s, img_c), "scene vs the same Gaussians as one dynamic set"
        plan_sd = RasterBatchPlan(B, Pd, LH, LW, DEV, static_P=Ps)
        img_sd, depth_sd = forward(plan_sd, dyn, cams, bg, depth=True, scene=sc, seed=40)
        rsd = compare_plan("ladder, scene + depth", plan_sd)
        np.testing.assert_array_equal(rsd["point_list"], r["point_list"])
        assert torch.equal(img_sd, img_s) and torch.equal(depth_sd, depth)

        # the per-frame API, frame 0
        rp = perframe("ladder, per-frame API", full[0][0].contiguous(), full[2][0].contiguous(), full[3], full[4], full[1][0].contiguous(),
                      cam_list[0], LH, LW, bg, seed=50)
        base, end = r["words"][4], r["words"][5]
        np.testing.assert_array_equal(rp["point_list"], r["point_list"][base:end])

    # compositing and backward of the plain variant (B = 3, lists merged from three runs) under the fp64 bounds
    scs = [dict(means3D=torch.from_numpy(means[b]), scales=torch.from_numpy(scales[b]), colors=torch.from_numpy(colors[b]), cam=cam_list[b],
                H=LH, W=LW, tanfovx=math.tan(cam_list[b].FovX / 2), tanfovy=math.tan(cam_list[b].FovY / 2), rotations=torch.from_numpy(rots),
                opacities=torch.from_numpy(opac)[:, None]) for b in range(B)]
    dL = torch.randn(B, 3, LH, LW, generator=torch.Generator().manual_seed(9))
    res = run_batched(scs, bg.cpu(), dL, capacity=plan.capacity, seed=60)
    for b, (fr, got, v) in enumerate(res):
        base, end = r["words"][4 + b], r["words"][5 + b]
        np.testing.assert_array_equal(v.get("vals_sorted", torch.zeros(0, dtype=torch.int32)).numpy(), r["point_list"][base:end])
        if b == 0:          # frame 1's lists take the same paths; the fp64 walk over a 16385-entry list takes a minute per frame
            check_frame(f"ladder frame {b}", fr, got, dL[b].to(DEV), want_restart=True)


# ------------------------------------------------------------------------------------------------- B. tile-table saturation
BH, BW, BF = 1080, 1920, 1000.0


def _big(g, n, kind):
    """Pixel centres, view depths and screen radii of n large Gaussians: 'wide' over the frame and past every edge, 'band' along
    the top edge (a CTA of them touches 3000-4096 tiles), 'pile' around the centre (tile lists above 2048)."""
    if kind == "wide":
        pix, r = g.uniform([-250, -250], [BW + 250, BH + 250], (n, 2)), g.uniform(100, 400, n)
    elif kind == "band":
        pix, r = np.stack([g.uniform(0, BW, n), g.uniform(0, 300, n)], 1), g.uniform(100, 150, n)
    else:
        pix, r = g.uniform([BW / 2 - 100, BH / 2 - 100], [BW / 2 + 100, BH / 2 + 100], (n, 2)), g.uniform(100, 150, n)
    return pix, g.uniform(2.0, 4.0, n), r


SPECIAL = [((BW / 2, BH / 2), 1300.0), ((-150.0, BH / 2), 300.0), ((BW + 150.0, BH / 2), 300.0), ((BW / 2, -150.0), 300.0),
           ((BW / 2, BH + 150.0), 300.0)]          # the whole grid, then clipped on the left, right, top and bottom edges


def _big_set(g, roles, special_at=()):
    pix, z, r = map(np.concatenate, zip(*[_big(g, n, k) for k, n in roles]))
    for i, (c, rad) in zip(special_at, SPECIAL):
        pix[i], r[i] = c, rad
    return pix, z, r


def _check_sampled_tiles(where, plan, img, colors, bg, r, b, g):
    """check_frame's forward tier (image, final_T, n_contrib on clear pixels) on every tile longer than 2048 and 24 others."""
    v = plan.views()[b]
    cnt = r["tile_count"][b]
    sel = cnt > rb.LONG
    nz = np.flatnonzero((cnt > 0) & ~sel)
    sel[g.choice(nz, min(24, nz.size), replace=False)] = True
    rg = v["ranges"].long().clone()
    rg[torch.from_numpy(~sel)] = 0
    fr = rf.Frame(v["xy"], v["conic_opacity"], colors, bg, rg, v["vals_sorted"].long(), plan.H, plan.W, device=DEV)
    fw = rf.forward(fr)
    tiles = torch.from_numpy(sel).to(DEV).reshape(r["gy"], r["gx"])
    px = tiles.repeat_interleave(16, 0).repeat_interleave(16, 1)[:plan.H, :plan.W]
    mask = px & ~fw["marginal"]
    check("K6 image", where, img, fw["image"][0], fw["image"][1], mask[None].expand(3, -1, -1))
    check("K6 final_T", where, v["final_T"].to(DEV), *fw["final_T"], mask)
    assert torch.equal(v["n_contrib"].to(DEV).long()[mask], fw["n_contrib"][mask]), f"{where}: n_contrib"
    assert int(mask.sum()) >= 0.99 * int(px.sum()), f"{where}: too many marginal pixels"
    return int(sel.sum()), int((cnt > rb.LONG).sum()), int(cnt.max())


def _saturation_report(where, r, P, straddle=None):
    ct = r["cta_tiles"]
    top = int(ct.max())
    mid = int(((ct > 3000) & (ct <= 4096)).sum())
    assert top > 4096, f"{where}: no CTA touches more than 4096 distinct tiles"
    assert mid >= 1, f"{where}: no CTA touches 3000-4096 distinct tiles"
    line = f"{where}: P = {P}, {r['instances']} instances; distinct tiles per CTA: max {top}, {mid} CTA(s) in (3000, 4096]"
    if straddle is not None:
        s = int(ct[:, straddle].max())
        assert s > 0
        line += f", the CTA across the dynamic / static boundary {s}"
    REACHED.append(line)


def _edges(r, xy, H, W):
    rc, tt = r["rect"].reshape(-1, 4), r["tiles_touched"].reshape(-1)
    x, y = xy.reshape(-1, 2)[:, 0], xy.reshape(-1, 2)[:, 1]
    vis = tt > 0
    assert (tt == r["T"]).any(), "no rect covers the whole grid"
    assert (vis & (x < 0) & (rc[:, 0] == 0)).any() and (vis & (x >= W) & (rc[:, 2] == r["gx"])).any()
    assert (vis & (y < 0) & (rc[:, 1] == 0)).any() and (vis & (y >= H) & (rc[:, 3] == r["gy"])).any()


def test_tile_table_saturation_1080p():
    B, P = 2, 3577                      # not a multiple of 256
    roles = [("wide", 256), ("band", 256), ("pile", 2300), ("wide", P - 2812)]
    g = np.random.default_rng(21)
    cam_list = [_camera(BH, BW, BF), _camera(BH, BW, BF, np.array([[1, 0, 0, 0.05], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1.0]]))]
    means = []
    for b in range(B):
        pix, z, rad = _big_set(g, roles, special_at=(5, 10, 11, 12, 3000))
        m = _means(cam_list[0], pix, z, BH, BW)
        means.append(np.concatenate([m, (rad * z / (3 * BF))[:, None].repeat(3, 1).astype(np.float32)], 1))
    means = np.stack(means)
    colors, opac = g.random((B, P, 3)).astype(np.float32), (0.05 + 0.5 * g.random(P)).astype(np.float32)
    rots = np.tile(np.array([1, 0, 0, 0], np.float32), (P, 1))
    cams, bg = _cams(cam_list), _t(g.random(3))
    dyn = (_t(means[..., :3]), _t(colors), _t(means[..., 3:]), _t(rots), _t(opac))
    with torch.no_grad():
        plan = RasterBatchPlan(B, P, BH, BW, DEV, capacity=12_000_000)
        img, _ = forward(plan, dyn, cams, bg, seed=70)
        r = compare_plan("saturation", plan)
        s = device_state(B, P, BH, BW, plan.capacity, plan.geom, plan.binning, plan.img)
        _edges(r, s["xy"], BH, BW)
        _saturation_report("saturation", r, P)
        for b in range(B):
            n, nlong, top = _check_sampled_tiles(f"saturation frame {b}", plan, img[b], dyn[1][b], bg, r, b, g)
            REACHED.append(f"saturation frame {b}: image checked on {n} tiles, all {nlong} longer than 2048 (longest {top})")

        # the player's case: a static set of large Gaussians after a dynamic set whose last CTA is partly static
        Pd = 2100
        pix, z, rad = _big_set(g, [("pile", 2300), ("wide", 100)])
        sm = _means(cam_list[0], pix, z, BH, BW)
        Ps = sm.shape[0]
        sc = GaussianScene(_t(sm), _t((rad * z / (3 * BF))[:, None].repeat(3, 1)), _t(np.tile(rots[:1], (Ps, 1))),
                           _t(0.05 + 0.5 * g.random(Ps)), _t(0.5 * g.standard_normal((Ps, 1, 3))), 0)
        sdyn = (dyn[0][:, :Pd].contiguous(), dyn[1][:, :Pd].contiguous(), dyn[2][:, :Pd].contiguous(), dyn[3][:Pd].contiguous(),
                dyn[4][:Pd].contiguous())
        plan_s = RasterBatchPlan(B, Pd, BH, BW, DEV, capacity=12_000_000, static_P=Ps)
        img_s, _ = forward(plan_s, sdyn, cams, bg, scene=sc, seed=80)
        rs = compare_plan("saturation, scene", plan_s)
        assert Pd % 256 != 0
        _saturation_report("saturation, scene", rs, Pd + Ps, straddle=Pd // 256)
        for b in range(B):
            cols = torch.cat([sdyn[1][b], plan_s.scene_rgb[b]]).contiguous()
            n, nlong, top = _check_sampled_tiles(f"saturation scene frame {b}", plan_s, img_s[b], cols, bg, rs, b, g)
            REACHED.append(f"saturation scene frame {b}: image checked on {n} tiles, all {nlong} longer than 2048 (longest {top})")


# ------------------------------------------------------------------------------------------------ C. scan rounds, capacity cuts
def test_scan_rounds_and_capacity_cuts_b8_1080p():
    B, P = 8, 20000
    g = np.random.default_rng(31)
    base = _camera(BH, BW, BF)
    cam_list = [_camera(BH, BW, BF, AWAY) if b == 5 else base for b in range(B)]
    frames = []
    for b in range(B):
        pix, z, rad = g.uniform([-20, -20], [BW + 20, BH + 20], (P, 2)), g.uniform(2.0, 4.0, P), g.uniform(3.0, 20.0, P)
        m = _means(base, pix, z, BH, BW)
        frames.append(np.concatenate([m, (rad * z / (3 * BF))[:, None].repeat(3, 1).astype(np.float32)], 1))
    frames = np.stack(frames)
    rots = np.tile(np.array([1, 0, 0, 0], np.float32), (P, 1))
    dyn = (_t(frames[..., :3]), _t(g.random((B, P, 3))), _t(frames[..., 3:]), _t(rots), _t(0.1 + 0.8 * g.random(P)))
    cams, bg = _cams(cam_list), _t(g.random(3))
    T = rb.grid(BH, BW)[2]
    rounds = -(-B * T // 4096)
    assert rounds == 16
    with torch.no_grad():
        plan = RasterBatchPlan(B, P, BH, BW, DEV, capacity=4_000_000)
        forward(plan, dyn, cams, bg, seed=90)
        r0 = compare_plan("scan, roomy", plan)
        assert r0["tile_count"][5].sum() == 0 and (r0["tile_count"].sum(1) > 0).sum() == B - 1
        total = r0["instances"]
        cnt = r0["tile_count"].reshape(-1)
        ends = np.cumsum(cnt)
        ks = [k for k in range(1, rounds) if cnt[4096 * k - 1] > 0 and cnt[4096 * k] > 0]
        assert ks, "no round boundary between two non-empty tiles"
        k = ks[len(ks) // 2]
        cuts = [("total", total), ("total - 1", total - 1), (f"end of tile {4096 * k - 1}", int(ends[4096 * k - 1])),
                ("inside frame 0", int(ends[T // 2]) - 1)]
        REACHED.append(f"scan: B = {B}, {B * T} tiles in {rounds} rounds of 4096, {total} instances, frame 5 culled")
        for name, cap in cuts:
            plan = RasterBatchPlan(B, P, BH, BW, DEV, capacity=cap)
            forward(plan, dyn, cams, bg, seed=100 + cap % 1000)
            r = compare_plan(f"scan, capacity {name}", plan)
            first_out = int(np.searchsorted(ends, cap, side="right"))
            assert r["words"][1] == int(cap < total)
            REACHED.append(f"scan: cut '{name}' at capacity {cap}: first tile left out {first_out} (frame {first_out // T}, round "
                           f"{first_out // 4096}), {r['words'][3]} tiles fit")
            if cap < total:
                assert not plan.check(wait=True) and plan.capacity > total
                forward(plan, dyn, cams, bg, seed=200 + cap % 1000)
                rr = compare_plan(f"scan, capacity {name}, grown", plan)
                assert rr["words"][1] == 0
                np.testing.assert_array_equal(rr["point_list"], r0["point_list"])
            else:
                assert plan.check(wait=True)
