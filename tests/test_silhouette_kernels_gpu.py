"""GPU: every launch of the soft silhouette (csrc/silhouette.cu) against the bounded fp64 reference of tests/silhouette_fp64.py, from
the kernels' own staged corners, boxes, per-pixel G and face gradients (derivation of the bounds in its docstring).

`ga_silhouette_forward` and `ga_silhouette_backward` are called through the C ABI with every output and the workspace inside
finite sentinels that must stay bit-identical; the workspace is read back through its layout (carve(), mirrored in
silhouette_fp64.workspace_layout).  Tiers, each |got - ref| <= bound on every clear element:
  setup        corners bit for bit against the fp32 restatement, boxes exactly, the empty box (1,0,1,0) for every dropped face.
  tile fwd     S per pixel, every face evaluated at every pixel of its fp64 box (a face missing from a tile list shows).
  partials     each tile's (S - M)^2 sum from the kernel's own S;  loss  within 1 ulp of their fp64 sum / (H W).
  tile bwd     G = w_b 2 (S - M) / (H W) exp(L) per pixel.
  face grad    the six corner gradients per (face, frame) from the kernel's own G; exact zeros for dropped faces.
  vertex grad  d_verts from the kernel's own fgrad; exact zeros for a vertex in no face or whose faces are all dropped.
  ceiling      on the long-edge scenes (a corner at ~5e5 px or just inside 2^20 px, an edge with both ends that far), the bound
               on x = +-d^2/sigma itself stays within 1e-4 max(1, |x|), and so does the kernel's S error.
Each bound must also reject a corrupted copy a plausible bug would produce.  Run with -s for the largest error / bound per tier and
the marginal fractions.
"""
import math

import numpy as np
import pytest
import torch

import silhouette_fp64 as sf
from gaussianavatar_b200 import _lib
from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, make_camera
from gaussianavatar_b200.mesh_render import cameras, vertex_face_csr

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PAD = 256
WORST = {}
MARG = {}
# A decision is marginal when its threshold lies within the value's bound: a band of relative width ~1e-7 around the truncation
# radius, a box side or an edge line.  That is a few pixels in 10^5 and a few faces in 10^3 on these meshes; the caps leave room
# and still fail if a bound blows up.
MARG_PIX, MARG_FACE = 2e-3, 2e-2
CEILING = 1e-4


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key, (r, where) in sorted(WORST.items()):
        print(f"\nsilhouette kernels: largest error/bound, {key}: {r:.3g} ({where})")
    for key, (n, tot) in sorted(MARG.items()):
        print(f"silhouette kernels: marginal {key}: {n} of {tot} ({n / max(tot, 1):.2e})")


class Sent:
    """n floats inside PAD finite sentinels on each side; `ok()` checks the sentinels are bit-identical."""

    def __init__(self, n, seed):
        g = torch.Generator(device=DEV).manual_seed(seed)
        self.buf = torch.randn(n + 2 * PAD, device=DEV, generator=g) * 1000.0
        self.before = self.buf.clone()
        self.t = self.buf[PAD:PAD + n]
        self.n = n

    def ok(self, where, whole=False):
        d = self.buf.view(torch.int32) != self.before.view(torch.int32)
        if not whole:
            d[PAD:PAD + self.n] = False
        assert int(d.sum()) == 0, f"{where}: sentinel words changed"


def ratio(got, ref, bound, mask=None):
    got = got.double()
    r = (got - ref).abs() / bound.clamp_min(1e-300)
    r = torch.where(bound == 0, torch.where(got == ref, 0.0, math.inf), r)
    r = torch.where(torch.isnan(got), math.inf, r)
    if mask is not None:
        r = r[mask.expand_as(r)]
    return float(r.max()) if r.numel() else 0.0


def check(key, where, got, ref, bound, mask=None):
    r = ratio(got, ref, bound, mask)
    if r > WORST.get(key, (-1.0, ""))[0]:
        WORST[key] = (r, where)
    assert r <= 1.0, f"{key}, {where}: error/bound {r:.4g}"


def rejects(what, bad, ref, bound, mask=None):
    assert ratio(bad, ref, bound, mask) > 1.0, f"self-check: the bound accepts {what}"


def count_marg(key, n, tot, cap):
    a, b = MARG.get(key, (0, 0))
    MARG[key] = (a + n, b + tot)
    assert n <= cap * tot + 2, f"marginal {key}: {n} of {tot}"


# ------------------------------------------------------------------------------------------------------------ scenes
def _cam(H, W, f):
    K = np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], np.float32)
    return cameras([make_camera(K, np.eye(4), H, W)])[0]


def _world(px, py, z, H, W, f):
    return [(px - W / 2 + 0.5) / f * z, (py - H / 2 + 0.5) / f * z, z]


def scene(kind, B, H, W, F=0, seed=0):
    """(verts [B,V,3] on the device, faces [F,3] int64, cams [B,40] on the device, (adj_off, adj_face) or None for the default
    CSR)."""
    g = np.random.default_rng(seed)
    csr = None
    if kind in ("smpl", "smplx"):
        from test_silhouette_gpu import _body, _verts
        poser, pose, transl = _body(kind, B)
        K = np.array([[1100 * min(H, W) / 1024, 0, W / 2], [0, 1100 * min(H, W) / 1024, H / 2], [0, 0, 1]], np.float32)
        cam = cameras([make_camera(K, TEST_POSE_EXTRINSIC, H, W)])[0]
        return _verts(poser, pose, transl).float().contiguous(), poser.faces.long().cpu().numpy(), cam[None].expand(B, -1).contiguous().to(DEV), None
    f = 1.2 * max(H, W)
    if kind == "rand":                       # F triangles of 1 to ~40 pixels scattered over (and a little beyond) the frame
        V = max(3, F // 2 + 3)
        px, py = g.uniform(-8, W + 8, V), g.uniform(-8, H + 8, V)
        X = np.array([_world(a, b, z, H, W, f) for a, b, z in zip(px, py, g.uniform(1.5, 2.5, V))])
        faces = np.zeros((F, 3), np.int64)
        for i in range(F):
            a = g.integers(0, V)
            d = np.hypot(px - px[a], py - py[a])
            near = np.argsort(d)[1:8]
            faces[i] = [a, *g.choice(near, 2, replace=False)]
    elif kind == "special":
        pts = []

        def tri(c, z=2.0):
            i = len(pts)
            pts.extend(_world(x, y, z, H, W, f) for x, y in c)
            return [i, i + 1, i + 2]

        faces = [tri([(3.3, 4.1), (3.6, 4.05), (3.4, 4.5)]),                      # sub-pixel
                 tri([(-3 * W, -3 * H), (4 * W, -2 * H), (0.5 * W, 5 * H)], 3.0),   # covers the frame
                 tri([(-2.5, 5.2), (-1.2, 9.7), (-1.9, 13.1)])]                      # off screen, its band entering
        faces.append(faces[0][:])                                                     # coincident duplicate
        c = tri([(10.2, 3.1), (14.6, 6.3), (8.8, 9.9)])
        faces.append(c)
        faces.append([c[0], c[1], len(pts)])
        pts.append([0.0, 0.0, 0.005])                                                 # behind the near plane
        faces.append([c[1], c[2], len(pts)])
        pts.append([float("nan"), 0.0, 2.0])                                         # NaN vertex
        faces.append([c[0], c[2], len(pts)])
        pts.append(_world(3e6, 5.0, 2.0, H, W, f))                                   # outside the guard band
        faces.append([c[0], c[0], c[1]])                                             # zero area
        hub = len(pts)                                                               # a vertex of valence 40
        pts.append(_world(0.6 * W, 0.55 * H, 2.0, H, W, f))
        ring = len(pts)
        for k in range(40):
            a = 2 * math.pi * k / 40
            pts.append(_world(0.6 * W + 6.3 * math.cos(a), 0.55 * H + 5.7 * math.sin(a), 2.0, H, W, f))
        faces += [[hub, ring + k, ring + (k + 1) % 40] for k in range(40)]
        pts.append([0.1, 0.1, 2.0])                                                  # in no face
        X, faces = np.array(pts), np.array(faces, np.int64)
        off, adj = vertex_face_csr(faces, len(X))
        adj = np.insert(adj, off[hub] + 1, adj[off[hub]])                            # a face listed twice at the hub
        off = off.copy()
        off[hub + 1:] += 1
        csr = (off, adj)
    elif kind.startswith("long"):            # corners ~far pixels away: one far corner, and edges with both ends far
        far = 5.2e5 if kind == "long5" else 1.04e6
        f = 100.0
        zf = 0.05
        pts, faces = [], []
        for k in range(12):
            a = g.uniform(0, 2 * math.pi)
            p0 = g.uniform([8, 8], [W - 8, H - 8])
            p1 = p0 + g.uniform(2, 6, 2)
            tip = p0 + far * np.array([math.cos(a), math.sin(a)])
            i = len(pts)
            pts += [_world(*p0, 2.0, H, W, f), _world(*p1, 2.0, H, W, f), _world(*tip, zf, H, W, f)]
            faces.append([i, i + 1, i + 2])
        for k in range(12):
            a = g.uniform(0, math.pi)
            d = np.array([math.cos(a), math.sin(a)])
            mid = g.uniform([10, 10], [W - 10, H - 10])
            i = len(pts)
            pts += [_world(*(mid - far * d), zf, H, W, f), _world(*(mid + far * d), zf, H, W, f),
                    _world(*(mid + g.uniform(3, 9) * np.array([-d[1], d[0]])), 2.0, H, W, f)]
            faces.append([i, i + 1, i + 2])
        X, faces = np.array(pts), np.array(faces, np.int64)
    shift = torch.tensor([[1e-3 * b, -7e-4 * b, 0.0] for b in range(B)], dtype=torch.float32)
    verts = (torch.from_numpy(np.asarray(X, np.float32))[None] + shift[:, None]).to(DEV).contiguous()
    cams = torch.stack([_cam(H, W, f)] * B).to(DEV).contiguous()
    return verts, np.asarray(faces, np.int64).reshape(-1, 3), cams, csr


def masks(B, H, W, seed=0):
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    m = np.stack([(((yy - H * 0.5) ** 2 + (xx - W * (0.45 + 0.02 * b)) ** 2) < (0.3 * min(H, W)) ** 2) * 255 for b in range(B)])
    m[:, ::7, ::5] = g.integers(100, 160, m[:, ::7, ::5].shape)
    return torch.from_numpy(m.astype(np.uint8)).to(DEV)


# ---------------------------------------------------------------------------------------------------------- launches
def run(verts, faces, cams, H, W, sigma, mask, w, csr=None, seed=0):
    L = _lib.lib()
    s = torch.cuda.current_stream().cuda_stream
    B, V = verts.shape[:2]
    F = len(faces)
    fz = torch.from_numpy(faces.astype(np.int32)).to(DEV).contiguous()
    off, adj = vertex_face_csr(faces, V) if csr is None else csr
    off, adj = torch.from_numpy(np.asarray(off, np.int32)).to(DEV), torch.from_numpy(np.asarray(adj, np.int32)).to(DEV)
    lay = sf.workspace_layout(B, F, H, W)
    assert L.ga_silhouette_workspace_bytes(B, V, F, H, W) == lay["total"]
    ws = Sent(lay["total"] // 4, seed)
    sil, loss = Sent(B * H * W, seed + 1), Sent(B, seed + 2)
    _lib.check(L.ga_silhouette_forward(B, V, F, H, W, sigma, verts.data_ptr(), fz.data_ptr(), cams.data_ptr(),
                                       None if mask is None else mask.data_ptr(), ws.t.data_ptr(), sil.t.data_ptr(),
                                       None if mask is None else loss.t.data_ptr(), s), "ga_silhouette_forward")
    torch.cuda.synchronize()
    ws.ok("workspace, forward")
    sil.ok("sil")
    loss.ok("loss", whole=mask is None)
    wb = ws.t.view(torch.uint8)

    def part(name, n, dt):
        return wb[lay[name]:lay[name] + n * 4].view(dt).clone()

    out = dict(B=B, V=V, F=F, H=H, W=W, sigma=sigma, verts=verts, faces=faces, cams=cams, mask=mask, off=off, adj=adj,
               sil=sil.t.view(B, H, W).clone(), loss=loss.t.clone(),
               boxes=part("boxes", 4 * B * F, torch.int32).view(B, F, 4).long(),
               xy=part("xy", 6 * B * F, torch.float32).view(B, F, 2, 3).transpose(2, 3).contiguous(),
               partial=part("partial", B * sf.cdiv(H, 16) * sf.cdiv(W, 16), torch.float32).view(B, -1))
    if mask is None:
        return out
    d = Sent(B * V * 3, seed + 3)
    _lib.check(L.ga_silhouette_backward(B, V, F, H, W, sigma, verts.data_ptr(), fz.data_ptr(), off.data_ptr(), adj.data_ptr(),
                                        cams.data_ptr(), mask.data_ptr(), w.data_ptr(), ws.t.data_ptr(), d.t.data_ptr(), s),
               "ga_silhouette_backward")
    torch.cuda.synchronize()
    ws.ok("workspace, backward")
    d.ok("d_verts")
    out.update(pix=part("pix", B * H * W, torch.float32).view(B, H, W), fgrad=part("fgrad", 6 * B * F, torch.float32).view(B, F, 6),
               d_verts=d.t.view(B, V, 3).clone(), w=w)
    return out


# ------------------------------------------------------------------------------------------------------------- tiers
def tier_setup(o, where):
    for b in range(o["B"]):
        xy, ok, box, unsure = sf.setup_f32(o["verts"][b].cpu().numpy(), o["faces"], o["cams"][b].cpu().numpy(), o["H"], o["W"], o["sigma"])
        got = o["xy"][b].cpu().numpy()
        fin = np.isfinite(xy)
        assert np.array_equal(got[fin].view(np.int32), xy[fin].view(np.int32)), f"{where}: corners"
        assert np.isnan(got[~fin]).all() if (~fin).any() else True
        gb = o["boxes"][b].cpu().numpy()
        sure = ~unsure
        assert np.array_equal(gb[sure], box[sure]), f"{where}: boxes"
        assert (gb[~ok & sure] == (1, 0, 1, 0)).all()
        assert ((gb[:, 0] <= gb[:, 1]) == (gb[:, 2] <= gb[:, 3])).all()


def frame_ref(o, b, rows=None, geom=None):
    ok = (o["boxes"][b, :, 0] <= o["boxes"][b, :, 1]).cpu()
    return sf.FrameRef(o["xy"][b].cpu().numpy(), ok.numpy(), o["H"], o["W"], o["sigma"], rows=rows, geom=geom, device=DEV)


def tier_forward(o, where, rows=None, ceiling=None):
    refs = []
    for b in range(o["B"]):
        fr = frame_ref(o, b, rows)
        r = fr.forward(ceiling=ceiling)
        got = o["sil"][b] if rows is None else o["sil"][b][torch.as_tensor(rows, device=DEV)]
        clear = ~r["marg"]
        if ceiling is not None:
            # the kernel's S against the exact function (the fp64-geometry reference's bound is ~1e-7 of x)
            ex = frame_ref(o, b, rows, geom="f64").forward()
            r["S_err"] = float((got.double() - ex["S"][0]).abs()[~ex["marg"]].max())
            print(f"\n{where} b{b}: largest |S - S_exact| {r['S_err']:.3g}, largest bound on x / ({ceiling:g} max(1, |x|)) "
                  f"{r['ceiling']:.3g}, marginal pixels {int(r['marg'].sum())} of {r['marg'].numel()}")
        count_marg("tile fwd pixels", int(r["marg"].sum()), r["marg"].numel(), MARG_PIX)
        check("tile fwd S", f"{where} b{b}", got, r["S"][0], r["S"][1], clear)
        if o["mask"] is not None and rows is None:
            M = (o["mask"][b] >= 128).double()
            pv, pe = sf.partials(o["sil"][b], M, o["H"], o["W"])
            check("partials", f"{where} b{b}", o["partial"][b], pv, pe)
            want = float(o["partial"][b].double().sum()) / (o["H"] * o["W"])
            got_l = float(o["loss"][b])
            assert abs(got_l - want) <= float(np.spacing(np.float32(abs(want)))), (where, got_l, want)
        refs.append((fr, r))
    return refs


def tier_backward(o, where, refs):
    for b in range(o["B"]):
        fr, r = refs[b]
        M = (o["mask"][b] >= 128).double()
        w_b = float(o["w"][b])
        G = fr.grad_pix(r["L"], M, w_b)
        clear = ~r["marg"]
        check("tile bwd G", f"{where} b{b}", o["pix"][b], G[0], G[1], clear)
        fg, fm = fr.face_grad(o["pix"][b], o["boxes"][b])
        count_marg("face grad faces", int(fm.sum()), fm.numel(), MARG_FACE)
        check("face grad", f"{where} b{b}", o["fgrad"][b], fg[0], fg[1], ~fm[:, None])
        dropped = o["boxes"][b, :, 0] > o["boxes"][b, :, 1]
        assert bool((o["fgrad"][b][dropped] == 0).all()), f"{where}: fgrad of a dropped face"
        vv, ve = sf.vertex_grad(o["fgrad"][b], o["verts"][b], o["faces"], o["off"], o["adj"], o["cams"][b], o["H"], o["W"])
        check("vertex grad", f"{where} b{b}", o["d_verts"][b], vv, ve)
        faces = torch.as_tensor(o["faces"], device=DEV)
        live = torch.zeros(o["V"], dtype=torch.bool, device=DEV)
        if len(o["faces"]):
            live[faces[~dropped].reshape(-1)] = True
        assert bool((o["d_verts"][b][~live] == 0).all()), f"{where}: d_verts of a vertex without a live face"
        yield b, fr, r, G, fg, fm, (vv, ve)


CASES = [("special", 1, 1, 1, 0, 1.0), ("special", 16, 17, 1, 0, 1.0), ("special", 37, 53, 3, 0, 0.25), ("special", 37, 53, 3, 0, 4.0),
         ("rand", 17, 16, 1, 0, 1.0), ("rand", 17, 16, 3, 1, 1.0), ("rand", 37, 53, 3, 255, 1.0), ("rand", 37, 53, 3, 256, 0.25),
         ("rand", 37, 53, 8, 257, 1.0), ("rand", 64, 80, 3, 513, 4.0)]


@pytest.mark.parametrize("kind,H,W,B,F,sigma", CASES)
def test_kernels_against_fp64(kind, H, W, B, F, sigma):
    verts, faces, cams, csr = scene(kind, B, H, W, F, seed=F + H)
    w = torch.tensor([1.0, 0.5, 2.0, 0.25, 1.5, 3.0, 0.75, 1.25][:B], device=DEV)
    where = f"{kind} {H}x{W} B{B} F{len(faces)} sigma {sigma}"
    o = run(verts, faces, cams, H, W, sigma, masks(B, H, W), w, csr)
    tier_setup(o, where)
    refs = tier_forward(o, where)
    for _ in tier_backward(o, where, refs):
        pass
    # without a mask the forward writes S only
    o2 = run(verts, faces, cams, H, W, sigma, None, None, csr, seed=9)
    assert torch.equal(o2["sil"], o["sil"])


@pytest.mark.parametrize("name,H,W,B", [("smpl", 540, 540, 8), ("smplx", 540, 540, 3), ("smpl", 96, 128, 1)])
def test_bodies_against_fp64(name, H, W, B):
    """Tiles hit by more than 256 faces (13776 SMPL faces, 20908 SMPL-X)."""
    verts, faces, cams, _ = scene(name, B, H, W)
    w = torch.linspace(0.5, 2.0, B, device=DEV)
    where = f"{name} {H}x{W} B{B}"
    o = run(verts, faces, cams, H, W, 1.0, masks(B, H, W), w)
    tier_setup(o, where)
    refs = tier_forward(o, where)
    assert int(refs[0][1]["count"].max()) > 0
    bx = o["boxes"][0]
    ty = torch.arange(sf.cdiv(H, 16), device=DEV)[:, None, None] * 16
    tx = torch.arange(sf.cdiv(W, 16), device=DEV)[None, :, None] * 16
    hits = ((bx[:, 0] <= bx[:, 1]) & (bx[:, 1] >= tx) & (bx[:, 0] < tx + 16) & (bx[:, 3] >= ty) & (bx[:, 2] < ty + 16)).sum(-1)
    if H == 540:
        assert int(hits.max()) > 256, int(hits.max())
    for _ in tier_backward(o, where, refs):
        pass


def test_wide_frame_sampled_rows():
    H, W = 1080, 1920
    verts, faces, cams, _ = scene("smpl", 1, H, W)
    o = run(verts, faces, cams, H, W, 1.0, None, None)
    tier_setup(o, "smpl 1080x1920")
    tier_forward(o, "smpl 1080x1920", rows=np.linspace(0, H - 1, 24).round().astype(np.int64))
    verts, faces, cams, csr = scene("special", 1, H, W)
    o = run(verts, faces, cams, H, W, 1.0, masks(1, H, W), torch.ones(1, device=DEV), csr)
    tier_setup(o, "special 1080x1920")
    refs = tier_forward(o, "special 1080x1920", rows=np.linspace(0, H - 1, 16).round().astype(np.int64))
    fr = frame_ref(o, 0)
    fg, fm = fr.face_grad(o["pix"][0], o["boxes"][0])               # one warp loops over the whole frame for face 1
    check("face grad", "special 1080x1920", o["fgrad"][0], fg[0], fg[1], ~fm[:, None])
    assert not bool(fm[1]) and int((o["boxes"][0, 1, 1] - o["boxes"][0, 1, 0] + 1) * (o["boxes"][0, 1, 3] - o["boxes"][0, 1, 2] + 1)) == H * W


@pytest.mark.parametrize("kind", ["long5", "long1e6"])
def test_long_edges_within_ceiling(kind):
    """Faces with a corner ~5e5 px or ~1.04e6 px away, and edges with both ends that far, crossing a 48 x 64 frame at sigma 1."""
    H, W = 48, 64
    verts, faces, cams, _ = scene(kind, 2, H, W, seed=3)
    w = torch.tensor([1.0, 0.5], device=DEV)
    o = run(verts, faces, cams, H, W, 1.0, masks(2, H, W), w)
    tier_setup(o, kind)
    x = o["xy"][0]
    assert float(x.double().norm(dim=-1).amax(1).min()) > 4e5        # every face has a far corner
    assert bool((o["boxes"][0, :, 0] <= o["boxes"][0, :, 1]).all())
    refs = tier_forward(o, kind, ceiling=CEILING)
    for b, (fr, r) in enumerate(refs):
        assert r["ceiling"] <= 1.0, f"{kind} b{b}: the bound on x exceeds the ceiling by {r['ceiling']:.3g}x"
        assert r["S_err"] <= CEILING
    for _ in tier_backward(o, kind, refs):
        pass


def test_self_checks_reject_corruptions():
    H, W = 96, 128
    verts, faces, cams, _ = scene("smpl", 2, H, W)
    w = torch.tensor([1.0, 0.5], device=DEV)
    o = run(verts, faces, cams, H, W, 1.0, masks(2, H, W), w)
    b = 1
    fr = frame_ref(o, b)
    r = fr.forward()
    clear = ~r["marg"]
    S = r["S"]
    # a face whose centroid pixel is clear and not saturated, left out of the tile holding that pixel
    bx = o["boxes"][b]
    cen = o["xy"][b].double().mean(1).round().long()
    inb = (cen[:, 0] >= 0) & (cen[:, 0] < W) & (cen[:, 1] >= 0) & (cen[:, 1] < H) & (bx[:, 0] <= bx[:, 1])
    cx, cy = cen[:, 0].clamp(0, W - 1), cen[:, 1].clamp(0, H - 1)
    score = torch.where(inb & clear[cy, cx], torch.exp(r["L"][0][cy, cx]), -1.0)
    f = int(score.argmax())
    assert float(score[f]) > 0
    tile = int(cy[f] // 16) * sf.cdiv(W, 16) + int(cx[f] // 16)
    rejects("a face left out of one tile", fr.forward(drop=(f, tile))["S"][0], S[0], S[1], clear)
    # a face whose box's last row runs through clear pixels that are not saturated, that row left out
    eL = torch.where(clear, torch.exp(r["L"][0]), -1.0)
    score = torch.full((bx.shape[0],), -1.0, dtype=torch.float64, device=DEV)
    for g in torch.nonzero(bx[:, 0] <= bx[:, 1]).reshape(-1)[::7].tolist():
        c0, c1, _, r1 = bx[g].tolist()
        score[g] = eL[r1, c0:c1 + 1].max()
    g = int(score.argmax())
    rejects("a box one row short", fr.forward(shrink=(g, bx.cpu()))["S"][0], S[0], S[1], clear)
    M = (o["mask"][b] >= 128).double()
    G = fr.grad_pix(r["L"], M, float(w[b]))
    rejects("w_b ignored", fr.grad_pix(r["L"], M, 1.0)[0], G[0], G[1], clear)
    fg, fm = fr.face_grad(o["pix"][b], bx)
    keep = ~fm[:, None].expand(-1, 6)
    rejects("t and 1 - t swapped", fr.face_grad(o["pix"][b], bx, swap_t=True)[0][0], fg[0], fg[1], keep)
    rejects("corners a and b swapped", fr.face_grad(o["pix"][b], bx, swap_ab=True)[0][0], fg[0], fg[1], keep)
    vv, ve = sf.vertex_grad(o["fgrad"][b], o["verts"][b], o["faces"], o["off"], o["adj"], o["cams"][b], H, W)
    nz = int(torch.nonzero(o["fgrad"][b].abs().sum(1) > 0)[0])
    bad = o["fgrad"][b].clone()
    bad[nz] = 0
    rejects("one face's fgrad zeroed", sf.vertex_grad(bad, o["verts"][b], o["faces"], o["off"], o["adj"], o["cams"][b], H, W)[0], vv, ve)
    rejects("the hx p_w proj[4k+3] term dropped",
            sf.vertex_grad(o["fgrad"][b], o["verts"][b], o["faces"], o["off"], o["adj"], o["cams"][b], H, W, drop_w_term=True)[0], vv, ve)
