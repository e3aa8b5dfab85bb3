"""CPU: the bounded fp64 soft-silhouette reference (tests/silhouette_fp64.py) against oracle/silhouette_oracle.py, its bounds against
numpy restatements of eval_face's expression tree (fp32 geometry, with and without contracted FMAs, and fp64 geometry), including
faces with corners far out in the guard band, and its workspace mirror against ga_silhouette_workspace_bytes."""
import numpy as np
import pytest
import torch

import silhouette_fp64 as sf
from oracle import silhouette_oracle as so
from oracle.mesh_oracle import fma32

f32 = np.float32


def emulate(xy, px, py, trunc, inv_sigma, geom, fma):
    """eval_face at pixel centres in numpy: x [n], live [n], edge [n], t, dx, dy [n] (float32 results)."""
    best = np.full(px.shape, np.inf)
    pos = np.ones(px.shape, bool)
    neg = np.ones(px.shape, bool)
    t_, dx_, dy_ = (np.zeros(px.shape, f32) for _ in range(3))
    edge = np.zeros(px.shape, np.int64)
    T = np.float64 if geom == "f64" else f32
    with np.errstate(all="ignore"):
        for k in range(3):
            k1 = (k + 1) % 3
            ax, ay, bx, by = (xy[:, i, j].astype(T) for i, j in ((k, 0), (k, 1), (k1, 0), (k1, 1)))
            ex, ey, wx, wy = bx - ax, by - ay, px.astype(T) - ax, py.astype(T) - ay
            if fma and geom == "f32":
                cr = fma32(ex, wy, -(ey * wx))
                t = fma32(wx, ex, wy * ey) / fma32(ex, ex, ey * ey)
            else:
                cr = ex * wy - ey * wx
                t = (wx * ex + wy * ey) / (ex * ex + ey * ey)
            t = np.minimum(np.maximum(t, T(0)), T(1))
            if fma and geom == "f32":
                dx, dy = fma32(-t, ex, wx), fma32(-t, ey, wy)
                d2 = fma32(dx, dx, dy * dy)
            else:
                dx, dy = wx - t * ex, wy - t * ey
                d2 = dx * dx + dy * dy
            pos &= cr >= 0
            neg &= cr <= 0
            take = d2 < best
            best = np.where(take, d2, best)
            t_, dx_, dy_ = (np.where(take, a.astype(f32), b) for a, b in ((t, t_), (dx, dx_), (dy, dy_)))
            edge = np.where(take, k, edge)
        inside = pos | neg
        live = inside | ~(best > trunc)
        b32 = best.astype(f32)
        x = np.where(inside, b32, -b32) * f32(inv_sigma)
    return x, live, edge, t_, dx_, dy_, inside


def softplus32(x):
    with np.errstate(all="ignore"):
        return np.where(x > 0, x + np.log1p(np.exp(-x)), np.log1p(np.exp(x))).astype(f32)


def _faces(kind, n, seed):
    """[n,3,2] float32 corners; 'far1' one corner at ~far pixels, 'far2' an edge crossing the frame with both ends far."""
    g = np.random.default_rng(seed)
    base = g.uniform(10, 50, (n, 3, 2))
    if kind == "small":
        return (base[:, :1] + g.uniform(-6, 6, (n, 3, 2))).astype(f32)
    far = 5.2e5 if kind.endswith("e5") else 1.04e6       # the second just inside the 2^20-pixel guard band
    if kind.startswith("far1"):
        c = base.copy()
        ang = g.uniform(0, 2 * np.pi, n)
        c[:, 2] = c[:, 0] + far * np.stack([np.cos(ang), np.sin(ang)], 1)
        return c.astype(f32)
    c = base.copy()                                     # both ends far, the edge passing near (30, 30)
    ang = g.uniform(0, np.pi, n)
    d = np.stack([np.cos(ang), np.sin(ang)], 1)
    mid = g.uniform(25, 35, (n, 2))
    c[:, 0], c[:, 1] = mid - far * d, mid + far * d
    c[:, 2] = mid + g.uniform(3, 12, (n, 1)) * np.stack([-d[:, 1], d[:, 0]], 1)
    return c.astype(f32)


KINDS = ["small", "far1e5", "far1e6", "far2e5", "far2e6"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("geom", ["f32", "f64"])
@pytest.mark.parametrize("sigma", [0.25, 1.0, 4.0])
def test_bound_holds_against_numpy_restatement(kind, geom, sigma):
    xy = _faces(kind, 24, seed=hash((kind, sigma)) % 1000)
    trunc, inv_sigma, r = sf.thresholds(sigma)
    fr = sf.FrameRef(xy, np.ones(len(xy), bool), 64, 64, sigma, geom=geom)
    worst, marg, tot, ceil_worst = 0.0, 0, 0, 0.0
    G = torch.linspace(-3e-4, 5e-4, 64 * 64, dtype=torch.float64)
    for f, c, rr in fr._pairs(all_rows=True):
        P = sf.eval_pairs(fr.xy, f, c, rr, trunc, inv_sigma, geom)
        mg = P["marg"] | (sf.box_marg(fr.xy, f, c, rr, r) & ~(P["dead"] & ~P["marg"]))
        tv, te, mn = sf.grad_terms(P, G[rr * 64 + c], inv_sigma)
        for fma in (False, True):
            x, live, edge, t, dx, dy, inside = emulate(xy[f.numpy()], c.numpy().astype(f32), rr.numpy().astype(f32), f32(trunc),
                                                       inv_sigma, geom, fma)
            clear = ~mg.numpy()
            assert np.array_equal(live[clear], (~P["dead"]).numpy()[clear])
            ok = clear & live
            xv, xe = P["x"][0].numpy(), P["x"][1].numpy()
            worst = max(worst, float((np.abs(x.astype(np.float64) - xv) / xe)[ok].max()))
            sv, se = P["sp"][0].numpy(), P["sp"][1].numpy()
            worst = max(worst, float((np.abs(softplus32(x).astype(np.float64) - sv) / se)[ok].max()))
            # the gradient terms of the edge the restatement chose
            okg = ok & ~mn.numpy()
            Gp = G[rr * 64 + c].numpy().astype(f32)
            with np.errstate(all="ignore"):
                sg = np.where(x >= 0, f32(1) / (f32(1) + np.exp(-x)), np.exp(x) / (f32(1) + np.exp(x))).astype(f32)
            coef = f32(-2) * Gp * sg * np.where(inside, f32(inv_sigma), f32(-inv_sigma))
            ca, cb = coef * (f32(1) - t), coef * t
            g = np.zeros((len(x), 6), f32)
            i = np.arange(len(x))
            e2 = (edge + 1) % 3
            g[i, 2 * edge], g[i, 2 * edge + 1] = ca * dx, ca * dy
            g[i, 2 * e2], g[i, 2 * e2 + 1] = cb * dx, cb * dy
            rg = np.abs(g.astype(np.float64) - tv.numpy()) / np.maximum(te.numpy(), 1e-300)
            rg[(te.numpy() == 0) & (g == tv.numpy())] = 0.0
            worst = max(worst, float(rg[okg].max()) if okg.any() else 0.0)
        marg += int(mg.sum())
        tot += mg.numel()
        xv, xe = P["x"]
        cl = ~mg & ~P["dead"]
        ceil_worst = max(ceil_worst, float((xe / (1e-4 * xv.abs().clamp_min(1.0)))[cl].max()))
    print(f"\n{kind} {geom} sigma {sigma}: error/bound {worst:.3g}, marginal {marg}/{tot}, bound/ceiling {ceil_worst:.3g}")
    assert worst <= 1.0
    assert marg <= (0.01 if kind == "small" or geom != "f32" else 0.1) * tot      # fp32 long edges: wide bounds, many marginal
    if kind == "small" or geom != "f32":
        assert ceil_worst <= 1.0
    elif sigma <= 1.0:
        assert ceil_worst > 1.0          # the fp32 geometry cannot keep a long edge's distance within the ceiling


def test_fp32_geometry_loses_long_edges():
    """The cancellation the fp64 geometry removes: the fp32 tree's x error on a long edge, against exact fp64."""
    worst = {}
    for kind in ("far1e5", "far2e6"):
        xy = _faces(kind, 24, seed=7)
        trunc, inv_sigma, _ = sf.thresholds(1.0)
        fr = sf.FrameRef(xy, np.ones(len(xy), bool), 64, 64, 1.0, geom="f64")
        err = []
        for f, c, rr in fr._pairs(all_rows=True):
            P = sf.eval_pairs(fr.xy, f, c, rr, trunc, inv_sigma, "f64")
            x32 = emulate(xy[f.numpy()], c.numpy().astype(f32), rr.numpy().astype(f32), f32(trunc), inv_sigma, "f32", False)[0]
            x64 = emulate(xy[f.numpy()], c.numpy().astype(f32), rr.numpy().astype(f32), f32(trunc), inv_sigma, "f64", False)[0]
            live = ~P["dead"] & ~P["marg"] & (P["x"][0].abs() < 10)
            err.append((np.abs(x32 - P["x"][0].numpy())[live.numpy()].max(), np.abs(x64 - P["x"][0].numpy())[live.numpy()].max()))
        worst[kind] = np.max(err, 0)
    print("\nlargest |x - exact| (fp32 geometry, fp64 geometry):", {k: [f"{a:.3g}" for a in v] for k, v in worst.items()})
    assert worst["far1e5"][0] > 1e-3 and worst["far2e6"][0] > 1e-2
    assert worst["far1e5"][1] < 1e-5 and worst["far2e6"][1] < 1e-5


def _mesh(seed, F=40):
    g = np.random.default_rng(seed)
    c = g.uniform(-2, 30, (F, 1, 2)) + g.uniform(-5, 5, (F, 3, 2))
    c[0] = [[-40, -30], [70, -20], [10, 80]]              # covers the frame
    c[1] = [[3.3, 4.1], [3.6, 4.05], [3.4, 4.5]]           # sub-pixel
    c[2] = c[3]                                            # coincident duplicate
    c[4] = [[-9, 5], [-6, 9], [-7.5, 12]]                  # off screen, its band entering the frame
    return c.astype(f32)


@pytest.mark.parametrize("sigma", [0.25, 1.0, 4.0])
def test_reference_matches_the_oracle(sigma):
    H, W = 24, 29
    xy = _mesh(int(sigma * 4))
    fr = sf.FrameRef(xy, np.ones(len(xy), bool), H, W, sigma)
    out = fr.forward()
    p = torch.stack(torch.meshgrid(torch.arange(W, dtype=torch.float64), torch.arange(H, dtype=torch.float64), indexing="xy"), -1).reshape(-1, 2)
    L = so.log_one_minus(torch.from_numpy(xy).double(), torch.ones(len(xy), dtype=torch.bool), p, sigma).reshape(H, W)
    clear = ~out["marg"]
    assert float(clear.double().mean()) > 0.95
    assert torch.allclose(out["L"][0][clear], L[clear], rtol=1e-13, atol=0)
    assert torch.allclose(out["S"][0][clear], -torch.expm1(L)[clear], rtol=1e-13, atol=0)
    assert int(out["count"].max()) >= 3


def test_self_checks_reject_corruptions():
    """Each corruption moves some clear element beyond its bound."""
    H, W, sigma = 24, 29, 1.0
    xy = _mesh(1)[1:]                                       # without the face covering the frame, where S = 1 hides the rest
    _, _, r = sf.thresholds(sigma)
    fr = sf.FrameRef(xy, np.ones(len(xy), bool), H, W, sigma)
    boxes = np.array([[max(0, int(np.ceil(x.min() - r))), min(W - 1, int(np.floor(x.max() + r))), max(0, int(np.ceil(y.min() - r))),
                       min(H - 1, int(np.floor(y.max() + r)))] for x, y in zip(xy[..., 0], xy[..., 1])])
    ref = fr.forward()
    clear = ~ref["marg"]

    def rejects(got, want, m):
        v, e = want
        return bool(((got - v).abs() > e)[m].any())

    face = 10
    tile = int((boxes[face, 2] // 16) * sf.cdiv(W, 16) + boxes[face, 0] // 16)
    assert rejects(fr.forward(drop=(face, tile))["S"][0], ref["S"], clear)
    assert rejects(fr.forward(shrink=(face, boxes))["S"][0], ref["S"], clear)
    G = torch.linspace(-1e-3, 2e-3, H * W, dtype=torch.float64).reshape(H, W)
    want, marg = fr.face_grad(G, boxes)
    for kw in (dict(swap_t=True), dict(swap_ab=True)):
        bad, _ = fr.face_grad(G, boxes, **kw)
        assert rejects(bad[0], want, ~marg[:, None].expand(-1, 6))
    assert float(marg.double().mean()) < 0.25


def test_workspace_mirror():
    from gaussianavatar_b200 import _lib
    L = _lib.lib()
    for B, V, F, H, W in ((1, 3, 0, 1, 1), (1, 5, 1, 16, 17), (3, 7, 255, 17, 16), (8, 100, 513, 37, 53), (8, 6890, 13776, 1080, 1920),
                          (2, 9, 257, 540, 540)):
        assert L.ga_silhouette_workspace_bytes(B, V, F, H, W) == sf.workspace_layout(B, F, H, W)["total"], (B, V, F, H, W)
