"""numpy restatement of the screen-space mesh renderer (csrc/mesh_render.cu, `ga_mesh_render`), in the kernel's operation order.

Every fp32 step is one numpy float32 operation (the kernel's explicitly rounded __f*_rn ops; its fused multiply-adds through
`fma32`, an exact emulation), every fp64 step is done in fp64, and the coverage is the same int64 arithmetic, so face_id and depth
compare bit for bit and rgb to the last few ulps.  What is assumed of pyrender (area-weighted normals, the BRDF, the headlight, the
near-plane rule) is listed in DESIGN.md §2: PARITY UNPINNED, as the reference's GL overlay is neither vendored nor run here."""
from __future__ import annotations

import numpy as np

f32, f64 = np.float32, np.float64
ZNEAR = f32(0.01)
GUARD = f32(1 << 20)
METALLIC, ROUGHNESS, LIGHT, PI = f32(0.2), f32(0.6), f32(3.0), f32(3.14159265358979)
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


def fma32(a, b, c):
    """fmaf(a, b, c) for float32 arrays: a * b is exact in fp64, the sum's error is recovered exactly (TwoSum), and a sum that lands
    on a float32 rounding midpoint is resolved by that error's sign (the one case where rounding fp64 -> fp32 twice differs)."""
    a, b, c = (np.asarray(x, f32) for x in (a, b, c))
    p = a.astype(f64) * b.astype(f64)
    c64 = c.astype(f64)
    s = p + c64
    bb = s - p
    err = (p - (s - bb)) + (c64 - bb)
    r = s.astype(f32)
    r64 = r.astype(f64)
    other = np.where(s > r64, np.nextafter(r, f32(np.inf)), np.nextafter(r, f32(-np.inf)))
    o64 = other.astype(f64)
    mid = (r64 != s) & (s - r64 == o64 - s)
    fix = mid & (err != 0) & (np.sign(err) == np.sign(o64 - s))
    return np.where(fix, other, r)


def xf_row(M, r, x, y, z):
    t = M[r] * x
    t = fma32(M[4 + r], y, t)
    t = fma32(M[8 + r], z, t)
    return t + M[12 + r]


def dot3(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def normalize3(a, fallback=None):
    """a [3,...] float32 / |a| where |a| > 0; elsewhere a itself, or `fallback` [3] when given."""
    l2 = dot3(a, a)
    ok = l2 > 0
    l = np.sqrt(np.where(ok, l2, f32(1)))
    out = np.where(ok, a / l, a)
    if fallback is not None:
        out = np.where(ok, out, np.asarray(fallback, f32).reshape((3,) + (1,) * (out.ndim - 1)))
    return out


def vertex_normals(X, faces, offsets, adj):
    """X [V,3] float32 -> normalised sums of the adjacent faces' cross products [V,3], summed in CSR order."""
    p0, p1, p2 = (X[faces[:, i]].T for i in range(3))
    a, c = p1 - p0, p2 - p0
    cross = np.stack([a[1] * c[2] - a[2] * c[1], a[2] * c[0] - a[0] * c[2], a[0] * c[1] - a[1] * c[0]])      # [3,F]
    V = X.shape[0]
    n = np.zeros((3, V), f32)
    deg = np.diff(offsets.astype(np.int64))
    for k in range(int(deg.max()) if V else 0):
        m = np.nonzero(deg > k)[0]
        n[:, m] = n[:, m] + cross[:, adj[offsets[m] + k]]
    return normalize3(n).T


def project(X, cam, H, W):
    """Screen positions of X [V,3]: (x, y) in 1/256 pixel, y up (int64), view-space z (float32), ok (z > znear, in the guard band)."""
    cam = np.asarray(cam, f32)
    view, proj = cam[:16], cam[16:32]
    px, py, pz = X[:, 0], X[:, 1], X[:, 2]
    tvz = xf_row(view, 2, px, py, pz)
    hx, hy, hw = xf_row(proj, 0, px, py, pz), xf_row(proj, 1, px, py, pz), xf_row(proj, 3, px, py, pz)
    with np.errstate(all="ignore"):
        p_w = f32(1) / (hw + f32(1e-7))
        ndc_x, ndc_y = hx * p_w, hy * p_w
        pixx = (((ndc_x.astype(f64) + 1.0) * W - 1.0) * 0.5).astype(f32)
        pixy = (((ndc_y.astype(f64) + 1.0) * H - 1.0) * 0.5).astype(f32)
        ok = (tvz > ZNEAR) & (np.abs(pixx) <= GUARD) & (np.abs(pixy) <= GUARD)
    x = np.where(ok, np.rint(np.where(ok, pixx, 0).astype(f64) * 256.0), 0).astype(np.int64)
    y = -np.where(ok, np.rint(np.where(ok, pixy, 0).astype(f64) * 256.0), 0).astype(np.int64)
    return x, y, tvz, ok


def edge(ax, ay, bx, by, px, py):
    return (bx - ax) * (py - ay) - (by - ay) * (px - ax)


def owns(e, dx, dy):
    return (e > 0) | ((e == 0) & ((dy < 0) | ((dy == 0) & (dx < 0))))


def setup_faces(faces, x, y, z, ok, H, W):
    """Per face: corners (counter-clockwise, y up) x, y [F,3], z [F,3], vertex ids [F,3], area, pixel box, and whether it is drawn."""
    v = np.asarray(faces, np.int64).copy()
    fx, fy, fz = x[v], y[v], z[v]
    area = edge(fx[:, 0], fy[:, 0], fx[:, 1], fy[:, 1], fx[:, 2], fy[:, 2])
    neg = area < 0
    for a in (fx, fy, fz, v):
        a[neg, 1], a[neg, 2] = a[neg, 2].copy(), a[neg, 1].copy()
    area = np.abs(area)
    c0 = np.maximum(0, (fx.min(1) + 255) >> 8)
    c1 = np.minimum(W - 1, fx.max(1) >> 8)
    r0 = np.maximum(0, (-fy.max(1) + 255) >> 8)
    r1 = np.minimum(H - 1, (-fy.min(1)) >> 8)
    drawn = ok[faces].all(1) & (area != 0) & (c0 <= c1) & (r0 <= r1)
    return dict(x=fx, y=fy, z=fz, v=v, area=area, c0=c0, c1=c1, r0=r0, r1=r1, drawn=drawn, front=~neg)


def edges_at(s, f, c, r):
    """Edge functions e[i] (opposite corner i) of faces f at the centres of pixels (c, r), and whether the faces own them."""
    px, py = 256 * c.astype(np.int64), -256 * r.astype(np.int64)
    x, y = s["x"][f], s["y"][f]
    e0 = edge(x[:, 1], y[:, 1], x[:, 2], y[:, 2], px, py)
    e1 = edge(x[:, 2], y[:, 2], x[:, 0], y[:, 0], px, py)
    e2 = edge(x[:, 0], y[:, 0], x[:, 1], y[:, 1], px, py)
    inside = owns(e2, x[:, 1] - x[:, 0], y[:, 1] - y[:, 0]) & owns(e0, x[:, 2] - x[:, 1], y[:, 2] - y[:, 1]) & \
        owns(e1, x[:, 0] - x[:, 2], y[:, 0] - y[:, 2])
    return (e0, e1, e2), inside


def inv_depth(s, f, e):
    A = s["area"][f].astype(f64)
    q = [(e[i].astype(f64) / A) / s["z"][f, i].astype(f64) for i in range(3)]
    return q, (q[0] + q[1]) + q[2]


def _covered(s, H, W, fs, rows=(0, 1), chunk=1 << 22):
    """Yields (face, column, row, edge functions) of every pixel centre a face of fs owns, in chunks; only in the rows
    rows[0] + k rows[1] (all rows by default)."""
    ro, rk = rows
    j0 = -((ro - s["r0"][fs]) // rk)                      # first k with ro + k rk >= r0
    nr = np.maximum(0, (s["r1"][fs] - ro) // rk - j0 + 1)
    wc = (s["c1"][fs] - s["c0"][fs] + 1)
    cnt = wc * nr
    ends = np.cumsum(cnt)
    lo = 0
    while lo < fs.size:
        start = ends[lo] - cnt[lo]
        hi = max(lo + 1, int(np.searchsorted(ends, start + chunk, side="right")))
        sel = np.arange(lo, hi)
        f = np.repeat(fs[sel], cnt[sel])
        k = np.arange(int(cnt[sel].sum()), dtype=np.int64) - np.repeat(ends[sel] - cnt[sel] - start, cnt[sel])
        w = np.repeat(wc[sel], cnt[sel])
        c = s["c0"][f] + k % w
        r = ro + rk * (np.repeat(j0[sel], cnt[sel]) + k // w)
        e, inside = edges_at(s, f, c, r)
        yield f[inside], c[inside], r[inside], tuple(x[inside] for x in e)
        lo = hi


def raster(s, H, W, rows=(0, 1)):
    """keys [H*W] uint64: the minimum over the faces covering each pixel centre of (fp32 depth bits << 32) | face (EMPTY outside
    the rows rows[0] + k rows[1])."""
    keys = np.full(H * W, EMPTY, np.uint64)
    for f, c, r, e in _covered(s, H, W, np.nonzero(s["drawn"])[0], rows):
        _, tot = inv_depth(s, f, e)
        d = (1.0 / tot).astype(f32)
        key = (d.view(np.uint32).astype(np.uint64) << np.uint64(32)) | f.astype(np.uint64)
        np.minimum.at(keys, r * W + c, key)
    return keys


def coverage(s, H, W, faces=None):
    """[H,W] int64: how many of the drawn faces (all, or those of the boolean mask `faces`) own each pixel centre."""
    sel = s["drawn"] if faces is None else s["drawn"] & faces
    n = np.zeros(H * W, np.int64)
    for f, c, r, _ in _covered(s, H, W, np.nonzero(sel)[0]):
        np.add.at(n, r * W + c, 1)
    return n.reshape(H, W)


def shade(n, l, v, base):
    """glTF 2.0 metallic-roughness BRDF (Appendix B) of one directional light; n, l, v [3,P] unit, base [3] -> [3,P] in [0,1]."""
    NdotL = dot3(n, l)
    h = normalize3(l + v, fallback=l)
    NdotV, NdotH, VdotH = np.fmax(dot3(n, v), f32(0)), np.fmax(dot3(n, h), f32(0)), np.fmax(dot3(v, h), f32(0))
    alpha = ROUGHNESS * ROUGHNESS
    a2 = alpha * alpha
    one_a2 = f32(1) - a2
    gv = np.sqrt(NdotV * NdotV * one_a2 + a2)
    gl = np.sqrt(NdotL * NdotL * one_a2 + a2)
    with np.errstate(all="ignore"):
        vis = f32(0.5) / (NdotL * gv + NdotV * gl)
    dd = NdotH * NdotH * (a2 - f32(1)) + f32(1)
    D = a2 / (PI * (dd * dd))
    t = f32(1) - VdotH
    t2 = t * t
    t5 = t2 * t2 * t
    one_m = f32(1) - METALLIC
    li = LIGHT * NdotL
    out = []
    for ch in range(3):
        b = f32(base[ch])
        f0 = f32(0.04) * one_m + b * METALLIC
        cdiff = b * f32(0.96) * one_m
        F = f0 + (f32(1) - f0) * t5
        c = li * ((f32(1) - F) * cdiff / PI + F * vis * D)
        out.append(np.fmin(np.fmax(c, f32(0)), f32(1)))
    out = np.stack(out)
    return np.where(NdotL > 0, out, f32(0))


def render_frame(X, faces, offsets, adj, cam, H, W, background=None, color=(1.0, 0.98, 0.94), rows=(0, 1)):
    """One frame: X [V,3], faces [F,3], CSR (offsets, adj), cam [40] -> rgb [3,H,W], face_id [H,W] int32, depth [H,W] float32.
    rows = (o, k): only the rows o + j k are computed (the others hold the background), for large frames of meshes with large faces."""
    X = np.asarray(X, f32)
    cam = np.asarray(cam, f32)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    normals = vertex_normals(X, faces, np.asarray(offsets, np.int64), np.asarray(adj, np.int64))
    x, y, z, ok = project(X, cam, H, W)
    s = setup_faces(faces, x, y, z, ok, H, W)
    keys = raster(s, H, W, rows)
    drawn = keys != EMPTY
    face_id = np.where(drawn, (keys & np.uint64(0xFFFFFFFF)).astype(np.int64), -1).astype(np.int32)
    depth = np.where(drawn, (keys >> np.uint64(32)).astype(np.uint32).view(f32), f32(0)).astype(f32)
    rgb = np.zeros((3, H * W), f32) if background is None else np.asarray(background, f32).reshape(3, H * W).copy()
    t = np.nonzero(drawn)[0]
    if t.size:
        f = face_id[t].astype(np.int64)
        c, r = t % W, t // W
        e, _ = edges_at(s, f, c, r)
        q, tot = inv_depth(s, f, e)
        w = [(q[i] / tot).astype(f32) for i in range(3)]
        vid = s["v"][f]
        nrm = (w[0] * normals[vid[:, 0]].T + w[1] * normals[vid[:, 1]].T) + w[2] * normals[vid[:, 2]].T
        P = (w[0] * X[vid[:, 0]].T + w[1] * X[vid[:, 1]].T) + w[2] * X[vid[:, 2]].T
        M = cam[:16]
        l = normalize3(np.array([-M[2], -M[6], -M[10]], f32))
        C = np.array([-((M[4 * k] * M[12] + M[4 * k + 1] * M[13]) + M[4 * k + 2] * M[14]) for k in range(3)], f32)
        v = normalize3(C[:, None] - P, fallback=l)
        nrm = normalize3(nrm, fallback=l)
        nrm = np.where(dot3(nrm, v) < 0, -nrm, nrm)
        base = [f32(c) for c in color]
        rgb[:, t] = shade(nrm, l[:, None], v, base)
    return rgb.reshape(3, H, W), face_id.reshape(H, W), depth.reshape(H, W)


def render(X, faces, offsets, adj, cams, H, W, background=None, color=(1.0, 0.98, 0.94)):
    """B frames: X [B,V,3], cams [B,40] -> rgb [B,3,H,W], face_id [B,H,W], depth [B,H,W]."""
    out = [render_frame(X[b], faces, offsets, adj, cams[b], H, W, None if background is None else background[b], color)
           for b in range(len(X))]
    return tuple(np.stack(o) for o in zip(*out))
