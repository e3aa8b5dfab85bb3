"""numpy restatement of the body-topology rig (gaussianavatar_b200.rig.extract_body_rig; csrc/body_rig.cu, `ga_mesh_shade_unlit`).

  subdivide        midpoint subdivision of a UV template, one face at a time with dictionaries (the library uses array sorts),
                   with the skin weights of the new vertices and the K-heaviest selection
  laplacian        ga_mesh_laplacian, fp32, in the kernel's order: bit for bit
  pushpull         ga_texture_pushpull, fp32, in the kernel's order: bit for bit
  shade_unlit      ga_mesh_shade_unlit on mesh_oracle's projection and coverage, the fp64 steps in the kernel's order
  layout_matrix    B of a ga_posmap_layout (face_id, bary) as a scipy sparse matrix, texels x vertices
  solve_fit        the fit's normal equations (B^T M B + lam L) d = B^T M (g - B x0), solved directly in fp64
"""
from __future__ import annotations

import numpy as np

from . import mesh_oracle as mo

f32, f64 = np.float32, np.float64


# ---- topology -----------------------------------------------------------------------------------------------------------------------
def _split(faces, n):
    """One midpoint split of faces [F,3] over n indices: (faces [4F,3], edges [(a, b)] in the order their midpoints were numbered
    n, n + 1, ...).  Edges are numbered in ascending (min, max) order."""
    edges = sorted({(min(a, b), max(a, b)) for f in faces.tolist() for a, b in ((f[0], f[1]), (f[1], f[2]), (f[2], f[0]))})
    mid = {e: n + i for i, e in enumerate(edges)}
    m = lambda a, b: mid[(min(a, b), max(a, b))]
    out = []
    for a, b, c in faces.tolist():
        ab, bc, ca = m(a, b), m(b, c), m(c, a)
        out += [(a, ab, ca), (ab, b, bc), (ca, bc, c), (ab, bc, ca)]
    return np.asarray(out, np.int64).reshape(-1, 3), edges


def subdivide(faces, uvs, faces_uv, weights, levels: int):
    """L midpoint subdivisions: (faces, uvs [fp64], faces_uv, weights [V,J] fp64, parents [(a, b) per new vertex, level by level])."""
    faces, faces_uv = np.asarray(faces, np.int64), np.asarray(faces_uv, np.int64)
    uvs, w = np.asarray(uvs, f64), np.asarray(weights, f64)
    parents = []
    for _ in range(levels):
        nf, e = _split(faces, w.shape[0])
        nt, et = _split(faces_uv, uvs.shape[0])
        w = np.concatenate([w, np.array([(w[a] + w[b]) / 2 for a, b in e]).reshape(-1, w.shape[1])])
        uvs = np.concatenate([uvs, np.array([(uvs[a] + uvs[b]) / 2 for a, b in et]).reshape(-1, 2)])
        parents += e
        faces, faces_uv = nf, nt
    return faces, uvs, faces_uv, w, parents


def top_k(weights, K: int):
    """(joints [V,K] uint8, weights [V,K] fp32): the K largest weights (ties to the lower joint), renormalised in fp64."""
    w = np.asarray(weights, f64)
    j = np.argsort(-w, axis=1, kind="stable")[:, :K]
    v = np.take_along_axis(w, j, 1)
    s = v.sum(1, keepdims=True)
    return j.astype(np.uint8), (v / np.where(s > 0, s, 1.0)).astype(f32)


def adjacency(faces, V: int):
    """Vertex adjacency CSR (offsets [V+1], adj) int32 of the faces' edges, neighbours ascending."""
    nb = [set() for _ in range(V)]
    for a, b, c in np.asarray(faces).tolist():
        for x, y in ((a, b), (b, c), (c, a)):
            nb[x].add(y)
            nb[y].add(x)
    off = np.zeros(V + 1, np.int64)
    off[1:] = np.cumsum([len(s) for s in nb])
    return off.astype(np.int32), np.array([u for s in nb for u in sorted(s)], np.int32)


# ---- kernels --------------------------------------------------------------------------------------------------------------------------
def laplacian(offsets, adj, x):
    """ga_mesh_laplacian in fp32, bit for bit."""
    x = np.asarray(x, f32)
    off = np.asarray(offsets, np.int64)
    deg = np.diff(off)
    s = np.zeros_like(x)
    for k in range(int(deg.max()) if deg.size else 0):
        m = np.nonzero(deg > k)[0]
        s[m] = s[m] + x[adj[off[m] + k]]
    return deg.astype(f32)[:, None] * x - s


def pushpull(image, mask):
    """ga_texture_pushpull of image [C,S,S] fp32 and mask [S,S], bit for bit."""
    image = np.asarray(image, f32)
    C, S = image.shape[0], image.shape[1]
    cov = np.asarray(mask) != 0
    vals, ws = [image], [cov.astype(f32)]
    while vals[-1].shape[1] > 1:
        n = vals[-1].shape[1]
        m = (n + 1) // 2
        v = np.zeros((C, 2 * m, 2 * m), f32)
        w = np.zeros((2 * m, 2 * m), f32)
        v[:, :n, :n] = np.where(ws[-1] > 0, vals[-1], f32(0))
        w[:n, :n] = ws[-1]
        s = np.zeros((C, m, m), f32)
        t = np.zeros((m, m), f32)
        have = np.zeros((m, m), bool)
        for i, j in ((0, 0), (0, 1), (1, 0), (1, 1)):
            wk, vk = w[i::2, j::2], v[:, i::2, j::2]
            on = wk > 0
            p = wk * vk
            s = np.where(on, np.where(have, s + p, p), s)
            t = np.where(on, np.where(have, t + wk, wk), t)
            have |= on
        with np.errstate(invalid="ignore", divide="ignore"):
            vals.append(np.where(have, s / np.where(have, t, f32(1)), f32(0)).astype(f32))
        ws.append(t)
    for l in range(len(vals) - 2, -1, -1):
        n = vals[l].shape[1]
        r = np.arange(n) // 2
        parent = vals[l + 1][:, r[:, None], r[None, :]]
        vals[l] = np.where(ws[l] > 0, vals[l], parent)
    if len(vals) == 1:
        vals[0] = np.where(cov, image, f32(0))
    return vals[0]


def shade_unlit(X, faces, cam, face_id, H, W, colors=None, uvs=None, texture=None, background=None):
    """ga_mesh_shade_unlit of one frame: X [V,3] fp32, face_id [H,W] -> rgb [3,H,W] fp32."""
    X = np.asarray(X, f32)
    x, y, z, ok = mo.project(X, cam, H, W)
    s = mo.setup_faces(np.asarray(faces, np.int64).reshape(-1, 3), x, y, z, ok, H, W)
    fid = np.asarray(face_id).reshape(-1)
    out = np.zeros((3, H * W), f32) if background is None else np.asarray(background, f32).reshape(3, H * W).copy()
    F = s["area"].shape[0]
    pix = np.nonzero((fid >= 0) & (fid < F))[0]
    pix = pix[s["drawn"][fid[pix]]]
    f = fid[pix]
    e, _ = mo.edges_at(s, f, pix % W, pix // W)
    q, tot = mo.inv_depth(s, f, e)
    w = [qi / tot for qi in q]
    v = s["v"][f]
    lerp = lambda a, k: (w[0] * a[v[:, 0], k] + w[1] * a[v[:, 1], k]) + w[2] * a[v[:, 2], k]
    if colors is not None:
        c = np.asarray(colors, f32).astype(f64)
        for ch in range(3):
            out[ch, pix] = lerp(c, ch).astype(f32)
        return out.reshape(3, H, W)
    uv = np.asarray(uvs, f32).astype(f64)
    T = np.asarray(texture, f32).astype(f64)
    Th, Tw = T.shape[:2]
    px, py = lerp(uv, 0) * Tw - 0.5, lerp(uv, 1) * Th - 0.5
    x0, y0 = np.floor(px), np.floor(py)
    fx, fy = px - x0, py - y0
    cl = lambda a, n: np.clip(np.nan_to_num(a, nan=0.0), 0, n - 1).astype(np.int64)
    c0, c1, r0, r1 = cl(x0, Tw), cl(x0 + 1, Tw), cl(y0, Th), cl(y0 + 1, Th)
    gx, gy = 1.0 - fx, 1.0 - fy
    for ch in range(3):
        top = gx * T[r0, c0, ch] + fx * T[r0, c1, ch]
        bot = gx * T[r1, c0, ch] + fx * T[r1, c1, ch]
        out[ch, pix] = (gy * top + fy * bot).astype(f32)
    return out.reshape(3, H, W)


# ---- the fit --------------------------------------------------------------------------------------------------------------------------
def layout_matrix(faces, face_id, bary, V):
    """B [S*S, V] (scipy CSR): row t = sum_i bary[t,i] e_{faces[face_id[t], i]}, empty where face_id is -1."""
    from scipy.sparse import csr_matrix
    fid = np.asarray(face_id).reshape(-1)
    t = np.nonzero(fid >= 0)[0]
    fc = np.asarray(faces, np.int64)[fid[t]]
    b = np.asarray(bary, f64).reshape(-1, 3)[t]
    return csr_matrix((b.reshape(-1), (np.repeat(t, 3), fc.reshape(-1))), shape=(fid.size, V))


def laplacian_matrix(offsets, adj, V):
    from scipy.sparse import csr_matrix, diags
    off = np.asarray(offsets, np.int64)
    A = csr_matrix((np.ones(off[-1]), np.asarray(adj, np.int64)[:off[-1]], off), shape=(V, V))
    return diags(np.diff(off).astype(f64)) - A


def solve_fit(Bm, mask, g, x0, Lm, lam):
    """x = x0 + d with d minimising sum_{t in M} |(B(x0 + d))_t - g_t|^2 + lam d^T L d, by a direct fp64 solve of the normal equations.
    Bm [T,V] sparse, mask [T] bool, g [T,3] (rows outside the mask are ignored), x0 [V,3], Lm [V,V] sparse.  Vertices the system leaves
    undetermined (no data in their component) keep d = 0."""
    from scipy.sparse import diags
    from scipy.sparse.linalg import spsolve
    Mm = diags(np.asarray(mask, f64).reshape(-1))
    x0 = np.asarray(x0, f64)
    r = np.where(np.asarray(mask).reshape(-1, 1), np.asarray(g, f64) - Bm @ x0, 0.0)
    A = (Bm.T @ Mm @ Bm + lam * Lm).tocsc()
    rhs = Bm.T @ (Mm @ r)
    free = np.asarray(abs(A).sum(1)).reshape(-1) > 0
    # a component without data has A = lam L there, singular: pin it at d = 0
    from scipy.sparse.csgraph import connected_components
    ncomp, lab = connected_components(abs(A) > 0, directed=False)
    has = np.zeros(ncomp, bool)
    has[lab[np.asarray(Bm.T @ np.asarray(mask, f64).reshape(-1)).reshape(-1) > 0]] = True
    keep = free & has[lab]
    d = np.zeros_like(x0)
    idx = np.nonzero(keep)[0]
    if idx.size:
        d[idx] = spsolve(A[idx][:, idx], rhs[idx]).reshape(-1, 3)
    return x0 + d
