"""numpy restatement of the mesh extraction kernels (csrc/tsdf.cu: `ga_tsdf_integrate`, `ga_tsdf_mesh_count` / `ga_tsdf_mesh_emit`).

Integration runs in the kernel's order, every fp32 step one numpy float32 operation (the kernel's explicitly rounded __f*_rn ops; its
fused multiply-adds through mesh_oracle.fma32), so the pixel each sample reads, the weights and carve counts match exactly and the
sdf and colour sums bit for bit.  The mesher restates the case-table rule, the classification and the emission order (vertices by
owner and slot, faces by cube, tetrahedron and triangle), so faces compare exactly and vertices and colours to fp32 rounding.
There is no reference code for this feature: it is defined here (DESIGN.md §2)."""
from __future__ import annotations

import numpy as np

from .mesh_oracle import xf_row

f32, f64 = np.float32, np.float64
ZCULL = f32(0.2)

# cube corner c at p + (c & 1, (c >> 1) & 1, (c >> 2) & 1); tetrahedron t = (0, e_a, e_a + e_b, 7) for the axis order PERM[t]
PERM = ((0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0))
EDGE_V = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))
SLOT_MASKS = (1, 2, 4, 3, 5, 6, 7)          # slot -> d as a corner mask: x, y, z, xy, xz, yz, xyz
POPC = np.array([bin(m).count("1") for m in range(128)], np.int64)


def corner_offset(c):
    return np.array([c & 1, (c >> 1) & 1, (c >> 2) & 1], np.int64)


def tet_corners(t):
    a, b = PERM[t][0], PERM[t][1]
    return (0, 1 << a, (1 << a) | (1 << b), 7)


def _local_edge(i, j):
    return EDGE_V.index((min(i, j), max(i, j)))


def case_table():
    """(ntri [6,16], edges [6,16,2,3] local edge ids (-1 unused), corner [6,4], owner [6,6] cube corner, slot [6,6]): one triangle
    for one or three inside vertices, the quad ac, ad, bd, bc split along ac-bd for two, each wound so that its normal at the edge
    midpoints points from the inside vertices' centroid to the outside vertices'."""
    ntri = np.zeros((6, 16), np.int64)
    edges = np.full((6, 16, 2, 3), -1, np.int64)
    corner = np.array([tet_corners(t) for t in range(6)], np.int64)
    owner = np.zeros((6, 6), np.int64)
    slot = np.zeros((6, 6), np.int64)
    for t in range(6):
        cs = tet_corners(t)
        pos = [corner_offset(c) for c in cs]
        for e, (i, j) in enumerate(EDGE_V):
            owner[t, e] = cs[i]
            slot[t, e] = SLOT_MASKS.index(cs[j] ^ cs[i])
        for c in range(16):
            ins = [v for v in range(4) if (c >> v) & 1]
            outs = [v for v in range(4) if not (c >> v) & 1]
            if len(ins) in (1, 3):
                lone, rest = (ins[0], outs) if len(ins) == 1 else (outs[0], ins)
                tris = [[_local_edge(lone, r) for r in rest]]
            elif len(ins) == 2:
                (a, b), (cc, d) = ins, outs
                ac, ad, bd, bc = _local_edge(a, cc), _local_edge(a, d), _local_edge(b, d), _local_edge(b, cc)
                tris = [[ac, ad, bd], [ac, bd, bc]]
            else:
                tris = []
            for k, tri in enumerate(tris):
                P = [pos[EDGE_V[e][0]] + pos[EDGE_V[e][1]] for e in tri]
                n = np.cross(P[1] - P[0], P[2] - P[0])
                o = len(ins) * sum(pos[v] for v in outs) - len(outs) * sum(pos[v] for v in ins)
                if n @ o < 0:
                    tri = [tri[0], tri[2], tri[1]]
                edges[t, c, k] = tri
            ntri[t, c] = len(tris)
    return ntri, edges, corner, owner, slot


# ---- state ------------------------------------------------------------------------------------------------------------------------
def new_state(dims):
    """Zeroed state of a grid (nx, ny, nz): dict of [nz,ny,nx] planes."""
    nx, ny, nz = dims
    z = lambda dt: np.zeros((nz, ny, nx), dt)
    return dict(sdf=z(f32), weight=z(np.int32), carve=z(np.int32), r=z(f32), g=z(f32), b=z(f32), cw=z(np.int32))


def sample_positions(origin, voxel, dims):
    """World positions (x, y, z) [nz,ny,nx] float32 of the samples: origin + voxel * index, one rounding per step."""
    nx, ny, nz = dims
    o = np.asarray(origin, f32)
    v = f32(voxel)
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    return (o[0] + v * i.astype(f32), o[1] + v * j.astype(f32), o[2] + v * k.astype(f32))


def project(cam, H, W, x, y, z):
    """(pixx, pixy, view z) float32 of world points: the Gaussian preprocess's projection and ndc2Pix (mesh_project.cuh)."""
    cam = np.asarray(cam, f32)
    view, proj = cam[:16], cam[16:32]
    vz = xf_row(view, 2, x, y, z)
    hx, hy, hw = xf_row(proj, 0, x, y, z), xf_row(proj, 1, x, y, z), xf_row(proj, 3, x, y, z)
    with np.errstate(all="ignore"):
        p_w = f32(1) / (hw + f32(1e-7))
        ndc_x, ndc_y = hx * p_w, hy * p_w
        pixx = (((ndc_x.astype(f64) + 1.0) * W - 1.0) * 0.5).astype(f32)
        pixy = (((ndc_y.astype(f64) + 1.0) * H - 1.0) * 0.5).astype(f32)
    return pixx, pixy, vz


def integrate(state, origin, voxel, trunc, cams, depth, image, final_T):
    """Folds the views in order into `state` (in place, and returned): cams [B,40], depth [B,2,H,W], image [B,3,H,W] (bg 0),
    final_T [B,H,W]."""
    dims = state["sdf"].shape[::-1]
    x, y, z = sample_positions(origin, voxel, dims)
    tau = f32(trunc)
    depth, image, final_T = (np.asarray(a, f32) for a in (depth, image, final_T))
    H, W = depth.shape[2], depth.shape[3]
    S = state
    for v in range(len(cams)):
        pixx, pixy, vz = project(cams[v], H, W, x, y, z)
        with np.errstate(all="ignore"):
            fc, fr = np.rint(pixx), np.rint(pixy)
            ok = (vz > ZCULL) & (fc >= 0) & (fc < f32(W)) & (fr >= 0) & (fr < f32(H))
        c = np.where(ok, fc, 0).astype(np.int64)
        r = np.where(ok, fr, 0).astype(np.int64)
        d = depth[v, 1][r, c]
        carve = ok & (d == 0)
        S["carve"] += carve.astype(np.int32)
        with np.errstate(all="ignore"):
            eta = d - vz
            upd = ok & (d != 0) & ~(eta < -tau)
            s = np.fmin(f32(1), eta / tau)
            w = S["weight"]
            new = (S["sdf"] * w.astype(f32) + s) / (w + 1).astype(f32)
        S["sdf"] = np.where(upd, new, S["sdf"]).astype(f32)
        S["weight"] = (w + upd).astype(np.int32)
        col = upd & (np.abs(eta) < tau)
        a = f32(1) - final_T[v][r, c]
        for ch, key in enumerate("rgb"):
            with np.errstate(all="ignore"):
                add = S[key] + image[v, ch][r, c] / a
            S[key] = np.where(col, add, S[key]).astype(f32)
        S["cw"] = (S["cw"] + col).astype(np.int32)
    return S


def classify(state, min_carve=1):
    """The mesher's sample values [nz,ny,nx] float32: +1 on the outer layer and where carve >= min_carve, -1 where weight = 0,
    otherwise sdf.  Inside iff < 0."""
    v = np.where(state["carve"] >= min_carve, f32(1), np.where(state["weight"] == 0, f32(-1), state["sdf"])).astype(f32)
    v[0], v[-1], v[:, 0], v[:, -1], v[:, :, 0], v[:, :, -1] = 1, 1, 1, 1, 1, 1
    return v


def mean_colors(state):
    """Mean colour [nz,ny,nx,3] float32 (0 where the colour weight is 0) and the colour weight."""
    cw = state["cw"]
    n = np.where(cw > 0, cw, 1).astype(f32)
    return np.stack([np.where(cw > 0, state[k] / n, f32(0)) for k in "rgb"], -1).astype(f32), cw


def mesh(state, origin, voxel, min_carve=1):
    """(verts [V,3] float32, faces [F,3] int32, colors [V,3] float32) of a fused state."""
    col, cw = mean_colors(state)
    return mesh_from_values(classify(state, min_carve), origin, voxel, col, cw)


def mesh_from_values(values, origin, voxel, colors=None, cw=None):
    """Marching tetrahedra of sample values [nz,ny,nx] (inside iff < 0; the outer layer must be outside for a closed mesh), in the
    kernels' order.  colors [nz,ny,nx,3] / cw [nz,ny,nx]: per-sample mean colours and colour weights (default: none)."""
    values = np.asarray(values, f32)
    nz, ny, nx = values.shape
    N = values.size
    s = values.reshape(-1)
    inside = s < 0
    col = np.zeros((N, 3), f32) if colors is None else np.asarray(colors, f32).reshape(N, 3)
    has = np.zeros(N, bool) if cw is None else np.asarray(cw).reshape(N) > 0
    idx = np.arange(N, dtype=np.int64)
    i, j, k = idx % nx, (idx // nx) % ny, idx // (nx * ny)
    ijk = np.stack([i, j, k], 1)
    strides = np.array([1, nx, nx * ny], np.int64)

    def present(c):
        o = corner_offset(c)
        return (i + o[0] < nx) & (j + o[1] < ny) & (k + o[2] < nz)

    def nb(c):
        return idx + corner_offset(c) @ strides

    cross = np.zeros((N, 7), bool)
    for sl, m in enumerate(SLOT_MASKS):
        ok = present(m)
        q = np.where(ok, nb(m), 0)
        cross[:, sl] = ok & (inside != inside[q])
    cnt = cross.sum(1)
    voff = np.concatenate([[0], np.cumsum(cnt)])[:-1]
    vmask = (cross * (1 << np.arange(7))).sum(1)

    p, sl = np.nonzero(cross)                          # row-major: by owner, then slot
    m = np.array(SLOT_MASKS, np.int64)[sl]
    d = np.stack([m & 1, (m >> 1) & 1, (m >> 2) & 1], 1)
    q = p + d @ strides
    s0, s1 = s[p], s[q]
    t = s0 / (s0 - s1)
    g = ijk[p].astype(f32) + t[:, None] * d.astype(f32)
    verts = np.asarray(origin, f32)[None, :] + f32(voxel) * g
    c0, c1 = col[p], col[q]
    h0, h1 = has[p][:, None], has[q][:, None]
    x0 = np.where(h0, c0, c1)
    x1 = np.where(h1, c1, c0)
    colors_out = (x0 + t[:, None] * (x1 - x0)).astype(f32)

    ntri, edges, corner, owner, slot = case_table()
    cubes = np.nonzero(present(7))[0]
    inb = inside.astype(np.int64)
    keys, tris = [], []
    for tt in range(6):
        cs = sum(inb[nb(int(corner[tt, v]))[cubes]] << v for v in range(4))
        for kk in range(2):
            sel = ntri[tt, cs] > kk
            cc, cse = cubes[sel], cs[sel]
            ids = []
            for qq in range(3):
                e = edges[tt, cse, kk, qq]
                own = cc + np.array([corner_offset(int(o)) @ strides for o in range(8)])[owner[tt, e]]
                sl_ = slot[tt, e]
                below = vmask[own] & ((1 << sl_) - 1)
                ids.append(voff[own] + POPC[below])
            tris.append(np.stack(ids, 1) if ids[0].size else np.zeros((0, 3), np.int64))
            keys.append(np.stack([cc, np.full(cc.size, tt), np.full(cc.size, kk)], 1))
    keys = np.concatenate(keys)
    tris = np.concatenate(tris)
    order = np.lexsort((keys[:, 2], keys[:, 1], keys[:, 0]))
    return verts.astype(f32), tris[order].astype(np.int32), colors_out
