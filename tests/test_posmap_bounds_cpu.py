"""CPU: the bound models of tests/test_posmap_kernels_gpu.py checked where they are written.

The vertex-posing kernels of csrc/posmap.cu (forward, the backward's per-CTA slots, its finish) are restated here in fp32, in
their operation order, as fp64 tensors rounded to fp32 after every operation (fmaf where the kernels call it).  Those emulations
must lie within the bounds the GPU file holds the kernels to, and every corruption the GPU file's self-checks name (a row group
of the pose-blend offset dropped, a frame's vertex from its neighbour, d_feat of every joint dropped, the last CTA's slot left
out, the homogeneous column of d_A dropped) must be rejected by the same bounds when it is made in the emulation.  The fill,
weight-map and fill-backward emulations, which the GPU file holds the kernels to bit for bit, must agree with
oracle/posefit_oracle.fill and its autograd within the fp32 rounding of those expressions.
"""
import numpy as np
import pytest
import torch

import raster_fp64 as rf
from test_posmap_kernels_gpu import (KV, Mesh, case_pose, csr_reference, d_verts_of, fill_bwd_emulation, fill_emulation, finish_model,
                                     group_offset, pose_model, slot_model, vertex_model, weights_emulation)
from test_step_kernels_gpu import E8F, gam, ratio, rejects

CPU = "cpu"


def f(x):
    return x.float().double()


def fma(a, b, c):
    return rf.fma32(a, b, c)


# ===================================================================================================== fp32 emulations
def emu_rodrigues(r):
    """rodrigues(): r [n, 3] -> R, and (n, theta, s, c, K, K2) for the backward."""
    n = f(r + E8F)
    th = f(torch.sqrt(f(f(f(n[:, 0] * n[:, 0]) + f(n[:, 1] * n[:, 1])) + f(n[:, 2] * n[:, 2]))))
    d = f(r / th[:, None])
    s, c = f(torch.sin(th)), f(torch.cos(th))
    z = torch.zeros_like(d[:, 0])
    K = torch.stack([z, -d[:, 2], d[:, 1], d[:, 2], z, -d[:, 0], -d[:, 1], d[:, 0], z], 1).view(-1, 3, 3)
    K2 = f(K[:, :, 0, None] * K[:, None, 0, :])
    for k in (1, 2):
        K2 = f(K2 + f(K[:, :, k, None] * K[:, None, k, :]))
    I = torch.eye(3, dtype=r.dtype)[None]
    R = f(f(I + f(s[:, None, None] * K)) + f(f(1 - c)[:, None, None] * K2))
    return R, (n, th, s, c, K, K2)


def emu_aff_mul(A, B):
    C = torch.empty_like(B)
    for c in range(4):
        t = f(f(f(A[..., :, 0] * B[..., 0, c, None]) + f(A[..., :, 1] * B[..., 1, c, None])) + f(A[..., :, 2] * B[..., 2, c, None]))
        C[..., :, c] = f(t + A[..., :, 3]) if c == 3 else t
    return C


def emu_pose_phase(m, full):
    """pose_phase: (R [B, J, 3, 3], L, G (chain_product, right to left), A [B, J, 3, 4], feat [B, kF])."""
    B, J, P = full.shape[0], m.J, m.parents
    r = full.double().view(B * J, 3)
    R, _ = emu_rodrigues(r)
    R = R.view(B, J, 3, 3)
    Jr = m.Jr.double()
    rel = torch.stack([Jr[j] if P[j] < 0 else f(Jr[j] - Jr[P[j]]) for j in range(J)])
    L = torch.cat([R, rel[None, :, :, None].expand(B, J, 3, 1)], -1)
    G = []
    for j in range(J):
        g = L[:, j]
        q = P[j]
        while q >= 0:
            g = emu_aff_mul(L[:, q], g)
            q = P[q]
        G.append(g)
    G = torch.stack(G, 1)
    GJ = f(f(f(G[..., 0] * Jr[None, :, None, 0]) + f(G[..., 1] * Jr[None, :, None, 1])) + f(G[..., 2] * Jr[None, :, None, 2]))
    A = torch.cat([G[..., :3], f(G[..., 3] - GJ)[..., None]], -1)
    feat = f(R[:, 1:] - torch.eye(3, dtype=R.dtype)).reshape(B, -1)
    return R, L, G, A, feat


def emu_offset(m, feat, groups, drop=None):
    """sum_r feat[r] pd[r, :] as `groups` row groups of FMA chains added from 0 in order (4 in the forward, 8 in pass 1)."""
    pd = m.posedirs.double()
    off = torch.zeros(feat.shape[0], pd.shape[1], dtype=torch.float64)
    for g in range(groups):
        acc = torch.zeros_like(off)
        for r in range(g, m.kF, groups):
            acc = fma(feat[:, r, None], pd[r][None], acc)
        if g != drop:
            off = f(off + acc)
    return off.view(feat.shape[0], m.V, 3)


def emu_blend(m, A):
    """blend_transform: T [B, V, 12], a kJ-term fmaf chain from 0."""
    w = m.weights.double()
    A12 = A.reshape(A.shape[0], m.J, 12)
    T = torch.zeros(A.shape[0], m.V, 12, dtype=torch.float64)
    for j in range(m.J):
        T = fma(w[None, :, j, None], A12[:, None, j], T)
    return T


def emu_vertices(m, full, transl, drop=None):
    B = full.shape[0]
    _, _, _, A, feat = emu_pose_phase(m, full)
    x = f(m.v_shaped.double()[None] + emu_offset(m, feat, 4, drop))
    T = emu_blend(m, A).view(B, m.V, 3, 4)
    tr = transl.double()[:, None, :]
    o = f(f(f(f(f(T[..., 0] * x[:, :, None, 0]) + f(T[..., 1] * x[:, :, None, 1])) + f(T[..., 2] * x[:, :, None, 2])) + T[..., 3]) + tr)
    return o


def emu_slots(m, full, g, no_homogeneous=False):
    """Pass 1: slots [ctas, B, kN] of d_verts g [B, V, 3]."""
    B, V, J = full.shape[0], m.V, m.J
    _, _, _, A, feat = emu_pose_phase(m, full)
    T = emu_blend(m, A).view(B, V, 3, 4)
    dx = f(f(f(T[:, :, 0, :3] * g[..., 0, None]) + f(T[:, :, 1, :3] * g[..., 1, None])) + f(T[:, :, 2, :3] * g[..., 2, None]))
    x = f(m.v_shaped.double()[None] + emu_offset(m, feat, 8))
    gx = torch.cat([f(g[..., :, None] * x[..., None, :]), g[..., :, None]], -1)          # [B, V, 3, 4]
    if no_homogeneous:
        gx[..., 3] = 0.0
    gx = gx.reshape(B, V, 12)
    w = m.weights.double()
    pd = m.posedirs.double().view(m.kF, V, 3)
    out = []
    for c in range(m.ctas):
        vs = range(KV * c, min(V, KV * c + KV))
        dA = torch.zeros(B, J, 12, dtype=torch.float64)
        for v in vs:
            dA = fma(w[v][None, :, None], gx[:, v, None, :], dA)
        pdc = torch.zeros(m.kF, 3 * KV, dtype=torch.float64)
        dxc = torch.zeros(B, 3 * KV, dtype=torch.float64)
        nv = len(vs)
        pdc[:, :3 * nv] = pd[:, KV * c:KV * c + nv].reshape(m.kF, -1)
        dxc[:, :3 * nv] = dx[:, KV * c:KV * c + nv].reshape(B, -1)
        lane = torch.arange(32)                                                            # lane l: columns l, l + 32, l + 64
        s = f(f(f(pdc[:, None, lane] * dxc[None, :, lane]) + f(pdc[:, None, lane + 32] * dxc[None, :, lane + 32]))
              + f(pdc[:, None, lane + 64] * dxc[None, :, lane + 64]))                   # [kF, B, 32]
        for o in (16, 8, 4, 2, 1):
            s = f(s + s[..., lane ^ o])
        dt = torch.zeros(B, 3, dtype=torch.float64)
        for v in vs:
            dt = f(dt + g[:, v])
        out.append(torch.cat([dA.reshape(B, 12 * J), s[..., 0].T, dt], -1))
    return torch.stack(out)


def emu_rodrigues_bwd(r, gR):
    """rodrigues_bwd() of csrc/smpl_math.cuh."""
    _, (n, th, s, c, K, K2) = emu_rodrigues(r)
    gs = torch.zeros_like(th)
    g1c = torch.zeros_like(th)
    gRf, Kf, K2f = gR.reshape(-1, 9), K.reshape(-1, 9), K2.reshape(-1, 9)
    for i in range(9):
        gs, g1c = fma(gRf[:, i], Kf[:, i], gs), fma(gRf[:, i], K2f[:, i], g1c)
    t = torch.zeros_like(gR)
    for k in range(3):
        t = f(t + f(f(gR[:, :, k, None] * K[:, None, :, k]) + f(K[:, k, :, None] * gR[:, None, k, :])))
    gK = f(f(s[:, None, None] * gR) + f(f(1 - c)[:, None, None] * t)).reshape(-1, 9)
    gd = torch.stack([f(gK[:, 7] - gK[:, 5]), f(gK[:, 2] - gK[:, 6]), f(gK[:, 3] - gK[:, 1])], 1)
    dot = f(f(f(gd[:, 0] * r[:, 0]) + f(gd[:, 1] * r[:, 1])) + f(gd[:, 2] * r[:, 2]))
    gth = f(f(f(gs * c) + f(g1c * s)) - f(dot / f(th * th)))
    return f(f(gd / th[:, None]) + f(f(gth[:, None] * n) / th[:, None]))


def emu_finish(m, full, slots, last=None, no_feat=False):
    """Pass 2 of slots [ctas, B, kN] (the first `last` slots when given): (d_pose [B, 3 kT], d_transl [B, 3])."""
    B, J, kT, kF, P = full.shape[0], m.J, m.kT, m.kF, m.parents
    S = torch.zeros(slots.shape[1:], dtype=torch.float64)
    for c in range(slots.shape[0] if last is None else last):
        S = f(S + slots[c])
    _, L, G, _, _ = emu_pose_phase(m, full)
    Jr = m.Jr.double()
    dA = S[:, :12 * J].view(B, J, 3, 4)
    dG = torch.cat([f(dA[..., :3] - f(dA[..., 3:] * Jr[None, :, None, :])), dA[..., 3:]], -1)
    dG = list(dG.unbind(1))
    dR = [None] * J
    for j in range(J - 1, -1, -1):
        q = P[j]
        if q < 0:
            dR[j] = dG[j][..., :3]
            continue
        Gp = G[:, q]
        dR[j] = f(f(f(Gp[:, 0, :3, None] * dG[j][:, None, 0, :3]) + f(Gp[:, 1, :3, None] * dG[j][:, None, 1, :3]))
                  + f(Gp[:, 2, :3, None] * dG[j][:, None, 2, :3]))
        Lj = L[:, j]
        u = f(f(f(f(dG[j][:, :, None, 0] * Lj[:, None, :, 0]) + f(dG[j][:, :, None, 1] * Lj[:, None, :, 1]))
                + f(dG[j][:, :, None, 2] * Lj[:, None, :, 2])) + f(dG[j][:, :, None, 3] * Lj[:, None, :, 3]))
        dG[q] = torch.cat([f(dG[q][..., :3] + u), f(dG[q][..., 3:] + dG[j][..., 3:])], -1)
    gR = torch.stack(dR[:kT], 1)
    if not no_feat:
        df = S[:, 12 * J:12 * J + kF].view(B, J - 1, 3, 3)[:, :kT - 1]
        gR = torch.cat([gR[:, :1], f(gR[:, 1:] + df)], 1)
    r = full.double().view(B, J, 3)[:, :kT].reshape(B * kT, 3)
    return emu_rodrigues_bwd(r, gR.reshape(B * kT, 3, 3)).view(B, 3 * kT), S[:, -3:]


# ============================================================================================================== the tests
def within(what, got, ref, bound):
    r = ratio(got, ref, bound)
    assert r <= 1.0, f"{what}: error/bound {r:.4g}"


CASES = [("smpl", 33, "random", 3), ("smpl", 1, "pi", 2), ("smpl", 70, "zero", 1), ("smpl", 40, "tiny1e-7", 2),
         ("smplx", 31, "flat_hands", 2), ("smplx", 65, "2pi", 1), ("smplx", 33, "canonical", 2)]


@pytest.mark.parametrize("body,V,kind,B", CASES)
def test_vertex_emulations_lie_within_the_bounds(body, V, kind, B):
    """Tiers (a)-(c) of the GPU file on fp32 emulations of the kernels, and the GPU file's corruptions rejected."""
    from oracle import posefit_oracle as pfo
    m = Mesh(body, V, CPU)
    gen = torch.Generator().manual_seed(V + B)
    full, transl = case_pose(body, kind, B, gen)
    where = f"{body} V={V} {kind} B={B}"
    pm = pose_model(full, m.Jr, m.parents)
    vm = vertex_model(m, pm, transl)
    full64 = full.double().requires_grad_(True)
    tr64 = transl.double().requires_grad_(True)
    ref = pfo.vertices(m.oracle_body(), full64, tr64)
    got = emu_vertices(m, full, transl)
    within(f"{where} vertices", got, ref.detach(), vm.ob)
    if kind not in ("zero", "tiny1e-7"):
        rejects(f"{where}: row group 3 dropped", emu_vertices(m, full, transl, drop=3), ref.detach(), vm.ob)
        drop = torch.einsum("bvrc,bvc->bvr", vm.T[..., :3], group_offset(m, pm, 3))
        rejects(f"{where}: row group 3 dropped (fp64)", ref.detach() - drop, ref.detach(), vm.ob)
    if B >= 2:
        bad = got.clone()
        bad[:, V - 1] = got[:, V - 1].roll(1, 0)
        rejects(f"{where}: the last vertex from the neighbouring frame", bad, ref.detach(), vm.ob)

    for gk in ("random", "last"):
        g = d_verts_of(gk, B, V, gen).double()
        slots, eslots = slot_model(m, vm, g)
        es = emu_slots(m, full, g)
        within(f"{where} {gk} slots", es, slots, eslots)
        want_p, want_t = torch.autograd.grad((ref * g).sum(), (full64, tr64), retain_graph=True)
        want_p = want_p[:, :3 * m.kT]
        edp, edt = finish_model(m, pm, slots, eslots)
        dp, dt = emu_finish(m, full, es)
        within(f"{where} {gk} d_pose", dp, want_p, edp)
        within(f"{where} {gk} d_transl", dt, want_t, edt)
        both = torch.cat([want_p, want_t], 1), torch.cat([edp, edt], 1)
        rejects(f"{where} {gk}: d_feat dropped", emu_finish(m, full, es, no_feat=True)[0], want_p, edp)
        rejects(f"{where} {gk}: the last slot left out", torch.cat(emu_finish(m, full, es, last=m.ctas - 1), 1), *both)
        rejects(f"{where} {gk}: the homogeneous column dropped", emu_finish(m, full, emu_slots(m, full, g, no_homogeneous=True))[0],
                want_p, edp)


@pytest.mark.parametrize("S", [8, 33])
@pytest.mark.parametrize("body", ["smpl", "smplx"])
def test_fill_emulations_agree_with_the_oracle(body, S):
    """fill_emulation / weights_emulation against posefit_oracle.fill (gamma(3) on sum |w| |x|), fill_bwd_emulation against its
    autograd (gamma(ceil(n / 32) + 5) on sum |w| |g| for a vertex of n entries); corner 0's weights for every corner rejected."""
    from oracle import posefit_oracle as pfo
    from oracle import posmap_oracle as po
    from test_posmap_kernels_gpu import body_arrays, body_model
    _, _, t = body_model(body)
    a = body_arrays(body, CPU)
    faces, W = a["faces"], a["weights"]
    V = W.shape[0]
    fid, bary = po.layout(t[2].astype(np.float32)[t[3]], S)
    fid_t, bary_t = torch.from_numpy(fid.astype(np.int32)), torch.from_numpy(bary.astype(np.float32))
    gen = torch.Generator().manual_seed(S)
    B = 2
    verts = torch.randn(B, V, 3, generator=gen).double()
    want = pfo.fill(verts, t[1], fid, bary)
    wb = bary_t.double().reshape(-1, 3)
    absfill = torch.einsum("ni,bnic->bcn", wb.abs(), verts.abs()[:, faces.long()[fid_t.reshape(-1).clamp(min=0).long()]])
    bound = (gam(3) * absfill * (fid_t.reshape(-1) >= 0)).view(B, 3, S, S)
    got = fill_emulation(verts.float().double(), faces, fid_t, bary_t)
    within(f"{body} S={S} fill", got, want, bound)
    rejects(f"{body} S={S}: fill with corner 0's weights", fill_emulation(verts, faces, fid_t, bary_t, corner0=True), want, bound)
    J = W.shape[1]
    Wp = torch.cat([W.double(), torch.zeros(V, -J % 3, dtype=torch.float64)], 1)            # the weight map is the fill of W's columns
    ref_w = torch.cat([pfo.fill(Wp[None, :, k:k + 3], t[1], fid, bary)[0] for k in range(0, Wp.shape[1], 3)], 0)[:J].permute(1, 2, 0)
    abs_w = torch.cat([pfo.fill(Wp.abs()[None, :, k:k + 3], t[1], fid, np.abs(bary))[0] for k in range(0, Wp.shape[1], 3)], 0)[:J]
    within(f"{body} S={S} weights", weights_emulation(W, faces, fid_t, bary_t), ref_w, gam(3) * abs_w.permute(1, 2, 0) + 3 * 2.0 ** -149)         # subnormal skinning weights round absolutely
    d = torch.randn(B, 3, S, S, generator=gen).double()
    vx = torch.zeros(B, V, 3, dtype=torch.float64, requires_grad=True)
    want_b, = torch.autograd.grad((pfo.fill(vx, t[1], fid, bary) * d).sum(), vx)
    off, ent = csr_reference(faces, fid_t, V)
    cnt = (off[1:] - off[:-1]).double()
    ab, = torch.autograd.grad((pfo.fill(vx, t[1], fid, np.abs(bary)) * d.abs()).sum(), vx)
    bound_b = gam(torch.ceil(cnt / 32) + 5)[None, :, None] * ab
    got_b = fill_bwd_emulation(off, ent, bary_t, d.float().double(), V)
    within(f"{body} S={S} fill backward", got_b, want_b, bound_b)
    if bool((cnt > 0).any()):
        rejects(f"{body} S={S}: fill backward with corner 0's weights", fill_bwd_emulation(off, ent, bary_t, d, V, corner0=True),
                want_b, bound_b)
