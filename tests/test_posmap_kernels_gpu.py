"""GPU: every launch of csrc/posmap.cu but the layout, element by element against fp64 or bit for bit.

Covered: posed vertices (ga_smpl_vertices / ga_smplx_vertices), both passes of their backward (the per-CTA workspace slots and the
finished d_pose / d_transl), the fill and the texel weight map (ga_posmap_fill / ga_posmap_weights, bit for bit), the vertex ->
(texel, corner) CSR and the fill's backward (ga_posmap_vertex_csr / ga_posmap_fill_backward, bit for bit), and the Python path
(PoseMapper / SmplxPoseMapper autograd, vertices_backward, fill_backward) across MAX_FRAMES_PER_CALL chunks.

Conventions, helpers and the Rodrigues / kinematic-chain bounds are those of tests/test_step_kernels_gpu.py: C-ABI calls with
outputs inside finite sentinels that must stay bit-identical, NaN in every input element a kernel must not read, |got - ref| <=
bound for every element with an a-priori gamma(c) bound counted along the kernel's code path, and a corrupted copy of each output
that the same bound must reject.  The fp64 references start from the exact fp32 arrays the kernels receive (a mapper's v_shaped,
rest joints, posedirs [kF, 3V] and weights), sliced to V vertices, so the ragged last 32-vertex CTA is exercised at every tail.
The bound models below run on whatever device their inputs are on; tests/test_posmap_bounds_cpu.py checks them against fp32
emulations of the kernels.

Run with -s to print the largest error / bound ratio per output.
"""
import functools
import types

import numpy as np
import pytest
import torch

import raster_fp64 as rf
from test_step_kernels_gpu import (FO, NAN, PAD, POSES, SMPL_PARENTS, SMPLX_PARENTS, U, WORST, Rnd, cdiv, chain_bounds, check, full_pose,
                                   gam, nan_buf, p, rejects, rest_relative_bwd_bounds, reverse_walk_bounds, rod_model, rodrigues_bwd_model,
                                   sentinel, stream, untouched)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KV = 32                                     # vertices per CTA of the vertex kernels (kVertsPerCta)
KEY = "posmap"                              # WORST keys of this file
ETA = 2.0 ** -149                           # the smallest fp32 subnormal: a rounding that underflows errs by up to ETA / 2


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for key in sorted(k for k in WORST if k.startswith(KEY)):
        r, where = WORST.pop(key)
        print(f"\nposmap kernels: largest error/bound, {key}: {r:.3g} ({where})")


def _lib():
    from gaussianavatar_b200 import _lib
    return _lib


# ================================================================================================================= body arrays
@functools.lru_cache(maxsize=None)
def body_model(body):
    """(model fields, betas, UV template) of the synthetic SMPL / SMPL-X body the position-map tests use."""
    from gaussianavatar_b200 import synthetic as syn
    if body == "smpl":
        b, t = syn.make_body(0), syn.make_uv_template(0)
        return syn.smpl_mesh_model(b, t), b.betas[0], t
    b, t = syn.make_smplx_body(0), syn.make_smplx_uv_template(0)
    return syn.smplx_mesh_model(b, t, syn.smplx_posedirs(0)), b.betas[0], t


def body_arrays(body, device):
    """The fp32 arrays a mapper hands the kernels (BodyPoser's v_shaped, rest_joints, posedirs [kF, 3V], weights, faces)."""
    from gaussianavatar_b200.body import body_of, shaped_vertices
    model, betas, _ = body_model(body)
    bd = body_of(body)
    V, nf = model["v_template"].shape[0], bd.pose_features
    return dict(v_shaped=shaped_vertices(model, betas).float().to(device), rest_joints=bd.rest_joints(model, betas).to(device),
                posedirs=torch.from_numpy(np.asarray(model["posedirs"], np.float32).reshape(V * 3, nf).T.copy()).to(device),
                weights=torch.from_numpy(np.asarray(model["weights"], np.float32)).to(device),
                faces=torch.from_numpy(np.asarray(model["f"]).astype(np.int32)).to(device))


class Mesh:
    """A body's arrays cut to its first V vertices, posedirs repacked to [kF, 3V]."""

    def __init__(self, body, V, device):
        a = body_arrays(body, device)
        self.body, self.V = body, V
        self.J = 55 if body == "smplx" else 24
        self.kT = 22 if body == "smplx" else 24
        self.kF = 9 * (self.J - 1)
        self.parents = SMPLX_PARENTS if body == "smplx" else SMPL_PARENTS
        self.Jr = a["rest_joints"]
        self.v_shaped = a["v_shaped"][:V].contiguous()
        self.posedirs = a["posedirs"][:, :3 * V].contiguous()
        self.weights = a["weights"][:V].contiguous()
        self.ctas = cdiv(V, KV)
        self.kN = 12 * self.J + self.kF + 3            # floats per (CTA, frame) workspace slot

    def oracle_body(self):
        """posefit_oracle's Body, in fp64 from these fp32 arrays (not recomputed from the model)."""
        return types.SimpleNamespace(v_shaped=self.v_shaped.double(), J=self.Jr.double(), weights=self.weights.double(),
                                     posedirs=self.posedirs.double().T.reshape(self.V, 3, self.kF), parents=self.parents)


# ================================================================================================================ bound models
def pose_model(full, Jr, parents):
    """The pose phase (pose_phase of posmap.cu) in fp64 with bounds: R_j (Rodrigues model), the chain of any association
    (chain_product multiplies right to left), A = rest_relative(G) (gamma(4) on |G_t| + |G_R| |J|), feat = R - I (the Rodrigues
    bound plus one rounding)."""
    B, J = full.shape[0], len(parents)
    r = full.double().reshape(B * J, 3)
    rnd = Rnd()
    R, _ = rod_model(r.clone(), rnd)
    eR = rnd.bound(R).detach().view(B, J, 3, 3)
    R = R.detach().view(B, J, 3, 3)
    Jd = Jr.double()
    L, dL, G, EG = chain_bounds(R, eR, Jd, parents, any_order=True)
    GR, Gt = G[..., :3], G[..., 3]
    A = G.clone()
    A[..., 3] = Gt - (GR * Jd[None, :, None, :]).sum(-1)
    EA = EG.clone()
    EA[..., 3] = EG[..., 3] + (EG[..., :3] * Jd.abs()[None, :, None, :]).sum(-1) \
        + gam(4) * (Gt.abs() + (GR.abs() * Jd.abs()[None, :, None, :]).sum(-1))
    feat = (R[:, 1:] - torch.eye(3, dtype=R.dtype, device=R.device)).reshape(B, -1)
    efeat = eR[:, 1:].reshape(B, -1) + U * feat.abs()
    return types.SimpleNamespace(R=R, L=L, dL=dL, G=G, EG=EG, A=A, EA=EA, feat=feat, efeat=efeat, full=full)


def vertex_model(m, pm, transl):
    """Posed vertices in fp64 and their bounds along vertices_kernel's code path.

    off = posedirs^T feat: four row groups, each a sequential FMA chain of ceil(kF / 4) terms, then the four added:
    gamma(ceil(kF / 4) + 3) sum |feat| |pd|, plus sum |pd| e_feat.  x = v_shaped + off, one rounding.  T = sum_j w_j A_j, a
    kJ-term FMA chain: gamma(kJ) sum |w| |A| plus sum |w| e_A, plus kJ ETA (SMPL's synthetic weights reach 2e-45, so products
    underflow: every rounding errs by u |x| + ETA / 2).  The output T_R x + T_t + transl, three products and four adds:
    gamma(5) on the absolute values, plus |x| e_T and |T_R| e_x.  First order: FO."""
    B, V, J = pm.full.shape[0], m.V, m.J
    w, pd = m.weights.double(), m.posedirs.double()
    A12, EA12 = pm.A.reshape(B, J, 12), pm.EA.reshape(B, J, 12)
    T = torch.einsum("vj,bjq->bvq", w, A12).view(B, V, 3, 4)
    eT = (gam(J) * torch.einsum("vj,bjq->bvq", w.abs(), A12.abs()) + torch.einsum("vj,bjq->bvq", w.abs(), EA12) + J * ETA).view(B, V, 3, 4)
    off = (pm.feat @ pd).view(B, V, 3)
    e_off = (gam(cdiv(m.kF, 4) + 3) * (pm.feat.abs() @ pd.abs()) + pm.efeat @ pd.abs()).view(B, V, 3)
    x = m.v_shaped.double()[None] + off
    e_x = e_off + U * x.abs()
    tr = transl.double()[:, None, :]
    out = (T[..., :3] * x[:, :, None, :]).sum(-1) + T[..., 3] + tr
    ob = gam(5) * ((T[..., :3].abs() * x.abs()[:, :, None, :]).sum(-1) + T[..., 3].abs() + tr.abs()) \
        + (eT[..., :3] * x.abs()[:, :, None, :]).sum(-1) + eT[..., 3] + (T[..., :3].abs() * e_x[:, :, None, :]).sum(-1)
    return types.SimpleNamespace(T=T, eT=eT, x=x, e_x=e_x, out=out, ob=FO * ob)


def group_offset(m, pm, g):
    """The posedirs offset of row group g alone (rows g, g + 4, ...), carried through T_R: what dropping that group changes."""
    B = pm.full.shape[0]
    return (pm.feat[:, g::4] @ m.posedirs.double()[g::4]).view(B, m.V, 3)


def _per_cta(t, m):
    """[B, V, ...] -> [B, ctas, 32, ...], zero past V."""
    pad = m.ctas * KV - m.V
    t = torch.cat([t, t.new_zeros(t.shape[0], pad, *t.shape[2:])], 1)
    return t.view(t.shape[0], m.ctas, KV, *t.shape[2:])


def slot_model(m, vm, g):
    """Pass 1 of the vertex backward: each CTA's slot [d_A (12 J) | d_feat (kF) | d_transl (3)] per frame, fp64, and bounds.

    x_v and T_v enter within their forward bounds (pass 1 forms x with eight row groups, fewer roundings than the forward's four).
    d_A_j = sum_v w_vj g_v [x_v; 1]^T: an FMA chain over the CTA's nv vertices of products g x (one rounding): gamma(nv + 1).
    d_feat[r] = sum pd[r, 3v + c] dx_vc with dx = T_R^T g (three products, two adds: gamma(3) on |T_R|^T |g|): per lane three
    columns (three products, two adds), then a five-level butterfly: gamma(8).  d_transl = sum_v g_v: gamma(nv).  Each also
    carries ETA per rounding for underflow (subnormal weights make subnormal terms of d_A).
    Returns (slots, bounds) [ctas, B, kN]."""
    B, J, ctas = g.shape[0], m.J, m.ctas
    nv = torch.tensor([min(KV, m.V - KV * c) for c in range(ctas)], dtype=torch.float64, device=g.device)
    gc = _per_cta(g, m)                                                                    # [B, ctas, 32, 3]
    X = _per_cta(torch.cat([vm.x, torch.ones_like(vm.x[..., :1])], -1), m)
    eX = _per_cta(torch.cat([vm.e_x, torch.zeros_like(vm.x[..., :1])], -1), m)
    wc = _per_cta(m.weights.double()[None], m)[0]                                         # [ctas, 32, J]
    gx = (gc[..., :, None] * X[..., None, :]).flatten(-2)                                  # [B, ctas, 32, 12]
    gxa = (gc.abs()[..., :, None] * X.abs()[..., None, :]).flatten(-2)
    egx = (gc.abs()[..., :, None] * eX[..., None, :]).flatten(-2)
    dA = torch.einsum("cvj,bcvq->cbjq", wc, gx).reshape(ctas, B, 12 * J)
    edA = (gam(nv + 1)[:, None, None, None] * torch.einsum("cvj,bcvq->cbjq", wc.abs(), gxa)
           + torch.einsum("cvj,bcvq->cbjq", wc.abs(), egx) + (2 * nv + 1)[:, None, None, None] * ETA).reshape(ctas, B, 12 * J)
    TR, eTR = vm.T[..., :3], vm.eT[..., :3]
    dx = torch.einsum("bvrc,bvr->bvc", TR, g)
    e_dx = gam(3) * torch.einsum("bvrc,bvr->bvc", TR.abs(), g.abs()) + torch.einsum("bvrc,bvr->bvc", eTR, g.abs())
    pdc = _per_cta(m.posedirs.double().view(m.kF, m.V, 3), m)                              # [kF, ctas, 32, 3]
    dxc, edxc = _per_cta(dx, m), _per_cta(e_dx, m)
    df = torch.einsum("fcvk,bcvk->cbf", pdc, dxc)
    edf = gam(8) * torch.einsum("fcvk,bcvk->cbf", pdc.abs(), dxc.abs()) + torch.einsum("fcvk,bcvk->cbf", pdc.abs(), edxc) + 3 * KV * ETA
    dt = gc.sum(2).transpose(0, 1)
    edt = gam(nv)[:, None, None] * gc.abs().sum(2).transpose(0, 1) + nv[:, None, None] * ETA
    return torch.cat([dA, df, dt], -1), torch.cat([edA, edf, edt], -1)


def finish_model(m, pm, slots, eslots):
    """Pass 2: the slots added in CTA order (gamma(ctas) on sum |slot| and ctas ETA, plus the slot bounds), d_A -> d_G (gamma(2)), the reverse
    walk, dR + d_feat (one add), then rodrigues_bwd under its own rounding model.  Returns FO-scaled bounds (d_pose [B, 3 kT],
    d_transl [B, 3])."""
    B, J, kT, kF = slots.shape[1], m.J, m.kT, m.kF
    S = slots.sum(0)
    eS = gam(m.ctas) * slots.abs().sum(0) + eslots.sum(0) + m.ctas * ETA
    dA, eA = S[:, :12 * J].view(B, J, 3, 4), eS[:, :12 * J].view(B, J, 3, 4)
    dG, eG = rest_relative_bwd_bounds(dA, eA, m.Jr.double())
    dLR, eLR = reverse_walk_bounds(pm.G, pm.EG, pm.L, pm.dL, dG, eG, m.parents)
    gR = torch.stack(dLR[:kT], 1)
    egR = torch.stack(eLR[:kT], 1)
    df = S[:, 12 * J:12 * J + kF].view(B, J - 1, 3, 3)[:, :kT - 1]
    edf = eS[:, 12 * J:12 * J + kF].view(B, J - 1, 3, 3)[:, :kT - 1]
    gR = torch.cat([gR[:, :1], gR[:, 1:] + df], 1)
    egR = torch.cat([egR[:, :1], egR[:, 1:] + edf + U * gR[:, 1:].abs()], 1)
    rnd = Rnd()
    r = pm.full.double().view(B, J, 3)[:, :kT].reshape(B * kT, 3)
    dr = rodrigues_bwd_model(r, rnd.known(gR.reshape(B * kT, 3, 3), egR.reshape(B * kT, 3, 3)), rnd)
    return FO * rnd.bound(dr).detach().view(B, 3 * kT), FO * eS[:, -3:]


def finish_ref(m, full, sums):
    """d_pose [B, 3 kT] and d_transl of total slot sums [B, kN] in fp64 (autograd through the oracle's Rodrigues and the chain):
    what pass 2 computes, so a corrupted sum can be carried to d_pose."""
    from oracle import posefit_oracle as pfo
    B, J, kF = full.shape[0], m.J, m.kF
    r = full.double().reshape(B * J, 3).clone().requires_grad_(True)
    R = pfo.rotations(r).view(B, J, 3, 3)
    Jd = m.Jr.double()
    rel = Jd.clone()
    rel[1:] = Jd[1:] - Jd[m.parents[1:]]
    L = torch.cat([R, rel[None, :, :, None].expand(B, J, 3, 1)], -1)
    G = [L[:, 0]]
    for j in range(1, J):
        Gp = G[m.parents[j]]
        G.append(torch.cat([Gp[..., :3] @ L[:, j, :, :3], (Gp[..., :3] @ L[:, j, :, 3:] + Gp[..., 3:])], -1))
    G = torch.stack(G, 1)
    A = torch.cat([G[..., :3], (G[..., 3] - (G[..., :3] * Jd[None, :, None, :]).sum(-1))[..., None]], -1)
    feat = (R[:, 1:] - torch.eye(3, dtype=R.dtype, device=R.device)).reshape(B, kF)
    loss = (A * sums[:, :12 * J].view(B, J, 3, 4)).sum() + (feat * sums[:, 12 * J:12 * J + kF]).sum()
    d, = torch.autograd.grad(loss, r)
    return d.view(B, 3 * J)[:, :3 * m.kT], sums[:, -3:]


# ============================================================================================== vertices, forward and backward
def case_pose(body, kind, B, gen):
    """(full pose [B, 3 J], transl [B, 3]) fp32 on gen's device: a POSES kind, flat_hands, or posmap.canonical_pose."""
    J = 55 if body == "smplx" else 24
    if kind == "canonical":
        from gaussianavatar_b200.posmap import canonical_pose
        full = canonical_pose(body).to(gen.device).expand(B, -1).contiguous()
    else:
        full = full_pose(kind, B, J, gen)
    return full, 0.3 * torch.randn(B, 3, device=gen.device, generator=gen)


def d_verts_of(kind, B, V, gen):
    g = torch.randn(B, V, 3, device=gen.device, generator=gen)
    if kind == "last":                           # only vertex V - 1, in the ragged last CTA
        g[:, :V - 1] = 0.0
    elif kind == "first":
        g[:, 1:] = 0.0
    return g


def vertex_inputs(m, full, transl):
    """pose / rest_pose / transl rows followed by two NaN frames; v_shaped, weights, posedirs followed by NaN."""
    B = full.shape[0]
    pose = nan_buf(B + 2, 3 * m.kT)
    pose[:B] = full[:, :3 * m.kT]
    rest = None
    if m.J == 55:
        rest = nan_buf(B + 2, 99)
        rest[:B] = full[:, 66:]
    tr = nan_buf(B + 2, 3)
    tr[:B] = transl
    vs = nan_buf(m.V + PAD, 3)
    vs[:m.V] = m.v_shaped
    w = nan_buf(m.V + PAD, m.J)
    w[:m.V] = m.weights
    pd = nan_buf(m.kF * 3 * m.V + PAD)
    pd[:m.kF * 3 * m.V] = m.posedirs.reshape(-1)
    Jr = nan_buf(m.J + 4, 3)
    Jr[:m.J] = m.Jr
    return dict(pose=pose, rest=rest, transl=tr, v_shaped=vs, weights=w, posedirs=pd, Jr=Jr)


def poses_args(m, ins):
    return (p(ins["pose"]),) if m.J == 24 else (p(ins["pose"]), p(ins["rest"]))


def vertices_launch(m, ins, B, out):
    L = _lib().lib()
    fn = L.ga_smpl_vertices if m.J == 24 else L.ga_smplx_vertices
    return fn(B, m.V, *poses_args(m, ins), p(ins["transl"]), p(ins["Jr"]), p(ins["v_shaped"]), p(ins["posedirs"]), p(ins["weights"]),
              p(out), stream())


def ws_bytes(m, B):
    L = _lib().lib()
    return (L.ga_smpl_vertices_backward_workspace_bytes if m.J == 24 else L.ga_smplx_vertices_backward_workspace_bytes)(B, m.V)


def backward_launch(m, ins, B, d_verts, ws, nbytes, dp, dt):
    L = _lib().lib()
    fn = L.ga_smpl_vertices_backward if m.J == 24 else L.ga_smplx_vertices_backward
    return fn(B, m.V, *poses_args(m, ins), p(ins["Jr"]), p(ins["v_shaped"]), p(ins["posedirs"]), p(ins["weights"]), p(d_verts),
              ws if isinstance(ws, int) else p(ws), nbytes, p(dp), p(dt), stream())


VS = {"smpl": [1, 31, 32, 33, 95, 97, 6890], "smplx": [1, 31, 32, 33, 95, 97, 10475]}
BS = [1, 3, 8]
VERT_CASES = [(body, V, "random", BS[i % 3]) for body in ("smpl", "smplx") for i, V in enumerate(VS[body][:-1])] + \
    [(body, VS[body][-1], kind, BS[i % 3]) for body in ("smpl", "smplx")
     for i, kind in enumerate(POSES + ["canonical"] + (["flat_hands"] if body == "smplx" else []))] + \
    [(body, 33, kind, 8) for body in ("smpl", "smplx") for kind in ("zero", "pi")]
BIG_FEAT = ("pi", "2pi", "random", "canonical", "flat_hands")       # poses whose pose-blend offset of one row group is far above the bound


@pytest.mark.parametrize("body,V,kind,B", VERT_CASES)
def test_vertices_and_backward(body, V, kind, B):
    """Tier (a) ga_smpl(x)_vertices (bounds: vertex_model), tier (b) each workspace slot of the backward's pass 1 (slot_model), tier
    (c) d_pose / d_transl against fp64 autograd through oracle/posefit_oracle.vertices (finish_model), for d_verts random, only on
    vertex V - 1 and only on vertex 0."""
    from oracle import posefit_oracle as pfo
    m = Mesh(body, V, DEV)
    gen = torch.Generator(device=DEV).manual_seed(V * 31 + B + len(kind) + m.J)
    full, transl = case_pose(body, kind, B, gen)
    where = f"{body} V={V} {kind} B={B}"
    ins = vertex_inputs(m, full, transl)
    n3 = B * V * 3

    # (a) forward
    out = sentinel(gen, n3 + PAD)
    out0 = out.clone()
    _lib().check(vertices_launch(m, ins, B, out), "ga_smpl(x)_vertices")
    torch.cuda.synchronize()
    untouched(f"{where} verts", out, out0, 0, n3)
    got = out[:n3].view(B, V, 3)
    pm = pose_model(full, m.Jr, m.parents)
    vm = vertex_model(m, pm, transl)
    ob = m.oracle_body()
    full64 = full.double().requires_grad_(True)
    tr64 = transl.double().requires_grad_(True)
    ref = pfo.vertices(ob, full64, tr64)
    check(f"{KEY} vertices", where, got, ref.detach(), vm.ob)
    bad = got.double().clone()
    bad[:, V - 1] = out0[:n3].view(B, V, 3)[:, V - 1].double()
    rejects(f"{where}: the last vertex not written", bad, ref.detach(), vm.ob)
    if B >= 2:
        bad = got.double().clone()
        bad[:, V - 1] = got[:, V - 1].double().roll(1, 0)
        rejects(f"{where}: the last vertex taken from the neighbouring frame", bad, ref.detach(), vm.ob)
    if kind in BIG_FEAT:
        drop = torch.einsum("bvrc,bvc->bvr", vm.T[..., :3], group_offset(m, pm, 3))
        rejects(f"{where}: row group 3 of the pose-blend offset dropped", ref.detach() - drop, ref.detach(), vm.ob)

    # (b), (c) backward
    need = ws_bytes(m, B)
    assert need == m.ctas * B * m.kN * 4
    for gk in ("random", "last", "first"):
        w2 = f"{where} d_verts {gk}"
        g = d_verts_of(gk, B, V, gen)
        gb = nan_buf(n3 + PAD)
        gb[:n3] = g.reshape(-1)
        ws = sentinel(gen, need // 4 + PAD)
        ws0 = ws.clone()
        dp, dt = sentinel(gen, B * 3 * m.kT + PAD), sentinel(gen, B * 3 + PAD)
        dp0, dt0 = dp.clone(), dt.clone()
        _lib().check(backward_launch(m, ins, B, gb, ws, need, dp, dt), "ga_smpl(x)_vertices_backward")
        torch.cuda.synchronize()
        untouched(f"{w2} workspace", ws, ws0, 0, need // 4)
        untouched(f"{w2} d_pose", dp, dp0, 0, B * 3 * m.kT)
        untouched(f"{w2} d_transl", dt, dt0, 0, B * 3)
        slots, eslots = slot_model(m, vm, g.double())
        got_s = ws[:need // 4].view(m.ctas, B, m.kN)
        J12 = 12 * m.J
        check(f"{KEY} bwd slot d_A", w2, got_s[..., :J12], slots[..., :J12], FO * eslots[..., :J12])
        check(f"{KEY} bwd slot d_feat", w2, got_s[..., J12:-3], slots[..., J12:-3], FO * eslots[..., J12:-3])
        check(f"{KEY} bwd slot d_transl", w2, got_s[..., -3:], slots[..., -3:], FO * eslots[..., -3:])
        if gk != "first" or m.ctas == 1:
            bad = got_s.double().clone()
            bad[-1] = 0.0
            rejects(f"{w2}: the last CTA's slot not written", bad, slots, FO * eslots)

        want_p, want_t = torch.autograd.grad((ref * g.double()).sum(), (full64, tr64), retain_graph=True)
        want_p = want_p[:, :3 * m.kT]
        edp, edt = finish_model(m, pm, slots, eslots)
        got_p, got_t = dp[:B * 3 * m.kT].view(B, 3 * m.kT), dt[:B * 3].view(B, 3)
        check(f"{KEY} bwd d_pose", w2, got_p, want_p, edp)
        check(f"{KEY} bwd d_transl", w2, got_t, want_t, edt)
        S = slots.sum(0)
        J12, kF = 12 * m.J, m.kF
        # one joint's d_feat term dropped: the trained joint whose d_feat stands out most against its d_pose bound (near theta = 0
        # the Rodrigues backward's 1 / theta terms widen that bound)
        df = S[:, J12:J12 + kF].view(B, m.J - 1, 9)[:, :m.kT - 1]
        j = 1 + int((df.abs().amax(2) / edp.view(B, m.kT, 3)[:, 1:].amax(2)).amax(0).argmax())
        S1 = S.clone()
        S1[:, J12 + 9 * (j - 1):J12 + 9 * j] = 0.0
        rejects(f"{w2}: joint {j}'s d_feat term dropped", finish_ref(m, full, S1)[0], want_p, edp)
        if gk != "first" or m.ctas == 1:
            bp, bt = finish_ref(m, full, slots[:-1].sum(0))
            rejects(f"{w2}: the last CTA's slot left out of the sum", torch.cat([bp, bt], 1), torch.cat([want_p, want_t], 1),
                    torch.cat([edp, edt], 1))
        S1 = S.clone()
        S1[:, :J12].view(B, m.J, 3, 4)[..., 3] = 0.0
        rejects(f"{w2}: the homogeneous column of d_A dropped", finish_ref(m, full, S1)[0], want_p, edp)


@pytest.mark.parametrize("body", ["smpl", "smplx"])
def test_vertices_argument_checks(body):
    """B = 0 is a no-op that writes nothing; the backward rejects B = 9, a workspace one byte short and a misaligned workspace,
    leaving its outputs untouched."""
    V = 97
    m = Mesh(body, V, DEV)
    gen = torch.Generator(device=DEV).manual_seed(5)
    full, transl = case_pose(body, "random", 9, gen)
    ins = vertex_inputs(m, full, transl)
    out = sentinel(gen, 9 * V * 3 + PAD)
    out0 = out.clone()
    assert vertices_launch(m, ins, 0, out) == 0
    torch.cuda.synchronize()
    untouched(f"{body} B=0 verts", out, out0, 0, 0)
    assert vertices_launch(m, ins, 9, out) != 0
    g = torch.randn(9 * V * 3 + PAD, device=DEV, generator=gen)
    dp, dt = sentinel(gen, 9 * 3 * m.kT + PAD), sentinel(gen, 9 * 3 + PAD)
    dp0, dt0 = dp.clone(), dt.clone()
    need = ws_bytes(m, 8)
    assert ws_bytes(m, 9) == 0
    ws = torch.zeros(need + 16, dtype=torch.uint8, device=DEV)
    for what, B, ptr_off, nbytes in (("B = 9", 9, 0, need + 16), ("one byte short", 8, 0, need - 1), ("misaligned", 8, 2, need + 14)):
        rc = backward_launch(m, ins, B, g, ws.data_ptr() + ptr_off, nbytes, dp, dt)
        torch.cuda.synchronize()
        assert rc != 0, f"{body}: {what} accepted"
        untouched(f"{body} {what} d_pose", dp, dp0, 0, 0)
        untouched(f"{body} {what} d_transl", dt, dt0, 0, 0)


# ======================================================================================================== fill and weight map
def layout(corners, S):
    corners = torch.as_tensor(np.ascontiguousarray(corners, np.float32)).to(DEV)
    fid = torch.empty(S, S, dtype=torch.int32, device=DEV)
    bary = torch.empty(S, S, 3, device=DEV)
    _lib().check(_lib().lib().ga_posmap_layout(corners.shape[0], S, p(corners), p(fid), p(bary), stream()), "ga_posmap_layout")
    bary[fid < 0] = NAN                         # the fill, the weight map and the fill backward never read an uncovered texel's
    return fid, bary


def template_layout(body, S):
    _, _, t = body_model(body)
    return layout(t[2].astype(np.float32)[t[3]], S)


def fill_emulation(verts, faces, fid, bary, corner0=False):
    """ga_posmap_fill in fp32, in the kernel's order: three fmaf from 0, corner 0 first; +0.0 where nothing covers the texel.
    verts [B, V, 3] -> [B, 3, S, S] (fp64 tensors holding fp32 values).  corner0: every corner weighted by bary[0] (a self-check)."""
    B, S = verts.shape[0], fid.shape[0]
    cov = (fid >= 0).reshape(-1)
    tri = faces.long()[fid.reshape(-1)[cov].long()]                                       # [n, 3]
    w = bary.reshape(-1, 3)[cov].double()
    o = torch.zeros(B, tri.shape[0], 3, dtype=torch.float64, device=verts.device)
    for i in range(3):
        o = rf.fma32(w[None, :, 0 if corner0 else i, None], verts[:, tri[:, i]].double(), o)
    out = torch.zeros(B, S * S, 3, dtype=torch.float64, device=verts.device)
    out[:, cov] = o
    return out.permute(0, 2, 1).reshape(B, 3, S, S)


def weights_emulation(W, faces, fid, bary):
    """ga_posmap_weights in fp32: out[t, j] = three fmaf from 0, corner 0 first; +0.0 where nothing covers t.  -> [S, S, J]."""
    S, J = fid.shape[0], W.shape[1]
    cov = (fid >= 0).reshape(-1)
    tri = faces.long()[fid.reshape(-1)[cov].long()]
    w = bary.reshape(-1, 3)[cov].double()
    o = torch.zeros(tri.shape[0], J, dtype=torch.float64, device=W.device)
    for i in range(3):
        o = rf.fma32(w[:, i, None], W[tri[:, i]].double(), o)
    out = torch.zeros(S * S, J, dtype=torch.float64, device=W.device)
    out[cov] = o
    return out.view(S, S, J)


def bit_equal(key, where, got, want):
    """got (fp32) bit-identical to want (fp32 values held in fp64): +0.0 and -0.0 differ."""
    n = int((got.view(torch.int32) != want.float().view(torch.int32)).sum())
    check(key, where, got, want, torch.zeros_like(want))
    assert n == 0, f"{key}, {where}: {n} elements differ in their bits"


@pytest.mark.parametrize("S", [1, 2, 15, 16, 17, 100, 512])
@pytest.mark.parametrize("body", ["smpl", "smplx"])
def test_fill_and_weights_bit_for_bit(body, S):
    """ga_posmap_fill at B = 1, 8, 9, 33 (no frame limit: grid.y is B) and ga_posmap_weights (J = 24 / 55), bit for bit against
    fill_emulation / weights_emulation.  NaN in the vertices no face uses (SMPL-X's last 25), in frames past B and in the
    barycentric weights of uncovered texels; uncovered texels must be +0.0."""
    a = body_arrays(body, DEV)
    faces, W = a["faces"], a["weights"]
    V, J = W.shape
    gen = torch.Generator(device=DEV).manual_seed(S + J)
    fid, bary = template_layout(body, S)
    used = torch.zeros(V, dtype=torch.bool, device=DEV)
    used[faces.long().reshape(-1)] = True
    assert body == "smpl" or int((~used).sum()) == 25
    n = S * S
    covered = bool((fid >= 0).any())
    for B in (1, 8, 9, 33):
        where = f"{body} S={S} B={B}"
        verts = nan_buf(B + 2, V, 3)
        verts[:B] = torch.randn(B, V, 3, device=DEV, generator=gen) * 0.5 + torch.tensor([0.0, 0.2, 0.0], device=DEV)
        verts[:, ~used] = NAN
        out = sentinel(gen, B * 3 * n + PAD)
        out0 = out.clone()
        _lib().check(_lib().lib().ga_posmap_fill(B, S, V, p(verts), p(faces), p(fid), p(bary), p(out), stream()), "ga_posmap_fill")
        torch.cuda.synchronize()
        untouched(f"{where} fill", out, out0, 0, B * 3 * n)
        got = out[:B * 3 * n].view(B, 3, S, S)
        want = fill_emulation(verts[:B], faces, fid, bary)
        bit_equal(f"{KEY} fill", where, got, want)
        assert bool((got[:, :, fid < 0].view(torch.int32) == 0).all())
        if covered:
            rejects(f"{where}: every corner weighted by corner 0's bary", fill_emulation(verts[:B], faces, fid, bary, corner0=True),
                    want, torch.zeros_like(want))
    Wb = nan_buf(V + PAD, J)
    Wb[:V] = W
    Wb[:V][~used] = NAN
    out = sentinel(gen, n * J + PAD)
    out0 = out.clone()
    _lib().check(_lib().lib().ga_posmap_weights(S, J, p(Wb), p(faces), p(fid), p(bary), p(out), stream()), "ga_posmap_weights")
    torch.cuda.synchronize()
    untouched(f"{body} S={S} weights", out, out0, 0, n * J)
    got = out[:n * J].view(S, S, J)
    want = weights_emulation(W, faces, fid, bary)
    bit_equal(f"{KEY} weights", f"{body} S={S}", got, want)
    assert bool((got[fid < 0].view(torch.int32) == 0).all())
    if covered:
        rejects(f"{body} S={S}: the joint columns shifted by one", torch.roll(want, 1, -1), want, torch.zeros_like(want))


# ====================================================================================================== CSR and fill backward
CSR_TARGETS = [3000, 65, 0, 1, 31, 32, 33, 64]     # entries of chosen vertices: several thousand, <= 32 and > 32 lanes' worth


def counted_mesh(S, V, seed):
    """A UV layout of S x S texels (the square triangulation of test_posmap_cpu with one cell per texel, a tenth of its faces
    removed so that some texels are uncovered) and mesh faces over V vertices chosen so that vertex 0 has CSR_TARGETS[0] entries,
    vertex V - 1 CSR_TARGETS[1], and six more vertices the others.  Returns (faces [F, 3] int32, face_id, bary, {vertex: count})."""
    from test_posmap_cpu import _square_triangulation
    g = np.random.default_rng(seed)
    corners = _square_triangulation(S, seed, 0.0)
    corners = corners[g.random(corners.shape[0]) >= 0.1]
    fid, bary = layout(corners, S)
    F = corners.shape[0]
    nf = np.bincount(fid[fid >= 0].long().cpu().numpy(), minlength=F)
    others = g.choice(np.arange(1, V - 1), 6, replace=False)
    targets = dict(zip([0, V - 1, *others.tolist()], CSR_TARGETS))
    pool = np.setdiff1d(np.arange(V), list(targets))
    faces = g.choice(pool, (F, 3))
    ones = g.permutation(np.nonzero(nf == 1)[0])
    k = 0
    for v, c in targets.items():                 # corner 0 of c distinct single-texel faces
        faces[ones[k:k + c], 0] = v
        k += c
    assert k <= ones.size
    return torch.from_numpy(faces.astype(np.int32)).to(DEV), fid, bary, targets


def csr_reference(faces, fid, V):
    """(offsets [V + 1], entries [n]): each vertex's entries 3 t + i, ascending."""
    t = torch.nonzero(fid.reshape(-1) >= 0)[:, 0]
    tri = faces.long()[fid.reshape(-1)[t].long()]                                         # [n_t, 3]
    e = (3 * t[:, None] + torch.arange(3, device=t.device)).reshape(-1)
    v = tri.reshape(-1)
    order = torch.argsort(v * (3 * fid.numel()) + e)
    counts = torch.bincount(v, minlength=V)
    offsets = torch.cat([counts.new_zeros(1), counts.cumsum(0)])
    return offsets.int(), e[order].int()


def fill_bwd_emulation(offsets, entries, bary, d_out, V, corner0=False):
    """ga_posmap_fill_backward in fp32: per (vertex, frame) lane l accumulates entries l, l + 32, ... with fmaf from 0, then
    xor-shuffle adds at offsets 16, 8, 4, 2, 1; lane 0's sum.  -> [B, V, 3] (fp64 tensors holding fp32 values)."""
    B, n = d_out.shape[0], d_out.shape[-1] * d_out.shape[-2]
    g = d_out.reshape(B, 3, n).double()
    bf = bary.reshape(-1).double()
    off = offsets.long()
    cnt = off[1:] - off[:-1]
    lane = torch.arange(32, device=d_out.device)
    a = torch.zeros(B, V, 32, 3, dtype=torch.float64, device=d_out.device)
    ent = entries.long()
    for k in range(cdiv(int(cnt.max()), 32) if V else 0):
        j = lane[None] + 32 * k                                                            # [1, 32]
        ok = j < cnt[:, None]                                                              # [V, 32]
        e = torch.where(ok, off[:-1, None] + j, torch.zeros_like(j))
        ti = ent[e.clamp(max=ent.numel() - 1)]
        w = bf[3 * (ti // 3) if corner0 else ti]
        gv = g[:, :, ti // 3].permute(0, 2, 3, 1)                                           # [B, V, 32, 3]
        a = torch.where(ok[None, :, :, None], rf.fma32(w[None, :, :, None], gv, a), a)
    for o in (16, 8, 4, 2, 1):
        a = (a + a[:, :, lane ^ o]).float().double()
    return a[:, :, 0]


@pytest.mark.parametrize("V", [1023, 1024, 1025, 2049, 6890, 10475])
def test_csr_and_fill_backward_bit_for_bit(V):
    """ga_posmap_vertex_csr: offsets are the exclusive cumsum of the per-vertex counts for every vertex (the scan's carry across
    1024-vertex blocks), entries each vertex's ascending list, nothing written past offsets[V] / V + 1; vertices with 0, 1, 31, 32,
    33, 64, 65 and 3000 entries.  ga_posmap_fill_backward at B = 1 and 8, bit for bit against fill_bwd_emulation."""
    S = 128
    faces, fid, bary, targets = counted_mesh(S, V, seed=V)
    gen = torch.Generator(device=DEV).manual_seed(V)
    n3 = 3 * S * S
    offsets = torch.randint(-2 ** 30, 2 ** 30, (V + 1 + PAD,), device=DEV, generator=gen, dtype=torch.int32)
    entries = torch.randint(-2 ** 30, 2 ** 30, (n3 + PAD,), device=DEV, generator=gen, dtype=torch.int32)
    o0, e0 = offsets.clone(), entries.clone()
    _lib().check(_lib().lib().ga_posmap_vertex_csr(S, V, p(faces), p(fid), p(offsets), p(entries), stream()), "ga_posmap_vertex_csr")
    torch.cuda.synchronize()
    off_ref, ent_ref = csr_reference(faces, fid, V)
    n = int(off_ref[-1])
    assert n < n3
    untouched(f"V={V} offsets", offsets, o0, 0, V + 1)
    untouched(f"V={V} entries", entries, e0, 0, n)
    assert torch.equal(offsets[:V + 1], off_ref), f"V={V}: {int((offsets[:V + 1] != off_ref).sum())} offsets differ"
    assert torch.equal(entries[:n], ent_ref), f"V={V}: {int((entries[:n] != ent_ref).sum())} entries differ"
    cnt = (off_ref[1:] - off_ref[:-1]).cpu()
    for v, c in targets.items():
        assert int(cnt[v]) == c, (V, v, int(cnt[v]), c)

    for B in (1, 8):
        where = f"V={V} S={S} B={B}"
        d_out = nan_buf(B + 1, 3, S, S)
        d_out[:B] = torch.randn(B, 3, S, S, device=DEV, generator=gen)
        d_out[:, :, fid < 0] = NAN
        dv = sentinel(gen, B * V * 3 + PAD)
        dv0 = dv.clone()
        _lib().check(_lib().lib().ga_posmap_fill_backward(B, S, V, p(offsets), p(entries), p(bary), p(d_out), p(dv), stream()),
                     "ga_posmap_fill_backward")
        torch.cuda.synchronize()
        untouched(f"{where} d_verts", dv, dv0, 0, B * V * 3)
        got = dv[:B * V * 3].view(B, V, 3)
        want = fill_bwd_emulation(off_ref, ent_ref, bary, d_out[:B], V)
        bit_equal(f"{KEY} fill backward", where, got, want)
        rejects(f"{where}: every corner weighted by corner 0's bary", fill_bwd_emulation(off_ref, ent_ref, bary, d_out[:B], V, corner0=True),
                want, torch.zeros_like(want))


# ======================================================================================================== the Python path
@pytest.mark.parametrize("body", ["smpl", "smplx"])
def test_python_path_chunks_bit_equal_to_the_c_abi(body):
    """PoseMapper / SmplxPoseMapper autograd (_PoseMap), vertices_backward and fill_backward at B = 11 (two MAX_FRAMES_PER_CALL
    chunks, one shared workspace) bit-equal to C-ABI calls on frames 0-7 and 8-10; the mapper hands the kernels body_arrays."""
    from gaussianavatar_b200.posmap import MAX_FRAMES_PER_CALL, PoseMapper, SmplxPoseMapper, vertices_backward
    model, betas, t = body_model(body)
    S, B = 32, 11
    mapper = (PoseMapper if body == "smpl" else SmplxPoseMapper)(model, betas, t, S, device=DEV)
    a = body_arrays(body, DEV)
    for k, v in (("v_shaped", mapper.v_shaped), ("rest_joints", mapper.rest_joints), ("posedirs", mapper.posedirs),
                 ("weights", mapper.weights), ("faces", mapper.faces)):
        assert torch.equal(a[k], v), k
    m = Mesh(body, mapper.V, DEV)
    gen = torch.Generator(device=DEV).manual_seed(11)
    full, transl = case_pose(body, "random", B, gen)
    pose = full[:, :3 * m.kT].contiguous().requires_grad_(True)
    rest = full[:, 66:].contiguous() if m.J == 55 else None
    tr = transl.clone().requires_grad_(True)
    maps = mapper(pose, tr) if m.J == 24 else mapper(pose, rest, tr)
    d_maps = torch.randn(B, 3, S, S, device=DEV, generator=gen)
    maps.backward(d_maps)
    dv_py = mapper.fill_backward(d_maps)
    dp_py, dt_py = vertices_backward(mapper, pose.detach(), rest, dv_py)
    torch.cuda.synchronize()
    assert MAX_FRAMES_PER_CALL == 8
    offsets, entries = mapper.vertex_csr()
    L = _lib().lib()
    for s, e in ((0, 8), (8, 11)):
        nb = e - s
        ins = vertex_inputs(m, full[s:e], transl[s:e])
        verts = torch.empty(nb, m.V, 3, device=DEV)
        _lib().check(vertices_launch(m, ins, nb, verts), "vertices")
        mp = torch.empty(nb, 3, S, S, device=DEV)
        _lib().check(L.ga_posmap_fill(nb, S, m.V, p(verts), p(mapper.faces), p(mapper.face_id), p(mapper.bary), p(mp), stream()), "fill")
        dm = d_maps[s:e].contiguous()
        dv = torch.empty(nb, m.V, 3, device=DEV)
        _lib().check(L.ga_posmap_fill_backward(nb, S, m.V, p(offsets), p(entries), p(mapper.bary), p(dm), p(dv), stream()), "fill bwd")
        need = ws_bytes(m, nb)
        ws = torch.empty(need, dtype=torch.uint8, device=DEV)
        dp, dt = torch.empty(nb, 3 * m.kT, device=DEV), torch.empty(nb, 3, device=DEV)
        _lib().check(backward_launch(m, ins, nb, dv, ws, need, dp, dt), "vertices bwd")
        torch.cuda.synchronize()
        for name, got, want in (("maps", maps.detach()[s:e], mp), ("fill_backward", dv_py[s:e], dv), ("d_pose", pose.grad[s:e], dp),
                                ("d_transl", tr.grad[s:e], dt), ("vertices_backward d_pose", dp_py[s:e], dp),
                                ("vertices_backward d_transl", dt_py[s:e], dt)):
            assert torch.equal(got.view(torch.int32), want.view(torch.int32)), f"{body} frames {s}-{e - 1}: {name}"
