"""fp64 reference of the soft-silhouette kernels (csrc/silhouette.cu), launch by launch, with a running error bound (test helper).

It starts from what the kernels themselves stage or write: the projected fp32 corners (`FaceXY`) and pixel boxes of
`sil_setup_kernel`, the per-pixel G of the backward's tile pass (`pix`), the tile partials, the six corner gradients per face
(`fgrad`).  From those it evaluates the exact function in fp64 and bounds how far the kernel's fp32 expression tree may lie from it:

  setup        corners and boxes restated in numpy fp32 in the kernel's operation order (`project_f32`): they compare bit for bit.
  tile, fwd    L(p) = -sum_f softplus(x_f(p)) and S = -expm1(L), every face against every pixel of its fp64 box grown by one
               pixel, so a face whose truncation band reaches a pixel counts there whatever box or tile list the kernel made.
  partials     sum over a tile's pixels of (S - M)^2 from the kernel's own S.
  tile, bwd    G = w_b 2 (S - M) / (H W) exp(L).
  face grad    the six corner gradients, sum over the face's box of G D_f dx_f/dcorners, from the kernel's own G and corners.
  vertex grad  d_verts from the kernel's own fgrad through the projection's Jacobian.

Error bound.  Every value is carried as (v, e): v the fp64 value, e a bound on |kernel result - v|.  Each operation of the
kernel's tree adds u (|result| + e) with u = 2^-24 + 2^-53 for an fp32 operation (its rounding plus that of v), or 2^-52 for an fp64
one, plus 2^-126 (2^-1022) for underflow.  Counting a multiply and an add separately also covers a contracted FMA.  Products and
quotients propagate operand errors rigorously (first order plus the product terms).  Division and sqrtf are IEEE-rounded (the
library is built without --use_fast_math).  expf adds 2 ulp, log1pf and expm1f 1 ulp of their result (CUDA Math API, maximum
ulp error tables); their argument's error is propagated through the function's derivative over the whole interval.  Fixed-order
sums add gamma(depth) sum |terms|: L over the faces at a pixel (ascending face order, depth = the number of faces), block_sum
(5 shuffle levels + 8 warps), the face grad's lane stride plus its 5-level shuffle tree, the vertex CSR gather.

The per-edge geometry of `eval_face` (w = p - a, t, q = a + t e, d^2 and the inside test) is modelled in fp64 from the fp32 corners
with d^2, t and p - q rounded to fp32 once (GEOM = "f64", what the kernel does), or in fp32 ("f32", the kernel's first form, whose
bound on a long edge is what the accuracy ceiling rejects).

Decisions are marginal when the threshold lies within the value's bound: the truncation d^2 > sigma ln(1/eps - 1) (against the
kernel's fp32 threshold), the inside test (any edge's cross product within its bound of 0 changes the verdict), box membership
(a pixel within its bound of a box side) and, for the gradient, the nearest edge: when two edges' d^2 intervals overlap and their
gradient terms differ by more than their bounds plus 1e-3 of the pair's largest term (the two edges at a corner agree that closely; across the
medial axis inside a face they do not).  Where the candidates agree, the bound is their hull.  A pixel (face) with a marginal pair is excluded from the element-wise checks
and counted.

Written in torch: it runs on the CPU for small meshes and in fp64 on the GPU for production frames.
"""
import math

import numpy as np
import torch

from oracle.mesh_oracle import xf_row

U32 = 2.0 ** -24 + 2.0 ** -53
U64 = 2.0 ** -52
ETA32 = 2.0 ** -126
ETA64 = 2.0 ** -1022
ULP = 2.0 ** -23                              # one ulp of a normal fp32 result, relative
LN_INV_EPS_F = float(np.float32(9.21024036697585))
ZNEAR = np.float32(0.01)
GUARD = np.float32(1 << 20)
TILE = 16
GEOM = "f64"                                  # how eval_face evaluates its per-edge geometry


def gam(n, u=U32):
    n = torch.as_tensor(n, dtype=torch.float64)
    return n * u / (1 - n * u)


def align_up(x, a=256):
    return (x + a - 1) // a * a


def cdiv(a, b):
    return -(-a // b)


def workspace_layout(B, F, H, W):
    """carve(): byte offsets of boxes int4[B F], xy FaceXY[B F] (6 floats), pix float[B H W], partial float[B tiles], fgrad
    float[B F 6], each at the next 256-byte boundary, and the total."""
    off, out = 0, {}
    for name, n in (("boxes", 16 * B * F), ("xy", 24 * B * F), ("pix", 4 * B * H * W), ("partial", 4 * B * cdiv(H, TILE) * cdiv(W, TILE)),
                    ("fgrad", 24 * B * F)):
        off = align_up(off)
        out[name] = off
        off += n
    out["total"] = align_up(off)
    return out


def thresholds(sigma):
    """The kernels' fp32 constants: (trunc_d2 = sigma * 9.2102404f, inv_sigma = 1.f / sigma, r = sqrtf(trunc_d2))."""
    s = np.float32(sigma)
    trunc = np.float32(s * np.float32(LN_INV_EPS_F))
    return float(trunc), float(np.float32(1) / s), float(np.sqrt(trunc))


# ------------------------------------------------------------------------------------------------------------- setup
def project_f32(X, cam, H, W):
    """mesh_project.cuh's project() in numpy fp32 (explicitly rounded ops, fmaf emulated exactly): pixx, pixy [V] f32, ok [V]."""
    X = np.asarray(X, np.float32)
    cam = np.asarray(cam, np.float32)
    view, proj = cam[:16], cam[16:32]
    x, y, z = X[:, 0], X[:, 1], X[:, 2]
    with np.errstate(all="ignore"):
        vz = xf_row(view, 2, x, y, z)
        hx, hy, hw = xf_row(proj, 0, x, y, z), xf_row(proj, 1, x, y, z), xf_row(proj, 3, x, y, z)
        p_w = np.float32(1) / (hw + np.float32(1e-7))
        pixx = (((hx * p_w).astype(np.float64) + 1.0) * W - 1.0) * 0.5
        pixy = (((hy * p_w).astype(np.float64) + 1.0) * H - 1.0) * 0.5
        pixx, pixy = pixx.astype(np.float32), pixy.astype(np.float32)
        ok = (vz > ZNEAR) & (np.abs(pixx) <= GUARD) & (np.abs(pixy) <= GUARD)
    return pixx, pixy, ok


def setup_f32(X, faces, cam, H, W, sigma):
    """sil_setup_kernel for one frame: xy [F,3,2] f32, ok [F], boxes [F,4] int64 (c0, c1, r0, r1; (1,0,1,0) when empty) and
    area_unsure [F] (an fp32 area whose zero test a contracted FMA could decide the other way: not held to the box check)."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    pixx, pixy, vok = project_f32(X, cam, H, W)
    xy = np.stack([pixx[faces], pixy[faces]], -1)                          # [F,3,2]
    ok = vok[faces].all(1)
    x, y = xy[..., 0], xy[..., 1]
    with np.errstate(all="ignore"):
        a, b, c, d = x[:, 1] - x[:, 0], y[:, 2] - y[:, 0], y[:, 1] - y[:, 0], x[:, 2] - x[:, 0]
        p, q = a.astype(np.float64) * b, c.astype(np.float64) * d          # exact
        area = p - q
        area32 = a * b - c * d
        unsure = np.abs(area) <= 2 * U32 * (np.abs(p) + np.abs(q))
        ok = ok & (area32 != 0) & np.isfinite(area32)
        _, _, r = thresholds(sigma)
        r = np.float32(r)
        x0, x1 = x.min(1) - r, x.max(1) + r
        y0, y1 = y.min(1) - r, y.max(1) + r
        box = np.stack([np.maximum(0, np.ceil(np.where(ok, x0, 0))), np.minimum(W - 1, np.floor(np.where(ok, x1, 0))),
                        np.maximum(0, np.ceil(np.where(ok, y0, 0))), np.minimum(H - 1, np.floor(np.where(ok, y1, 0)))], 1).astype(np.int64)
    empty = ~ok | (box[:, 0] > box[:, 1]) | (box[:, 2] > box[:, 3])
    box[empty] = (1, 0, 1, 0)
    return xy, ok, box, unsure & vok[faces].all(1)


# ---------------------------------------------------------------------------------------------- tracked operations
class Ops:
    """(v, e) arithmetic with the rounding unit of one precision."""

    def __init__(self, u, eta):
        self.u, self.eta = u, eta

    def rnd(self, v, d):
        return v, d + self.u * (v.abs() + d) + self.eta

    def add(self, a, b):
        return self.rnd(a[0] + b[0], a[1] + b[1])

    def sub(self, a, b):
        return self.rnd(a[0] - b[0], a[1] + b[1])

    def mul(self, a, b):
        return self.rnd(a[0] * b[0], a[0].abs() * b[1] + b[0].abs() * a[1] + a[1] * b[1])

    def div(self, a, b):
        den = b[0].abs() * (b[0].abs() - b[1])
        d = torch.where(den > 0, (a[1] * b[0].abs() + a[0].abs() * b[1]) / den.clamp_min(1e-300), torch.full_like(den, math.inf))
        return self.rnd(a[0] / b[0], d)


F32, F64 = Ops(U32, ETA32), Ops(U64, ETA64)


def exact(v):
    return v, torch.zeros_like(v)


def to32(a):
    return F32.rnd(a[0], a[1])


def clamp01(a):
    v, e = a
    t = v.clamp(0.0, 1.0)
    e = torch.where((v - e >= 1.0) | (v + e <= 0.0), torch.zeros_like(e), e)      # clearly clamped: exactly 0 or 1
    return t, e


def expf(a):
    v, e = a
    g = torch.exp(v)
    return g, g * ((1 + 2 * ULP + U64) * torch.exp(e) - 1) + 2 * ETA32


def log1pf(a):
    """a in (0, 1]."""
    v, e = a
    prop = e / (1 + (v - e).clamp_min(0.0))
    r = torch.log1p(v)
    return r, prop + (ULP + U64) * (r.abs() + prop) + ETA32


def expm1f(a):
    v, e = a
    r = torch.expm1(v)
    prop = torch.exp(v) * torch.expm1(e)
    return r, prop + (ULP + U64) * (r.abs() + prop) + ETA32


def _both(x, pos, neg):
    """A branch on x > 0 (>= 0): both branches compute the same function, and the kernel may take either where x's interval
    contains 0, so there the larger bound holds.  Each branch's argument is clamped to <= 1 on the side it is not taken, where
    it only matters within x's bound of 0."""
    v, e = x
    ev = torch.where(v > 0, pos[1], neg[1])
    ev = torch.where(v.abs() <= e, torch.maximum(pos[1], neg[1]), ev)
    return torch.where(v > 0, pos[0], neg[0]), ev


def softplus(x):
    """x > 0 ? x + log1pf(expf(-x)) : log1pf(expf(x))."""
    v, e = x
    pos = F32.add(x, log1pf(expf(((-v).clamp(max=1.0), e))))
    neg = log1pf(expf((v.clamp(max=1.0), e)))
    return _both(x, pos, neg)


def sigmoid(x):
    """x >= 0 ? 1 / (1 + expf(-x)) : expf(x) / (1 + expf(x))."""
    v, e = x
    one = exact(torch.ones_like(v))
    gp, gn = expf(((-v).clamp(max=1.0), e)), expf((v.clamp(max=1.0), e))
    pos = F32.div(one, F32.add(one, gp))
    neg = F32.div(gn, F32.add(one, gn))
    return _both(x, pos, neg)


def vmin(a, b):
    """The kernel's fp32 min of two tracked values lies in [min(a - ea, b - eb), min(a + ea, b + eb)]."""
    lo = torch.minimum(a[0] - a[1], b[0] - b[1])
    hi = torch.minimum(a[0] + a[1], b[0] + b[1])
    v = torch.minimum(a[0], b[0])
    return v, torch.maximum(v - lo, hi - v)


# --------------------------------------------------------------------------------------------------------- eval_face
def edge_geom(ax, ay, bx, by, px, py, geom):
    """One edge a -> b at pixel centres (px, py): cross product, t, p - q and d^2 as tracked values in the given model."""
    O = F32 if geom == "f32" else F64
    ax, ay, bx, by, px, py = map(exact, (ax, ay, bx, by, px, py))
    ex, ey = O.sub(bx, ax), O.sub(by, ay)
    wx, wy = O.sub(px, ax), O.sub(py, ay)
    cr = O.sub(O.mul(ex, wy), O.mul(ey, wx))
    t = clamp01(O.div(O.add(O.mul(wx, ex), O.mul(wy, ey)), O.add(O.mul(ex, ex), O.mul(ey, ey))))
    dx, dy = O.sub(wx, O.mul(t, ex)), O.sub(wy, O.mul(t, ey))
    d2 = O.add(O.mul(dx, dx), O.mul(dy, dy))
    if geom == "f64":
        t, dx, dy = to32(t), to32(dx), to32(dy)
    return dict(cr=cr, t=t, dx=dx, dy=dy, d2=d2)


def eval_pairs(xy, f, c, r, trunc, inv_sigma, geom, swap_t=False, swap_ab=False):
    """Faces f (into xy [F,3,2] fp64 holding the fp32 corners) at pixels (c, r): the tracked x, softplus, sigmoid, liveness and
    the marginal decisions, and the per-edge terms the gradient needs."""
    cx, cy = xy[f, :, 0], xy[f, :, 1]
    px, py = c.double(), r.double()
    E = [edge_geom(cx[:, k], cy[:, k], cx[:, (k + 1) % 3], cy[:, (k + 1) % 3], px, py, geom) for k in range(3)]
    ge = [(e["cr"][0] - e["cr"][1] >= 0, e["cr"][0] + e["cr"][1] >= 0) for e in E]
    le = [(e["cr"][0] + e["cr"][1] <= 0, e["cr"][0] - e["cr"][1] <= 0) for e in E]
    ins_lo = (ge[0][0] & ge[1][0] & ge[2][0]) | (le[0][0] & le[1][0] & le[2][0])
    ins_hi = (ge[0][1] & ge[1][1] & ge[2][1]) | (le[0][1] & le[1][1] & le[2][1])
    cr = torch.stack([e["cr"][0] for e in E])
    inside = (cr >= 0).all(0) | (cr <= 0).all(0)
    marg_in = ins_lo != ins_hi
    best = vmin(vmin(E[0]["d2"], E[1]["d2"]), E[2]["d2"])
    d2v = torch.stack([e["d2"][0] for e in E])
    d2e = torch.stack([e["d2"][1] for e in E])
    m = d2v.argmin(0)
    best32 = to32(best) if geom == "f64" else best
    dead = ~inside & (best[0] > trunc)
    marg_tr = ~inside & ((best[0] - best[1] > trunc) != (best[0] + best[1] > trunc))
    sgn = torch.where(inside, 1.0, -1.0).double()
    x = F32.mul((sgn * best32[0], best32[1]), exact(torch.full_like(sgn, inv_sigma)))
    sp = softplus(x)
    cand = (d2v - d2e) <= (d2v + d2e).min(0).values[None]
    return dict(E=E, inside=inside, dead=dead, marg=marg_in | marg_tr, x=x, sp=sp, m=m, cand=cand, sgn=sgn,
                swap_t=swap_t, swap_ab=swap_ab)


def grad_terms(P, G, inv_sigma):
    """The six corner-gradient terms [n,6] of each pair and their bounds, G the kernel's own per-pixel G (exact), and whether the
    nearest-edge choice is marginal (candidates whose terms disagree beyond their bounds)."""
    n = G.shape[0]
    sig = sigmoid(P["x"])
    coef = F32.mul(F32.mul(exact(-2.0 * G), sig), exact(P["sgn"] * inv_sigma))
    one = exact(torch.ones_like(G))
    vals, errs = [], []
    for k in range(3):
        e = P["E"][k]
        t = e["t"]
        if P["swap_t"]:
            t = F32.sub(one, t)
        ca, cb = F32.mul(coef, F32.sub(one, t)), F32.mul(coef, t)
        a, b = (k + 1) % 3, k
        if not P["swap_ab"]:
            a, b = b, a
        tv = torch.zeros(n, 6, dtype=torch.float64, device=G.device)
        te = torch.zeros_like(tv)
        for corner, cc in ((a, ca), (b, cb)):
            for j, d in ((0, e["dx"]), (1, e["dy"])):
                v, er = F32.mul(cc, d)
                tv[:, 2 * corner + j] = v
                te[:, 2 * corner + j] = er
        vals.append(tv)
        errs.append(te)
    V, Er = torch.stack(vals), torch.stack(errs)                          # [3,n,6]
    idx = P["m"][None, :, None].expand(1, n, 6)
    ref, eref = V.gather(0, idx)[0], Er.gather(0, idx)[0]
    diff = (V - ref[None]).abs()
    cand = P["cand"][:, :, None]
    # near a corner the two edges meeting there give nearly the same terms (t at or near its clamp): their hull is the bound
    agree = (diff <= Er + eref[None] + 1e-3 * torch.maximum(V.abs().amax(2, keepdim=True), ref.abs().amax(1, keepdim=True)[None])) | ~cand
    marg = ~agree.all(2).all(0)
    bound = torch.where(cand, diff + Er, torch.zeros_like(Er)).amax(0)
    return ref, torch.maximum(bound, eref), marg


# ---------------------------------------------------------------------------------------------------------- pairs
def pair_list(xy, ok, H, W, r, rows=None, limit=1 << 21):
    """Chunks of (face, column, row) over every pixel of each ok face's fp64 box grown by one pixel (only the rows `rows`, a
    sorted tensor, when given)."""
    dev = xy.device
    x, y = xy[..., 0], xy[..., 1]
    fs = torch.nonzero(ok).reshape(-1)
    c0 = torch.ceil(x[fs].amin(1) - r - 1).clamp(0, W - 1).long()
    c1 = torch.floor(x[fs].amax(1) + r + 1).clamp(-1, W - 1).long()
    r0 = torch.ceil(y[fs].amin(1) - r - 1).clamp(0, H - 1).long()
    r1 = torch.floor(y[fs].amax(1) + r + 1).clamp(-1, H - 1).long()
    rows = torch.arange(H, device=dev) if rows is None else torch.as_tensor(rows, device=dev).long()
    j0 = torch.searchsorted(rows, r0)
    j1 = torch.searchsorted(rows, r1, right=True)
    nc = (c1 - c0 + 1).clamp_min(0)
    nr = (j1 - j0).clamp_min(0)
    cnt = nc * nr
    keep = cnt > 0
    fs, c0, nc, j0, cnt = fs[keep], c0[keep], nc[keep], j0[keep], cnt[keep]
    ends = torch.cumsum(cnt, 0)
    lo = 0
    while lo < fs.numel():
        start = int(ends[lo] - cnt[lo])
        hi = max(lo + 1, int(torch.searchsorted(ends, torch.tensor(start + limit, device=dev), right=True)))
        sel = slice(lo, hi)
        k = torch.arange(int(cnt[sel].sum()), device=dev) - torch.repeat_interleave(ends[sel] - cnt[sel] - start, cnt[sel])
        w = torch.repeat_interleave(nc[sel], cnt[sel])
        f = torch.repeat_interleave(fs[sel], cnt[sel])
        c = torch.repeat_interleave(c0[sel], cnt[sel]) + k % w
        rr = rows[torch.repeat_interleave(j0[sel], cnt[sel]) + k // w]
        yield f, c, rr
        lo = hi


def box_marg(xy, f, c, r, rr):
    """Pairs within their bound of one of the face's box sides (the arguments of the kernel's ceilf / floorf)."""
    x, y = xy[f, :, 0], xy[f, :, 1]
    out = torch.zeros_like(c, dtype=torch.bool)
    for lo, hi, p in ((x.amin(1), x.amax(1), c.double()), (y.amin(1), y.amax(1), r.double())):
        for s, sgn in ((lo, -1.0), (hi, 1.0)):
            v = s + sgn * rr
            e = U32 * (s.abs() + rr) + 2 * U32 * rr
            out |= (p - v).abs() <= e
    return out


# ------------------------------------------------------------------------------------------------------------ tiers
class FrameRef:
    """One frame: xy [F,3,2] (the kernel's fp32 corners), ok [F] (its boxes non-empty), H, W, sigma, rows (None: all)."""

    def __init__(self, xy, ok, H, W, sigma, rows=None, geom=None, device="cpu"):
        self.xy = torch.as_tensor(np.asarray(xy, np.float32)).double().to(device).reshape(-1, 3, 2)
        self.ok = torch.as_tensor(np.asarray(ok)).to(device).reshape(-1)
        self.F = self.xy.shape[0]
        self.H, self.W, self.sigma = int(H), int(W), float(sigma)
        self.trunc, self.inv_sigma, self.r = thresholds(sigma)
        self.rr = math.sqrt(self.trunc)
        self.rows = None if rows is None else torch.as_tensor(rows, device=device).long()
        self.geom = GEOM if geom is None else geom
        self.dev = device

    def _pairs(self, all_rows=False):
        return pair_list(self.xy, self.ok, self.H, self.W, self.rr, None if all_rows else self.rows)

    def forward(self, drop=None, shrink=None, ceiling=None):
        """L and S (v, e) per pixel [n_rows, W], the marginal pixels, the number of live faces per pixel and, with `ceiling`, the
        largest bound on x relative to ceiling max(1, |x|) over clear live pairs.  drop = (face, tile): that face left out of that
        tile's pixels; shrink = face: its kernel box one row shorter (boxes [F,4] given as shrink = (face, boxes))."""
        nr = self.H if self.rows is None else self.rows.numel()
        rowpos = torch.full((self.H,), -1, dtype=torch.long, device=self.dev)
        rowpos[torch.arange(self.H, device=self.dev) if self.rows is None else self.rows] = torch.arange(nr, device=self.dev)
        Lv = torch.zeros(nr * self.W, dtype=torch.float64, device=self.dev)
        Le, La, cnt = torch.zeros_like(Lv), torch.zeros_like(Lv), torch.zeros_like(Lv)
        marg = torch.zeros(nr * self.W, dtype=torch.bool, device=self.dev)
        worst = 0.0
        tiles_x = cdiv(self.W, TILE)
        for f, c, r in self._pairs():
            P = eval_pairs(self.xy, f, c, r, self.trunc, self.inv_sigma, self.geom)
            live = ~P["dead"]
            if drop is not None:
                live &= ~((f == drop[0]) & ((r // TILE) * tiles_x + c // TILE == drop[1]))
            if shrink is not None:
                live &= ~((f == shrink[0]) & (r == int(shrink[1][shrink[0], 3])))
            mg = P["marg"] | (box_marg(self.xy, f, c, r, self.r) & ~(P["dead"] & ~P["marg"]))
            o = rowpos[r] * self.W + c
            sv, se = P["sp"]
            Lv.index_add_(0, o, torch.where(live, sv, 0.0))
            Le.index_add_(0, o, torch.where(live, se, 0.0))
            La.index_add_(0, o, torch.where(live, sv.abs() + se, 0.0))
            cnt.index_add_(0, o, live.double())
            marg[o[mg]] = True
            if ceiling is not None:
                xv, xe = P["x"]
                rel = xe / (ceiling * xv.abs().clamp_min(1.0))
                clear = live & ~mg
                if bool(clear.any()):
                    worst = max(worst, float(rel[clear].max()))
        L = (-Lv, Le + gam(cnt) * La)
        S = expm1f(L)
        S = (-S[0], S[1])
        sh = (nr, self.W)
        out = dict(L=(L[0].reshape(sh), L[1].reshape(sh)), S=(S[0].reshape(sh), S[1].reshape(sh)), marg=marg.reshape(sh),
                   count=cnt.reshape(sh))
        if ceiling is not None:
            out["ceiling"] = worst
        return out

    def grad_pix(self, L, M, w_b):
        """G = w_b (2 (S - M) / (H W)) expf(L) (every row)."""
        S = expm1f(L)
        S = (-S[0], S[1])
        M = exact(M.double())
        q = F32.div((2.0 * F32.sub(S, M)[0], 2.0 * F32.sub(S, M)[1]), exact(torch.full_like(M[0], float(self.H * self.W))))
        return F32.mul(F32.mul(exact(torch.full_like(M[0], float(w_b))), q), expf(L))

    def face_grad(self, G, boxes, swap_t=False, swap_ab=False, zero_face=None):
        """fgrad (v, e) [F,6] from the kernel's own G [H,W] and boxes [F,4] (the lane-stride depth), and the marginal faces."""
        G = torch.as_tensor(G).double().to(self.dev).reshape(-1)
        boxes = torch.as_tensor(boxes).to(self.dev).long().reshape(-1, 4)
        gv = torch.zeros(self.F, 6, dtype=torch.float64, device=self.dev)
        ge, ga = torch.zeros_like(gv), torch.zeros_like(gv)
        marg = torch.zeros(self.F, dtype=torch.bool, device=self.dev)
        for f, c, r in self._pairs(all_rows=True):
            P = eval_pairs(self.xy, f, c, r, self.trunc, self.inv_sigma, self.geom, swap_t, swap_ab)
            live = ~P["dead"]
            tv, te, mn = grad_terms(P, G[r * self.W + c], self.inv_sigma)
            mg = P["marg"] | (box_marg(self.xy, f, c, r, self.r) & ~(P["dead"] & ~P["marg"])) | (mn & live)
            z = live[:, None]
            gv.index_add_(0, f, torch.where(z, tv, 0.0))
            ge.index_add_(0, f, torch.where(z, te, 0.0))
            ga.index_add_(0, f, torch.where(z, tv.abs() + te, 0.0))
            marg[f[mg]] = True
        n = ((boxes[:, 1] - boxes[:, 0] + 1) * (boxes[:, 3] - boxes[:, 2] + 1)).clamp_min(0)
        depth = cdiv(n, 32) + 5
        if zero_face is not None:
            gv[zero_face] = 0.0
        return (gv, ge + gam(depth)[:, None] * ga), marg


def partials(S, M, H, W):
    """Per tile: sum of (S - M)^2 over its pixels from the kernel's own S [H,W] (v, e), tiles in blockIdx order."""
    S, M = torch.as_tensor(S).double(), torch.as_tensor(M).double()
    th, tw = cdiv(H, TILE), cdiv(W, TILE)
    d = F32.sub(exact(S), exact(M))
    sq = F32.mul(d, d)
    pad = lambda a: torch.nn.functional.pad(a, (0, tw * TILE - W, 0, th * TILE - H))
    blk = lambda a: pad(a).reshape(th, TILE, tw, TILE).sum((1, 3)).reshape(-1)
    v, e = blk(sq[0]), blk(sq[1])
    return v, e + gam(5 + 8) * blk(sq[0].abs() + sq[1])


def vertex_grad(fgrad, X, faces, adj_off, adj_face, cam, H, W, drop_w_term=False):
    """d_verts (v, e) [V,3] of one frame from the kernel's own fgrad [F,6], fp32 verts X [V,3], the CSR and the camera."""
    dev = fgrad.device
    fgrad = fgrad.double()
    faces = torch.as_tensor(faces, device=dev).long().reshape(-1, 3)
    off = torch.as_tensor(adj_off, device=dev).long()
    adj = torch.as_tensor(adj_face, device=dev).long()
    V = off.numel() - 1
    vtx = torch.repeat_interleave(torch.arange(V, device=dev), off[1:] - off[:-1])
    prev = torch.cat([torch.full((1,), -1, device=dev, dtype=torch.long), adj[:-1]])
    first = torch.cat([torch.ones(1, dtype=torch.bool, device=dev), vtx[1:] != vtx[:-1]])
    keep = first | (adj != prev)
    fv = faces[adj]
    i = torch.where(fv[:, 0] == vtx, 0, torch.where(fv[:, 1] == vtx, 1, 2))
    gx = fgrad[adj, 2 * i] * keep
    gy = fgrad[adj, 2 * i + 1] * keep
    n = torch.zeros(V, dtype=torch.float64, device=dev).index_add_(0, vtx, keep.double())
    sx_ = torch.zeros(V, dtype=torch.float64, device=dev).index_add_(0, vtx, gx)
    sy_ = torch.zeros_like(sx_).index_add_(0, vtx, gy)
    ax = torch.zeros_like(sx_).index_add_(0, vtx, gx.abs())
    ay = torch.zeros_like(sx_).index_add_(0, vtx, gy.abs())
    gX, gY = (sx_, gam(n) * ax), (sy_, gam(n) * ay)
    X = torch.as_tensor(X, device=dev).double().reshape(-1, 3)
    cam = torch.as_tensor(cam, device=dev).double().reshape(-1)
    proj = cam[16:32]

    def row(rw):
        x, y, z = (exact(X[:, k]) for k in range(3))
        t = F32.mul(exact(proj[rw].expand(V)), x)
        t = F32.add(F32.mul(exact(proj[4 + rw].expand(V)), y), t)
        t = F32.add(F32.mul(exact(proj[8 + rw].expand(V)), z), t)
        return F32.add(t, exact(proj[12 + rw].expand(V)))

    hx, hy = row(0), row(1)
    one = exact(torch.ones(V, dtype=torch.float64, device=dev))
    p_w = F32.div(one, F32.add(row(3), exact(torch.full((V,), float(np.float32(1e-7)), dtype=torch.float64, device=dev))))
    sx = F32.mul(F32.mul((gX[0] * 0.5, gX[1] * 0.5), exact(torch.full((V,), float(W), dtype=torch.float64, device=dev))), p_w)
    sy = F32.mul(F32.mul((gY[0] * 0.5, gY[1] * 0.5), exact(torch.full((V,), float(H), dtype=torch.float64, device=dev))), p_w)
    out_v, out_e = [], []
    for k in range(3):
        p3 = exact(proj[4 * k + 3].expand(V))
        tx = F32.mul(F32.mul(hx, p_w), p3)
        ty = F32.mul(F32.mul(hy, p_w), p3)
        if drop_w_term:
            tx, ty = exact(torch.zeros(V, dtype=torch.float64, device=dev)), exact(torch.zeros(V, dtype=torch.float64, device=dev))
        a = F32.mul(sx, F32.sub(exact(proj[4 * k].expand(V)), tx))
        b = F32.mul(sy, F32.sub(exact(proj[4 * k + 1].expand(V)), ty))
        s = F32.add(a, b)
        out_v.append(s[0])
        out_e.append(s[1])
    zero = (gX[0] == 0) & (gY[0] == 0) & (gX[1] == 0) & (gY[1] == 0)
    v, e = torch.stack(out_v, 1), torch.stack(out_e, 1)
    return (torch.where(zero[:, None], 0.0, v), torch.where(zero[:, None], 0.0, e))
