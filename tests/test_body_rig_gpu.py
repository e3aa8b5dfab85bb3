"""GPU: the body-topology rig.  ga_mesh_laplacian and ga_texture_pushpull bit for bit against oracle/body_rig_oracle.py at ragged
sizes (inside sentinels, two runs identical), ga_mesh_shade_unlit against the oracle, the fit's known answers and its agreement with
an fp64 direct solve, a smooth function of UV through the textured resolve, rigs of tube-bodied SMPL / SMPL-X / stage-2 avatars
against the TSDF rig (silhouette IoU and unlit PSNR), and tools/extract_mesh.py --topology body on a saved checkpoint."""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from gaussianavatar_b200 import _lib  # noqa: E402
from gaussianavatar_b200 import mesh_extract as me  # noqa: E402
from gaussianavatar_b200 import rig as rg  # noqa: E402
from gaussianavatar_b200 import synthetic as syn  # noqa: E402
from gaussianavatar_b200._lib import ptr  # noqa: E402
from gaussianavatar_b200.mesh_render import MeshRenderer  # noqa: E402
from gaussianavatar_b200.posmap import CANO_TRANSL, canonical_pose  # noqa: E402
from body_rig_fixture import tube_avatar, tube_model  # noqa: E402
from oracle import body_rig_oracle as bo  # noqa: E402
from test_mesh_extract_gpu import _state  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
f32 = np.float32
GUARD = 64
# the body rig's silhouette IoU may fall this far below the TSDF rig's, its unlit PSNR this many dB (DESIGN.md §2)
IOU_GAP = 0.01
PSNR_GAP = 1.0
# ga_mesh_shade_unlit against the oracle: the same fp64 steps in the same order, rounded to fp32 once; one fp32 ulp at 1
UNLIT_TOL = 2.0 ** -23


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _guarded(n, dtype=torch.float32, fill=float("nan")):
    buf = torch.full((n + 2 * GUARD,), fill, dtype=dtype, device=DEV)
    return buf, buf[GUARD:GUARD + n]


def _guards_intact(buf, fill):
    g = torch.cat([buf[:GUARD], buf[-GUARD:]])
    return bool(torch.isnan(g).all()) if fill != fill else bool((g == fill).all())


# ---- kernels ---------------------------------------------------------------------------------------------------------------------------
def _ragged_csr(V, seed):
    """A random symmetric adjacency over V vertices with some degree-0 vertices and one vertex of high degree."""
    rng = np.random.default_rng(seed)
    E = 3 * V
    a, b = rng.integers(0, V, E), rng.integers(0, V, E)
    keep = (a != b) & (a % 7 != 3) & (b % 7 != 3)
    if V > 10:
        a, b = np.concatenate([a[keep], np.zeros(V // 2, np.int64)]), np.concatenate([b[keep], np.arange(1, V // 2 + 1)])
    else:
        a, b = a[keep], b[keep]
    pairs = np.unique(np.concatenate([np.stack([a, b], 1), np.stack([b, a], 1)]), axis=0) if len(a) else np.zeros((0, 2), np.int64)
    off = np.zeros(V + 1, np.int64)
    np.cumsum(np.bincount(pairs[:, 0], minlength=V), out=off[1:])
    return off.astype(np.int32), pairs[:, 1].astype(np.int32)


@pytest.mark.parametrize("case", ["V1", "V257", "V4099", "smpl_L1"])
def test_laplacian_matches_oracle_bit_for_bit(case):
    if case == "smpl_L1":
        topo = rg.body_topology(syn.make_uv_template(0), syn.make_body(0).lbs_weights, 1)
        off, adj, V = topo.offsets, topo.adj, topo.V
    else:
        V = int(case[1:])
        off, adj = _ragged_csr(V, V)
    x = (np.random.default_rng(V).normal(size=(V, 3)) * 10).astype(f32)
    want = bo.laplacian(off, adj, x)
    o, a, xd = (torch.from_numpy(t).to(DEV) for t in (off, np.concatenate([adj, [0]]).astype(np.int32), x))
    outs = []
    for _ in range(2):
        buf, y = _guarded(3 * V)
        _lib.check(_lib.lib().ga_mesh_laplacian(V, ptr(o), ptr(a), ptr(xd), ptr(y), _stream()), "ga_mesh_laplacian")
        torch.cuda.synchronize()
        assert _guards_intact(buf, float("nan"))
        outs.append(y.cpu().numpy().reshape(V, 3))
    assert np.array_equal(outs[0].view(np.int32), want.view(np.int32))
    assert np.array_equal(outs[0].view(np.int32), outs[1].view(np.int32))
    print(f"{case}: V {V}, degree 0 .. {np.diff(off).max()}, {int((np.diff(off) == 0).sum())} isolated")


@pytest.mark.parametrize("S", [1, 7, 64, 512])
@pytest.mark.parametrize("cover", ["random", "one", "none", "all"])
def test_pushpull_matches_oracle_bit_for_bit(S, cover):
    rng = np.random.default_rng(S)
    C = 3 if S != 7 else 4
    img = rng.random((C, S, S)).astype(f32)
    mask = {"random": rng.random((S, S)) < 0.3, "one": np.zeros((S, S), bool), "none": np.zeros((S, S), bool),
            "all": np.ones((S, S), bool)}[cover]
    if cover == "one":
        mask[S - 1, S // 3] = True
    img[:, ~mask] = np.nan
    want = bo.pushpull(img, mask)
    L = _lib.lib()
    n = L.ga_texture_pushpull_workspace_bytes(S, C)
    ws = torch.empty(max(n, 1), dtype=torch.uint8, device=DEV)
    im, mk = torch.from_numpy(img).to(DEV), torch.from_numpy(mask.astype(np.uint8)).to(DEV)
    outs = []
    for _ in range(2):
        buf, out = _guarded(C * S * S, fill=-7.0)
        _lib.check(L.ga_texture_pushpull(S, C, ptr(im), ptr(mk), ptr(ws), n, ptr(out), _stream()), "ga_texture_pushpull")
        torch.cuda.synchronize()
        assert _guards_intact(buf, -7.0)
        outs.append(out.cpu().numpy().reshape(C, S, S))
    assert np.array_equal(outs[0].view(np.int32), want.view(np.int32)) and np.isfinite(outs[0]).all()
    assert np.array_equal(outs[0].view(np.int32), outs[1].view(np.int32))


def _tube_scene(B=3, size=80, levels=1):
    """The SMPL tube's canonical mesh (subdivided) split at its UV seams (X [V,3] device, faces, glTF texcoords), its topology and B
    size x size cameras around it."""
    import types
    model, template, betas = tube_model("smpl")
    topo = rg.body_topology(template, model["weights"], levels)
    x = rg.subdivide_points(torch.from_numpy(template[0]).float(), topo).to(DEV) + torch.tensor(CANO_TRANSL, device=DEV)
    vid, tex, faces = rg.seam_split(types.SimpleNamespace(faces=topo.faces, uv_faces=topo.uv_faces, uvs=topo.uvs))
    cams = me.fusion_cameras(x.mean(0).cpu().numpy(), 1.0, B, size)
    return x[torch.from_numpy(vid).to(DEV)].contiguous(), faces, tex, topo, cams.to(DEV)


@pytest.mark.parametrize("mode", ["colors", "texture"])
def test_shade_unlit_matches_oracle(mode):
    H = W = 80
    X, faces, tex, _, cams = _tube_scene(3, H)
    V = X.shape[0]
    rng = np.random.default_rng(1)
    colors = rng.random((V, 3)).astype(f32)
    texture = rng.random((37, 53, 3)).astype(f32)
    mr = MeshRenderer(faces, V, device=DEV)
    Xb = X[None].expand(3, -1, -1).contiguous()
    bg = torch.rand(3, 3, H, W, device=DEV)
    kw = dict(colors=colors) if mode == "colors" else dict(uvs=tex, texture=texture)
    rgb, fid, _ = mr.render_unlit(Xb, cams, H, W, background=bg, **kw)
    rgb2, _, _ = mr.render_unlit(Xb, cams, H, W, background=bg, **kw)
    assert torch.equal(rgb, rgb2)
    one, _, _ = mr.render_unlit(Xb[1:2], cams[1:2], H, W, background=bg[1:2], **kw)
    assert torch.equal(one[0], rgb[1])                        # a frame does not depend on the batch it is drawn in
    worst = 0.0
    for b in range(3):
        want = bo.shade_unlit(X.cpu().numpy(), faces, cams[b].cpu().numpy(), fid[b].cpu().numpy(), H, W, background=bg[b].cpu().numpy(),
                              **({"colors": colors} if mode == "colors" else {"uvs": tex, "texture": texture}))
        got = rgb[b].cpu().numpy()
        drawn = fid[b].cpu().numpy() >= 0
        assert drawn.sum() > 100 and np.array_equal(got[:, ~drawn], bg[b].cpu().numpy()[:, ~drawn])
        worst = max(worst, float(np.abs(got - want).max()))
    print(f"{mode}: max |device - oracle| {worst:.3g}")
    assert worst <= UNLIT_TOL


def test_smooth_uv_function_through_the_textured_resolve():
    """A texture sampled from f(u, v) at texel centres, drawn through the resolve, matches f at each pixel's own (u, v) within the
    bilinear error bound h^2/8 (max|f_uu| + max|f_vv|); a v flip, a half-texel shift or a u/v transpose is far outside it."""
    H = W = 160
    S = 128
    X, faces, tex, _, cams = _tube_scene(4, H)
    k1, k2 = 2.0 * np.pi * 1.3, 2.0 * np.pi
    f = lambda u, v: np.stack([0.5 + 0.4 * np.sin(k1 * u), 0.5 + 0.4 * np.cos(k2 * v), u * (1 - v)], 0)
    r, c = np.meshgrid(np.arange(S), np.arange(S), indexing="ij")
    texture = f((c + 0.5) / S, 1.0 - (r + 0.5) / S).transpose(1, 2, 0).astype(f32)        # row r is template v = 1 - (r + 0.5) / S
    uv_template = np.stack([tex[:, 0], 1.0 - tex[:, 1], np.zeros(len(tex))], 1).astype(f32)
    mr = MeshRenderer(faces, X.shape[0], device=DEV)
    Xb = X[None].expand(4, -1, -1).contiguous()
    got, fid, _ = mr.render_unlit(Xb, cams, H, W, uvs=tex, texture=texture)
    uv, _, _ = mr.render_unlit(Xb, cams, H, W, colors=uv_template)
    got, uv, drawn = got.cpu().numpy(), uv.cpu().numpy().astype(np.float64), (fid >= 0).cpu().numpy()
    want = np.stack([f(uv[b, 0], uv[b, 1]) for b in range(4)])
    err = np.abs(got - want).transpose(1, 0, 2, 3)[:, drawn]
    h = 1.0 / S
    bound = h * h / 8 * np.array([0.4 * k1 ** 2, 0.4 * k2 ** 2, 0.0]) + 1e-6
    print(f"pixels {int(drawn.sum())}: max error per channel {err.max(1)}, bound {bound}")
    assert drawn.sum() > 1000 and (err.max(1) <= bound).all()


# ---- the fit ----------------------------------------------------------------------------------------------------------------------------
def _fit_setup(levels=1, S=128):
    from gaussianavatar_b200.body import SMPL
    from gaussianavatar_b200.posmap import PoseMapper
    model, template, betas = tube_model("smpl")
    poser = PoseMapper(model, betas, template, 1, device=DEV, body=SMPL)
    topo = rg.body_topology(template, poser.weights, levels)
    pose, rest = SMPL.split(canonical_pose("smpl").to(DEV))
    x0 = rg.subdivide_points(poser.posed(pose, rest, torch.tensor([CANO_TRANSL], device=DEV))[0], topo)
    layout = rg.UVLayout(topo.faces, topo.uvs, topo.uv_faces, topo.V, S, DEV)
    rng = np.random.default_rng(levels)
    M = ((layout.face_id >= 0).cpu().numpy() & (rng.random((S, S)) < 0.8)).astype(f32)
    return topo, layout, x0, torch.from_numpy(M).to(DEV)


def test_fit_known_answers_on_the_device():
    topo, layout, x0, M = _fit_setup()
    g = layout.fill(x0)
    x, rel = rg.fit_body_mesh(layout, topo, x0, g, M)
    assert torch.equal(x, x0) and float(rel) == 0.0
    c = torch.tensor([0.03, -0.02, 0.01], device=DEV)[:, None, None]
    x, rel = rg.fit_body_mesh(layout, topo, x0, g + c, M)
    x2, _ = rg.fit_body_mesh(layout, topo, x0, g + c, M)
    assert torch.equal(x, x2)
    err = (x - x0 - c.reshape(1, 3)).abs().max().item()
    print(f"constant offset: max |x - (x0 + c)| {err:.3g}, relative residual {float(rel):.3g}")
    assert err < 1e-5


@pytest.mark.parametrize("levels", [0, 1, 2])
def test_fit_agrees_with_an_fp64_direct_solve(levels):
    topo, layout, x0, M = _fit_setup(levels)
    g = layout.fill(x0) + 0.01 * torch.randn(3, layout.S, layout.S, generator=torch.Generator(device=DEV).manual_seed(0), device=DEV)
    x, rel = rg.fit_body_mesh(layout, topo, x0, g, M)
    Bm = bo.layout_matrix(topo.faces, layout.face_id.cpu().numpy(), layout.bary.cpu().numpy(), topo.V)
    Lm = bo.laplacian_matrix(topo.offsets, topo.adj, topo.V)
    want = bo.solve_fit(Bm, M.cpu().numpy().reshape(-1) > 0, g.reshape(3, -1).t().double().cpu().numpy(), x0.double().cpu().numpy(), Lm,
                        rg.FIT_LAMBDA)
    d_ref = want - x0.double().cpu().numpy()
    err = np.abs(x.double().cpu().numpy() - want).max() / np.abs(d_ref).max()
    print(f"L {levels}: V {topo.V}, CG relative residual after {rg.FIT_ITERATIONS} iterations {float(rel):.3g}, "
          f"max |x - x_fp64| / max |d| {err:.3g}")
    assert err < 2e-2


# ---- end to end ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("body,stage", [("smpl", 1), ("smplx", 1), ("smpl", 2)])
def test_body_rig_end_to_end(body, stage):
    m, mapper, template, pose, transl, rest = tube_avatar(body, stage)
    before = _state(m)
    rigs = {L: rg.extract_body_rig(m, template, subdiv=L, influences=4, pose_mapper=mapper) for L in (0, 1, 2)}
    after = _state(m)
    assert before.keys() == after.keys() and all(torch.equal(before[k], after[k]) for k in before)
    res = [rigs[L].fit["residual_rms"] for L in (0, 1, 2)]
    cg = [rigs[L].fit["cg_relative_residual"] for L in (0, 1, 2)]
    print(f"{body} stage {stage}: fit RMS over M (L 0, 1, 2) {['%.4g' % r for r in res]}, CG relative residual "
          f"{['%.3g' % r for r in cg]}, |M| {rigs[1].fit['texels']}")
    assert res[1] <= res[0] * (1 + 1e-3) and res[2] <= res[1] * (1 + 1e-3)
    rig = rigs[1]
    w = rig.weights.double()
    assert (rig.joints.long() < m.body.joints).all() and (w.sum(1) - 1).abs().max() < 1e-6
    S = int(m.model_parms.query_posmap_size)
    assert tuple(rig.texture.shape) == (S, S, 3) and rig.texture.dtype == torch.uint8
    tsdf = rg.extract_rigged_mesh(m, res=256, views=64, size=512, influences=4, pose_mapper=mapper)
    with torch.no_grad():
        means, scales, _ = me.posed_gaussians(m, pose, transl, rest, mapper)
    origin, voxel, dims, _ = me.fusion_grid(means, scales, 256, 4)
    center = np.asarray(origin) + 0.5 * voxel * (np.asarray(dims) - 1)
    held_out = me.fusion_cameras(center, 0.5 * voxel * float(np.linalg.norm(np.asarray(dims) - 1)), 8, 512)
    full = m.body.join(pose[None], rest.reshape(1, -1)) if m.body.rest_width else pose[None]
    mo = rg.bake_poses(m._rest_joints, full, transl[None], 30.0, "y")
    out = {}
    for name, r in (("body", rig), ("tsdf", tsdf)):
        v = torch.from_numpy(rg.pose_rig(r, mo, 0)).float().to(DEV)
        out[name] = (me.silhouette_iou(m, pose, transl, v, r.faces, held_out, 512, 512, rest, mapper),
                     rg.unlit_psnr(m, r, v, pose, transl, held_out, 512, 512, rest, mapper))
    (ib, pb), (it, pt) = out["body"], out["tsdf"]
    print(f"{body} stage {stage}: IoU body min {min(ib):.4f} mean {np.mean(ib):.4f}, tsdf min {min(it):.4f} mean {np.mean(it):.4f}; "
          f"PSNR body min {min(pb):.2f} mean {np.mean(pb):.2f}, tsdf min {min(pt):.2f} mean {np.mean(pt):.2f} dB; "
          f"V body {rig.verts.shape[0]} tsdf {tsdf.verts.shape[0]}")
    assert min(ib) >= min(it) - IOU_GAP
    assert np.mean(pb) >= np.mean(pt) - PSNR_GAP


def test_tool_end_to_end(tmp_path):
    from dataset_fixture import write_synthetic_dataset
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams, OptimizationParams
    from test_rig_cpu import accessor, read_glb
    mp = write_synthetic_dataset(str(tmp_path), seed=0)
    smpl = os.path.join(mp.smpl_model_path, "SMPL_NEUTRAL.pkl")
    template = syn.make_uv_template(0)
    with open(smpl, "wb") as fh:                      # the same body with the fields the body rig needs (weights, faces, posedirs)
        pickle.dump(syn.smpl_mesh_model(syn.make_body(0), template), fh)
    syn.write_uv_template_obj(os.path.join(mp.project_path, "assets", "template_mesh_smpl_uv.obj"), template)
    torch.manual_seed(0)
    m = AvatarModel(mp, NetworkParams(nf=8), OptimizationParams(), train=True)
    m.training_setup()
    with torch.no_grad():
        sd = m.net.state_dict()
        sd["decoder.conv8N.bias"] = torch.tensor([-5.3])
        m.net.load_state_dict(sd, strict=False)
    m.save(7)
    base = [sys.executable, os.path.join(ROOT, "tools", "extract_mesh.py"), "-s", mp.source_path, "-m", mp.model_path, "--project_path",
            mp.project_path, "--smpl_model", smpl, "--query_posmap_size", str(mp.query_posmap_size), "--inp_posmap_size",
            str(mp.inp_posmap_size), "--epoch", "7", "--format", "glb", "--frame", "0", "--frame", "2", "--iou", "--psnr"]
    r = subprocess.run(base + ["--topology", "body", "--out", str(tmp_path / "rig")], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    rec = json.loads([x for x in r.stdout.splitlines() if x.startswith("{")][-1])
    print("tool (body)", rec)
    assert len(rec["iou"]) == 2 and len(rec["psnr"]) == 2 and all(np.isfinite(rec["psnr"])) and rec["fit"]["texels"] > 0
    g, binc = read_glb(rec["mesh"])
    prim = g["meshes"][0]["primitives"][0]
    assert "TEXCOORD_0" in prim["attributes"] and g["extensionsUsed"] == ["KHR_materials_unlit"]
    assert accessor(g, binc, prim["indices"]).size == 3 * rec["faces"]
    r = subprocess.run(base + ["--res", "64", "--views", "16", "--size", "128", "--out", str(tmp_path / "tsdf")], capture_output=True,
                       text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    rec = json.loads([x for x in r.stdout.splitlines() if x.startswith("{")][-1])
    print("tool (tsdf)", rec)
    assert len(rec["psnr"]) == 2 and all(np.isfinite(rec["psnr"])) and "fit" not in rec
