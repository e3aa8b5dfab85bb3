"""CPU: the body-topology rig.  The fit oracle's known answers (zero and constant offsets, a dense least-squares solve on a small
mesh), the push-pull and Laplacian oracles' properties, the library's subdivision against the oracle's (V, F, Euler characteristic,
welded seams, skin weights), the new C-ABI entries' refusals, a textured .glb round trip and the tool's new arguments."""
import ctypes
import io
import os
import struct
import sys
import zlib

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from gaussianavatar_b200 import rig as rg  # noqa: E402
from gaussianavatar_b200 import synthetic as syn  # noqa: E402
from gaussianavatar_b200.body import SMPL_JOINT_NAMES, SMPL_PARENTS  # noqa: E402
from oracle import body_rig_oracle as bo  # noqa: E402
from oracle import posmap_oracle as po  # noqa: E402
import test_rig_cpu as trc  # noqa: E402

trc._N.setdefault("VEC2", 2)
f32 = np.float32


def _grid(R=6, C=7, seed=0):
    """A small open grid mesh in the plane z = 0 with a two-island UV layout (synthetic._grid_uv_template) and random weights."""
    rng = np.random.default_rng(seed)
    v = np.stack(np.meshgrid(np.linspace(0, 1, C), np.linspace(0, 1, R)), -1).reshape(-1, 2)
    verts = np.concatenate([v, np.zeros((R * C, 1))], 1)
    t = syn._grid_uv_template((R, C), C // 2, rng, 0.2, verts)
    w = rng.random((R * C, 24)) ** 4
    return t, w / w.sum(1, keepdims=True)


def _euler(V, faces):
    e = np.unique(np.sort(np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]), axis=1), axis=0)
    return V - len(e) + len(faces), len(e)


# ---- topology -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("levels", [0, 1, 2])
def test_subdivision_matches_the_oracle_and_keeps_the_topology(levels):
    t, w = _grid()
    topo = rg.body_topology(t, w, levels)
    of, ouv, oft, ow, _ = bo.subdivide(t[1], t[2], t[3], w, levels)
    assert np.array_equal(topo.faces, of) and np.array_equal(topo.uv_faces, oft)
    assert np.array_equal(topo.uvs, ouv) and np.array_equal(topo.weights, ow)
    V0, F0 = t[0].shape[0], t[1].shape[0]
    chi0, E0 = _euler(V0, t[1])
    chi, E = _euler(topo.V, topo.faces)
    assert chi == chi0 and len(topo.faces) == F0 * 4 ** levels
    if levels == 1:
        assert topo.V == V0 + E0
    # the UV seam stays welded in 3D: vertices on it (new midpoints included) carry two texture coordinates and one position
    pairs = np.unique(np.stack([topo.faces.reshape(-1), topo.uv_faces.reshape(-1)], 1), axis=0)
    uvs_per_vertex = np.bincount(pairs[:, 0], minlength=topo.V)
    seam = np.nonzero(uvs_per_vertex == 2)[0]
    assert uvs_per_vertex.max() == 2 and len(seam) == 6 * 2 ** levels - (2 ** levels - 1)
    assert levels == 0 or seam.max() >= V0
    off, adj = bo.adjacency(topo.faces, topo.V)
    assert np.array_equal(topo.offsets, off) and np.array_equal(topo.adj, adj)
    j, ww = rg.top_influences(topo.weights, 4)
    oj, oww = bo.top_k(topo.weights, 4)
    assert np.array_equal(j, oj) and np.array_equal(ww, oww)
    assert np.abs(ww.astype(np.float64).sum(1) - 1).max() < 1e-6


def test_smpl_template_subdivision_counts():
    t = syn.make_uv_template(0)
    w = syn.make_body(0).lbs_weights.double().numpy()
    chi0, E0 = _euler(6890, t[1])
    topo = rg.body_topology(t, w, 1)
    assert topo.V == 6890 + E0 and len(topo.faces) == 4 * len(t[1]) and _euler(topo.V, topo.faces)[0] == chi0
    # a new vertex's weights are its edge's mean: still a partition of unity
    assert np.abs(topo.weights.sum(1) - w.sum(1).mean()).max() < 1e-5


# ---- kernels' oracles ----------------------------------------------------------------------------------------------------------------
def test_laplacian_oracle_is_the_graph_laplacian():
    t, w = _grid()
    topo = rg.body_topology(t, w, 1)
    x = np.random.default_rng(1).normal(size=(topo.V, 3)).astype(f32)
    want = bo.laplacian_matrix(topo.offsets, topo.adj, topo.V) @ x.astype(np.float64)
    got = bo.laplacian(topo.offsets, topo.adj, x)
    assert got.dtype == f32 and np.abs(got - want).max() < 1e-5
    assert np.abs(bo.laplacian(topo.offsets, topo.adj, np.ones_like(x))).max() == 0


@pytest.mark.parametrize("S", [1, 2, 7, 64])
def test_pushpull_oracle_keeps_covered_texels_and_stays_in_range(S):
    rng = np.random.default_rng(S)
    img = rng.random((3, S, S)).astype(f32)
    mask = rng.random((S, S)) < 0.2
    mask.flat[rng.integers(S * S)] = True
    img[:, ~mask] = np.nan                        # uncovered texels are never read
    out = bo.pushpull(img, mask)
    assert np.array_equal(out[:, mask].view(np.int32), img[:, mask].view(np.int32)) and np.isfinite(out).all()
    for c in range(3):
        lo, hi = img[c, mask].min(), img[c, mask].max()
        assert (out[c] >= lo).all() and (out[c] <= hi).all()
    one = np.zeros((S, S), bool)
    one[S // 2, S - 1] = True
    o1 = bo.pushpull(img if mask[S // 2, S - 1] else np.where(one, 0.25, img).astype(f32), one)
    assert np.all(o1 == o1[:, S // 2, S - 1][:, None, None])      # a single covered texel fills the whole map
    assert np.array_equal(bo.pushpull(img, np.zeros((S, S), bool)), np.zeros((3, S, S), f32))


# ---- the fit ------------------------------------------------------------------------------------------------------------------------
def _fit_problem(levels=1, S=24):
    t, w = _grid()
    topo = rg.body_topology(t, w, levels)
    fid, bary = po.layout(topo.uvs.astype(f32)[topo.uv_faces], S)
    Bm = bo.layout_matrix(topo.faces, fid, bary, topo.V)
    rng = np.random.default_rng(3)
    x0 = rng.normal(size=(topo.V, 3)) * 0.1
    mask = (np.asarray(fid).reshape(-1) >= 0) & (rng.random(S * S) < 0.7)
    Lm = bo.laplacian_matrix(topo.offsets, topo.adj, topo.V)
    return topo, Bm, x0, mask, Lm


@pytest.mark.parametrize("lam", [1e-3, 0.1, 10.0])
def test_fit_known_answers(lam):
    topo, Bm, x0, mask, Lm = _fit_problem()
    g = Bm @ x0
    assert np.abs(bo.solve_fit(Bm, mask, g, x0, Lm, lam) - x0).max() < 1e-12
    c = np.array([0.3, -0.2, 0.05])
    x = bo.solve_fit(Bm, mask, g + c, x0, Lm, lam)
    covered = np.asarray(Bm.sum(0)).reshape(-1) > 0
    # B c = c up to the fp32 barycentric weights' rounding (each row sums to 1 within a few 1e-8)
    assert np.abs(x[covered] - (x0[covered] + c)).max() < 1e-6


def test_fit_matches_a_dense_least_squares_solve():
    topo, Bm, x0, mask, Lm = _fit_problem(0, 16)
    rng = np.random.default_rng(5)
    g = Bm @ x0 + rng.normal(size=(Bm.shape[0], 3)) * 0.01
    lam = 0.1
    x = bo.solve_fit(Bm, mask, g, x0, Lm, lam)
    # min |M (B (x0 + d) - g)|^2 + lam |D d|^2 with D the edge-difference matrix (D^T D = L), as one stacked dense system
    e = np.unique(np.sort(np.concatenate([topo.faces[:, [0, 1]], topo.faces[:, [1, 2]], topo.faces[:, [2, 0]]]), axis=1), axis=0)
    D = np.zeros((len(e), topo.V))
    D[np.arange(len(e)), e[:, 0]], D[np.arange(len(e)), e[:, 1]] = 1.0, -1.0
    Bd = Bm.toarray()[mask]
    A = np.concatenate([Bd, np.sqrt(lam) * D])
    rhs = np.concatenate([g[mask] - Bd @ x0, np.zeros((len(e), 3))])
    d, *_ = np.linalg.lstsq(A, rhs, rcond=None)
    assert np.abs(x - (x0 + d)).max() < 1e-9


# ---- C ABI ----------------------------------------------------------------------------------------------------------------------------
def test_abi_refuses_bad_arguments_before_any_launch():
    from gaussianavatar_b200 import _lib
    L = _lib.lib()
    p = ctypes.c_void_p(256)
    before = _lib.launch_count()
    for V in (0, -1, (1 << 24) + 1):
        assert L.ga_mesh_laplacian(V, p, p, p, p, None) != 0
    for nul in range(4):
        ptrs = [p] * 4
        ptrs[nul] = None
        assert L.ga_mesh_laplacian(10, *ptrs, None) != 0 and "NULL" in L.ga_last_error().decode()
    assert L.ga_texture_pushpull_workspace_bytes(1, 3) == 0 and L.ga_texture_pushpull_workspace_bytes(513, 3) == 0
    assert L.ga_texture_pushpull_workspace_bytes(7, 5) == 0 and L.ga_texture_pushpull_workspace_bytes(512, 3) > 0
    need = L.ga_texture_pushpull_workspace_bytes(64, 3)
    for S, C, ws in ((0, 3, need), (513, 3, need), (64, 0, need), (64, 5, need), (64, 3, need - 1)):
        assert L.ga_texture_pushpull(S, C, p, p, p, ws, p, None) != 0
        assert L.ga_last_error().decode().startswith("ga_texture_pushpull")
    assert L.ga_texture_pushpull(64, 3, p, p, ctypes.c_void_p(260), need, p, None) != 0      # misaligned workspace
    for nul in range(4):
        ptrs = [p] * 4
        ptrs[nul] = None
        assert L.ga_texture_pushpull(64, 3, *ptrs[:3], need, ptrs[3], None) != 0 and "NULL" in L.ga_last_error().decode()
    base = [1, 10, 4, 8, 8, p, p, p, p]
    for args in ([0] + base[1:], [9] + base[1:], base[:1] + [0] + base[2:], base[:3] + [0] + base[4:]):
        assert L.ga_mesh_shade_unlit(*args, p, None, None, 0, 0, None, p, None) != 0
    assert L.ga_mesh_shade_unlit(*base, p, p, p, 4, 4, None, p, None) != 0                 # colours and a texture
    assert L.ga_mesh_shade_unlit(*base, None, None, None, 4, 4, None, p, None) != 0        # neither
    assert L.ga_mesh_shade_unlit(*base, None, p, p, 0, 4, None, p, None) != 0              # an empty texture
    assert L.ga_mesh_shade_unlit(*base, None, p, None, 4, 4, None, p, None) != 0           # coordinates without a texture
    assert L.ga_mesh_shade_unlit(*base[:8], None, p, None, None, 0, 0, None, p, None) != 0  # no face_id
    assert _lib.launch_count() == before


# ---- glb ----------------------------------------------------------------------------------------------------------------------------
def decode_png(data: bytes) -> np.ndarray:
    """An 8-bit RGB, filter-0 PNG (what rig.encode_png writes) -> [H,W,3] uint8, checking every chunk's CRC."""
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    f = io.BytesIO(data[8:])
    idat, hdr = b"", None
    while True:
        n, = struct.unpack(">I", f.read(4))
        tag, body, crc = f.read(4), f.read(n), struct.unpack(">I", f.read(4))[0]
        assert zlib.crc32(tag + body) & 0xFFFFFFFF == crc
        if tag == b"IHDR":
            hdr = struct.unpack(">IIBBBBB", body)
        elif tag == b"IDAT":
            idat += body
        elif tag == b"IEND":
            break
    W, H, depth, ctype = hdr[:4]
    assert depth == 8 and ctype == 2
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(H, 1 + 3 * W)
    assert (raw[:, 0] == 0).all()
    return raw[:, 1:].reshape(H, W, 3)


def _textured_rig(K=4, levels=1):
    a = syn.make_avatar_assets(2000, 64, seed=0)
    sk = rg.skeleton(a.rest_joints, np.linalg.inv(a.cano_joint_mats.double().numpy()), SMPL_PARENTS)
    t = syn.make_uv_template(0)
    topo = rg.body_topology(t, syn.make_body(0).lbs_weights.double().numpy(), levels)
    x = torch.from_numpy(rg.subdivide_points(torch.from_numpy(t[0]).float(), topo).numpy())
    j, w = rg.top_influences(topo.weights, K)
    tex = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (32, 32, 3)).astype(np.uint8))
    return rg.RiggedMesh(x, torch.from_numpy(topo.faces.astype(np.int32)), torch.rand(topo.V, 3), torch.from_numpy(j), torch.from_numpy(w),
                         tuple(SMPL_PARENTS), SMPL_JOINT_NAMES, **sk, uvs=topo.uvs, uv_faces=topo.uv_faces, texture=tex)


@pytest.mark.parametrize("K", [4, 8])
def test_textured_glb_round_trip(tmp_path, K):
    rig = _textured_rig(K)
    path = tmp_path / "body.glb"
    rg.write_glb(path, rig)
    g, binc = trc.read_glb(path)
    prim = g["meshes"][0]["primitives"][0]
    at = prim["attributes"]
    assert sorted(at) == sorted(["POSITION", "TEXCOORD_0"] + [f"{n}_{s}" for n in ("JOINTS", "WEIGHTS") for s in range(K // 4)])
    P, T = trc.accessor(g, binc, at["POSITION"]), trc.accessor(g, binc, at["TEXCOORD_0"])
    idx = trc.accessor(g, binc, prim["indices"]).reshape(-1, 3)
    vid, tex, faces = rg.seam_split(rig)
    assert len(P) == len(T) == len(vid) > rig.verts.shape[0] and np.array_equal(idx, faces)
    assert np.array_equal(P, rig.verts.numpy()[vid]) and (T >= 0).all() and (T <= 1).all()
    # every (vertex, uv) corner of the rig is one written vertex: same position, u kept, v flipped
    f, tf = rig.faces.numpy().reshape(-1), rig.uv_faces.reshape(-1)
    assert np.array_equal(P[idx.reshape(-1)], rig.verts.numpy()[f])
    assert np.allclose(T[idx.reshape(-1)], np.stack([rig.uvs[tf, 0], 1 - rig.uvs[tf, 1]], 1), atol=1e-7)
    Wt = np.concatenate([trc.accessor(g, binc, at[f"WEIGHTS_{s}"]) for s in range(K // 4)], 1)
    Jt = np.concatenate([trc.accessor(g, binc, at[f"JOINTS_{s}"]) for s in range(K // 4)], 1)
    assert np.abs(Wt.astype(np.float64).sum(1) - 1).max() < 1e-6 and Jt.max() < 24 and np.array_equal(Jt, rig.joints.numpy()[vid])
    assert g["extensionsUsed"] == ["KHR_materials_unlit"]
    mat = g["materials"][prim["material"]]
    assert "KHR_materials_unlit" in mat["extensions"] and mat["pbrMetallicRoughness"]["metallicFactor"] == 0.0
    texd = g["textures"][mat["pbrMetallicRoughness"]["baseColorTexture"]["index"]]
    smp = g["samplers"][texd["sampler"]]
    assert smp == {"magFilter": 9729, "minFilter": 9729, "wrapS": 33071, "wrapT": 33071}
    img = g["images"][texd["source"]]
    view = g["bufferViews"][img["bufferView"]]
    assert img["mimeType"] == "image/png"
    png = binc[view["byteOffset"]:view["byteOffset"] + view["byteLength"]]
    assert np.array_equal(decode_png(png), rig.texture.numpy())
    # the skinned bind pose is the mesh
    assert np.abs(rg.pose_rig(rig) - rig.verts.double().numpy()).max() < 1e-5


def test_untextured_rig_is_written_as_before(tmp_path):
    rig, _ = trc._toy_rig(4)
    rg.write_glb(tmp_path / "a.glb", rig)
    g, _ = trc.read_glb(tmp_path / "a.glb")
    assert not any(k in g for k in ("materials", "images", "textures", "samplers", "extensionsUsed"))
    assert "COLOR_0" in g["meshes"][0]["primitives"][0]["attributes"]


# ---- tool ---------------------------------------------------------------------------------------------------------------------------
def test_tool_arguments():
    import extract_mesh as tool
    base = ["-s", "d", "-m", "m", "--epoch", "1", "--out", "o"]
    a = tool.parse(base + ["--format", "glb", "--topology", "body", "--smpl_model", "S.pkl", "--psnr", "--iou", "--frame", "0"])
    assert a.topology == "body" and a.subdiv is None and a.psnr and a.iou
    a = tool.parse(base + ["--format", "glb", "--topology", "body", "--subdiv", "2", "--smpl_model", "S.pkl", "--uv_template", "t.obj"])
    assert a.subdiv == 2 and a.uv_template == "t.obj"
    assert tool.parse(base + ["--format", "glb", "--psnr", "--frame", "1"]).topology == "tsdf"
    for bad in (["--format", "glb", "--topology", "body"], ["--format", "glb", "--subdiv", "1"],
                ["--format", "glb", "--topology", "body", "--smpl_model", "S.pkl", "--subdiv", "3"],
                ["--frame", "0", "--psnr"], ["--frame", "0", "--topology", "body", "--smpl_model", "S.pkl"],
                ["--format", "glb", "--topology", "mesh"]):
        with pytest.raises(SystemExit):
            tool.parse(base + bad)
