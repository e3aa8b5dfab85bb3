"""CPU: mesh extraction.  The marching-tetrahedra case table and the Kuhn split, oracle/tsdf_oracle.py's mesher on analytic fields
(sphere, torus, two spheres) and its integration of ray-cast sphere depth maps, the C ABI's refusals (before any launch), the tool's
argument handling, and PLY / OBJ round trips."""
import ctypes
import importlib.util
import os
import sys
from collections import Counter

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gaussianavatar_b200 import _lib  # noqa: E402
from gaussianavatar_b200 import mesh_extract as me  # noqa: E402
from oracle import tsdf_oracle as to  # noqa: E402

f32 = np.float32


# ---- mesh checks shared with the GPU tests ------------------------------------------------------------------------------------------
def directed_edges(faces):
    f = np.asarray(faces, np.int64)
    return np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])


def closed_manifold(faces) -> bool:
    """Every undirected edge is in exactly two faces, used once in each direction."""
    e = Counter(map(tuple, directed_edges(faces)))
    return bool(e) and all(n == 1 for n in e.values()) and all(e.get((b, a), 0) == 1 for a, b in e)


def euler(verts, faces) -> int:
    return len(verts) - len(directed_edges(faces)) // 2 + len(faces)


def components(nv, faces) -> int:
    parent = np.arange(nv)

    def find(a):
        while parent[a] != a:
            parent[a] = parent[parent[a]]
            a = parent[a]
        return a
    for a, b in directed_edges(faces):
        ra, rb = find(a), find(b)
        if ra != rb:
            parent[ra] = rb
    used = np.unique(np.asarray(faces).reshape(-1))
    return len({find(v) for v in used})


def signed_volume(verts, faces):
    v = np.asarray(verts, np.float64)[np.asarray(faces, np.int64)]
    return float(np.einsum("ij,ij->i", v[:, 0], np.cross(v[:, 1], v[:, 2])).sum() / 6.0)


def _field(fn, n, voxel, trunc):
    org = np.full(3, -0.5 * voxel * (n - 1), f32)
    x, y, z = to.sample_positions(org, voxel, (n, n, n))
    v = np.clip(fn(x.astype(np.float64), y.astype(np.float64), z.astype(np.float64)) / trunc, -1, 1).astype(f32)
    v[0], v[-1], v[:, 0], v[:, -1], v[:, :, 0], v[:, :, -1] = 1, 1, 1, 1, 1, 1
    return v, org


# ---- case table -------------------------------------------------------------------------------------------------------------------
def test_case_table_separates_and_faces_outward():
    ntri, edges, corner, owner, slot = to.case_table()
    g = np.random.default_rng(0)
    for t in range(6):
        pos = np.array([to.corner_offset(int(c)) for c in corner[t]], np.float64)
        assert abs(np.linalg.det(pos[1:] - pos[0])) == 1.0                # a proper tetrahedron
        for c in range(16):
            ins = [v for v in range(4) if (c >> v) & 1]
            outs = [v for v in range(4) if not (c >> v) & 1]
            crossing = {to._local_edge(a, b) for a in ins for b in outs}
            used = {int(e) for k in range(ntri[t, c]) for e in edges[t, c, k]}
            assert used == crossing and ntri[t, c] == (0 if not crossing else 1 if len(crossing) == 3 else 2)
            for trial in range(4):                                          # midpoints, then random crossings along the edges
                tt = np.full(6, 0.5) if trial == 0 else g.uniform(0.05, 0.95, 6)
                P = {e: pos[to.EDGE_V[e][0]] + tt[e] * (pos[to.EDGE_V[e][1]] - pos[to.EDGE_V[e][0]]) for e in range(6)}
                for k in range(ntri[t, c]):
                    a, b, cc = (P[int(e)] for e in edges[t, c, k])
                    n = np.cross(b - a, cc - a)
                    assert np.linalg.norm(n) > 0
                    # the triangle's plane separates the tetrahedron's inside vertices from its outside ones, facing outward
                    assert all(n @ (pos[v] - a) < 0 for v in ins) and all(n @ (pos[v] - a) > 0 for v in outs), (t, c, k, trial)
            for e in range(6):
                i, j = to.EDGE_V[e]
                assert owner[t, e] == corner[t, i]
                assert to.SLOT_MASKS[slot[t, e]] == corner[t, j] ^ corner[t, i]


def test_kuhn_split_is_conforming():
    """Every cube face is cut along the same diagonal from both cubes that share it, and the six tetrahedra fill the cube."""
    _, _, corner, _, _ = to.case_table()
    vols = [abs(np.linalg.det(np.array([to.corner_offset(int(c)) for c in corner[t][1:]], np.float64))) / 6 for t in range(6)]
    assert np.isclose(sum(vols), 1.0)

    def diagonals(axis, side):
        """Cube-face diagonals (as pairs of face-local corner positions) the tetrahedra draw on the face {x_axis = side}."""
        out = set()
        for t in range(6):
            on = [to.corner_offset(int(c)) for c in corner[t] if ((int(c) >> axis) & 1) == side]
            for a in on:
                for b in on:
                    d = b - a
                    if np.count_nonzero(d) == 2:
                        key = tuple(sorted([tuple(np.delete(a, axis)), tuple(np.delete(b, axis))]))
                        out.add(key)
        return out
    for axis in range(3):
        assert diagonals(axis, 1) == diagonals(axis, 0) and len(diagonals(axis, 0)) == 1


# ---- oracle mesher on analytic fields -----------------------------------------------------------------------------------------------
def test_sphere_is_closed_with_the_right_volume():
    n, voxel, r = 40, 0.08, 1.0
    v, org = _field(lambda x, y, z: np.sqrt(x * x + y * y + z * z) - r, n, voxel, 4 * voxel)
    V, F, _ = to.mesh_from_values(v, org, voxel)
    assert closed_manifold(F) and euler(V, F) == 2
    vol = signed_volume(V, F)
    assert abs(vol / (4 / 3 * np.pi * r ** 3) - 1) < 0.01, vol                 # inscribed facets: a slight underestimate
    assert np.abs(np.linalg.norm(V.astype(np.float64), axis=1) - r).max() < voxel


def test_torus_has_euler_characteristic_zero():
    n, voxel, R, a = 48, 0.06, 0.9, 0.35
    v, org = _field(lambda x, y, z: np.sqrt((np.sqrt(x * x + z * z) - R) ** 2 + y * y) - a, n, voxel, 4 * voxel)
    V, F, _ = to.mesh_from_values(v, org, voxel)
    assert closed_manifold(F) and euler(V, F) == 0 and signed_volume(V, F) > 0


def test_two_spheres_give_two_components():
    n, voxel = 48, 0.06
    v, org = _field(lambda x, y, z: np.minimum(np.sqrt((x - 0.7) ** 2 + y * y + z * z), np.sqrt((x + 0.7) ** 2 + y * y + z * z)) - 0.5,
                    n, voxel, 4 * voxel)
    V, F, _ = to.mesh_from_values(v, org, voxel)
    assert closed_manifold(F) and components(len(V), F) == 2 and euler(V, F) == 4


# ---- oracle integration of ray-cast sphere depth maps ------------------------------------------------------------------------------
def sphere_views(cams, H, W, center, r, color):
    """Analytic depth pass of an opaque sphere: (depth [B,2,H,W], image [B,3,H,W] with bg 0, final_T [B,H,W]).  Pixel (c, r) is the
    ray through view-space (c + 0.5 - W/2, r + 0.5 - H/2, f) of fusion_cameras' centred intrinsics."""
    B = len(cams)
    depth = np.zeros((B, 2, H, W), f32)
    image = np.zeros((B, 3, H, W), f32)
    final_T = np.ones((B, H, W), f32)
    for b in range(B):
        M = np.asarray(cams[b][:16], np.float64).reshape(4, 4).T          # column-vector world -> view
        tanx = float(cams[b][32])
        f = 0.5 * W / tanx
        R, t = M[:3, :3], M[:3, 3]
        C = -R.T @ t
        cc, rr = np.meshgrid(np.arange(W), np.arange(H))
        d = np.stack([(cc + 0.5 - W / 2) / f, (rr + 0.5 - H / 2) / f, np.ones_like(cc, float)], -1) @ R   # world directions, view z = 1
        oc = C - np.asarray(center, np.float64)
        A = (d * d).sum(-1)
        Bq = 2 * (d @ oc)
        disc = Bq * Bq - 4 * A * (oc @ oc - r * r)
        hit = disc > 0
        s = np.where(hit, (-Bq - np.sqrt(np.where(hit, disc, 0))) / (2 * A), 0)
        depth[b, 1] = np.where(hit, s, 0)
        depth[b, 0] = depth[b, 1]
        final_T[b] = np.where(hit, 0, 1)
        for ch in range(3):
            image[b, ch] = np.where(hit, color[ch], 0)
    return depth, image, final_T


def test_oracle_fusion_of_a_ray_cast_sphere():
    n, r = 32, 0.6
    voxel = 2.0 / (n - 1)
    org = np.full(3, -1.0, f32)
    dims = (n, n, n)
    cams = me.fusion_cameras(np.zeros(3), np.sqrt(3.0), 24, 160).numpy()
    depth, image, final_T = sphere_views(cams, 160, 160, np.zeros(3), r, (0.25, 0.5, 0.75))
    S = to.integrate(to.new_state(dims), org, voxel, 4 * voxel, cams, depth, image, final_T)
    x, y, z = to.sample_positions(org, voxel, dims)
    dist = np.sqrt(x.astype(np.float64) ** 2 + y ** 2 + z ** 2)
    assert (S["carve"][dist > r + voxel] >= 1).all()                      # carving removes everything outside
    assert (S["carve"][dist < r - voxel] == 0).all()
    V, F, C = to.mesh(S, org, voxel)
    assert closed_manifold(F) and euler(V, F) == 2
    # eta is a difference of view depths, not a Euclidean distance: views at an oblique angle to the surface overstate it, so a vertex
    # can sit a little more than a voxel off (1.13 voxels here); on average it is a quarter of a voxel
    err = np.abs(np.linalg.norm(V.astype(np.float64), axis=1) - r)
    assert err.max() < 1.25 * voxel and err.mean() < 0.35 * voxel
    assert np.abs(C - np.array([0.25, 0.5, 0.75], f32)).max() < 1e-6


# ---- C ABI refusals ---------------------------------------------------------------------------------------------------------------
def _desc(**kw):
    d = dict(nx=8, ny=8, nz=8, origin=(0.0, 0.0, 0.0), voxel=0.1, trunc=0.4)
    d.update(kw)
    return _lib.GaTsdfDesc(d["nx"], d["ny"], d["nz"], (ctypes.c_float * 3)(*d["origin"]), d["voxel"], d["trunc"])


BAD_DESCS = [
    (dict(nx=1), "outside [2, 512]"), (dict(ny=513), "outside [2, 512]"), (dict(nz=0), "outside [2, 512]"),
    (dict(voxel=0.0), "voxel size"), (dict(voxel=float("nan")), "voxel size"), (dict(voxel=-1.0), "voxel size"),
    (dict(trunc=0.0), "truncation"), (dict(trunc=float("inf")), "truncation"), (dict(origin=(0.0, float("nan"), 0.0)), "origin"),
]


@pytest.mark.parametrize("bad,message", BAD_DESCS)
def test_cabi_refuses_bad_grids_before_any_launch(bad, message):
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    L = _lib.lib()
    fake = 256                     # never dereferenced
    d = ctypes.byref(_desc(**bad))
    before = L.ga_launch_count()
    assert L.ga_tsdf_state_bytes(d) == 0 and L.ga_tsdf_mesh_workspace_bytes(d) == 0
    assert L.ga_tsdf_reset(d, fake, None) != 0 and message in L.ga_last_error().decode()
    assert L.ga_tsdf_integrate(d, 1, 16, 16, fake, fake, fake, fake, fake, None) != 0 and message in L.ga_last_error().decode()
    assert L.ga_tsdf_mesh_count(d, fake, 1, fake, 1 << 30, fake, None) != 0 and message in L.ga_last_error().decode()
    assert L.ga_tsdf_mesh_emit(d, fake, 1, fake, 1 << 30, 4, 4, fake, fake, fake, None) != 0 and message in L.ga_last_error().decode()
    assert L.ga_launch_count() == before


@pytest.mark.parametrize("case,message", [
    ("B=0", "views outside [1, 8]"), ("B=9", "views outside [1, 8]"), ("H=0", "outside [1, 16384]"), ("NULL depth", "NULL pointer"),
    ("NULL state", "NULL pointer"), ("NULL desc", "NULL grid descriptor"), ("min_carve=0", "min_carve 0"),
    ("NULL totals", "NULL pointer"), ("small workspace", "workspace of"), ("negative capacity", "negative capacity"),
    ("NULL verts", "NULL pointer"),
])
def test_cabi_refuses_bad_arguments_before_any_launch(case, message):
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    L = _lib.lib()
    fake = 256
    d = ctypes.byref(_desc())
    before = L.ga_launch_count()
    if case in ("B=0", "B=9", "H=0", "NULL depth", "NULL state", "NULL desc"):
        B = {"B=0": 0, "B=9": 9}.get(case, 2)
        H = 0 if case == "H=0" else 16
        rc = L.ga_tsdf_integrate(None if case == "NULL desc" else d, B, H, 16, fake, None if case == "NULL depth" else fake, fake, fake,
                                 None if case == "NULL state" else fake, None)
    elif case in ("min_carve=0", "NULL totals", "small workspace"):
        rc = L.ga_tsdf_mesh_count(d, fake, 0 if case == "min_carve=0" else 1, fake, 16 if case == "small workspace" else 1 << 30,
                                  None if case == "NULL totals" else fake, None)
    else:
        rc = L.ga_tsdf_mesh_emit(d, fake, 1, fake, 1 << 30, -1 if case == "negative capacity" else 4, 4,
                                 None if case == "NULL verts" else fake, fake, fake, None)
    assert rc != 0 and message in L.ga_last_error().decode()
    assert L.ga_launch_count() == before


def test_state_bytes():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    assert _lib.lib().ga_tsdf_state_bytes(ctypes.byref(_desc(nx=40, ny=48, nz=64))) == 28 * 40 * 48 * 64


# ---- tool ---------------------------------------------------------------------------------------------------------------------------
def _tool():
    spec = importlib.util.spec_from_file_location("extract_mesh_tool", os.path.join(ROOT, "tools", "extract_mesh.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("extra,message", [
    ([], "give --frame K (repeatable) or --motion CLIP"),
    (["--frame", "0", "--motion", "c.npz", "--fps", "10"], "not both"),
    (["--frame", "0", "--fps", "10"], "go with --motion"),
    (["--motion", "c.npz"], "--motion needs --fps"),
    (["--motion", "c.npz", "--fps", "0"], "must be positive"),
    (["--frame", "0", "--res", "513"], "--res 513 outside 2..512"),
    (["--frame", "0", "--min_carve", "0"], "must be positive"),
    (["--frame", "0", "--format", "stl"], "invalid choice"),
    (["--frame", "0", "--stage", "2"], "--stage 2 needs"),
])
def test_tool_arguments(tmp_path, capsys, extra, message):
    tool = _tool()
    with pytest.raises(SystemExit) as e:
        tool.parse(["-s", str(tmp_path), "-m", str(tmp_path), "--epoch", "1", "--out", str(tmp_path / "o")] + extra)
    assert e.value.code == 2 and message in capsys.readouterr().err


def test_tool_accepts_frames_and_motion(tmp_path):
    tool = _tool()
    a = tool.parse(["-s", "S", "-m", "M", "--epoch", "3", "--frame", "0", "--frame", "4", "--out", "o", "--iou", "--format", "obj"])
    assert a.frame == [0, 4] and a.iou and a.format == "obj" and (a.res, a.views, a.size, a.trunc, a.min_carve) == (256, 64, 512, 4.0, 1)
    a = tool.parse(["-s", "S", "-m", "M", "--epoch", "3", "--motion", "c.npz", "--fps", "10", "--align_to", "1", "--out", "o"])
    assert a.motion == "c.npz" and a.fps == 10 and a.align_to == 1 and a.frame is None


# ---- files --------------------------------------------------------------------------------------------------------------------------
def read_ply(path):
    """(verts [V,3] float32, faces [F,3] int32, colours [V,3] uint8) of a binary little-endian PLY as write_ply writes it."""
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    header = data[:end].decode("ascii").split("\n")
    assert header[0] == "ply" and header[1] == "format binary_little_endian 1.0"
    nv = int(next(h for h in header if h.startswith("element vertex")).split()[-1])
    nf = int(next(h for h in header if h.startswith("element face")).split()[-1])
    vt = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    ft = np.dtype([("n", "u1"), ("v", "<i4", (3,))])
    v = np.frombuffer(data, vt, nv, end)
    f = np.frombuffer(data, ft, nf, end + nv * vt.itemsize)
    assert end + nv * vt.itemsize + nf * ft.itemsize == len(data) and (f["n"] == 3).all()
    return (np.stack([v["x"], v["y"], v["z"]], 1), f["v"].astype(np.int32), np.stack([v["red"], v["green"], v["blue"]], 1))


def read_obj(path):
    vs, fs = [], []
    for line in open(path):
        p = line.split()
        if p and p[0] == "v":
            vs.append([float(x) for x in p[1:7]])
        elif p and p[0] == "f":
            fs.append([int(x) - 1 for x in p[1:4]])
    v = np.array(vs, np.float64).reshape(-1, 6)
    return v[:, :3], np.array(fs, np.int32).reshape(-1, 3), v[:, 3:]


def test_ply_and_obj_round_trip(tmp_path):
    g = np.random.default_rng(1)
    V = g.normal(size=(50, 3)).astype(f32)
    F = g.integers(0, 50, size=(70, 3)).astype(np.int32)
    C = g.uniform(-0.1, 1.1, size=(50, 3)).astype(f32)
    C[0] = [np.nan, 0.5 / 255, 1.0]
    me.write_ply(tmp_path / "m.ply", V, F, C)
    v, f, c = read_ply(tmp_path / "m.ply")
    assert np.array_equal(v, V) and np.array_equal(f, F)
    q = np.clip(np.nan_to_num(C * f32(255) + f32(0.5), nan=0), 0, 255).astype(np.uint8)
    assert np.array_equal(c, q) and list(c[0]) == [0, 1, 255]
    me.write_obj(tmp_path / "m.obj", V, F, C)
    v, f, c = read_obj(tmp_path / "m.obj")
    assert np.array_equal(v.astype(f32), V) and np.array_equal(f, F)
    assert np.allclose(c[1:], C[1:], atol=1e-5)
