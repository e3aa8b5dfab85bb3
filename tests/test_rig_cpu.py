"""CPU: the skin-weight oracle (known answers, neighbour sets against scipy's cKDTree), ga_skin_weights' argument refusals, the glTF
skeleton's identities on the synthetic SMPL and SMPL-X subjects, a .glb round trip through a minimal reader, and the tool's
arguments for --format glb."""
import ctypes
import json
import os
import struct
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gaussianavatar_b200 import rig as rg  # noqa: E402
from gaussianavatar_b200 import synthetic as syn  # noqa: E402
from gaussianavatar_b200.body import SMPL_JOINT_NAMES, SMPL_PARENTS, SMPLX_JOINT_NAMES, SMPLX_PARENTS  # noqa: E402
from oracle import skin_oracle as so  # noqa: E402


# ---- oracle -------------------------------------------------------------------------------------------------------------------------
def test_vertex_on_a_mean_with_k1_takes_that_gaussians_top_K():
    rng = np.random.default_rng(0)
    means = rng.normal(size=(50, 3)).astype(np.float32)
    lbs = rng.random((50, 24)).astype(np.float32)
    j, w = so.skin_weights(means[[7, 20]], means, lbs, 24, 1, 4)
    for r, g in enumerate((7, 20)):
        top = np.argsort(-lbs[g].astype(np.float64), kind="stable")[:4]
        assert list(j[r]) == list(top)
        assert np.allclose(w[r], lbs[g, top] / lbs[g, top].astype(np.float64).sum(), atol=1e-7)


def test_equidistant_ties_go_to_the_lower_index():
    means = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    idx, d2 = so.nearest(np.zeros((1, 3), np.float32), means, 2)
    assert list(idx[0]) == [0, 1] and d2[0, 0] == d2[0, 1]
    lbs = np.zeros((4, 24), np.float32)
    lbs[:, 5] = lbs[:, 3] = 0.5                         # equal weights: joint 3 before joint 5
    j, w = so.skin_weights(np.zeros((1, 3), np.float32), means, lbs, 24, 2, 4)
    assert list(j[0]) == [3, 5, 0, 0] and list(w[0]) == [0.5, 0.5, 0.0, 0.0]


def test_K_truncation_renormalises():
    lbs = np.zeros((1, 24), np.float32)
    lbs[0, [2, 9, 11, 17]] = [0.4, 0.3, 0.2, 0.1]
    j, w = so.skin_weights(np.zeros((1, 3), np.float32), np.zeros((1, 3), np.float32), lbs, 24, 1, 2)
    assert list(j[0]) == [2, 9] and np.allclose(w[0], [4 / 7, 3 / 7], atol=1e-7)
    assert abs(float(w[0].astype(np.float64).sum()) - 1.0) < 1e-6


def test_smplx_56th_column_and_all_zero_rule():
    lbs = np.zeros((2, 56), np.float32)
    lbs[0, 55] = 1.0                                    # the padding column never counts: the blend is zero
    lbs[1, 40] = 1.0
    v = np.array([[0, 0, 0], [5, 5, 5]], np.float32)
    m = np.array([[0, 0, 0], [5, 5, 5]], np.float32)
    j, w = so.skin_weights(v, m, lbs, 55, 1, 4)
    assert list(j[0]) == [0, 0, 0, 0] and list(w[0]) == [1.0, 0.0, 0.0, 0.0]
    assert list(j[1]) == [40, 0, 0, 0] and list(w[1]) == [1.0, 0.0, 0.0, 0.0]


def test_blend_is_inverse_distance_weighted():
    means = np.array([[0, 0, 0], [0.1, 0, 0]], np.float32)
    lbs = np.zeros((2, 24), np.float32)
    lbs[0, 1], lbs[1, 2] = 1.0, 1.0
    v = np.array([[0.02, 0, 0]], np.float32)
    j, w = so.skin_weights(v, means, lbs, 24, 2, 4)
    d2 = so.dist2(v, means)[0].astype(np.float64)
    c = 1 / (d2 + 1e-6)
    assert list(j[0][:2]) == [1, 2] and np.allclose(w[0][:2], c / c.sum(), atol=1e-7)


@pytest.mark.parametrize("k", [1, 8, 16])
def test_oracle_neighbour_sets_match_ckdtree(k):
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(k)
    means = rng.normal(size=(3000, 3)).astype(np.float32)
    verts = rng.normal(size=(500, 3)).astype(np.float32)
    idx, d2 = so.nearest(verts, means, k)
    dd, ii = cKDTree(means.astype(np.float64)).query(verts.astype(np.float64), k)
    ii = ii.reshape(len(verts), k)
    dd = dd.reshape(len(verts), k)
    assert np.array_equal(np.sort(idx, 1), np.sort(ii, 1))
    assert np.allclose(np.sqrt(d2.astype(np.float64)), dd, rtol=1e-5, atol=1e-6)


def test_abi_refuses_bad_arguments_before_any_launch():
    from gaussianavatar_b200 import _lib
    L = _lib.lib()
    p = ctypes.c_void_p(16)
    before = _lib.launch_count()
    for args in [(0, 10, 24, 24, 4, 4), (10, 0, 24, 24, 4, 4), (10, 10, 24, 24, 0, 4), (10, 10, 24, 24, 17, 4), (10, 3, 24, 24, 4, 4),
                 (10, 10, 24, 24, 4, 0), (10, 10, 24, 24, 4, 9), (10, 10, 25, 24, 4, 4), (10, 10, 24, 300, 4, 4), (10, 10, 2, 2, 1, 4)]:
        assert L.ga_skin_weights(*args, p, p, p, p, p, None) != 0, args
        assert L.ga_last_error().decode().startswith("ga_skin_weights")
    for nul in range(5):
        ptrs = [p] * 5
        ptrs[nul] = None
        assert L.ga_skin_weights(10, 10, 24, 24, 4, 4, *ptrs, None) != 0
        assert "NULL" in L.ga_last_error().decode()
    assert _lib.launch_count() == before


# ---- skeleton -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("body", ["smpl", "smplx"])
def test_skeleton_identities(body):
    a = syn.make_avatar_assets(2000, 64, seed=0, body=body)
    parents = SMPLX_PARENTS if body == "smplx" else SMPL_PARENTS
    inv = np.linalg.inv(a.cano_joint_mats.double().numpy())
    sk = rg.skeleton(a.rest_joints, inv, parents)
    G = rg.node_globals(parents, sk["translations"], sk["rotations"])
    assert np.abs(G @ sk["ibm"] - np.eye(4)).max() < 1e-5
    rng = np.random.default_rng(1)
    Jr = a.rest_joints.double().numpy()
    for _ in range(3):
        pose = (rng.normal(size=3 * len(parents)) * 0.4).astype(np.float32)
        t = rng.normal(size=3).astype(np.float32) * 0.1
        m = rg.bake_poses(a.rest_joints, pose[None], t[None], 30.0, "y")
        loc = sk["translations"].copy()
        loc[0] = m.root_translation[0]
        Gp = rg.node_globals(parents, loc, m.rotations[0])
        want = syn.joint_transforms_np(Jr, pose.astype(np.float64), t.astype(np.float64), parents) @ inv
        assert np.abs(Gp @ sk["ibm"] - want).max() < 1e-5
    assert len(SMPL_JOINT_NAMES) == 24 and len(SMPLX_JOINT_NAMES) == 55 and len(set(SMPLX_JOINT_NAMES)) == 55


def test_quaternion_round_trip():
    rng = np.random.default_rng(2)
    R = syn.rodrigues_np(rng.normal(size=(200, 3)) * 2.0)
    R[:4] = [np.eye(3), np.diag([1.0, -1, -1]), np.diag([-1.0, 1, -1]), np.diag([-1.0, -1, 1])]
    q = rg.quat_from_matrix(R)
    assert np.allclose(np.linalg.norm(q, axis=1), 1.0) and (q[:, 3] >= 0).all()
    assert np.abs(rg.matrix_from_quat(q) - R).max() < 1e-7          # the shifted norm leaves R 1e-8 off orthonormal


# ---- glb ----------------------------------------------------------------------------------------------------------------------------
def read_glb(path):
    """(json dict, BIN bytes) of a .glb, checking the header and chunk layout."""
    data = open(path, "rb").read()
    magic, version, length = struct.unpack_from("<III", data, 0)
    assert magic == 0x46546C67 and version == 2 and length == len(data) and length % 4 == 0
    jl, jt = struct.unpack_from("<II", data, 12)
    assert jt == 0x4E4F534A and jl % 4 == 0
    js = data[20:20 + jl]
    assert js.rstrip(b" ") == js.rstrip() and js.decode().strip()[-1] == "}"
    bl, bt = struct.unpack_from("<II", data, 20 + jl)
    assert bt == 0x004E4942 and bl % 4 == 0 and 28 + jl + bl == len(data)
    return json.loads(js), data[28 + jl:28 + jl + bl]


_DT = {5126: np.float32, 5121: np.uint8, 5125: np.uint32}
_N = {"SCALAR": 1, "VEC3": 3, "VEC4": 4, "MAT4": 16}


def accessor(g, binc, i):
    a = g["accessors"][i]
    v = g["bufferViews"][a["bufferView"]]
    dt = np.dtype(_DT[a["componentType"]])
    off = v.get("byteOffset", 0) + a.get("byteOffset", 0)
    n = a["count"] * _N[a["type"]]
    assert off % dt.itemsize == 0 and n * dt.itemsize <= v["byteLength"] and off + v["byteLength"] <= len(binc)
    assert v["byteOffset"] + v["byteLength"] <= g["buffers"][0]["byteLength"] == len(binc)
    out = np.frombuffer(binc, dt, n, off).reshape(a["count"], -1)
    if "min" in a:
        assert np.allclose(out.min(0), a["min"]) and np.allclose(out.max(0), a["max"])
    return out


def _toy_rig(K, seed=0):
    a = syn.make_avatar_assets(2000, 64, seed=0)
    inv = np.linalg.inv(a.cano_joint_mats.double().numpy())
    sk = rg.skeleton(a.rest_joints, inv, SMPL_PARENTS)
    rng = np.random.default_rng(seed)
    V = 300
    verts = a.query_points[:V].clone()
    faces = torch.from_numpy(rng.integers(0, V, (500, 3)).astype(np.int32))
    lbs = a.query_lbs.numpy()
    j, w = so.skin_weights(verts.numpy(), a.query_points.numpy(), lbs, 24, 8, K)
    return rg.RiggedMesh(verts, faces, torch.rand(V, 3), torch.from_numpy(j), torch.from_numpy(w), tuple(SMPL_PARENTS),
                         SMPL_JOINT_NAMES, **sk), a


@pytest.mark.parametrize("K,up", [(4, None), (8, "z"), (4, "-y")])
def test_glb_round_trip(tmp_path, K, up):
    rig, a = _toy_rig(K)
    motion = None
    if up is not None:
        pose, t = syn.synthetic_poses(5, seed=1)
        motion = rg.bake_poses(a.rest_joints, pose, t, 24.0, up)
    path = tmp_path / "a.glb"
    rg.write_glb(path, rig, motion)
    g, binc = read_glb(path)
    assert g["asset"]["version"] == "2.0"
    prim = g["meshes"][0]["primitives"][0]
    at = prim["attributes"]
    assert sorted(at) == sorted(["POSITION", "COLOR_0"] + [f"{n}_{s}" for n in ("JOINTS", "WEIGHTS") for s in range(K // 4)])
    P = accessor(g, binc, at["POSITION"])
    assert np.array_equal(P, rig.verts.numpy())
    idx = accessor(g, binc, prim["indices"])
    assert g["accessors"][prim["indices"]]["componentType"] == 5125 and idx.max() < len(P)
    Jt = np.concatenate([accessor(g, binc, at[f"JOINTS_{s}"]) for s in range(K // 4)], 1)
    Wt = np.concatenate([accessor(g, binc, at[f"WEIGHTS_{s}"]) for s in range(K // 4)], 1)
    assert Jt.max() < 24 and np.abs(Wt.astype(np.float64).sum(1) - 1).max() < 1e-6 and (Wt >= 0).all()
    skin = g["skins"][0]
    assert skin["joints"] == list(range(1, 25)) and skin["skeleton"] == 1
    ibm = accessor(g, binc, skin["inverseBindMatrices"]).reshape(24, 4, 4)
    assert np.allclose(np.transpose(ibm, (0, 2, 1)), rig.ibm, atol=1e-6)            # column-major
    nodes = g["nodes"]
    assert nodes[0]["mesh"] == 0 and nodes[0]["skin"] == 0
    for j in range(24):
        kids = [1 + i for i, p in enumerate(SMPL_PARENTS) if p == j]
        assert nodes[1 + j].get("children", []) == kids
        assert np.allclose(nodes[1 + j]["rotation"], rig.rotations[j]) and np.allclose(nodes[1 + j]["translation"], rig.translations[j])
    G = rg.node_globals(SMPL_PARENTS, np.array([n["translation"] for n in nodes[1:]]), np.array([n["rotation"] for n in nodes[1:]]))
    assert np.abs(G @ np.transpose(ibm, (0, 2, 1)) - np.eye(4)).max() < 1e-5
    if motion is None:
        assert "animations" not in g
        return
    an = g["animations"][0]
    assert len(an["channels"]) == 25 and all(s["interpolation"] == "LINEAR" for s in an["samplers"])
    times = accessor(g, binc, an["samplers"][0]["input"]).ravel()
    assert len(times) == 5 and (np.diff(times) > 0).all()
    for ch in an["channels"]:
        out = accessor(g, binc, an["samplers"][ch["sampler"]]["output"])
        assert len(out) == 5
        if ch["target"]["path"] == "rotation":
            assert np.abs(np.linalg.norm(out.astype(np.float64), axis=1) - 1).max() < 1e-6
    # up folded into the root only: the glTF-posed vertices are the clip-world pose turned by U, and the clip's up goes to +Y
    U = rg.UP_ROTATIONS[up]
    assert np.allclose(U @ {"z": [0, 0, 1], "-y": [0, -1, 0]}[up], [0, 1, 0])
    flat = rg.bake_poses(a.rest_joints, pose, t, 24.0, "y")
    for i in (0, 4):
        assert np.abs(rg.pose_rig(rig, motion, i) - rg.pose_rig(rig, flat, i) @ U.T).max() < 1e-5
    assert np.allclose(motion.rotations[:, 1:], flat.rotations[:, 1:] * np.sign((motion.rotations[:, 1:] * flat.rotations[:, 1:]).sum(-1,
                                                                                                                         keepdims=True)))


def test_pose_rig_at_bind_is_the_mesh():
    rig, _ = _toy_rig(4)
    assert np.abs(rg.pose_rig(rig) - rig.verts.double().numpy()).max() < 1e-5


# ---- tool ---------------------------------------------------------------------------------------------------------------------------
def test_tool_arguments():
    import extract_mesh as tool
    base = ["-s", "d", "-m", "m", "--epoch", "1", "--out", "o"]
    a = tool.parse(base + ["--format", "glb"])
    assert a.frame is None and a.motion is None and a.influences is None
    a = tool.parse(base + ["--format", "glb", "--motion", "c.npz", "--fps", "30", "--up", "z", "--influences", "8"])
    assert a.up == "z" and a.influences == 8
    for bad in (["--format", "glb", "--frame", "0", "--motion", "c.npz", "--fps", "3"], ["--format", "glb", "--up", "z"],
                ["--format", "glb", "--influences", "6"], ["--frame", "0", "--influences", "8"], ["--frame", "0", "--up", "y"],
                ["--format", "glb", "--motion", "c.npz"], ["--format", "glb", "--fps", "3"], ["--format", "ply"]):
        with pytest.raises(SystemExit):
            tool.parse(base + bad)
    assert rg.default_up("a.npz", None) == "z" and rg.default_up("a.npz", 0) == "-y" and rg.default_up("smpl_parms.pth", None) == "-y"
