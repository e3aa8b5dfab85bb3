"""GPU: mesh extraction.  ga_tsdf_integrate against oracle/tsdf_oracle.py (ray-cast sphere depth maps and the real depth pass of a
random scene, grids 32^3 and 40 x 48 x 64), fusion split over launches of 1, 3 and 8 views, the mesher against the oracle on the
device's own grid (order, sentinels, repeatability), a shell of opaque Gaussians end to end, synthetic SMPL / SMPL-X avatars (stage 1
and a stage-2 model) against their own silhouettes from held-out cameras, and tools/extract_mesh.py on a saved checkpoint."""
import json
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from gaussianavatar_b200 import mesh_extract as me  # noqa: E402
from gaussianavatar_b200 import synthetic as syn  # noqa: E402
from gaussianavatar_b200.rasterizer import RasterBatchPlan, rasterize_batch_depth  # noqa: E402
from gaussianavatar_b200.animate import final_transmittance  # noqa: E402
from oracle import tsdf_oracle as to  # noqa: E402
from test_mesh_extract_cpu import closed_manifold, euler, read_ply, sphere_views  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
f32 = np.float32
# IoU of the mesh's coverage against the avatar's own alpha >= 0.5 surface from 8 held-out 512^2 cameras, res 256, 64 views: observed
# 0.900-0.926 on an H100 (DESIGN.md §2)
IOU_MIN = 0.89


def _planes(vol):
    return {k: v.cpu().numpy() for k, v in vol.fields().items()}


def _near_boundary(cams, H, W, origin, voxel, dims):
    """Samples whose projection in some view lies within 1e-4 px of a pixel-rounding boundary (x.5)."""
    x, y, z = to.sample_positions(origin, voxel, dims)
    out = np.zeros(x.shape, bool)
    for c in cams:
        px, py, vz = to.project(c, H, W, x, y, z)
        for p in (px, py):
            fr = np.abs(p - np.floor(p) - 0.5)
            out |= (vz > 0.2) & (fr < 1e-4)
    return out


def _compare(vol, S, near):
    got = _planes(vol)
    keep = ~near
    for k in ("weight", "carve", "cw"):
        assert np.array_equal(got[k][keep], S[k][keep]), k
    for k in ("sdf", "r", "g", "b"):
        assert np.array_equal(got[k][keep].view(np.int32), S[k][keep].view(np.int32)), k
    return int(near.sum())


def _scene_views(dims_seed):
    """The real depth pass of a random scene from its camera and two turned copies: (cams [3,40], depth, image, final_T) on the device."""
    from scenes import random_scene
    from gaussianavatar_b200.mesh_render import cameras
    sc = random_scene(P=3000, H=96, W=96, seed=dims_seed, aniso=True)
    cams = cameras([sc["cam"]] * 3)
    for b, ang in ((1, 0.3), (2, -0.25)):                  # rotate the world about the y axis for the other two views
        R = torch.tensor([[np.cos(ang), 0, np.sin(ang), 0], [0, 1, 0, 0], [-np.sin(ang), 0, np.cos(ang), 0], [0, 0, 0, 1]], dtype=torch.float32)
        view = R.t() @ cams[b, :16].reshape(4, 4)
        full = R.t() @ cams[b, 16:32].reshape(4, 4)
        cams[b, :16], cams[b, 16:32] = view.reshape(-1), full.reshape(-1)
    cams = cams.to(DEV)
    plan = RasterBatchPlan(3, 3000, 96, 96, DEV)
    n = lambda t: t.to(DEV).unsqueeze(0).expand(3, *t.shape).contiguous()
    with torch.no_grad():
        img, depth = rasterize_batch_depth(n(sc["means3D"]), n(sc["colors"]), n(sc["scales"]), sc["rotations"].to(DEV),
                                           sc["opacities"].to(DEV), cams, torch.zeros(3, device=DEV), plan)
    assert plan.check(wait=True)
    return cams, depth, img, final_transmittance(plan).clone(), sc


@pytest.mark.parametrize("dims", [(32, 32, 32), (40, 48, 64)])
def test_integrate_matches_oracle_on_sphere_depth(dims):
    H = W = 96
    voxel = 2.0 / (max(dims) - 1)
    origin = np.array([-1.0, -1.1, -0.9], f32)
    cams = me.fusion_cameras([0.0, 0.0, 0.0], 1.8, 11, H).numpy()
    depth, image, final_T = sphere_views(cams, H, W, [0.05, -0.02, 0.03], 0.6, (0.2, 0.6, 0.9))
    g = np.random.default_rng(1)
    image = (image * g.uniform(0.5, 1.0, image.shape)).astype(f32)
    final_T = np.where(final_T == 0, g.uniform(0, 0.5, final_T.shape), final_T).astype(f32)
    vol = me.TsdfVolume(origin, voxel, dims, 4 * voxel)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    vol.integrate(t(depth), t(image), t(final_T), t(cams))
    S = to.integrate(to.new_state(dims), origin, voxel, 4 * voxel, cams, depth, image, final_T)
    near = _compare(vol, S, _near_boundary(cams, H, W, origin, voxel, dims))
    print(f"sphere {dims}: {near} samples within 1e-4 px of a rounding boundary excluded")
    assert _planes(vol)["weight"].sum() > 0 and _planes(vol)["carve"].sum() > 0


@pytest.mark.parametrize("dims", [(32, 32, 32), (40, 48, 64)])
def test_integrate_matches_oracle_on_a_scene_depth_pass(dims):
    cams, depth, img, final_T, sc = _scene_views(5)
    m = sc["means3D"].numpy()
    lo, hi = m.min(0) - 0.05, m.max(0) + 0.05
    voxel = float(np.float32((hi - lo).max() / (max(dims) - 1)))
    origin = lo.astype(f32)
    vol = me.TsdfVolume(origin, voxel, dims, 3 * voxel)
    vol.integrate(depth, img, final_T, cams)
    h = lambda x: x.cpu().numpy()
    S = to.integrate(to.new_state(dims), origin, voxel, 3 * voxel, h(cams), h(depth), h(img), h(final_T))
    near = _compare(vol, S, _near_boundary(h(cams), 96, 96, origin, voxel, dims))
    print(f"scene {dims}: {near} samples within 1e-4 px of a rounding boundary excluded")
    assert _planes(vol)["weight"].sum() > 0 and _planes(vol)["cw"].sum() > 0


def test_views_per_launch_do_not_change_the_grid():
    H = W = 64
    cams = me.fusion_cameras([0.0, 0.0, 0.0], 1.7, 24, H)
    depth, image, final_T = (torch.from_numpy(a).to(DEV) for a in sphere_views(cams.numpy(), H, W, [0, 0, 0], 0.6, (0.3, 0.4, 0.5)))
    cams = cams.to(DEV)
    states = []
    for per in (1, 3, 8):
        vol = me.TsdfVolume([-1, -1, -1], 2 / 39, (40, 40, 40), 8 / 39)
        for s in range(0, 24, per):
            vol.integrate(depth[s:s + per], image[s:s + per], final_T[s:s + per], cams[s:s + per])
        states.append(vol.state.clone())
    assert torch.equal(states[0], states[1]) and torch.equal(states[0], states[2])


def test_mesher_matches_oracle_order_sentinels_and_repeats():
    import ctypes
    from gaussianavatar_b200 import _lib
    cams, depth, img, final_T, sc = _scene_views(2)
    dims, voxel = (40, 48, 64), 0.03
    origin = np.array([-0.7, -1.0, -0.6], f32)
    vol = me.TsdfVolume(origin, voxel, dims, 3 * voxel)
    H = W = 64
    sph = me.fusion_cameras([0.0, -0.3, 0.2], 0.9, 16, H)
    d2, i2, t2 = (torch.from_numpy(a).to(DEV) for a in sphere_views(sph.numpy(), H, W, [0.0, -0.3, 0.2], 0.5, (0.9, 0.1, 0.4)))
    vol.integrate(d2, i2, t2, sph.to(DEV))
    planes = _planes(vol)
    for min_carve in (1, 3):
        V, F, C = vol.mesh(min_carve)
        V2, F2, C2 = vol.mesh(min_carve)
        assert torch.equal(V, V2) and torch.equal(F, F2) and torch.equal(C, C2)
        wv, wf, wc = to.mesh(planes, origin, voxel, min_carve)
        assert np.array_equal(F.cpu().numpy(), wf)
        assert np.allclose(V.cpu().numpy(), wv, rtol=0, atol=1e-6) and np.allclose(C.cpu().numpy(), wc, rtol=0, atol=1e-6)
        assert closed_manifold(wf) and len(wf) > 100
    # sentinels: outputs written exactly up to V and F, guards past them untouched, and smaller capacities respected
    L = _lib.lib()
    d = ctypes.byref(vol.desc)
    ws = torch.empty(L.ga_tsdf_mesh_workspace_bytes(d), dtype=torch.uint8, device=DEV)
    tot = torch.zeros(2, dtype=torch.int32, device=DEV)
    _lib.check(L.ga_tsdf_mesh_count(d, vol.state.data_ptr(), 1, ws.data_ptr(), ws.numel(), tot.data_ptr(), None))
    nV, nF = (int(x) for x in tot.cpu())
    V, F, C = vol.mesh(1)
    for capV, capF in ((nV, nF), (nV // 2, nF // 3)):
        g = 64
        vb = torch.full((nV + g, 3), float("nan"), device=DEV)
        cb = torch.full((nV + g, 3), float("nan"), device=DEV)
        fb = torch.full((nF + g, 3), -7, dtype=torch.int32, device=DEV)
        _lib.check(L.ga_tsdf_mesh_emit(d, vol.state.data_ptr(), 1, ws.data_ptr(), ws.numel(), capV, capF, vb.data_ptr(), cb.data_ptr(),
                                       fb.data_ptr(), None))
        torch.cuda.synchronize()
        assert torch.equal(vb[:capV], V[:capV]) and torch.equal(cb[:capV], C[:capV]) and torch.equal(fb[:capF], F[:capF])
        assert torch.isnan(vb[capV:]).all() and torch.isnan(cb[capV:]).all() and (fb[capF:] == -7).all()


def _shell(n=40000, r=0.5, sigma=0.006, color=(0.8, 0.3, 0.1)):
    d = me.fibonacci_directions(n)
    means = torch.from_numpy(d * r).float()
    return means, torch.full((n, 3), sigma), torch.tensor(color).expand(n, 3).contiguous()


def test_shell_of_opaque_gaussians_end_to_end():
    r, sigma, color = 0.5, 0.006, (0.8, 0.3, 0.1)
    means, scales, colors = _shell(r=r, sigma=sigma, color=color)
    n = means.shape[0]
    fake = types.SimpleNamespace(fix_rotation=torch.tensor([[1.0, 0, 0, 0]], device=DEV).expand(n, 4).contiguous(),
                                 fix_opacity=torch.ones(n, 1, device=DEV))
    M, Sc, Co = (t.to(DEV)[None] for t in (means, scales, colors))
    origin, voxel, dims, trunc = me.fusion_grid(M, Sc, 96, 4)
    vol = me.TsdfVolume(origin, voxel, dims, trunc)
    center = np.asarray(vol.origin) + 0.5 * voxel * (np.asarray(dims) - 1)
    cams = me.fusion_cameras(center, 0.5 * voxel * float(np.linalg.norm(np.asarray(dims) - 1)), 32, 384).to(DEV)
    for s, e, img, depth, fT in me.render_views(fake, M, Sc, Co, cams, 384, 384):
        vol.integrate(depth, img, fT, cams[s:e])
    V, F, C = (t.cpu().numpy() for t in vol.mesh())
    assert closed_manifold(F) and euler(V, F) == 2
    err = np.abs(np.linalg.norm(V.astype(np.float64), axis=1) - r)
    print(f"shell: voxel {voxel:.4g}, max |r - |v|| {err.max():.4g}, mean {err.mean():.4g}")
    assert err.max() < voxel + 3 * sigma
    assert np.abs(C - np.array(color, f32)).max() <= 1 / 255


def _avatar(body, stage=1, N=20000, S=256, inp=32):
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams
    from gaussianavatar_b200.workload import load_poses
    a = syn.make_avatar_assets(N, S, seed=0, body=body)
    pose, transl, _ = load_poses(4)
    if body == "smplx":
        pose = pose[:, :66].contiguous()
    fields = dict(train_stage=2, inp_posmap_size=inp) if stage == 2 else {}
    torch.manual_seed(0)
    m = AvatarModel.from_assets(a, [], pose, transl, batch_size=1, train=False, net_parms=NetworkParams(nf=8), **fields)
    with torch.no_grad():
        sd = m.net.state_dict()
        sd["decoder.conv8N.bias"] = torch.tensor([-5.3])
        m.net.load_state_dict(sd, strict=False)
    mapper = None
    if stage == 2:
        from gaussianavatar_b200.posmap import PoseMapper
        t = syn.make_uv_template(0)
        mapper = PoseMapper(syn.smpl_mesh_model(a.body, t), a.body.betas[0], t, inp, device=DEV)
    rest = syn.synthetic_smplx_poses(1, seed=0)[1].to(DEV) if body == "smplx" else None
    return m, mapper, pose[1].to(DEV), transl[1].to(DEV), rest


def _state(m):
    sd = {("net." + k): v.detach().cpu().clone() for k, v in m.net.state_dict().items()}
    if hasattr(m, "pose_encoder"):
        sd.update({("enc." + k): v.detach().cpu().clone() for k, v in m.pose_encoder.state_dict().items()})
    sd["bn"] = m.net.bn_running.detach().cpu().clone()
    sd["geo"] = m.geo_feature.detach().cpu().clone()
    return sd


@pytest.mark.parametrize("body,stage", [("smpl", 1), ("smplx", 1), ("smpl", 2)])
def test_avatar_mesh_is_closed_and_matches_its_silhouette(body, stage):
    m, mapper, pose, transl, rest = _avatar(body, stage)
    before = _state(m)
    V, F, C = me.extract_mesh(m, pose, transl, rest, res=256, views=64, size=512, pose_mapper=mapper)
    after = _state(m)
    assert before.keys() == after.keys() and all(torch.equal(before[k], after[k]) for k in before)
    Fn = F.cpu().numpy()
    assert closed_manifold(Fn) and len(Fn) > 1000
    assert (C >= -1e-6).all() and (C <= 1 + 1e-6).all()
    with torch.no_grad():
        means, scales, _ = me.posed_gaussians(m, pose, transl, rest, mapper)
    origin, voxel, dims, _ = me.fusion_grid(means, scales, 256, 4)
    center = np.asarray(origin) + 0.5 * voxel * (np.asarray(dims) - 1)
    held_out = me.fusion_cameras(center, 0.5 * voxel * float(np.linalg.norm(np.asarray(dims) - 1)), 8, 512)   # not among the 64
    ious = me.silhouette_iou(m, pose, transl, V, F, held_out, 512, 512, rest, mapper)
    print(f"{body} stage {stage}: IoU {[round(x, 4) for x in ious]} min {min(ious):.4f}, V {V.shape[0]} F {F.shape[0]}")
    assert min(ious) >= IOU_MIN


def test_tool_end_to_end(tmp_path):
    from dataset_fixture import write_synthetic_dataset
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams, OptimizationParams
    mp = write_synthetic_dataset(str(tmp_path), seed=0)
    torch.manual_seed(0)
    m = AvatarModel(mp, NetworkParams(nf=8), OptimizationParams(), train=True)
    m.training_setup()
    with torch.no_grad():
        sd = m.net.state_dict()
        sd["decoder.conv8N.bias"] = torch.tensor([-5.3])
        m.net.load_state_dict(sd, strict=False)
    m.save(7)
    base = [sys.executable, os.path.join(ROOT, "tools", "extract_mesh.py"), "-s", mp.source_path, "-m", mp.model_path, "--project_path",
            mp.project_path, "--smpl_model", os.path.join(mp.smpl_model_path, "SMPL_NEUTRAL.pkl"), "--query_posmap_size",
            str(mp.query_posmap_size), "--inp_posmap_size", str(mp.inp_posmap_size), "--epoch", "7", "--res", "64", "--views", "16",
            "--size", "128"]
    out = tmp_path / "meshes"
    r = subprocess.run(base + ["--frame", "0", "--frame", "2", "--iou", "--out", str(out)], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    recs = [json.loads(line) for line in r.stdout.splitlines() if line.startswith("{")]
    assert [os.path.basename(x["mesh"]) for x in recs] == ["frame_00000.ply", "frame_00002.ply"]
    assert all(0.0 <= x["iou"] <= 1.0 for x in recs)
    print("tool IoU", [x["iou"] for x in recs])
    for x in recs:
        v, f, c = read_ply(x["mesh"])
        assert len(f) == x["faces"] > 0 and closed_manifold(f)
    clip = os.path.join(mp.test_folder, "smpl_parms.pth")
    out2 = tmp_path / "clip"
    r = subprocess.run(base + ["--motion", clip, "--clip_fps", "30", "--fps", "15", "--align_to", "1", "--format", "obj", "--out", str(out2)],
                       capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    names = sorted(os.listdir(out2))
    assert names and names == ["{:05d}.obj".format(i) for i in range(len(names))]
    from test_mesh_extract_cpu import read_obj
    v, f, c = read_obj(out2 / names[0])
    assert len(f) > 0 and closed_manifold(f)
