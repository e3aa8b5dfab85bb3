"""CPU: the animation player's oracle (sampler against scipy's Rotation / Slerp in fp64, packer against torchvision's save_image
PNG bytes), the clip loader, the time and alignment rules, and the C ABI's argument checks (which run before any launch)."""
import io
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import animate_oracle as ao  # noqa: E402
from gaussianavatar_b200 import animate as an  # noqa: E402

Rotation = pytest.importorskip("scipy.spatial.transform").Rotation
Slerp = pytest.importorskip("scipy.spatial.transform").Slerp


def _random_clip(T, J, seed, near_pi=False, antipodal=False):
    g = np.random.default_rng(seed)
    aa = Rotation.random(T * J, random_state=seed).as_rotvec().reshape(T, J, 3)
    if near_pi:        # angles within 1e-6 of pi, and exactly pi
        ax = g.normal(size=(T, J, 3))
        ax /= np.linalg.norm(ax, axis=-1, keepdims=True)
        ang = np.pi - g.uniform(0, 1e-6, size=(T, J, 1))
        ang[0, :3] = np.pi
        aa = ax * ang
    if antipodal:      # key i+1 = the same rotation as key i written the long way round (angle 2 pi - a about -axis)
        th = np.linalg.norm(aa[0], axis=-1, keepdims=True)
        aa[1] = -aa[0] / th * (2 * np.pi - th)
    aa = aa.astype(np.float32).astype(np.float64)
    trans = g.normal(0, 1, size=(T, 3)).astype(np.float32).astype(np.float64)
    return aa.reshape(T, J * 3), trans


def _scipy_sample(pose, trans, times, align):
    T = pose.shape[0]
    J = pose.shape[1] // 3
    tau = np.clip(times, 0, T - 1)
    out = np.zeros((len(times), J, 3, 3))
    Ra = Rotation.from_matrix(align[:9].reshape(3, 3))
    for j in range(J):
        rots = Rotation.from_rotvec(pose[:, 3 * j:3 * j + 3])
        if T == 1:
            r = Rotation.from_rotvec(np.repeat(pose[:, 3 * j:3 * j + 3], len(times), 0))
        else:
            r = Slerp(np.arange(T), rots)(tau)
        if j == 0:
            r = Ra * r
        out[:, j] = r.as_matrix()
    i0 = np.minimum(np.floor(tau).astype(int), T - 1)
    i1 = np.minimum(i0 + 1, T - 1)
    f = tau - i0
    v = trans[i0] + f[:, None] * (trans[i1] - trans[i0])
    return out, v @ align[:9].reshape(3, 3).T + align[9:]


def _mats(pose):
    n, w = pose.shape
    return Rotation.from_rotvec(pose.reshape(-1, 3)).as_matrix().reshape(n, w // 3, 3, 3)


@pytest.mark.parametrize("J", [24, 55])
@pytest.mark.parametrize("kind", ["random", "near_pi", "antipodal"])
def test_sampler_oracle_matches_scipy(J, kind):
    T = 6
    pose, trans = _random_clip(T, J, seed=J + len(kind), near_pi=kind == "near_pi", antipodal=kind == "antipodal")
    times = np.array([0.0, 0.25, 0.5, 1.0, 1.999999, 2.0, 3.7, T - 1.0, -3.0, T + 4.5, 0.1 + 1e-9])
    align = np.concatenate([Rotation.random(random_state=J).as_matrix().reshape(9), [0.3, -1.0, 2.0]])
    got_p, got_t = ao.motion_sample(pose, trans, times, align)
    want_R, want_t = _scipy_sample(pose, trans, times, align)
    assert np.abs(_mats(got_p) - want_R).max() < 1e-12
    assert np.abs(got_t - want_t).max() < 1e-12
    ang = np.linalg.norm(got_p.reshape(len(times), J, 3), axis=-1)
    assert (ang <= np.pi + 1e-12).all()


def test_sampler_single_key_and_integer_times():
    pose, trans = _random_clip(1, 24, seed=3)
    p, t = ao.motion_sample(pose, trans, np.array([0.0, 0.5, 7.0, -1.0]), an.IDENTITY_ALIGN)
    for k in range(4):
        assert np.abs(_mats(p[k:k + 1]) - _mats(pose)).max() < 1e-12
        assert np.array_equal(t[k], trans[0])
    pose, trans = _random_clip(5, 24, seed=4)
    p, t = ao.motion_sample(pose, trans, np.arange(5.0), an.IDENTITY_ALIGN)
    assert np.abs(_mats(p) - _mats(pose)).max() < 1e-12 and np.array_equal(t, trans)


def test_alignment_known_answers():
    g = np.random.default_rng(0)
    pose, trans = _random_clip(7, 24, seed=5)
    target_root, target_t = Rotation.random(random_state=9).as_rotvec(), g.normal(size=3)
    align = an.alignment(pose[0, :3], trans[0], target_root, target_t)
    p, t = ao.motion_sample(pose, trans, np.arange(7.0), align)
    assert np.abs(Rotation.from_rotvec(p[0, :3]).as_matrix() - Rotation.from_rotvec(target_root).as_matrix()).max() < 1e-12
    assert np.abs(t[0] - target_t).max() < 1e-12
    Ra = align[:9].reshape(3, 3)
    assert np.abs(Ra @ Ra.T - np.eye(3)).max() < 1e-12 and abs(np.linalg.det(Ra) - 1) < 1e-12
    # frame differences rotate rigidly: translations and relative root rotations
    assert np.abs((t - t[0]) - (trans - trans[0]) @ Ra.T).max() < 1e-12
    R0, Rc = Rotation.from_rotvec(pose[0, :3]).as_matrix(), Rotation.from_rotvec(pose[:, :3]).as_matrix()
    R = Rotation.from_rotvec(p[:, :3]).as_matrix()
    assert np.abs(R @ np.swapaxes(R[:1], 1, 2) - Ra @ Rc @ R0.T @ Ra.T).max() < 1e-12
    # other joints are not moved by the alignment
    assert np.abs(_mats(p)[:, 1:] - _mats(pose)[:, 1:]).max() < 1e-12


def test_sample_times_rule():
    assert np.array_equal(an.sample_times(10, 30, 30), np.arange(10.0))
    assert np.array_equal(an.sample_times(10, 120, 30), [0.0, 4.0, 8.0])
    t = an.sample_times(11, 30, 60, speed=0.5)
    assert len(t) == 41 and t[-1] == 10.0
    t = an.sample_times(4, 25, 30, speed=1.5)
    assert len(t) == int(np.floor(3 * 30 / (1.5 * 25))) + 1 and np.allclose(np.diff(t), 1.25)
    assert len(an.sample_times(1, 30, 60)) == 1
    with pytest.raises(ValueError, match="positive"):
        an.sample_times(5, 30, 0)


def _save_npz(path, **arrays):
    np.savez(path, **arrays)
    return str(path)


def test_motion_clip_formats(tmp_path):
    g = np.random.default_rng(1)
    T = 5
    h = g.normal(size=(T, 156))
    x = g.normal(size=(T, 165))
    tr = g.normal(size=(T, 3))
    smplh = _save_npz(tmp_path / "h.npz", poses=h, trans=tr, mocap_framerate=120.0, betas=np.zeros(16))
    smplx = _save_npz(tmp_path / "x.npz", poses=x, trans=tr, mocap_frame_rate=60.0)
    smplx_old = _save_npz(tmp_path / "x2.npz", poses=x, trans=tr, mocap_framerate=50.0)
    c = an.MotionClip.load(smplh, "smpl")
    assert c.fps == 120.0 and c.pose.shape == (T, 72) and c.pose.dtype == torch.float32
    assert np.array_equal(c.pose[:, :66].numpy(), h[:, :66].astype(np.float32)) and (c.pose[:, 66:] == 0).all()
    assert np.array_equal(c.trans.numpy(), tr.astype(np.float32))
    c = an.MotionClip.load(smplh, "smplx")
    assert c.pose.shape == (T, 165) and (c.pose[:, 66:75] == 0).all()
    assert np.array_equal(c.pose[:, 75:].numpy(), h[:, 66:].astype(np.float32))
    assert np.array_equal(c.pose[:, :66].numpy(), h[:, :66].astype(np.float32))
    c = an.MotionClip.load(smplx, "smplx")
    assert c.fps == 60.0 and np.array_equal(c.pose.numpy(), x.astype(np.float32))
    c = an.MotionClip.load(smplx, "smpl")
    assert c.pose.shape == (T, 72) and np.array_equal(c.pose[:, :66].numpy(), x[:, :66].astype(np.float32)) and (c.pose[:, 66:] == 0).all()
    assert an.MotionClip.load(smplx_old, "smplx").fps == 50.0
    assert an.MotionClip.load(smplx_old, "smplx", fps=24).fps == 24.0
    for body, w in (("smpl", 72), ("smplx", 165)):
        p = tmp_path / f"{body}.pth"
        bp = torch.randn(T, w)
        torch.save(dict(beta=torch.zeros(1, 10), body_pose=bp, trans=torch.from_numpy(tr)), p)
        c = an.MotionClip.load(p, body, fps=30)
        assert c.fps == 30.0 and torch.equal(c.pose, bp) and c.body == body
        with pytest.raises(ValueError, match="fps"):
            an.MotionClip.load(p, body)
        with pytest.raises(ValueError, match="body_pose"):
            an.MotionClip.load(p, "smplx" if body == "smpl" else "smpl", fps=30)


def test_motion_clip_errors(tmp_path):
    g = np.random.default_rng(2)
    tr = g.normal(size=(4, 3))
    with pytest.raises(ValueError, match="poses"):
        an.MotionClip.load(_save_npz(tmp_path / "a.npz", trans=tr, mocap_framerate=30.0), "smpl")
    with pytest.raises(ValueError, match="trans"):
        an.MotionClip.load(_save_npz(tmp_path / "b.npz", poses=g.normal(size=(4, 156)), mocap_framerate=30.0), "smpl")
    with pytest.raises(ValueError, match="poses"):
        an.MotionClip.load(_save_npz(tmp_path / "c.npz", poses=g.normal(size=(4, 72)), trans=tr, mocap_framerate=30.0), "smpl")
    with pytest.raises(ValueError, match="mocap_framerate"):
        an.MotionClip.load(_save_npz(tmp_path / "d.npz", poses=g.normal(size=(4, 156)), trans=tr), "smpl")
    with pytest.raises(ValueError, match="mocap_frame_rate"):
        an.MotionClip.load(_save_npz(tmp_path / "e.npz", poses=g.normal(size=(4, 165)), trans=tr), "smplx")
    with pytest.raises(ValueError, match="trans"):
        an.MotionClip.load(_save_npz(tmp_path / "f.npz", poses=g.normal(size=(4, 156)), trans=tr[:3], mocap_framerate=30.0), "smpl")
    with pytest.raises(ValueError, match="body"):
        an.MotionClip.load(_save_npz(tmp_path / "g.npz", poses=g.normal(size=(4, 156)), trans=tr, mocap_framerate=30.0), "mano")
    p = tmp_path / "noTrans.pth"
    torch.save(dict(body_pose=torch.zeros(4, 72)), p)
    with pytest.raises(ValueError, match="trans"):
        an.MotionClip.load(p, "smpl", fps=30)


def _boundary_values():
    k = np.arange(256, dtype=np.float64)
    centre = ((k - 0.5) / 255.0).astype(np.float32)          # x at which x * 255 + 0.5 lands on an integer
    vals = [centre, np.nextafter(centre, np.float32(np.inf)), np.nextafter(centre, np.float32(-np.inf)),
            (k / 255.0).astype(np.float32), np.nextafter((k / 255.0).astype(np.float32), np.float32(2)),
            np.nextafter((k / 255.0).astype(np.float32), np.float32(-2)),
            np.array([-1.0, -1e-8, -0.0, 0.0, 1.0, 1.0 + 1e-7, 2.0, 300.0, np.inf, -np.inf, np.nan], np.float32)]
    return np.concatenate(vals).astype(np.float32)


def test_packer_oracle_matches_save_image():
    from PIL import Image
    from torchvision.utils import save_image
    v = _boundary_values()
    g = np.random.default_rng(0)
    v = np.concatenate([v, g.uniform(-0.1, 1.1, size=3 * 40 * 40 - v.size % (3 * 40 * 40)).astype(np.float32)])
    n = v.size // 3 // 40 * 3 * 40
    img = v[:n].reshape(1, 3, -1, 40)
    buf = io.BytesIO()
    save_image(torch.from_numpy(img[0].copy()), buf, format="png")
    want = np.array(Image.open(io.BytesIO(buf.getvalue())).convert("RGB"))
    got = ao.frame_pack(img, channels=3)[0]
    finite = np.isfinite(img[0]).all(0)
    assert np.array_equal(got[finite], want[finite])
    assert (got[~np.isfinite(img[0]).transpose(1, 2, 0) & np.isnan(img[0]).transpose(1, 2, 0)] == 0).all()


def test_packer_oracle_rgba_known_answers():
    bg = np.array([1.0, 1.0, 1.0], np.float32)
    C = np.array([0.2, 0.5, 0.0], np.float32)
    for T in (np.float32(0.0), np.float32(0.25), np.float32(1.0), np.float32(0.999)):
        x = (C * (1 - T) + T * bg).astype(np.float32).reshape(1, 3, 1, 1)
        out = ao.frame_pack(x, np.full((1, 1, 1), T, np.float32), bg, channels=4)[0, 0, 0]
        A = ao.quant8(np.float32(1) - T)
        assert out[3] == A
        if A == 0:
            assert (out == 0).all()
        else:
            assert np.abs(out[:3].astype(int) - ao.quant8(C).astype(int)).max() <= 1


def test_cabi_rejects_bad_arguments():
    from gaussianavatar_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    L = _lib.lib()
    fake = 256         # never dereferenced: every call below must fail its checks before any launch
    bad_sample = [(0, 24, 1), (2, 23, 1), (2, 56, 1), (2, 24, 0), (2, 24, -1)]
    for T, J, n in bad_sample:
        assert L.ga_motion_sample(T, J, fake, fake, n, fake, fake, fake, fake, None) != 0
    assert L.ga_motion_sample(2, 24, fake, None, 1, fake, fake, fake, fake, None) != 0
    assert L.ga_motion_sample(2, 55, fake, fake, 1, fake, None, fake, fake, None) != 0
    assert b"joints" in L.ga_last_error() or b"NULL" in L.ga_last_error()
    for B, H, W, C in [(0, 4, 4, 3), (9, 4, 4, 3), (1, 0, 4, 3), (1, 4, 16385, 3), (1, 4, 4, 2), (1, 4, 4, 5)]:
        assert L.ga_frame_pack(B, H, W, C, fake, fake, fake, fake, None) != 0
    assert L.ga_frame_pack(1, 4, 4, 4, fake, None, fake, fake, None) != 0      # RGBA needs final_T
    assert L.ga_frame_pack(1, 4, 4, 4, fake, fake, None, fake, None) != 0      # ... and the background
    assert L.ga_frame_pack(1, 4, 4, 3, None, None, None, fake, None) != 0
    assert L.ga_frame_pack(1, 4, 4, 4, fake, fake, fake, fake + 1, None) != 0  # RGBA rows are written as 4-byte words
    assert L.ga_version() >= 106
