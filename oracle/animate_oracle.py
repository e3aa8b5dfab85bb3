"""numpy restatement of the animation player's two kernels (csrc/animate.cu).

motion_sample: the clip sampler in fp64 (tau clamp, per-joint quaternion slerp on the shortest path, normalised lerp above a dot of
1 - 1e-12, root alignment, axis-angle with w >= 0); returns fp64 so tests can compare the kernel's fp32 against it.
frame_pack: the byte packer in single float32 operations, in the kernel's order, so its bytes are exact.
"""
from __future__ import annotations

import numpy as np

NLERP_DOT = 1.0 - 1e-12


def quat_from_aa(v):
    """[..., 3] axis-angle -> [..., 4] unit quaternion (w, x, y, z)."""
    v = np.asarray(v, np.float64)
    th = np.linalg.norm(v, axis=-1)
    h = 0.5 * th
    with np.errstate(invalid="ignore", divide="ignore"):
        s = np.where(th > 1e-8, np.sin(h) / np.where(th > 0, th, 1.0), 0.5 - th * th / 48.0)
    return np.concatenate([np.cos(h)[..., None], s[..., None] * v], -1)


def quat_from_mat(R):
    """Shepperd's method on one 3x3 rotation (the kernel's branch order)."""
    R = np.asarray(R, np.float64).reshape(9)
    tr = R[0] + R[4] + R[8]
    if tr >= R[0] and tr >= R[4] and tr >= R[8]:
        s = 2.0 * np.sqrt(1.0 + tr)
        q = [0.25 * s, (R[7] - R[5]) / s, (R[2] - R[6]) / s, (R[3] - R[1]) / s]
    elif R[0] >= R[4] and R[0] >= R[8]:
        s = 2.0 * np.sqrt(1.0 + R[0] - R[4] - R[8])
        q = [(R[7] - R[5]) / s, 0.25 * s, (R[1] + R[3]) / s, (R[2] + R[6]) / s]
    elif R[4] >= R[8]:
        s = 2.0 * np.sqrt(1.0 + R[4] - R[0] - R[8])
        q = [(R[2] - R[6]) / s, (R[1] + R[3]) / s, 0.25 * s, (R[5] + R[7]) / s]
    else:
        s = 2.0 * np.sqrt(1.0 + R[8] - R[0] - R[4])
        q = [(R[3] - R[1]) / s, (R[2] + R[6]) / s, (R[5] + R[7]) / s, 0.25 * s]
    q = np.asarray(q)
    return q / np.linalg.norm(q)


def quat_mul(a, b):
    aw, ax, ay, az = np.moveaxis(a, -1, 0)
    bw, bx, by, bz = np.moveaxis(b, -1, 0)
    return np.stack([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                     aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw], -1)


def slerp(a, b, f):
    """a, b [..., 4] unit quaternions, f [...] -> [..., 4]."""
    d = np.sum(a * b, -1)
    b = np.where((d < 0)[..., None], -b, b)
    d = np.abs(d)
    f = np.broadcast_to(np.asarray(f, np.float64), d.shape)
    near = d > NLERP_DOT
    om = np.arccos(np.clip(np.where(near, 0.0, d), -1.0, 1.0))
    so = np.where(near, 1.0, np.sin(om))
    ca = np.where(near, 1.0 - f, np.sin((1.0 - f) * om) / so)
    cb = np.where(near, f, np.sin(f * om) / so)
    q = ca[..., None] * a + cb[..., None] * b
    return q / np.linalg.norm(q, axis=-1, keepdims=True)


def quat_to_aa(q):
    q = np.where((q[..., :1] < 0), -q, q)
    s = np.linalg.norm(q[..., 1:], axis=-1)
    with np.errstate(invalid="ignore", divide="ignore"):
        g = np.where(s > 0, 2.0 * np.arctan2(s, q[..., 0]) / np.where(s > 0, s, 1.0), 0.0)
    return g[..., None] * q[..., 1:]


def motion_sample(key_pose, key_trans, times, align):
    """key_pose [T,J*3], key_trans [T,3] (the kernel reads them as fp32), times [n], align [12] -> (pose [n,J*3], trans [n,3]) fp64."""
    kp = np.asarray(key_pose, np.float32).astype(np.float64)
    kt = np.asarray(key_trans, np.float32).astype(np.float64)
    T = kp.shape[0]
    J = kp.shape[1] // 3
    align = np.asarray(align, np.float64).reshape(12)
    tau = np.clip(np.nan_to_num(np.asarray(times, np.float64), nan=0.0), 0.0, T - 1)
    i0 = np.minimum(np.floor(tau).astype(np.int64), T - 1)
    i1 = np.minimum(i0 + 1, T - 1)
    f = tau - i0
    q0 = quat_from_aa(kp[i0].reshape(-1, J, 3))
    q1 = quat_from_aa(kp[i1].reshape(-1, J, 3))
    q = slerp(q0, q1, np.repeat(f[:, None], J, 1))
    R = align[:9].reshape(3, 3)
    q[:, 0] = quat_mul(np.broadcast_to(quat_from_mat(R), q[:, 0].shape), q[:, 0])
    pose = quat_to_aa(q).reshape(-1, J * 3)
    v = kt[i0] + f[:, None] * (kt[i1] - kt[i0])
    trans = v @ R.T + align[9:]
    return pose, trans


def quant8(x):
    """save_image's mul(255).add_(0.5).clamp_(0, 255).to(uint8) in float32, NaN -> 0."""
    x = np.asarray(x, np.float32)
    y = (x * np.float32(255.0)).astype(np.float32)
    y = (y + np.float32(0.5)).astype(np.float32)
    with np.errstate(invalid="ignore"):
        y = np.where(np.isnan(y), np.float32(0), np.clip(y, np.float32(0), np.float32(255)))
    return y.astype(np.uint8)


def frame_pack(image, final_T=None, bg=None, channels=3):
    """image [B,3,H,W] fp32 (C + T bg), final_T [B,H,W], bg [3] -> uint8 [B,H,W,channels]."""
    img = np.asarray(image, np.float32)
    if channels == 3:
        return np.ascontiguousarray(quant8(img).transpose(0, 2, 3, 1))
    Tr = np.asarray(final_T, np.float32)
    bg = np.asarray(bg, np.float32).reshape(3)
    a = (np.float32(1.0) - Tr).astype(np.float32)
    A = quant8(a)
    out = np.zeros(img.shape[:1] + img.shape[2:] + (4,), np.uint8)
    with np.errstate(divide="ignore", invalid="ignore"):
        for c in range(3):
            num = (img[:, c] - (Tr * bg[c]).astype(np.float32)).astype(np.float32)
            out[..., c] = quant8((num / a).astype(np.float32))
    out[..., 3] = A
    out[A == 0] = 0
    return out
