"""numpy restatement of ga_skin_weights (csrc/skin.cu; the rule is in include/gavatar.h).

The squared distance is the kernel's fp32 expression ((dx dx + dy dy) + dz dz) with every operation rounded to fp32, so the
neighbour sets agree bit for bit; the blend, the selection and the renormalisation are the kernel's fp64 operations in its order.
"""
from __future__ import annotations

import numpy as np

EPS2 = 1e-6          # eps^2, eps = 1e-3 world units


def dist2(verts, means) -> np.ndarray:
    """[V,N] fp32 squared distances, d = mean - vertex."""
    v, m = np.asarray(verts, np.float32), np.asarray(means, np.float32)
    dx, dy, dz = (m[None, :, a] - v[:, None, a] for a in range(3))
    return (dx * dx + dy * dy) + dz * dz


def nearest(verts, means, k: int):
    """(indices [V,k] int64, d2 [V,k] fp32) of the k nearest means, ascending by distance, equal distances to the lower index."""
    d2 = dist2(verts, means)
    idx = np.argsort(d2, axis=1, kind="stable")[:, :k]
    return idx, np.take_along_axis(d2, idx, 1)


def skin_weights(verts, means, lbs, J: int, k: int, K: int):
    """(joints [V,K] uint8, weights [V,K] fp32) of ga_skin_weights; lbs [N,ld] with J <= ld."""
    lbs = np.asarray(lbs, np.float32)
    idx, d2 = nearest(verts, means, k)
    V = idx.shape[0]
    c = 1.0 / (d2.astype(np.float64) + EPS2)
    den = np.zeros(V)
    num = np.zeros((V, J))
    for i in range(k):                                  # neighbour order, as the kernel sums
        den = den + c[:, i]
        num = num + c[:, i:i + 1] * lbs[idx[:, i], :J].astype(np.float64)
    w = num / den[:, None]
    order = np.argsort(-w, axis=1, kind="stable")[:, :K]  # heaviest first, equal weights to the lower joint
    sw = np.take_along_axis(w, order, 1)
    keep = sw > 0
    sw = np.where(keep, sw, 0.0)
    sj = np.where(keep, order, 0)
    total = np.zeros(V)
    for s in range(K):
        total = total + sw[:, s]
    joints = sj.astype(np.uint8)
    weights = np.zeros((V, K), np.float32)
    ok = total > 0
    weights[ok] = (sw[ok] / total[ok, None]).astype(np.float32)
    weights[~ok, 0] = 1.0
    return joints, weights
