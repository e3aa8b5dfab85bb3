"""Seeded static Gaussian scenes, and 3DGS's point_cloud.ply / cameras.json written with numpy (test helper, not product)."""
import json

import numpy as np
import torch


def random_static(Ps, degree, seed=0, center=(0.0, -0.2, 0.0), spread=(1.2, 1.4, 1.0), scale_mean=0.03, opacity=(0.1, 0.95)):
    """Raw (pre-activation, as 3DGS stores them) parameters of Ps anisotropic Gaussians: xyz, f_dc [Ps,3], f_rest [Ps,3,M-1]
    (channel-major), opacity logits, log scales, unnormalised quaternions (w first)."""
    g = np.random.default_rng(seed)
    M = (degree + 1) ** 2
    xyz = (g.random((Ps, 3)) - 0.5) * 2 * np.asarray(spread) + np.asarray(center)
    o = g.uniform(*opacity, size=Ps)
    rot = g.normal(size=(Ps, 4))
    rot *= g.uniform(0.5, 2.0, size=(Ps, 1))
    return dict(xyz=xyz.astype(np.float32), f_dc=g.normal(0.0, 0.5, size=(Ps, 3)).astype(np.float32),
                f_rest=g.normal(0.0, 0.2, size=(Ps, 3, M - 1)).astype(np.float32),
                opacity=np.log(o / (1 - o)).astype(np.float32),
                scale=np.log(scale_mean * np.exp(0.5 * g.normal(size=(Ps, 3)))).astype(np.float32), rot=rot.astype(np.float32),
                degree=degree)


def activated(raw):
    """The GaussianScene fields of raw parameters (fp64 activations rounded to fp32)."""
    P, M = raw["xyz"].shape[0], (raw["degree"] + 1) ** 2
    shs = np.zeros((P, M, 3), np.float64)
    shs[:, 0] = raw["f_dc"]
    shs[:, 1:] = raw["f_rest"].astype(np.float64).transpose(0, 2, 1)
    rot = raw["rot"].astype(np.float64)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32))
    return dict(means3D=t(raw["xyz"]), scales=t(np.exp(raw["scale"].astype(np.float64))),
                rotations=t(rot / np.linalg.norm(rot, axis=1, keepdims=True)),
                opacities=t(1 / (1 + np.exp(-raw["opacity"].astype(np.float64)))), shs=t(shs), sh_degree=raw["degree"])


def scene_of(raw):
    from gaussianavatar_b200.scene import GaussianScene
    return GaussianScene(**activated(raw))


def write_ply(path, raw, shuffle_seed=None, extra=True, fmt="binary_little_endian", drop=None, n_rest=None):
    """3DGS's save_ply layout (x y z nx ny nz f_dc_* f_rest_* opacity scale_* rot_*, float32), optionally with the properties in a
    shuffled order, an extra property, a property dropped, or n_rest f_rest columns instead of all."""
    P = raw["xyz"].shape[0]
    rest = raw["f_rest"].reshape(P, -1)
    cols = [("x", raw["xyz"][:, 0]), ("y", raw["xyz"][:, 1]), ("z", raw["xyz"][:, 2])]
    cols += [(n, np.zeros(P, np.float32)) for n in ("nx", "ny", "nz")]
    cols += [(f"f_dc_{i}", raw["f_dc"][:, i]) for i in range(3)]
    k = rest.shape[1] if n_rest is None else n_rest
    cols += [(f"f_rest_{i}", rest[:, i] if i < rest.shape[1] else np.zeros(P, np.float32)) for i in range(k)]
    cols += [("opacity", raw["opacity"])]
    cols += [(f"scale_{i}", raw["scale"][:, i]) for i in range(3)]
    cols += [(f"rot_{i}", raw["rot"][:, i]) for i in range(4)]
    if extra:
        cols.append(("semantic_id", np.arange(P, dtype=np.float32)))
    if drop:
        cols = [c for c in cols if c[0] != drop]
    if shuffle_seed is not None:
        order = np.random.default_rng(shuffle_seed).permutation(len(cols))
        cols = [cols[i] for i in order]
    end = ">" if fmt == "binary_big_endian" else "<"
    arr = np.empty(P, dtype=[(n, end + "f4") for n, _ in cols])
    for n, v in cols:
        arr[n] = v
    head = "ply\nformat {} 1.0\nelement vertex {}\n{}end_header\n".format(fmt, P, "".join(f"property float {n}\n" for n, _ in cols))
    with open(path, "wb") as f:
        f.write(head.encode("ascii"))
        if fmt == "ascii":
            f.write("\n".join(" ".join(repr(float(x)) for x in row) for row in arr.tolist()).encode("ascii"))
        else:
            f.write(arr.tobytes())


def write_cameras_json(path, cams):
    """cams: (K [3,3], E [4,4] world->camera, width, height) -> 3DGS's cameras.json (position = centre, rotation = camera->world)."""
    out = []
    for i, (K, E, w, h) in enumerate(cams):
        E = np.asarray(E, np.float64)
        C2W = np.linalg.inv(E)
        out.append(dict(id=i, img_name=f"{i:05d}", width=int(w), height=int(h), position=C2W[:3, 3].tolist(),
                        rotation=C2W[:3, :3].tolist(), fy=float(K[1][1]), fx=float(K[0][0])))
    with open(path, "w") as f:
        json.dump(out, f)
