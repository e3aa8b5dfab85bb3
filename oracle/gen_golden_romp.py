"""ORACLE — TEST INFRASTRUCTURE ONLY.  Generates tests/golden/romp_split.npz by running the reference's own capture-to-folder code
(/root/reference/scripts/sample_romp2gsavatar.py, read-only, never copied) on synthetic captures.  Run in the build container only:

    python oracle/gen_golden_romp.py

That script runs on import (hard-coded paths, copies), so its `load_smpl_param` and the statements of its non-snap split branch
are lifted out of its syntax tree with `ast` and executed against a synthetic capture directory.  Per case (frame count, pose keys
`thetas` or `global_orient` + `body_pose`, betas [1,10] or [10]) the fixture holds the input poses, the image names, the train /
test image names and both smpl_parms.pth dictionaries (beta, body_pose, trans).
"""
import ast
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = "/root/reference/scripts/sample_romp2gsavatar.py"
OUT = os.path.join(ROOT, "tests", "golden", "romp_split.npz")

# (name, frames, pose keys, betas shape)
CASES = [("n7_split", 7, "split", (1, 10)), ("n10_thetas", 10, "thetas", (1, 10)), ("n23_split", 23, "split", (10,)),
         ("n23_thetas", 23, "thetas", (10,)), ("n100_thetas", 100, "thetas", (1, 10))]


def reference_parts():
    """(load_smpl_param, the code of the non-snap split branch) from the reference script's syntax tree."""
    tree = ast.parse(open(SCRIPT).read())
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "load_smpl_param")
    branch = next(n for n in tree.body if isinstance(n, ast.If) and isinstance(n.test, ast.Name) and n.test.id == "snap")
    ns = {"np": np, "torch": torch}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), SCRIPT, "exec"), ns)
    return ns["load_smpl_param"], compile(ast.Module(body=branch.orelse, type_ignores=[]), SCRIPT, "exec")


def poses_for(n, keys, beta_shape, seed):
    g = np.random.default_rng(seed)
    th = (g.normal(0, 0.2, (n, 72))).astype(np.float32)
    p = dict(betas=g.normal(0, 0.5, beta_shape).astype(np.float32), transl=g.normal(0, 0.3, (n, 3)).astype(np.float32))
    if keys == "thetas":
        p["thetas"] = th
    else:
        p["global_orient"], p["body_pose"] = th[:, :3].copy(), th[:, 3:].copy()
    return p


def main():
    load_smpl_param, split_code = reference_parts()
    out = {}
    for k, (name, n, keys, beta_shape) in enumerate(CASES):
        poses = poses_for(n, keys, beta_shape, seed=100 + k)
        names = [f"{i:06d}.png" for i in range(n)]
        with tempfile.TemporaryDirectory() as d:
            os.makedirs(os.path.join(d, "images"))
            for x in names:
                open(os.path.join(d, "images", x), "wb").close()
            ns = {"os": os, "all_image_path": os.path.join(d, "images"), "print": lambda *a, **kw: None}
            exec(split_code, ns)
            path = os.path.join(d, "poses.npz")
            np.savez(path, **poses)
            train = load_smpl_param(path, ns["train_list"])
            test = load_smpl_param(path, ns["test_list"])
        for key, v in poses.items():
            out[f"{name}/poses/{key}"] = v
        out[f"{name}/names"] = np.array(names)
        out[f"{name}/train_names"] = np.array(ns["train_split_name"], dtype="<U16").reshape(-1)
        out[f"{name}/test_names"] = np.array(ns["test_split_name"], dtype="<U16").reshape(-1)
        for part, prm in (("train", train), ("test", test)):
            for key in ("beta", "body_pose", "trans"):
                out[f"{name}/{part}/{key}"] = prm[key].numpy()
    np.savez_compressed(OUT, **out)
    print(OUT, len(out), "arrays")


if __name__ == "__main__":
    sys.exit(main())
