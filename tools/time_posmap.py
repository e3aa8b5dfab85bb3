"""Cost of the device position maps (csrc/posmap.cu).  Run on the GPU box:
    python tools/time_posmap.py > posmap.json
  1. `ga_smpl_vertices` at B = 2 and 8 against its byte floor: posedirs (207 x 20670 fp32, 17.1 MB) read once per call, which is
     5.1 us at the H100 SXM data sheet's 3.35 TB/s (computed from bytes, not measured);
  2. `ga_posmap_fill` at S = 128 and 512 (B = 2), and the one-off `ga_posmap_layout` at S = 512, on the synthetic UV template
     (13416 faces; SMPL's has 13776);
  3. a stage-2 training step with maps built on the device (ModelParams.inp_posmap_from_pose) against the same step with the maps
     read from inp_map/ files (written by tools/pose_maps.py, already in device memory as part of the batch), alternating block by
     block: at the test sizes (700 Gaussians, 48^2 UV, 32^2 input maps, 64^2 frames) and at 200k Gaussians (512^2 UV, 128^2 input
     maps, 1024^2 frames).  B = 2 frames per step.
Kernel times are CUDA events around many back-to-back launches; the card's name, power limit and max SM clock are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from gaussianavatar_b200 import _lib, synthetic as syn  # noqa: E402
from gaussianavatar_b200._lib import ptr  # noqa: E402
from gaussianavatar_b200.posmap import PoseMapper  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return dict(gpu=torch.cuda.get_device_name(0), nvidia_smi=q)


def time_us(fn, iters, rounds=5):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b) * 1e3 / iters)
    return statistics.median(out), out


def kernels(res):
    s = torch.cuda.current_stream().cuda_stream
    L = _lib.lib()
    t = syn.make_uv_template(0)
    body = syn.make_body(0)
    model = syn.smpl_mesh_model(body, t)
    m = PoseMapper(model, body.betas[0], t, 512)
    V = m.V
    floor_us = 207 * 3 * V * 4 / HBM_BYTES_PER_S * 1e6
    for B in (2, 8):
        pose, transl = syn.synthetic_poses(B, seed=1)
        pose, transl = pose.cuda(), transl.cuda()
        out = torch.empty(B, V, 3, device="cuda")
        med, rounds = time_us(lambda: _lib.check(L.ga_smpl_vertices(B, V, ptr(pose), ptr(transl), ptr(m.rest_joints), ptr(m.v_shaped),
                                                                   ptr(m.posedirs), ptr(m.weights), ptr(out), s)), 500)
        nbytes = 207 * 3 * V * 4 + V * 24 * 4 + V * 12 + B * V * 12
        res[f"smpl_vertices_B{B}"] = dict(us=med, rounds_us=rounds, posedirs_floor_us=floor_us, all_bytes=nbytes,
                                          tb_per_s=nbytes / (med * 1e-6) / 1e12)
    corners = torch.from_numpy(t[2].astype("float32")[t[3]]).cuda().contiguous()
    for S in (128, 512):
        mm = m if S == 512 else PoseMapper(model, body.betas[0], t, S)
        verts = mm.vertices(*syn.synthetic_poses(2, seed=1))
        out = torch.empty(2, 3, S, S, device="cuda")
        med, rounds = time_us(lambda: _lib.check(L.ga_posmap_fill(2, S, V, ptr(verts), ptr(mm.faces), ptr(mm.face_id), ptr(mm.bary), ptr(out), s)),
                              500)
        res[f"posmap_fill_S{S}_B2"] = dict(us=med, rounds_us=rounds, covered=float((mm.face_id >= 0).float().mean()))
    fid = torch.empty(512, 512, dtype=torch.int32, device="cuda")
    bary = torch.empty(512, 512, 3, device="cuda")
    med, rounds = time_us(lambda: _lib.check(L.ga_posmap_layout(corners.shape[0], 512, ptr(corners), ptr(fid), ptr(bary), s)), 20)
    res["posmap_layout_S512"] = dict(us=med, rounds_us=rounds, faces=int(corners.shape[0]))


def steps(res, name, N, S, inp, side, n_steps, blocks):
    from posmap_fixture import write_posmap_dataset
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.config import NetworkParams, OptimizationParams
    from gaussianavatar_b200.trainer import AvatarTrainer
    from gaussianavatar_b200.workload import to_cuda
    with tempfile.TemporaryDirectory() as tmp:
        mp_on = write_posmap_dataset(tmp, N=N, S=S, num_frames=4, side=side, inp=inp)
        subprocess.run([sys.executable, os.path.join(ROOT, "tools", "pose_maps.py"), os.path.join(mp_on.source_path, "train"), "--smpl_model",
                        os.path.join(mp_on.smpl_model_path, "SMPL_NEUTRAL.pkl"), "--uv_template",
                        os.path.join(mp_on.project_path, "assets", "template_mesh_smpl_uv.obj"), "--size", str(inp)], check=True, capture_output=True)
        mp_off = type(mp_on)(**{**vars(mp_on), "inp_posmap_from_pose": False})
        runs = {}
        for key, mp in (("files", mp_off), ("device", mp_on)):
            torch.manual_seed(0)
            m = AvatarModel(mp, NetworkParams(), OptimizationParams(), train=True)
            with torch.no_grad():          # ~5 mm Gaussians at the start, as bench.py's workload (an untrained net's are far larger)
                sd = m.net.state_dict(); sd["decoder.conv8N.bias"] = torch.tensor([-5.3]); m.net.load_state_dict(sd, strict=False)
            tr = AvatarTrainer(m, use_graph=False)
            items = [m.train_dataset[i] for i in range(2)]
            batch = {k: (torch.stack([torch.as_tensor(it[k]) for it in items]) if not isinstance(items[0][k], (int, float)) else [it[k] for it in items])
                     for k in items[0]}
            batch["pose_idx"] = torch.tensor([0, 1])
            batch = to_cuda(batch, torch.device("cuda"))[0]
            for i in range(3):
                tr.step(batch, 3000 + i, epoch=1)
            tr.finish()
            runs[key] = (tr, batch)
        torch.cuda.synchronize()
        times = {"files": [], "device": []}
        for blk in range(blocks):
            for key in (("files", "device") if blk % 2 == 0 else ("device", "files")):
                tr, batch = runs[key]
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for i in range(n_steps):
                    tr.step(batch, 3000 + i, epoch=1)
                tr.finish()
                b.record()
                b.synchronize()
                times[key].append(a.elapsed_time(b) / n_steps)
        res[f"stage2_step_{name}"] = dict(N=N, S=S, inp=inp, side=side, B=2, steps_per_block=n_steps,
                                          ms_files=times["files"], ms_device=times["device"],
                                          median_ms_files=statistics.median(times["files"]), median_ms_device=statistics.median(times["device"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--blocks", type=int, default=6)
    a = ap.parse_args()
    res = card()
    kernels(res)
    print(json.dumps(res), file=sys.stderr, flush=True)
    steps(res, "test_size", 700, 48, 32, 64, a.steps, a.blocks)
    steps(res, "200k", 200_000, 512, 128, 1024, a.steps, a.blocks)
    res["card_after"] = card()["nvidia_smi"]
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
