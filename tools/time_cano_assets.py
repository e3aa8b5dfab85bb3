"""Cost of the canonical-asset kernels (csrc/posmap.cu).  Run on the GPU box:
    python tools/time_cano_assets.py > cano_assets.json
  1. `ga_smplx_vertices` at B = 2 and 8 against its byte floor: posedirs (486 x 31425 fp32, 61.1 MB) read once per call, which is
     18.2 us at the H100 SXM data sheet's 3.35 TB/s (computed from bytes, not measured);
  2. `ga_posmap_weights` at S = 512 with J = 24 and 55 (the map it writes is 25.2 / 57.7 MB);
  3. the whole canonical build (`posmap.canonical_assets`) at S = 512 for each body on the synthetic models and UV templates, host
     set-up included, timed with a device synchronise.
Kernel times are CUDA events around many back-to-back launches; the card's name, power limit and max SM clock are read in the same run.
"""
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from gaussianavatar_b200 import _lib, synthetic as syn  # noqa: E402
from gaussianavatar_b200._lib import ptr  # noqa: E402
from gaussianavatar_b200.posmap import PoseMapper, SmplxPoseMapper, canonical_assets  # noqa: E402
from time_posmap import HBM_BYTES_PER_S, card, time_us  # noqa: E402


def main():
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    res = card()
    s = torch.cuda.current_stream().cuda_stream
    L = _lib.lib()
    bx, tx = syn.make_smplx_body(0), syn.make_smplx_uv_template(0)
    mx_model = syn.smplx_mesh_model(bx, tx, syn.smplx_posedirs(0))
    mx = SmplxPoseMapper(mx_model, bx.betas[0], tx, 512)
    V = mx.V
    pd_bytes = 486 * 3 * V * 4
    for B in (2, 8):
        pose, rest, transl = (x.cuda().contiguous() for x in syn.synthetic_smplx_poses(B, seed=1))
        out = torch.empty(B, V, 3, device="cuda")
        med, rounds = time_us(lambda: _lib.check(L.ga_smplx_vertices(B, V, ptr(pose), ptr(rest), ptr(transl), ptr(mx.rest_joints),
                                                                    ptr(mx.v_shaped), ptr(mx.posedirs), ptr(mx.weights), ptr(out), s)), 500)
        nbytes = pd_bytes + V * 55 * 4 + V * 12 + B * V * 12
        res[f"smplx_vertices_B{B}"] = dict(us=med, rounds_us=rounds, posedirs_mb=pd_bytes / 1e6,
                                           posedirs_floor_us=pd_bytes / HBM_BYTES_PER_S * 1e6, all_bytes=nbytes,
                                           tb_per_s=nbytes / (med * 1e-6) / 1e12)
    bs, ts = syn.make_body(0), syn.make_uv_template(0)
    ms = PoseMapper(syn.smpl_mesh_model(bs, ts), bs.betas[0], ts, 512)
    for m in (ms, mx):
        J = m.JOINTS
        out = torch.empty(512, 512, J, device="cuda")
        med, rounds = time_us(lambda: _lib.check(L.ga_posmap_weights(512, J, ptr(m.weights), ptr(m.faces), ptr(m.face_id), ptr(m.bary),
                                                                    ptr(out), s)), 200)
        nbytes = out.numel() * 4
        res[f"posmap_weights_S512_J{J}"] = dict(us=med, rounds_us=rounds, out_bytes=nbytes, tb_per_s_out=nbytes / (med * 1e-6) / 1e12)
    for body, model, b, t in (("smpl", syn.smpl_mesh_model(bs, ts), bs, ts), ("smplx", mx_model, bx, tx)):
        canonical_assets(model, b.betas[0], t, 512, body=body)
        torch.cuda.synchronize()
        ms_ = []
        for _ in range(5):
            t0 = time.perf_counter()
            canonical_assets(model, b.betas[0], t, 512, body=body)
            torch.cuda.synchronize()
            ms_.append((time.perf_counter() - t0) * 1e3)
        res[f"canonical_assets_S512_{body}"] = dict(median_ms=statistics.median(ms_), rounds_ms=ms_)
    res["card_after"] = card()["nvidia_smi"]
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
