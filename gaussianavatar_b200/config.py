"""Plain-data mirrors of the reference's option groups (/root/reference arguments/__init__.py:55-144) so callers that
do not go through argparse (benchmarks, tests, synthetic runs) can build an AvatarModel.  Field names and defaults are
the reference's; `arguments.ModelParams(...).extract(args)` namespaces work unchanged too (duck-typed)."""
from __future__ import annotations

import os
from dataclasses import dataclass, field


@dataclass
class ModelParams:
    source_path: str = ""
    model_path: str = ""
    project_path: str = field(default_factory=os.getcwd)
    smpl_model_path: str = ""
    smplx_model_path: str = ""
    test_folder: str = ""
    stage1_out_path: str = ""
    save_epoch: int = 30
    train_stage: int = 1
    dataset_type: str = "peeplesnapshot"
    smpl_gender: str = "neutral"
    smpl_type: str = "smpl"
    no_mask: int = 0
    fixed_inp: int = 0
    train_mode: int = 0
    cam_static: int = 1
    white_background: bool = True
    batch_size: int = 2
    query_posmap_size: int = 512
    inp_posmap_size: int = 128
    # stage 2: build each frame's input position map on the device from its SMPL pose instead of reading inp_map/*.npz
    # (not a reference option; read with getattr(..., False) so the reference's own namespaces keep working)
    inp_posmap_from_pose: bool = False
    # train against metric depth maps, <split>/depths/<name>.npy (float32 metres) or .png (uint16 millimetres); not a reference
    # option, read with getattr(..., False)
    depth_maps: bool = False
    # render with 3DGS's `antialiasing` setting (Mip-Splatting's screen-space filter: each splat's opacity is scaled so that its
    # footprint does not depend on the 0.3 px^2 dilation) in training and every render of the avatar; not a reference option, read
    # with getattr(..., False).  A checkpoint does not record it: render an avatar with the mode it was trained with
    antialiasing: bool = False
    # learn each training frame's exposure and white balance, c' = A c + t per frame with training frame 0 fixed at [I | 0]
    # (DESIGN.md §4); not a reference option, read with getattr(..., False)
    train_exposure: bool = False


@dataclass
class NetworkParams:
    c_pose: int = 64
    c_geom: int = 64
    hsize: int = 128
    nf: int = 32
    up_mode: str = "upconv"
    use_dropout: int = 0
    pos_encoding: int = 0
    num_emb_freqs: int = 6
    posemb_incl_input: int = 0
    geom_layer_type: str = "conv"
    gaussian_kernel_size: int = 5


@dataclass
class OptimizationParams:
    epochs: int = 200
    lambda_dssim: float = 0.2
    lambda_scale: float = 3e-2
    lambda_lpips: float = 0.2
    lambda_pose: float = 10
    lambda_rgl: float = 1e1
    log_iter: int = 2000
    lpips_start_iter: int = 30
    pose_op_start_iter: int = 1800
    lr_net: float = 3e-3
    lr_geomfeat: float = 5e-4
    sched_milestones: list = field(default_factory=lambda: [66, 133])
    # weight of the masked L1 depth loss when the batches carry `depth` (ModelParams.depth_maps); not a reference option, read
    # with getattr(..., 1.0).  An unmeasured starting point, not a tuned value
    lambda_depth: float = 1.0
    # Adam learning rate of the per-frame exposure table (ModelParams.train_exposure), falling log-linearly from init to final over
    # the stage's steps, as 3DGS's exposure optimiser does; not reference options, read with getattr
    exposure_lr_init: float = 0.01
    exposure_lr_final: float = 0.001
