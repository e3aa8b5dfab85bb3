"""The frame-by-frame rasterizer loop AvatarModel takes for more than 8 frames, which renders consecutive frames on two alternating
side streams."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def test_frame_loop_renders_each_frame_as_the_batched_rasterizer_does():
    """An inference model renders frames 0-7 as one batch of 8 and frame 8 alone through render_free_stage1 (the batched rasterizer),
    then the same 9 frames' Gaussians together, which takes the frame-by-frame loop.  The skinning kernel takes at most 8 frames, so
    the 9 frames' Gaussians are the two calls' own.  Every frame is rasterized from the same Gaussians by the same kernels in both
    paths: the images are bit-identical."""
    from gaussianavatar_b200 import synthetic as syn
    from gaussianavatar_b200.avatar_model import AvatarModel
    from gaussianavatar_b200.camera import TEST_POSE_EXTRINSIC, TEST_POSE_K, make_camera, scaled_intrinsics
    from gaussianavatar_b200.workload import load_poses
    N, S, side, F = 4000, 64, 128, 9
    pose, transl, _ = load_poses(F)
    torch.manual_seed(0)
    m = AvatarModel.from_assets(syn.make_avatar_assets(N, S, seed=0), [], pose, transl, train=False, device=DEV, inp_posmap_size=32)
    with torch.no_grad():
        sd = m.net.state_dict()
        sd["decoder.conv8N.bias"] = torch.tensor([-5.3])        # small Gaussians, as in the benchmark workload
        m.net.load_state_dict(sd, strict=False)
    cam = make_camera(scaled_intrinsics(TEST_POSE_K, side), TEST_POSE_EXTRINSIC, side, side).to(DEV)

    def frames(lo, hi):
        B = hi - lo
        return dict(pose_data=pose[lo:hi].to(DEV), transl_data=transl[lo:hi].to(DEV), FovX=[cam.FovX] * B, FovY=[cam.FovY] * B,
                    height=[cam.height] * B, width=[cam.width] * B, world_view_transform=cam.world_view_transform[None].expand(B, -1, -1),
                    full_proj_transform=cam.full_proj_transform[None].expand(B, -1, -1), camera_center=cam.camera_center[None].expand(B, -1))

    paths = []              # which rasterizer path each render took

    def recording_path(name):
        method = getattr(m, name)

        def wrapper(*args):
            paths.append(name)
            return method(*args)
        return wrapper

    for name in ("_render_batched", "_render_frames_one_by_one"):
        setattr(m, name, recording_path(name))

    gaussians = []          # (means, scales, colors) that render_free_stage1 hands the rasterizer, one entry per call
    render_frames = m._render_frames

    def recording_gaussians(batch, means, scales, colors):
        gaussians.append((means, scales, colors))
        return render_frames(batch, means, scales, colors)

    m._render_frames = recording_gaussians
    with torch.no_grad():
        batched = torch.cat([m.render_free_stage1(frames(0, 8), 59400), m.render_free_stage1(frames(8, F), 59400)])
        means, scales, colors = (torch.cat(t) for t in zip(*gaussians))
        loop = render_frames(frames(0, F), means, scales, colors)
    torch.cuda.synchronize()
    assert paths == ["_render_batched", "_render_batched", "_render_frames_one_by_one"], paths
    assert loop.shape == batched.shape == (F, 3, side, side)
    for b in range(F):
        assert torch.equal(loop[b], batched[b]), (b, (loop[b] - batched[b]).abs().mean().item(), (loop[b] - batched[b]).abs().max().item())
    assert (loop < 0.999).any()                                               # the body is on screen (white background)
    assert (loop[0] - loop[F - 1]).abs().mean().item() > 1e-4                 # and the frames differ
