"""GPU: the synchronous overflow retry (`RasterBatchPlan.render_checked`) through each of its callers.  Every caller starts with a
binning buffer of 64 instances, far too few, so its first forward overflows; the buffer grows and the render runs again.  What it
returns must be bit for bit what an ample buffer renders: AvatarModel's inference render, the animation player's eager path (a
stage-2 actor) and mesh extraction's view renders."""
import os
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from gaussianavatar_b200 import animate as an  # noqa: E402
from gaussianavatar_b200 import mesh_extract as me  # noqa: E402
from gaussianavatar_b200 import rasterizer as rz  # noqa: E402
from test_animate_gpu import SIDE, _avatar, _cameras, _clip  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TINY = 64
PLAN = rz.RasterBatchPlan


def _tiny_plans(monkeypatch, module):
    """Makes every RasterBatchPlan that `module` constructs start with a TINY binning buffer; returns the list of those plans."""
    made = []

    def plan(*args, **kw):
        made.append(PLAN(*args, **dict(kw, capacity=TINY)))
        return made[-1]
    monkeypatch.setattr(module, "RasterBatchPlan", plan)
    return made


def test_avatar_model_render_retries(monkeypatch):
    m, _ = _avatar("smpl")
    clip = _clip("smpl")
    anim = an.Animator(m, _cameras("orbit"), SIDE, SIDE)
    sched = anim.schedule(clip, 30.0)
    pose, trans = anim.sample(clip, sched)
    batch = {"pose_data": pose[1:2], "transl_data": trans[1:2], "_cams": sched.cams[1:2].to(DEV), "height": [SIDE], "width": [SIDE]}
    with torch.no_grad():
        want = m.render_free_stage1(batch, 59400).clone()
        m.__dict__.pop("_raster_plans")
        made = _tiny_plans(monkeypatch, rz)
        got = m.render_free_stage1(batch, 59400)
    assert len(made) == 1 and made[0].capacity > TINY
    assert torch.equal(got, want)


def _frames(anim, clip):
    frames, depth = [], []
    for _, f, d in anim.frames(clip, 30.0):
        frames.append(f.clone())                        # the pinned buffers are reused two chunks later
        depth.append(d.clone())
    return torch.cat(frames), torch.cat(depth)


def test_animation_eager_path_retries():
    """The stage-2 decoder's BatchNorm sums are accumulated with atomics, so two decodes of one frame may differ in the last bits:
    each frame's Gaussians are decoded once and reused by both players, which leaves the rasterizer as the only difference."""
    m, mapper = _avatar("smpl", stage=2)
    clip = _clip("smpl", T=3)
    decode, memo = m._stage2_from_pose, {}

    def decoded(mapper_, pose, transl, rest, placement=None):
        key = (pose.cpu().numpy().tobytes(), transl.cpu().numpy().tobytes())
        if key not in memo:
            memo[key] = decode(mapper_, pose, transl, rest, placement=placement)
        return memo[key]
    m._stage2_from_pose = decoded
    ample = an.Animator(m, _cameras("orbit"), SIDE, SIDE, chunk=2, channels=4, pose_mapper=mapper, depth=True)
    want = _frames(ample, clip)
    tiny = an.Animator(m, _cameras("orbit"), SIDE, SIDE, chunk=2, channels=4, pose_mapper=mapper, depth=True, capacity=TINY)
    got = _frames(tiny, clip)
    assert ample.overflows == 0 and tiny.overflows >= 1
    assert got[0].shape[0] == want[0].shape[0] >= 2
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def test_mesh_extraction_views_retry(monkeypatch):
    n = 8000
    means = torch.from_numpy(me.fibonacci_directions(n) * 0.5).float().to(DEV)[None]
    scales = torch.full((1, n, 3), 0.01, device=DEV)
    colors = torch.tensor([0.8, 0.3, 0.1], device=DEV).expand(1, n, 3).contiguous()
    fake = types.SimpleNamespace(fix_rotation=torch.tensor([[1.0, 0, 0, 0]], device=DEV).expand(n, 4).contiguous(),
                                 fix_opacity=torch.ones(n, 1, device=DEV))
    cams = me.fusion_cameras([0.0, 0.0, 0.0], 0.6, 10, 128).to(DEV)

    def views():
        return [(s, e, img.clone(), depth.clone(), fT.clone()) for s, e, img, depth, fT in me.render_views(fake, means, scales, colors,
                                                                                                           cams, 128, 128)]
    want = views()
    made = _tiny_plans(monkeypatch, me)
    got = views()
    assert len(made) == 2 and all(p.capacity > TINY for p in made)
    assert [(s, e) for s, e, *_ in got] == [(s, e) for s, e, *_ in want] == [(0, 8), (8, 10)]
    for g, w in zip(got, want):
        assert all(torch.equal(a, b) for a, b in zip(g[2:], w[2:]))
