"""render_frames (dreamscene_b200.video) against the reference's video loop (harness/video_ref.py) driven by the
per-view path, render_scene without augmentation + disparity_from_depth_alpha: every frame bit for bit, for every
views_per_pass, through an empty view, a pass that overflows its pair capacity, deterministic mode, reserved groups'
live prefixes, and the empty inputs."""
import math

import numpy as np
import pytest
import torch

from dreamscene_b200 import rasterizer as R
from dreamscene_b200.reserve import ReservedGroup
from dreamscene_b200.video import render_frames
from harness import cameras, video_ref
from tests import util_scene as U

pytestmark = pytest.mark.gpu

NAMES = ("_xyz", "_opacity", "_scaling", "_rotation", "_features_dc", "_features_rest")


def _groups(sizes, M, seed=0, radius=0.6, log_scale=-3.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    return [{"_xyz": r(n, 3) * radius, "_opacity": r(n, 1) * 2, "_scaling": r(n, 3) * 0.5 + log_scale,
             "_rotation": r(n, 4), "_features_dc": r(n, 1, 3), "_features_rest": r(n, M - 1, 3) * 0.3}
            for n in sizes]


def _away(H, W):
    """A camera at the orbit's radius that looks away from the scene (right and forward of an orbit pose negated)."""
    pose = cameras.orbit_pose(3.5, 60.0, 20.0)
    pose[:3, 0] *= -1
    pose[:3, 2] *= -1
    return cameras.camera_from_pose(pose, 0.6, H, W)


def _views(N, M, H=80, W=88, seed=0):
    """N views around the scene: sh_degree cycling over what M allows, black / white / random backgrounds, one view at
    scale_modifier 1.3 and one that sees nothing (view 7)."""
    g = torch.Generator().manual_seed(seed)
    degs = [d for d in range(4) if (d + 1) ** 2 <= M]
    out = []
    for v in range(N):
        cam = _away(H, W) if v == 7 else cameras.orbit_camera(radius=2.5 + 0.05 * v, theta_deg=40.0 + 3 * v,
                                                               phi_deg=29.0 * v, fovx=0.7, height=H, width=W)
        bg = [(0.0, 0.0, 0.0), (1.0, 1.0, 1.0)][v % 3] if v % 3 < 2 else tuple(float(x) for x in torch.rand(3, generator=g))
        out.append(U.cuda_settings(cam, degs[v % len(degs)], bg=bg, scale_modifier=1.3 if v == 11 else 1.0))
    return out


def _reference(groups, S, monkeypatch):
    monkeypatch.setattr(R, "_pair_mode", "sync")       # every per-view render waits for its own pair count
    with torch.no_grad():
        img, dep = video_ref.frames(video_ref.native_render(groups), S)
    return np.stack(img), np.stack(dep)


def _check(out, ref):
    rgb, depth = out
    assert rgb.is_pinned() and depth.is_pinned() and rgb.dtype == depth.dtype == torch.uint8
    np.testing.assert_array_equal(rgb.numpy(), ref[0])
    np.testing.assert_array_equal(depth.numpy(), ref[1])


LAYOUTS = {"object": ([3000], 16), "scene": ([900, 40, 1500, 1, 700, 2600], 4)}
_refs: dict = {}


@pytest.mark.parametrize("vpp", [1, 5, 16])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_frames_equal_the_reference_loop(layout, vpp, monkeypatch):
    sizes, M = LAYOUTS[layout]
    groups = _groups(sizes, M, seed=len(sizes))
    S = _views(37, M, seed=M)
    if layout not in _refs:
        _refs[layout] = _reference(groups, S, monkeypatch)
    ref = _refs[layout]
    out = render_frames(groups, S, views_per_pass=vpp)
    _check(out, ref)
    rgb, depth = out
    # the view looking away: the quantised background, and an all-zero depth frame
    bg = S[7].bg.cpu().numpy().astype(np.float32)
    assert (rgb[7].numpy() == (bg * 255).round().astype(np.uint8)).all() and not depth[7].any()
    assert len({tuple(s.bg.tolist()) for s in S}) > 3 and {s.sh_degree for s in S} == set(range(int(math.sqrt(M))))
    assert depth[0].max() == 255 and rgb.numpy().std() > 10


def test_frames_do_not_depend_on_views_per_pass_at_any_image_size():
    """H % 16 != 0: a pass of one view is written unpadded, a pass of several stacked in padded tile rows; B*H*W odd:
    the last pixels of a pass are stored byte by byte."""
    groups = _groups([2500, 300], 9, seed=6)
    S = _views(9, 9, H=71, W=87, seed=3)
    a = render_frames(groups, S, views_per_pass=1)
    for vpp in (4, 16):
        b = render_frames(groups, S, views_per_pass=vpp)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), vpp
    assert a[0].shape == (9, 71, 87, 3) and a[1][0].max() == 255 and not a[1][7].any()


def test_overflowing_pass_is_rendered_again(monkeypatch):
    """Cameras from far to close: the first pass fixes the capacity (2x its pairs, at least 4 per Gaussian and 2^20),
    and a later, closer pass produces more pairs than that.  It is re-issued; the frames are still the reference's."""
    P, H, W = 50_003, 256, 256
    groups = _groups([P], 4, seed=5, log_scale=-3.0)
    dist = [30.0, 20.0, 10.0, 6.0, 3.5, 2.2, 1.6, 1.3]
    S = [U.cuda_settings(cameras.orbit_camera(radius=r, theta_deg=60.0, phi_deg=10.0 * k, fovx=0.7, height=H, width=W),
                         1, bg=(0.2, 0.3, 0.4)) for k, r in enumerate(dist)]
    d = R._device_state(torch.device("cuda", torch.cuda.current_device()))
    monkeypatch.setattr(d, "user_capacity", False)
    R.flush_checks()
    grown = []                                                      # pair counts of the passes that overflowed
    grow = R._Device.grow
    monkeypatch.setattr(R._Device, "grow", lambda self, pairs: grown.append(pairs) or grow(self, pairs))
    out = render_frames(groups, S, views_per_pass=2)
    assert grown and min(grown) > max(1 << 20, 4 * 2 * P)           # a pass overflowed and was re-issued
    monkeypatch.setattr(R._Device, "grow", grow)
    _check(out, _reference(groups, S, monkeypatch))


def test_deterministic_mode_gives_the_same_frames():
    groups = _groups([900, 2000], 9, seed=3)
    S = _views(20, 9, seed=1)
    a = render_frames(groups, S, views_per_pass=7)
    torch.use_deterministic_algorithms(True)
    try:
        b = render_frames(groups, S, views_per_pass=7)
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_reserved_groups_live_prefixes_give_the_packed_frames():
    plain = _groups([1200, 500], 4, seed=8)
    reserved = []
    for g in plain:
        r = ReservedGroup.from_tensors(g["_xyz"], g["_features_dc"], g["_features_rest"], g["_opacity"], g["_scaling"],
                                       g["_rotation"], capacity=2 * g["_xyz"].shape[0] + 17)
        with torch.no_grad():
            for k in NAMES:
                getattr(r, k)[r.live_count:] = float("nan")
        reserved.append(r)
    S = _views(9, 4, seed=2)
    a = render_frames([r.rows() for r in reserved], S, views_per_pass=4)
    b = render_frames(plain, S, views_per_pass=4)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_empty_inputs(monkeypatch):
    rgb, depth = render_frames(_groups([100], 4), [])
    assert rgb.shape == (0, 0, 0, 3) and depth.shape == (0, 0, 0, 1)
    S = _views(5, 4, seed=4)
    empty = _groups([0, 0], 4)
    rgb, depth = render_frames(empty, S, views_per_pass=2)
    assert rgb.shape == (5, 80, 88, 3) and depth.shape == (5, 80, 88, 1)
    for v, s in enumerate(S):
        assert (rgb[v].numpy() == (s.bg.cpu().numpy() * 255).round().astype(np.uint8)).all()
    assert not depth.any()
    _check((rgb, depth), _reference(empty, S, monkeypatch))
