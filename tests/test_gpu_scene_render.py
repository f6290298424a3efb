"""render_scene (dreamscene_b200.scene): the views of a training step rendered straight from the raw parameter groups,
against the two-op path it replaces, assemble_scene(noise="fused", views=B) + rasterize_views, with the same seed."""
import pytest
import torch

from harness import cameras
from tests import util_scene as U

pytestmark = pytest.mark.gpu

NAMES = ("_xyz", "_opacity", "_scaling", "_rotation", "_features_dc", "_features_rest")


def _groups(sizes, M, seed=0, offset=(0.0, 0.0, 0.0)):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    out = []
    for n in sizes:
        d = {"_xyz": r(n, 3) * 0.6 + torch.tensor(offset, device="cuda"), "_opacity": r(n, 1) * 2,
             "_scaling": r(n, 3) * 0.5 - 3.0, "_rotation": r(n, 4), "_features_dc": r(n, 1, 3),
             "_features_rest": r(n, M - 1, 3) * 0.1}
        out.append({k: v.contiguous().requires_grad_(True) for k, v in d.items()})
    return out


def _clone(groups):
    return [{k: v.detach().clone().requires_grad_(True) for k, v in g.items()} for g in groups]


def _settings(B, H=96, W=80, degs=None, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for v in range(B):
        cam = cameras.orbit_camera(radius=3.5, theta_deg=50.0 + 7 * v, phi_deg=37.0 * v, fovx=0.6, height=H, width=W)
        deg = 3 if degs is None else degs[v % len(degs)]
        bg = tuple(float(x) for x in torch.rand(3, generator=g))
        out.append(U.cuda_settings(cam, deg, bg=bg))
    return out


def _two_op(groups, S, seed, shs_flags, scale_flags, means2D):
    """assemble_scene + rasterize_views; per-view flags pick each view's slices from the assemble with that view's
    augmentation (the Philox streams depend on the view only, so the slices are what a per-view flag would give)."""
    from dreamscene_b200.multiview import rasterize_views
    from dreamscene_b200.scene import assemble_scene
    B = len(S)
    cache = {}

    def get(sa, ca):
        if (sa, ca) not in cache:
            m, o, sc, r, sh = assemble_scene(groups, shs_aug=sa, scale_aug=ca, noise="fused", seed=seed, views=B)
            cache[(sa, ca)] = (m, o, sc if B > 1 else sc[None], r, sh if B > 1 else sh[None])
        return cache[(sa, ca)]

    m, o, _, r, _ = get(shs_flags[0], scale_flags[0])
    shs = [get(shs_flags[v], scale_flags[v])[4][v] for v in range(B)]
    scales = [get(shs_flags[v], scale_flags[v])[2][v] for v in range(B)]
    outs = rasterize_views(S, m, o, shs=shs, scales=scales, rotations=r, means2D=means2D)
    return outs, torch.stack(scales)


def _flags(f, B):
    return tuple(f) if isinstance(f, (list, tuple)) else (f,) * B


def _loss(outs, w, scales=None):
    loss = sum((w[0][v] * o[0]).sum() + (w[1][v] * o[2]).sum() for v, o in enumerate(outs))
    return loss + 3.0 * scales.mean() if scales is not None else loss


def _weights(B, H, W, seed=3):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(B, 3, H, W, device="cuda", generator=g), torch.randn(B, 2, H, W, device="cuda", generator=g))


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


@pytest.mark.parametrize("M,sizes,B,aug", [
    (1, [300, 0, 1, 777], 1, True),
    (4, [1000, 1, 513, 0, 4097], 4, True),
    (9, [129, 64, 1], 4, [True, False, True, False]),
    (16, [2000, 333], 4, False),
    (16, [1, 0, 1500, 250], 16, [v % 3 != 0 for v in range(16)]),
    (4, [2600], 16, True),
])
def test_forward_and_scales_bitwise_equal_to_assemble_plus_rasterize_views(M, sizes, B, aug):
    from dreamscene_b200.scene import render_scene
    degs = [d for d in range(4) if (d + 1) ** 2 <= M]
    S = _settings(B, degs=degs, seed=M)
    groups = _groups(sizes, M, seed=M + B)
    flags = _flags(aug, B)
    with torch.no_grad():
        outs, sc = render_scene(groups, S, shs_aug=aug, scale_aug=aug, seed=1234, return_scales=True)
        ref, ref_sc = _two_op(groups, S, 1234, flags, flags, None)
    assert torch.equal(sc, ref_sc)
    for v in range(B):
        for k in range(3):
            assert torch.equal(outs[v][k], ref[v][k]), (v, k)
    assert any(bool((o[1] > 0).any()) for o in outs)        # something is on screen


def test_shs_and_scale_augmentation_switch_independently():
    from dreamscene_b200.scene import render_scene
    S = _settings(3, degs=[1, 2])
    groups = _groups([800, 400], 9, seed=2)
    with torch.no_grad():
        outs, sc = render_scene(groups, S, shs_aug=True, scale_aug=[False, True, False], seed=9, return_scales=True)
        ref, ref_sc = _two_op(groups, S, 9, (True,) * 3, (False, True, False), None)
    assert torch.equal(sc, ref_sc)
    assert all(torch.equal(outs[v][k], ref[v][k]) for v in range(3) for k in range(3))


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("M,sizes,B,aug,with_scales", [
    (4, [1000, 1, 513, 0, 4097], 4, True, False),
    (16, [1500, 250], 4, [True, False, False, True], True),
    (9, [700, 129], 1, True, True),
    (1, [900], 3, False, False),
])
def test_backward_matches_the_two_op_path(det, M, sizes, B, aug, with_scales):
    from dreamscene_b200.scene import render_scene
    H, W = 96, 80
    S = _settings(B, H, W, degs=[d for d in range(4) if (d + 1) ** 2 <= M], seed=5)
    groups = _groups(sizes, M, seed=11)
    ref_groups = _clone(groups)
    w = _weights(B, H, W)
    flags = _flags(aug, B)
    m2 = [torch.zeros(sum(sizes), 3, device="cuda", requires_grad=True) for _ in range(B)]
    r2 = [torch.zeros(sum(sizes), 3, device="cuda", requires_grad=True) for _ in range(B)]
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        outs, sc = render_scene(groups, S, shs_aug=aug, scale_aug=aug, seed=77, means2D=m2, return_scales=True)
        _loss(outs, w, sc if with_scales else None).backward()
        ref, ref_sc = _two_op(ref_groups, S, 77, flags, flags, r2)
        _loss(ref, w, ref_sc if with_scales else None).backward()
    finally:
        torch.use_deterministic_algorithms(old)
    for g, r in zip(groups, ref_groups):
        for k in NAMES:
            if g[k].numel() == 0:
                continue
            assert torch.isfinite(g[k].grad).all(), k
            if float(r[k].grad.norm()) == 0.0:
                assert float(g[k].grad.norm()) == 0.0, k
            else:
                e = _rel(g[k].grad, r[k].grad)
                assert e < 2e-6, (k, e)
    for v in range(B):
        if det:
            assert torch.equal(m2[v].grad, r2[v].grad), v
        else:
            assert _rel(m2[v].grad, r2[v].grad) < 1e-5, v


def test_culled_and_empty_inputs_give_zero_finite_gradients():
    from dreamscene_b200.scene import render_scene
    S = _settings(3, degs=[1])
    culled = _groups([500, 0, 37], 4, seed=1)
    with torch.no_grad():
        for g in culled:
            g["_xyz"].fill_(1.0e4)                     # far outside every camera's view
    outs = render_scene(culled, S, seed=1)
    assert all(not bool((o[1] > 0).any()) for o in outs)
    sum(o[0].sum() + o[2].sum() for o in outs).backward()
    for g in culled:
        for k in NAMES:
            t = g[k].grad
            assert t is not None and torch.isfinite(t).all() and not bool(t.any()), k
    empty = _groups([0, 0], 4, seed=2)
    outs = render_scene(empty, S, seed=1)
    assert all(o[1].numel() == 0 for o in outs)
    sum(o[0].sum() + o[2].sum() for o in outs).backward()
    for g in empty:
        for k in NAMES:
            assert g[k].grad is not None and g[k].grad.numel() == 0


def test_culled_rows_get_zero_gradients_next_to_visible_ones():
    """Half the rows behind every camera: their leaf gradients are exactly zero (view 0 writes every row, later
    views add only into the rows they saw), unless the scale loss reaches them."""
    from dreamscene_b200.scene import render_scene
    S = _settings(4, degs=[0, 1])
    groups = _groups([3000], 4, seed=4)
    far = torch.zeros(3000, dtype=torch.bool, device="cuda")
    far[::2] = True
    with torch.no_grad():
        groups[0]["_xyz"][far] = 1.0e4
    m2 = [torch.zeros(3000, 3, device="cuda", requires_grad=True) for _ in range(4)]
    outs, sc = render_scene(groups, S, seed=3, means2D=m2, return_scales=True)
    assert not any(bool((o[1][far] > 0).any()) for o in outs) and all(bool((o[1] > 0).any()) for o in outs)
    sum(o[0].sum() for o in outs).backward(retain_graph=True)
    for k in NAMES:
        gr = groups[0][k].grad
        assert torch.isfinite(gr).all() and float(gr[far].abs().max()) == 0.0 and float(gr[~far].abs().max()) > 0, k
        groups[0][k].grad = None
    sc.sum().backward()                      # the scale loss reaches every row's _scaling, culled ones included
    assert bool((groups[0]["_scaling"].grad[far] != 0).all())


def test_deterministic_mode_gives_bitwise_identical_leaf_gradients():
    from dreamscene_b200.scene import render_scene
    S = _settings(4)
    w = _weights(4, 96, 80)
    grads = []
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(2):
            groups = _groups([4000, 1000], 16, seed=8)
            outs, sc = render_scene(groups, S, seed=5, return_scales=True)
            _loss(outs, w, sc).backward()
            grads.append([g[k].grad.clone() for g in groups for k in NAMES])
    finally:
        torch.use_deterministic_algorithms(old)
    assert all(torch.equal(a, b) for a, b in zip(*grads))


def test_peak_memory_is_lower_than_the_two_op_path_by_at_least_one_copy():
    from dreamscene_b200.scene import render_scene
    P, M, B, H = 200_000, 16, 4, 256
    S = _settings(B, H, H)
    groups = _groups([P], M, seed=6)
    w = _weights(B, H, H)

    def peak(fn):
        for g in groups:
            for v in g.values():
                v.grad = None
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fn()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    run_scene = lambda: _loss(render_scene(groups, S, seed=1), w).backward()
    run_two = lambda: _loss(_two_op(groups, S, 1, (True,) * B, (True,) * B, None)[0], w).backward()
    run_scene(); run_two()                   # capacities measured, workspaces allocated
    a, b = peak(run_scene), peak(run_two)
    print(f"peak allocated over forward+backward: render_scene {a / 2**20:.1f} MiB, two-op {b / 2**20:.1f} MiB")
    assert b - a >= B * P * 3 * M * 4, (a, b)


def test_three_adam_steps_stay_within_two_lr_per_step_of_the_two_op_path():
    from dreamscene_b200 import GaussianAdam
    from dreamscene_b200.scene import render_scene
    from harness.adam_ref import LRS, reference_adam
    B, H, W = 4, 96, 80
    S = _settings(B, H, W, degs=[3])
    init = _groups([5000, 1200], 16, seed=12)
    short = {"_xyz": "xyz", "_features_dc": "f_dc", "_features_rest": "f_rest", "_opacity": "opacity",
             "_scaling": "scaling", "_rotation": "rotation"}
    runs = []
    for path in ("scene", "two_op"):
        groups = [{k: torch.nn.Parameter(v.detach().clone()) for k, v in g.items()} for g in init]
        opts = [reference_adam({short[k]: v for k, v in g.items()}, GaussianAdam) for g in groups]
        for step in range(3):
            for o in opts:
                o.zero_grad(set_to_none=True)
            w = _weights(B, H, W, seed=20 + step)
            if path == "scene":
                outs, sc = render_scene(groups, S, seed=100 + step, return_scales=True)
            else:
                outs, sc = _two_op(groups, S, 100 + step, (True,) * B, (True,) * B, None)
            _loss(outs, w, sc).backward()
            for o in opts:
                o.step()
        runs.append(groups)
    differ, total = 0, 0
    for ga, gb in zip(*runs):
        for k in NAMES:
            d = (ga[k].detach() - gb[k].detach()).abs()
            assert d.numel() == 0 or float(d.max()) <= 2 * LRS[short[k]] * 3, (k, float(d.max()))
            differ += int((d > 0).sum()); total += d.numel()
    print(f"after 3 Adam steps {differ / total:.2e} of the parameter elements differ at all")
