"""Deterministic mode (torch.use_deterministic_algorithms(True)): the important score, every gradient and the
disparity backward are bitwise reproducible - across repeats, streams, CUDA-graph replays, retain_graph re-runs
and ways of splitting the work - and stay as accurate as the default fp32-atomic path."""
import contextlib
import math

import numpy as np
import pytest
import torch

from tests import util_scene as U
from tests.parity_budgets import BWD_REL
from tests.test_gpu_parity import run_oracle

pytestmark = pytest.mark.gpu

NAMES = ("means3D", "opacities", "shs", "scales", "rotations")


@contextlib.contextmanager
def deterministic(on=True):
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(old)


def fwd_bwd(sc, cam, deg, grads, score=True, scale_modifier=1.0, retain=False):
    """One forward + backward through the public surface -> dict of every output and gradient (device tensors)."""
    from dreamscene_b200 import GaussianRasterizer
    S = U.cuda_settings(cam, deg, score=score, scale_modifier=scale_modifier)
    t = {k: sc[k].detach().to("cuda").clone().requires_grad_(True) for k in NAMES}
    m2d = torch.zeros(t["means3D"].shape[0], 3, device="cuda", requires_grad=True)
    out = GaussianRasterizer(S)(means3D=t["means3D"], means2D=m2d, opacities=t["opacities"], shs=t["shs"],
                                scales=t["scales"], rotations=t["rotations"])
    res = dict(zip(("score", "color", "radii", "depth_alpha") if score else ("color", "radii", "depth_alpha"), out))
    gc, gd = (g.to("cuda") for g in grads)
    leaves = [t[k] for k in NAMES] + [m2d]
    g = torch.autograd.grad([res["color"], res["depth_alpha"]], leaves, [gc, gd], retain_graph=retain)
    res.update({f"d_{k}": v for k, v in zip(NAMES + ("means2D",), g)})
    if retain:
        g2 = torch.autograd.grad([res["color"], res["depth_alpha"]], leaves, [gc, gd])
        res.update({f"d2_{k}": v for k, v in zip(NAMES + ("means2D",), g2)})
    return res


def assert_bitwise(a, b, what=""):
    for k in a:
        assert torch.equal(a[k], b[k]), f"{what}{k} differs"


def grad_inputs(H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(3, H, W, generator=g) / (H * W), torch.randn(2, H, W, generator=g) / (H * W)


@pytest.mark.parametrize("P,H", [(10_000, 256), (100_000, 512)])
def test_repeats_side_stream_and_retain_graph_are_bitwise_equal(P, H):
    sc, cam, deg = U.make_inputs(P, H, H, seed=3, exact_knn=False)
    grads = grad_inputs(H, H, 4)
    with deterministic():
        runs = [fwd_bwd(sc, cam, deg, grads) for _ in range(3)]
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            side = fwd_bwd(sc, cam, deg, grads)
        torch.cuda.current_stream().wait_stream(s)
        again = fwd_bwd(sc, cam, deg, grads, retain=True)
    torch.cuda.synchronize()
    assert float(runs[0]["score"].abs().sum()) > 0 and float(runs[0]["d_means2D"].abs().sum()) > 0
    for r in runs[1:] + [side]:
        assert_bitwise(runs[0], r)
    for k in NAMES + ("means2D",):
        assert torch.equal(again[f"d_{k}"], runs[0][f"d_{k}"]) and torch.equal(again[f"d2_{k}"], runs[0][f"d_{k}"]), k


def test_cuda_graph_replay_is_bitwise_equal_to_eager():
    from dreamscene_b200 import GaussianRasterizer
    from dreamscene_b200 import rasterizer as R
    H = W = 128
    P = 8000
    sc, cam, deg = U.make_inputs(P, H, W, seed=8)
    S = U.cuda_settings(cam, deg, score=True)
    static = {k: sc[k].cuda().clone().requires_grad_(True) for k in NAMES}
    m2d = torch.zeros(P, 3, device="cuda", requires_grad=True)
    gc, gd = (g.cuda() for g in grad_inputs(H, W, 5))

    def fb(p):
        score, color, radii, da = GaussianRasterizer(S)(means3D=p["means3D"], means2D=m2d, opacities=p["opacities"],
                                                        shs=p["shs"], scales=p["scales"], rotations=p["rotations"])
        g = torch.autograd.grad([color, da], [p[k] for k in NAMES] + [m2d], [gc, gd])
        return (score, color, da) + tuple(g)

    with deterministic():
        fb(static)
        R.flush_checks()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            fb(static)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            g_out = fb(static)
        with torch.no_grad():
            static["means3D"].add_(0.01 * torch.randn_like(static["means3D"]))
            static["opacities"].mul_(0.9)
        for _ in range(2):
            graph.replay()
            torch.cuda.synchronize()
            e_out = fb(static)
            torch.cuda.synchronize()
            for a, b in zip(g_out, e_out):
                assert torch.equal(a, b)


def test_one_view_of_a_multi_view_call_equals_the_single_view_call():
    """The fixed-point sums depend only on the set of partials: view 0 rendered alongside view 1 (its own tensors)
    gives bit for bit what view 0 rendered alone gives, although the work is scheduled differently."""
    from dreamscene_b200 import GaussianRasterizer
    from dreamscene_b200.multiview import rasterize_views
    H = W = 192
    sc, cam0, deg = U.make_inputs(12000, H, W, seed=21, exact_knn=False)
    cam1 = U.make_inputs(12, H, W, phi=70.0)[1]
    grads = [grad_inputs(H, W, 30 + v) for v in range(2)]
    settings = [U.cuda_settings(c, deg, score=True) for c in (cam0, cam1)]
    with deterministic():
        per_view = [{k: sc[k].cuda().clone().requires_grad_(True) for k in NAMES} for _ in range(2)]
        m2d = [torch.zeros(12000, 3, device="cuda", requires_grad=True) for _ in range(2)]
        outs = rasterize_views(settings, **{k: [per_view[v][k] for v in range(2)] for k in NAMES}, means2D=m2d)
        torch.autograd.backward([outs[v][i] for v in range(2) for i in (1, 3)],
                                [grads[v][j].cuda() for v in range(2) for j in (0, 1)])
        single = fwd_bwd(sc, cam0, deg, grads[0])
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0], single["score"])
    for k in NAMES:
        assert torch.equal(per_view[0][k].grad, single[f"d_{k}"]), k
    assert torch.equal(m2d[0].grad, single["d_means2D"])


def _accuracy(sc, cam, deg, grads, scale_modifier=1.0):
    ref32 = run_oracle(sc, cam, deg, score=True, scale_modifier=scale_modifier, record=True)
    ref = run_oracle(sc, cam, deg, grads=grads, dtype=torch.float64, decisions=ref32["decisions"],
                     scale_modifier=scale_modifier)
    with deterministic():
        det = fwd_bwd(sc, cam, deg, grads, scale_modifier=scale_modifier)
    base = fwd_bwd(sc, cam, deg, grads, scale_modifier=scale_modifier)
    for k in NAMES + ("means2D",):
        assert U.rel_err(det[f"d_{k}"], ref["grads"][k]) < BWD_REL, k
        assert U.rel_err(det[f"d_{k}"], base[f"d_{k}"]) < 1e-5, k
    assert U.rel_err(det["score"], base["score"]) < 1e-5
    assert U.rel_err(det["score"], ref32["score"]) < 1e-4


def test_accuracy_cfg1_full_frame():
    sc, cam, deg = U.make_inputs(10_000, 256, 256)
    _accuracy(sc, cam, deg, grad_inputs(256, 256, 1))


def test_accuracy_screen_filling_gaussians_with_score():
    H, W = 135, 240
    sc, cam, deg = U.make_inputs(3000, H, W, seed=29)
    sc["scales"][:5] = 2.0
    sc["opacities"][:5] = 0.3
    _accuracy(sc, cam, deg, grad_inputs(H, W, 3), scale_modifier=0.7)


def test_dynamic_range_gives_every_gaussian_its_own_scale():
    """Incoming gradients 1e-8 on the left half of the image, 1 on the right: Gaussians that lie only in the left
    half must keep their precision (one global fixed-point scale would flush them to zero)."""
    H = W = 128
    sc, cam, deg = U.make_inputs(3000, H, W, seed=3)
    gc, gd = grad_inputs(H, W, 11)
    gc[:, :, :W // 2] *= 1e-8
    gd[:, :, :W // 2] *= 1e-8
    ref32 = run_oracle(sc, cam, deg, record=True)
    ref = run_oracle(sc, cam, deg, grads=(gc, gd), dtype=torch.float64, decisions=ref32["decisions"])
    with deterministic():
        det = fwd_bwd(sc, cam, deg, (gc, gd), score=False)
    rect = ref32["pre"]["rect"]                                  # [P, 4] tile rect (minx, miny, maxx, maxy)
    left = (ref32["radii"] > 0) & (rect[:, 2] <= (W // 16) // 2)
    assert int(left.sum()) > 50
    for k in ("means3D", "opacities", "scales", "means2D"):
        a = det[f"d_{k}"].cpu().double().reshape(len(left), -1)[left]
        b = ref["grads"][k].double().reshape(len(left), -1)[left]
        assert float(b.abs().max()) < 1e-6                       # these rows only ever saw the small gradients
        rn = b.norm(dim=1)
        keep = rn > 1e-2 * rn.max()
        row_err = (a - b).norm(dim=1)[keep] / rn[keep]
        assert float(row_err.max()) < 1e-4, (k, float(row_err.max()))


def test_headroom_screen_covering_gaussians_large_gradients_1024():
    H = W = 1024
    sc, cam, deg = U.make_inputs(20_000, H, W, seed=13, exact_knn=False)
    sc["scales"][:6] = 2.0
    sc["opacities"][:6] = 0.2
    gc, gd = grad_inputs(H, W, 6)
    grads = (gc * 1e8, gd * 1e8)
    with deterministic():
        det = fwd_bwd(sc, cam, deg, grads)
    base = fwd_bwd(sc, cam, deg, grads)
    assert int((det["radii"][:6] > 0).sum()) == 6
    for k in NAMES + ("means2D",):
        assert bool(torch.isfinite(det[f"d_{k}"]).all()), k
        assert U.rel_err(det[f"d_{k}"], base[f"d_{k}"]) < 1e-5, k


def test_nan_incoming_gradient_stays_non_finite_in_both_modes():
    H = W = 128
    sc, cam, deg = U.make_inputs(3000, H, W, seed=3)
    gc, gd = grad_inputs(H, W, 12)
    gc[1, 64, 64] = float("nan")
    with deterministic():
        det = fwd_bwd(sc, cam, deg, (gc, gd))
    base = fwd_bwd(sc, cam, deg, (gc, gd))
    bad_det = ~torch.isfinite(det["d_means2D"]).all(dim=1)
    bad_base = ~torch.isfinite(base["d_means2D"]).all(dim=1)
    assert int(bad_det.sum()) > 0 and torch.equal(bad_det, bad_base)
    for k in NAMES + ("means2D",):
        a, b = det[f"d_{k}"], base[f"d_{k}"]
        fa = torch.isfinite(a.reshape(a.shape[0], -1)).all(dim=1)
        assert torch.equal(fa, torch.isfinite(b.reshape(b.shape[0], -1)).all(dim=1)), k
        assert U.rel_err(a[fa], b[fa]) < 1e-5, k


def test_disparity_backward_is_repeatable_and_matches_autograd():
    from dreamscene_b200.postprocess import disparity_from_depth_alpha
    from tests.test_gpu_postprocess import _fake_depth_alpha, reference_disparity
    H, W, B = 256, 192, 4
    focals = [1 / (2 * math.tan(f / 2)) for f in (0.55, 0.96, 0.7, 0.96)]
    das = torch.stack([_fake_depth_alpha(H, W, 10 + k, k != 2) for k in range(B)])
    g = torch.Generator(device="cuda").manual_seed(9)
    gd = torch.randn(B, 1, H, W, device="cuda", generator=g)
    ga = torch.randn(B, 1, H, W, device="cuda", generator=g)
    outs = []
    with deterministic():
        for _ in range(3):
            x = das.clone().requires_grad_(True)
            d, a = disparity_from_depth_alpha(x, focals)
            torch.autograd.backward([d, a], [gd, ga])
            outs.append(x.grad)
    assert all(torch.equal(outs[0], o) for o in outs[1:])
    for k in range(B):
        x = das[k].clone().requires_grad_(True)
        d, a = reference_disparity(x, focals[k])
        torch.autograd.backward([d, a], [gd[k], ga[k]])
        err = float((outs[0][k] - x.grad).abs().max() / x.grad.abs().max())
        assert err < 1e-4, (k, err)


def _train_step(seed):
    """A scaled-down DreamScene scene step: assembly -> 4 views -> disparity -> L2 + tv -> backward ->
    densification statistics -> densify_and_prune."""
    from harness import cameras, synthetic
    from dreamscene_b200 import densify
    from dreamscene_b200.multiview import rasterize_views
    from dreamscene_b200.postprocess import disparity_from_depth_alpha
    from dreamscene_b200.scene import assemble_scene
    P, H, W, B = 6000, 96, 96, 4
    sc = synthetic.ball_scene(P, radius=0.5, sh_degree_max=1, seed=seed, opacity="sigmoid_normal", exact_knn=False)
    leaves = {"_xyz": sc["means3D"], "_opacity": torch.logit(sc["opacities"].clamp(1e-4, 1 - 1e-4)),
              "_scaling": sc["scales"].log(), "_rotation": sc["rotations"],
              "_features_dc": sc["shs"][:, :1], "_features_rest": sc["shs"][:, 1:]}
    leaves = {k: v.contiguous().cuda().requires_grad_(True) for k, v in leaves.items()}
    means, opac, scales, rots, shs = assemble_scene([leaves], noise="fused", seed=1234 + seed, views=B)
    cams = [cameras.orbit_camera(radius=3.5, phi_deg=90.0 * v, fovx=0.7, height=H, width=W) for v in range(B)]
    settings = [U.cuda_settings(c, 1) for c in cams]
    m2d = [torch.zeros(P, 3, device="cuda", requires_grad=True) for _ in range(B)]
    outs = rasterize_views(settings, means, opac, shs=[shs[v] for v in range(B)], scales=[scales[v] for v in range(B)],
                           rotations=rots, means2D=m2d)
    das = torch.stack([o[2] for o in outs])
    disp, _ = disparity_from_depth_alpha(das, [1 / (2 * math.tan(0.35))] * B)
    target = torch.linspace(0, 1, 3 * H * W, device="cuda").reshape(3, H, W)
    loss = sum(((o[0] - target) ** 2).mean() for o in outs)
    loss = loss + (disp[..., 1:, :] - disp[..., :-1, :]).abs().mean() + (disp[..., 1:] - disp[..., :-1]).abs().mean()
    loss.backward()
    accum = torch.zeros(P, 1, device="cuda")
    denom = torch.zeros(P, 1, device="cuda")
    maxr = torch.zeros(P, device="cuda")
    for v in range(B):
        densify.add_densification_stats(m2d[v].grad, outs[v][1], accum, denom, maxr)
    g = (accum / denom.clamp_min(1)).reshape(-1)
    thr = float(np.quantile(g.cpu().numpy(), 0.9))
    params = {"xyz": leaves["_xyz"], "f_dc": leaves["_features_dc"], "f_rest": leaves["_features_rest"],
              "opacity": leaves["_opacity"], "scaling": leaves["_scaling"], "rotation": leaves["_rotation"]}
    gen = torch.Generator(device="cuda").manual_seed(77)
    new_p, _, info = densify.densify_and_prune({k: v.detach() for k, v in params.items()}, None, accum, denom, thr,
                                               0.005, 1.0, 20, generator=gen)
    torch.cuda.synchronize()
    result = {f"grad{k}": v.grad.clone() for k, v in leaves.items()}
    result.update({f"m2d{v}": m2d[v].grad.clone() for v in range(B)})
    result.update(accum=accum, denom=denom, maxr=maxr, disp=disp.detach(),
                  **{f"new_{k}": v for k, v in new_p.items()})
    return result, info


def test_scene_train_step_is_bitwise_reproducible_under_torch_determinism():
    with deterministic():
        a, ia = _train_step(0)
        b, ib = _train_step(0)
    assert ia["cloned"] + ia["split_parents"] > 0
    assert (ia["kept"], ia["cloned"], ia["split_parents"], ia["points"]) == (ib["kept"], ib["cloned"], ib["split_parents"], ib["points"])
    assert set(a) == set(b)
    assert_bitwise(a, b)
