"""Densification statistics inside the scene backward and the replayed step (DESIGN.md f12): render_scene(densify_stats=)
and StepGraph(densify_stats=, keep_means2D=) against densify.add_densification_stats over the same call's stored
screen-space gradient and radii (bit for bit), against a torch restatement of the reference's formula, and across
replays, re-captures and the frozen-group refusal.  Three groups: 0 frozen, 1 gathers statistics, 2 trains without."""
import pytest
import torch

from dreamscene_b200 import densify
from tests.test_gpu_scene_render import NAMES, _clone, _groups
from tests.test_gpu_step_graph import _assert_state, _flags, _optimizers, _schedule, _step_settings, det_mode  # noqa: F401

pytestmark = pytest.mark.gpu

SIZES, FROZEN, B, M, H, W = [1200, 1500, 700], [True, False, False], 3, 16, 96, 80
ROWS = (1200, 2700)                     # group 1's packed rows
MODES = pytest.mark.parametrize("det_mode", [True, False], indirect=True)


def _init_stats(n, seed):
    """Non-trivial starting values: accum > 0, whole-number denom, max_radii2D around the radii's range."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.rand(n, 1, device="cuda", generator=g) * 1e-3, torch.randint(0, 5, (n, 1), device="cuda",
            generator=g).float(), torch.randint(0, 12, (n,), device="cuda", generator=g).float())


def _copy(st):
    return tuple(t.clone() for t in st)


def _eager(st, grad_rows, radii_rows):
    want = _copy(st)
    densify.add_densification_stats(grad_rows, radii_rows, *want)
    return want


def _torch_reference(st, grad_rows, radii_rows):
    """The reference's add_densification_stats (gs_renderer.py) and max_radii2D update, in torch."""
    accum, denom, mx = _copy(st)
    vis = radii_rows > 0
    accum[vis] += torch.norm(grad_rows[vis, :2], dim=-1, keepdim=True)
    denom[vis] += 1
    mx[vis] = torch.max(mx[vis], radii_rows[vis].float())
    return accum, denom, mx


def _equal(a, b):
    return all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(a, b))


def _loss(outs, seed=3):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return sum((torch.randn(o[0].shape, device="cuda", generator=g) * o[0]).sum() +
               (torch.randn(o[2].shape, device="cuda", generator=g) * o[2]).sum() for o in outs)


def _render(groups, S, stats, view, ports=True, frozen=FROZEN):
    from dreamscene_b200.scene import render_scene
    P = sum(SIZES)
    m2d = [torch.zeros(P, 3, device="cuda", requires_grad=True) for _ in range(B)] if ports else None
    outs = render_scene(groups, S, shs_aug=[True, False, True], scale_aug=[False, True, True], seed=77, means2D=m2d,
                        frozen=frozen, densify_stats=None if stats is None else [None, stats, None],
                        stats_view=view)
    _loss(outs).backward()
    return outs, m2d


@MODES
@pytest.mark.parametrize("view", [-1, 0])
def test_render_scene_statistics_equal_add_densification_stats(det_mode, view):
    S = _step_settings(B, H, W, M, 2)
    ga = _groups(SIZES, M, seed=5)
    gb, gc = _clone(ga), _clone(ga)
    init = _init_stats(SIZES[1], 9)
    st = _copy(init)
    outs, m2d = _render(ga, S, st, view)
    v = B - 1 if view == -1 else view
    a, b = ROWS
    grad, radii = m2d[v].grad[a:b], outs[v][1][a:b]
    assert int((radii > 0).sum()) > 100
    assert _equal(st, _eager(init, grad, radii))
    # the reference's formula: denom and max_radii2D exact; accum within two ulps - torch.norm rounds the square sum
    # without a fused multiply-add (one ulp of the norm), and the single addition rounds once more
    ra, rd, rm = _torch_reference(init, grad, radii)
    assert torch.equal(st[1], rd) and torch.equal(st[2], rm)
    ulp = torch.nextafter(ra.abs(), torch.full_like(ra, float("inf"))) - ra.abs()
    assert bool(((st[0] - ra).abs() <= 2 * ulp).all()), float(((st[0] - ra).abs() / ulp).max())
    # without means2D ports: no screen-space gradient is stored, the statistics are the same
    st2 = _copy(init)
    _render(gb, S, st2, view, ports=False)
    if det_mode:
        assert _equal(st2, st)
    # gradients and d_means2D as the frozen-only call (bit for bit in deterministic mode)
    _, m2d_c = _render(gc, S, None, view)
    if det_mode:
        for x, y, f in zip(ga, gc, FROZEN):
            for k in NAMES:
                assert (x[k].grad is None) if f else torch.equal(x[k].grad, y[k].grad), k
        for x, y in zip(ga, gb):
            for k in NAMES:
                assert (x[k].grad is None) == (y[k].grad is None) and (x[k].grad is None or torch.equal(x[k].grad, y[k].grad))
        assert all(torch.equal(x.grad, y.grad) for x, y in zip(m2d, m2d_c))


def test_retain_graph_adds_twice():
    from dreamscene_b200.scene import render_scene
    S = _step_settings(B, H, W, M, 1)
    g = _groups(SIZES, M, seed=6)
    init = _init_stats(SIZES[1], 4)
    st = _copy(init)
    m2d = [torch.zeros(sum(SIZES), 3, device="cuda", requires_grad=True) for _ in range(B)]
    outs = render_scene(g, S, seed=3, means2D=m2d, frozen=FROZEN, densify_stats=[None, st, None])
    loss = _loss(outs)
    g1 = torch.autograd.grad(loss, m2d, retain_graph=True)
    first = _copy(st)
    gm = torch.autograd.grad(loss, m2d)
    a, b = ROWS
    assert _equal(first, _eager(init, g1[B - 1][a:b], outs[B - 1][1][a:b]))
    assert _equal(st, _eager(first, gm[B - 1][a:b], outs[B - 1][1][a:b]))


def _graph_setup(keep, seed=31):
    from dreamscene_b200 import StepGraph
    g = _groups(SIZES, M, seed=seed)
    opts = _optimizers(g[1:])
    st = _init_stats(SIZES[1], 12)
    sg = StepGraph(g, opts, views=B, height=H, width=W, frozen=FROZEN, densify_stats=[None, st, None],
                   keep_means2D=keep)
    return g, opts, st, sg


def _graph_step(sg, opts, step, view, optimize=True):
    S = _step_settings(B, H, W, M, step, device="cpu" if step % 2 else "cuda")
    shs, sca = _flags(B, step)
    _schedule(opts, step)
    out = sg.render(S, shs_aug=shs, scale_aug=sca, seed=500 + step)
    gen = torch.Generator(device="cuda").manual_seed(step)
    ((torch.randn(out.image.shape, device="cuda", generator=gen) * out.image).sum() + out.disp.mean()).backward()
    sg.step(optimize=optimize, stats_view=view)
    return out


@MODES
def test_step_graph_statistics_follow_the_view_without_recapture(det_mode):
    g, opts, st, sg = _graph_setup(True)
    graphs = None
    a, b = ROWS
    for step, (view, optimize) in enumerate([(-1, True), (0, True), (None, True), (-1, False)]):
        before = _copy(st)
        out = _graph_step(sg, opts, step, view, optimize)
        if graphs is None:
            graphs = sg._graphs
        assert sg._graphs is graphs, step                  # no re-capture
        if view is None:
            assert _equal(st, before), step
        else:
            v = B - 1 if view == -1 else view
            assert _equal(st, _eager(before, sg.d_means2D[v, a:b], out.radii[v, a:b])), step
    sg.check()


@pytest.mark.parametrize("det_mode", [True], indirect=True)
def test_keep_means2D_false_same_state_less_memory(det_mode):
    import gc
    P = sum(SIZES)

    def run(keep):
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        g, opts, st, sg = _graph_setup(keep)
        for step in range(4):
            _graph_step(sg, opts, step, -1)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        assert (sg.d_means2D is None) == (not keep)
        res = ([{k: x[k].detach().clone() for k in NAMES} for x in g], opts, _copy(st), peak)
        del sg
        return res

    run(True)                                           # warm-up: library and allocator set-up
    gk, ok, sk, peak_keep = run(True)
    gn, on, sn, peak_none = run(False)
    assert _equal(sk, sn)
    for x, y in zip(gk, gn):
        assert all(torch.equal(x[k], y[k]) for k in NAMES)
    for oa, ob in zip(ok, on):
        for pa, pb in zip([p for grp in oa.param_groups for p in grp["params"]],
                          [p for grp in ob.param_groups for p in grp["params"]]):
            assert torch.equal(oa.state[pa]["exp_avg"], ob.state[pb]["exp_avg"])
            assert torch.equal(oa.state[pa]["exp_avg_sq"], ob.state[pb]["exp_avg_sq"])
    assert peak_keep - peak_none >= B * P * 12, (peak_keep, peak_none)


@pytest.mark.parametrize("det_mode", [True], indirect=True)
def test_densify_replaces_leaves_and_statistics_and_recaptures(det_mode):
    from dreamscene_b200 import GaussianAdam
    g, opts, st, sg = _graph_setup(False)
    for step in range(2):
        _graph_step(sg, opts, step, -1)
    graphs = sg._graphs
    names = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity",
             "scaling": "_scaling", "rotation": "_rotation"}
    params = {k: g[1][v].detach() for k, v in names.items()}
    new_p, _, info = densify.densify_and_prune(params, None, st[0], st[1], max_grad=float(st[0].div(st[1]).nanmedian()),
                                               min_opacity=0.005, extent=1.0, max_screen_size=None,
                                               generator=torch.Generator(device="cuda").manual_seed(1))
    n = info["points"]
    assert n != SIZES[1]
    old = _copy(st)
    g[1] = {v: new_p[k].contiguous().requires_grad_(True) for k, v in names.items()}
    new_st = (info["xyz_gradient_accum"], info["denom"], info["max_radii2D"])
    sg.groups = g
    sg.optimizers = [GaussianAdam([{"params": [g[1][k]], "lr": 1e-3, "name": k} for k in NAMES], lr=0.0, eps=1e-15),
                     opts[1]]
    sg.densify_stats = [None, new_st, None]
    S = _step_settings(B, H, W, M, 5)
    out = sg.render(S, seed=9)
    assert sg._graphs is not graphs
    out.image.sum().backward()
    sg.step(stats_view=-1)
    assert _equal(st, old)                                # the replaced tensors are left alone
    assert int(new_st[1].sum()) == int((out.radii[B - 1, SIZES[0]:SIZES[0] + n] > 0).sum()) > 0
    sg.check()


def test_frozen_group_statistics_are_refused_before_capture():
    from dreamscene_b200 import StepGraph
    from dreamscene_b200.scene import render_scene
    g = _groups(SIZES, M, seed=2)
    st = _init_stats(SIZES[0], 1)
    with pytest.raises(ValueError, match="frozen group 0"):
        StepGraph(g, _optimizers(g[1:]), views=B, height=H, width=W, frozen=FROZEN, densify_stats=[st, None, None])
    with pytest.raises(ValueError, match="frozen group 0"):
        render_scene(g, _step_settings(B, H, W, M, 0), frozen=FROZEN, densify_stats=[st, None, None])
