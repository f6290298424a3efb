"""Densification statistics gathered inside the backward of the two-step scene route: assemble_scene +
rasterize_views(densify_stats=scene.stats_rows(...)) against the reference's eager route - means2D ports, then one
add_densification_stats per trained group over the last view's gradient and radii.  The statistics are those of
add_densification_stats bit for bit; the leaf and port gradients are those of the call without statistics; without
ports the step stores no screen-space gradient.  Every test runs in default and in deterministic mode."""

import pytest
import torch

from tests.test_gpu_frozen_views import DEFAULT_MODE_REL, _loss, _weights
from tests.test_gpu_scene_render import NAMES, _clone, _groups, _rel, _settings
from tests.test_gpu_sds_step import _exact
from tests.test_gpu_step_graph import det_mode  # noqa: F401

pytestmark = pytest.mark.gpu
DET = pytest.mark.parametrize("det_mode", [False, True], ids=["default", "det"], indirect=True)


def _render(groups, S, noise, frozen, stats, ports, seed=1234, stats_view=-1):
    """assemble_scene + rasterize_views with the frozen groups' rows and the trained groups' statistics records
    passed explicitly; noise="torch" draws from a seeded generator, so every call sees the same draws."""
    from dreamscene_b200.multiview import rasterize_views
    from dreamscene_b200.scene import assemble_scene, frozen_rows, stats_rows
    B, P = len(S), sum(int(g["_xyz"].shape[0]) for g in groups)
    gen = torch.Generator(device="cuda").manual_seed(seed) if noise == "torch" else None
    m, o, sc, r, sh = assemble_scene(groups, noise=noise, seed=seed, generator=gen, views=B, frozen=frozen)
    m2d = [torch.zeros(P, 3, device="cuda", requires_grad=True) for _ in range(B)] if ports else None
    outs = rasterize_views(S, m, o, shs=list(sh.unbind(0)), scales=list(sc.unbind(0)), rotations=r, means2D=m2d,
                           frozen_rows=None if frozen is None else frozen_rows(groups, frozen),
                           densify_stats=None if stats is None else stats_rows(groups, stats), stats_view=stats_view)
    return outs, sc, m2d


def _start(n, seed, with_max=True):
    """Non-trivial starting statistics ([n,1] accum and denom as the reference keeps them, [n] max_radii2D)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.rand(n, 1, device="cuda", generator=g) * 3,
            torch.randint(0, 9, (n, 1), device="cuda", generator=g).float(),
            torch.rand(n, device="cuda", generator=g) * 20 if with_max else None)


def _copy(stats):
    return [None if s is None else tuple(None if t is None else t.clone() for t in s) for s in stats]


def _eager(stats, grad, radii, sizes):
    """The eager route: one add_densification_stats per trained group over its rows of one view's port gradient."""
    from dreamscene_b200.densify import add_densification_stats
    lo = 0
    for n, s in zip(sizes, stats):
        if s is not None and n:
            add_densification_stats(grad[lo:lo + n], radii[lo:lo + n], *s)
        lo += n


def _same(a, b, exact):
    if a is None or b is None:
        return a is None and b is None
    return _exact(a, b) if exact else _rel(a, b) < DEFAULT_MODE_REL


def _assert_stats(got, want, exact=True):
    for k, (a, b) in enumerate(zip(got, want)):
        if a is None:
            assert b is None
            continue
        assert _same(a[0], b[0], exact), k                 # accum: float atomics' rounding across calls (default mode)
        assert _exact(a[1], b[1]) and _same(a[2], b[2], True), k      # denom and max_radii2D come from the radii


# sizes and frozen flags: a trained group between frozen ones; two trained groups (one without max_radii2D) beside a
# frozen and an empty group; every group trained
LAYOUTS = {
    "frozen_beside": ([1500, 700, 900], [True, False, True]),
    "two_trained": ([1200, 1, 0, 700, 901], [False, True, True, False, True]),
    "all_trained": ([1000, 777], None),
}


@DET
@pytest.mark.parametrize("view", [0, -1], ids=["view0", "last"])
@pytest.mark.parametrize("noise", ["torch", "fused"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_statistics_equal_add_densification_stats_over_the_ports(det_mode, layout, noise, view):
    sizes, frozen = LAYOUTS[layout]
    B, M, H, W, P = 4, 16, 96, 80, sum(sizes)
    flags = frozen or [False] * len(sizes)
    S = _settings(B, H, W)
    g = _groups(sizes, M, seed=len(sizes))
    stats = [None if f else _start(n, k, with_max=k != 3) for k, (n, f) in enumerate(zip(sizes, flags))]
    start, want = _copy(stats), _copy(stats)
    outs, sc, m2d = _render(g, S, noise, frozen, stats, ports=True, stats_view=view)
    _loss(outs, sc, _weights(B, P, H, W)).backward()
    v = B - 1 if view == -1 else view
    _eager(want, m2d[v].grad, outs[v][1], sizes)
    _assert_stats(stats, want)
    assert all(s is None or not torch.equal(s[1], t[1]) for s, t in zip(stats, start))    # every record gathered


@DET
@pytest.mark.parametrize("noise", ["torch", "fused"])
@pytest.mark.parametrize("layout", ["frozen_beside", "two_trained"])
def test_gradients_unchanged_and_statistics_equal_without_ports(det_mode, layout, noise):
    """Three calls on clones of one scene: plain (ports, no statistics), ports + statistics, statistics without
    ports.  Every leaf gradient and port gradient is the plain call's (bitwise in deterministic mode, within float
    atomics' rounding otherwise), and the statistics of the two gathering calls agree (bitwise in deterministic mode)."""
    sizes, frozen = LAYOUTS[layout]
    B, M, H, W, P = 4, 16, 96, 80, sum(sizes)
    S = _settings(B, H, W)
    w = _weights(B, P, H, W, seed=9)
    base = _groups(sizes, M, seed=5)
    start = [None if f else _start(n, 40 + k) for k, (n, f) in enumerate(zip(sizes, frozen))]
    runs = {}
    for name, stats, ports in (("plain", None, True), ("ports", _copy(start), True), ("noports", _copy(start), False)):
        g = _clone(base)
        outs, sc, m2d = _render(g, S, noise, frozen, stats, ports)
        _loss(outs, sc, w).backward()
        runs[name] = (g, m2d, stats, outs)
    exact = det_mode
    ref_g, ref_m2d = runs["plain"][:2]
    for name in ("ports", "noports"):
        g = runs[name][0]
        for a, b, f in zip(ref_g, g, frozen):
            for k in NAMES:
                if f:
                    assert b[k].grad is None
                elif a[k].numel():
                    assert _same(b[k].grad, a[k].grad, exact), (name, k)
    for a, b in zip(ref_m2d, runs["ports"][1]):
        assert _same(b.grad, a.grad, exact)
    assert runs["noports"][1] is None
    _assert_stats(runs["noports"][2], runs["ports"][2], exact)
    # and both equal the eager route over the plain call's last-view port gradient
    want = _copy(start)
    _eager(want, ref_m2d[B - 1].grad, runs["plain"][3][B - 1][1], sizes)
    _assert_stats(runs["noports"][2], want, exact)


@DET
def test_no_backward_or_no_view_leaves_the_statistics_untouched_and_retain_graph_adds_twice(det_mode):
    from dreamscene_b200 import _lib
    sizes, frozen = LAYOUTS["frozen_beside"]
    B, M, H, W, P = 4, 4, 96, 80, sum(sizes)
    S = _settings(B, H, W, degs=[1, 0])
    w = _weights(B, P, H, W)
    g = _groups(sizes, M, seed=3)
    stats = [None, _start(sizes[1], 1), None]
    want = _copy(stats)
    # no backward: under no_grad, and a forward whose graph is dropped
    with torch.no_grad():
        _render(g, S, "fused", frozen, stats, ports=False)
    outs, sc, _ = _render(g, S, "fused", frozen, stats, ports=False)
    del outs, sc
    _assert_stats(stats, want)

    # the C entry point with stats_view = -1 gathers nothing (over a plain forward's saved state, without ports)
    outs, sc, m2d = _render(g, S, "fused", frozen, None, ports=True)
    loss = _loss(outs, sc, w)
    node = outs[0][0].grad_fn
    while not hasattr(node, "saved_buf"):          # the view of the stacked image -> the rasterize_views node
        node = node.next_functions[0][0]
    _spec, _B, _P, _W, Hs, cap, _wb, _nflat, det, fz = node.meta
    prm, vin = node.views
    radii, depth_alpha = node.saved_tensors[:2]
    packed = list(node.saved_tensors[2:])
    Hp = Hs // B
    g_color, g_da = torch.zeros(3, Hs, W, device="cuda"), torch.zeros(2, Hs, W, device="cuda")
    for v in range(B):
        g_color[:, v * Hp:v * Hp + H] = w[0][v]
        g_da[:, v * Hp:v * Hp + H] = w[1][v]
    out = (_lib.ViewGrads * B)()
    keep = []
    for v in range(B):
        # the packed inputs in rasterize_views' order: means3D, shs[B], opacities, scales[B], rotations
        d = [torch.zeros_like(packed[i]) for i in (0, 1 + v, 1 + B, 2 + B + v, 2 + 2 * B)]
        keep += d
        out[v] = _lib.ViewGrads(d[0].data_ptr(), None, d[1].data_ptr(), None, d[2].data_ptr(), d[3].data_ptr(),
                                d[4].data_ptr(), None, 0)
    lo = sizes[0]
    rec = (_lib.RowStats * 1)(_lib.RowStats(lo, sizes[1], *[t.data_ptr() for t in stats[1]]))
    rr = (_lib.RowRange * 2)(*[_lib.RowRange(a, n) for a, n in fz])
    ptr = _lib.ptr
    rc = _lib.load().b200gsr_backward_views_stats(
        B, prm, vin, ptr(radii), ptr(depth_alpha), ptr(g_color), ptr(g_da), ptr(node.saved_buf),
        node.saved_buf.numel(), cap, out, _lib.BWD_DETERMINISTIC if det else 0, rr, len(fz), rec, 1, -1,
        _lib.stream(radii.device))
    _lib.check(rc, "b200gsr_backward_views_stats")
    _assert_stats(stats, want)
    del loss

    # a retained graph's second backward adds the statistics a second time
    outs, sc, m2d = _render(g, S, "fused", frozen, stats, ports=True)
    loss = _loss(outs, sc, w)
    g1 = torch.autograd.grad(loss, m2d, retain_graph=True)
    g2 = torch.autograd.grad(loss, m2d)
    _eager(want, g1[B - 1], outs[B - 1][1], sizes)
    _eager(want, g2[B - 1], outs[B - 1][1], sizes)
    _assert_stats(stats, want)


@DET
def test_without_ports_the_step_peak_memory_drops(det_mode):
    """One step of the eager route (B means2D ports, then add_densification_stats) against one step that gathers in
    the backward without ports: the peak allocation drops by at least the B [P,3] float32 ports, B P 12 bytes."""
    sizes, frozen = [150000, 60000, 90000], [True, False, True]
    B, M, H, W, P = 4, 16, 256, 256, sum(sizes)
    S = _settings(B, H, W)
    w = _weights(B, P, H, W)
    g = _groups(sizes, M, seed=8)
    stats = [None, _start(sizes[1], 2), None]

    def step(backward):
        for grp in g:
            for t in grp.values():
                t.grad = None
        outs, sc, m2d = _render(g, S, "torch", frozen, stats if backward else None, ports=not backward)
        _loss(outs, sc, w).backward()
        if not backward:
            _eager(stats, m2d[B - 1].grad, outs[B - 1][1], sizes)

    peaks = {}
    for rep in range(2):
        for backward in (False, True):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            step(backward)
            torch.cuda.synchronize()
            peaks[backward] = torch.cuda.max_memory_allocated() - base
    assert peaks[False] - peaks[True] >= B * P * 12, peaks


@DET
@pytest.mark.parametrize("noise", ["torch", "fused"])
def test_scene_stages_reproduce_the_reference_slicing_on_the_last_view(det_mode, noise):
    """The scene stages in order - env, floor, both - on groups packed [object, floor, env], statistics accumulating
    across the stages.  Eager: ports, then the reference's slices of the last view (env at -len_env:, floor at
    -len_env - len_floor:-len_env).  In the backward: stats_rows of the trained groups, no ports."""
    from dreamscene_b200.densify import add_densification_stats
    names = ["object", "floor", "env"]
    sizes = [1300, 500, 900]
    B, M, H, W, P = 4, 16, 96, 80, sum(sizes)
    S = _settings(B, H, W)
    w = _weights(B, P, H, W, seed=4)
    ge = _groups(sizes, M, seed=12)
    gb = _clone(ge)
    se = {n: _start(k, 60 + i) for i, (n, k) in enumerate(zip(names, sizes))}
    sb = {n: tuple(t.clone() for t in s) for n, s in se.items()}
    len_env, len_floor = sizes[2], sizes[1]
    slices = {"env": slice(-len_env, None), "floor": slice(-len_env - len_floor, -len_env)}
    for stage, trained in enumerate((["env"], ["floor"], ["env", "floor"])):
        frozen = [n not in trained for n in names]
        outs, sc, m2d = _render(ge, S, noise, frozen, None, ports=True, seed=100 + stage)
        _loss(outs, sc, w).backward()
        for n in trained:
            add_densification_stats(m2d[B - 1].grad[slices[n]], outs[B - 1][1][slices[n]], *se[n])
        outs, sc, m2d = _render(gb, S, noise, frozen, [sb[n] if n in trained else None for n in names], ports=False,
                                seed=100 + stage)
        assert m2d is None
        _loss(outs, sc, w).backward()
        _assert_stats([sb[n] for n in names], [se[n] for n in names], exact=det_mode)
