"""Reserved-row parameter groups (DESIGN.md f13): StepGraph over ReservedGroups (live < capacity, dead rows NaN)
against StepGraph over plain groups cloned from the live prefixes, bit for bit in deterministic mode; densify, prune,
filter and opacity reset in place between replays against the f4 / f5 / reference-expression results, without a
re-capture; and the growth past the capacity, which re-captures exactly once."""
import pytest
import torch

from dreamscene_b200 import GaussianAdam
from dreamscene_b200 import densify as D
from dreamscene_b200 import filtering as F
from dreamscene_b200 import graph as G
from dreamscene_b200.reserve import ReservedGroup
from tests.test_gpu_scene_render import NAMES, _groups, _settings
from tests.test_gpu_step_graph import _flags, _step_settings, _weights, det_mode  # noqa: F401

pytestmark = pytest.mark.gpu

M, H, W = 16, 96, 80
LRS = {"_xyz": 1.6e-4, "_opacity": 0.05, "_scaling": 0.005, "_rotation": 0.001, "_features_dc": 0.0025,
       "_features_rest": 0.000125}
DET = pytest.mark.parametrize("det_mode", [True], indirect=True)


def _get(g, k):
    return g[k] if isinstance(g, dict) else getattr(g, k)


def _reserve(g, cap):
    """A ReservedGroup of the dict group's rows at capacity `cap`, dead leaf rows NaN."""
    r = ReservedGroup.from_tensors(g["_xyz"], g["_features_dc"], g["_features_rest"], g["_opacity"], g["_scaling"],
                                   g["_rotation"], capacity=cap)
    n = r.live_count
    with torch.no_grad():
        for k in NAMES:
            getattr(r, k)[n:] = float("nan")
    return r


def _plain(r):
    """A plain dict group cloned from a reserved group's live prefix."""
    return {k: _get(r.rows(), k).detach().clone().requires_grad_(True) for k in NAMES}


def _opt(g):
    return GaussianAdam([{"params": [_get(g, k)], "lr": LRS[k], "name": k} for k in NAMES], lr=0.0, eps=1e-15)


def _live_cols(x, groups, dim):
    """The live rows (along dim) of a capacity-layout tensor, packed; and the dead ones."""
    live, dead, s = [], [], 0
    for g in groups:
        n = int(_get(g, "_xyz").shape[0])
        k = g.live_count if isinstance(g, ReservedGroup) else n
        live.append(x.narrow(dim, s, k))
        dead.append(x.narrow(dim, s + k, n - k))
        s += n
    return torch.cat(live, dim), torch.cat(dead, dim)


def _bits(t):
    return t.detach().contiguous().view(torch.int32)


def _eq(a, b):
    return torch.equal(_bits(a), _bits(b))


def _loss(out, w):
    return (w[0] * out.image).sum() + (w[1] * out.disp).sum() + 0.3 * out.alpha.mean()


def _step(sg, S, seed, flags, w, target, optimize=True, stats_view=-1):
    shs, sca = flags
    if target is not None:
        sg.render(S, shs_aug=shs, scale_aug=sca, seed=seed, target_index=list(range(len(S))))
    else:
        out = sg.render(S, shs_aug=shs, scale_aug=sca, seed=seed)
        _loss(out, w).backward()
    snap = (sg.out.image.clone(), sg.out.disp.clone(), sg.out.alpha.clone(), sg.out.radii.clone())
    sg.step(optimize=optimize, stats_view=stats_view)
    return snap


def _assert_same_state(rgroups, pgroups, ropts, popts, rdead0):
    """Live parameters and moments equal bitwise; dead parameters unchanged, dead moments still zero."""
    for r, p, ro, po, d0 in zip(rgroups, pgroups, ropts, popts, rdead0):
        for k in NAMES:
            a = _get(r, k)
            n = r.live_count if isinstance(r, ReservedGroup) else a.shape[0]
            assert _eq(a[:n], _get(p, k)), k
            assert _eq(a[n:], d0[k]), k
            if ro is None:
                continue
            sa, sb = ro.state[a], po.state[_get(p, k)]
            assert float(sa["step"]) == float(sb["step"])
            for m in ("exp_avg", "exp_avg_sq"):
                assert _eq(sa[m][:n], sb[m]), (k, m)
                assert not sa[m][n:].any(), (k, m)


CASES = {                          # B, reserved per group, frozen, mode, statistics
    "b1": (1, [True, True], None, None, False),
    "b4_mixed_stats": (4, [True, False], None, None, True),
    "b4_reg": (4, [True, True], None, "reg", False),
    "b4_target": (4, [False, True], None, "target", False),
    "b4_frozen_plain_beside_reserved": (4, [False, True], [True, False], None, True),
}


@DET
@pytest.mark.parametrize("case", list(CASES))
def test_reserved_step_graph_equals_the_plain_one_on_the_live_rows(det_mode, case):
    B, res, frozen, mode, stats = CASES[case]
    base = _groups([900, 700], M, seed=11)
    rg = [_reserve(g, int(g["_xyz"].shape[0]) + 333) if r else {k: v.detach().clone().requires_grad_(True)
                                                                  for k, v in g.items()} for g, r in zip(base, res)]
    pg = [_plain(g) if isinstance(g, ReservedGroup) else {k: v.detach().clone().requires_grad_(True)
                                                          for k, v in g.items()} for g in rg]
    train = [not (frozen and frozen[k]) for k in range(2)]
    ropts = [_opt(g) if t else None for g, t in zip(rg, train)]
    popts = [_opt(g) if t else None for g, t in zip(pg, train)]
    kw = dict(views=B, height=H, width=W, frozen=frozen)
    target = None
    if mode == "reg":
        kw.update(tv_weight=0.5, tv_depth_weight=0.25, scale_weight=2.0)
    if mode == "target":
        target = torch.rand(B, 3, H, W, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
        kw.update(target=target, target_weight=10.0)
    rstats = pstats = None
    if stats:
        rstats = [g if isinstance(g, ReservedGroup) and t else None for g, t in zip(rg, train)]
        pstats = [(torch.zeros(int(g["_xyz"].shape[0]), 1, device="cuda"),
                   torch.zeros(int(g["_xyz"].shape[0]), 1, device="cuda"),
                   torch.zeros(int(g["_xyz"].shape[0]), device="cuda")) if s is not None else None
                  for g, s in zip(pg, rstats)]
    sr = G.StepGraph(rg, [o for o in ropts if o], densify_stats=rstats, **kw)
    sp = G.StepGraph(pg, [o for o in popts if o], densify_stats=pstats, **kw)
    w = _weights(B, H, W)
    dead0 = [{k: _get(g, k)[g.live_count:].detach().clone() if isinstance(g, ReservedGroup)
              else _get(g, k)[:0].detach().clone() for k in NAMES} for g in rg]
    for step in range(3):
        S = _step_settings(B, H, W, M, step)
        flags = _flags(B, step) if step else ([True] * B, [True] * B)
        a = _step(sr, S, 40 + step, flags, w, target)
        b = _step(sp, S, 40 + step, flags, w, target)
        for x, y in zip(a[:3], b[:3]):
            assert _eq(x, y)
        live, dead = _live_cols(a[3], rg, 1)
        assert torch.equal(live, b[3]) and not dead.any()
        if sr.d_means2D is not None:
            live, dead = _live_cols(sr.d_means2D, rg, 1)
            assert _eq(live, sp.d_means2D) and not dead.any()
        for k, (gr, gp) in enumerate(zip(sr.grads, sp.grads)):
            if gr is None:
                assert gp is None
                continue
            for name in NAMES:
                n = rg[k].live_count if isinstance(rg[k], ReservedGroup) else gr[name].shape[0]
                assert _eq(gr[name][:n], gp[name]) and not gr[name][n:].any(), name
        if mode == "reg":
            assert _eq(sr.reg_loss[:2], sp.reg_loss[:2])
            torch.testing.assert_close(sr.reg_loss[2], sp.reg_loss[2], rtol=1e-6, atol=0)
        if mode == "target":
            assert _eq(sr.loss, sp.loss)
        _assert_same_state(rg, pg, ropts, popts, dead0)
        if stats:
            for g, e in zip(rg, pstats):
                if e is not None:
                    n = g.live_count
                    for x, y in zip(g.stats, e):
                        assert _eq(x.view(-1)[:n], y.view(-1)) and not x.view(-1)[n:].any()


# ---- events between replays -----------------------------------------------------------------------------------------
class _CaptureSpy:
    """Counts the captures of each StepGraph instance."""
    def __init__(self, monkeypatch):
        self.counts = {}
        orig = G.StepGraph._capture

        def spy(sg, *a, **k):
            self.counts[id(sg)] = self.counts.get(id(sg), 0) + 1
            return orig(sg, *a, **k)
        monkeypatch.setattr(G.StepGraph, "_capture", spy)

    def of(self, sg):
        return self.counts.get(id(sg), 0)


def _snapshot(g, opt):
    n = g.live_count
    params = {k: getattr(g, _NAME[k])[:n].detach().clone() for k in _NAME}
    adam = {k: tuple(opt.state[getattr(g, _NAME[k])][m][:n].clone() for m in ("exp_avg", "exp_avg_sq")) for k in _NAME}
    stats = {name: t[:n].clone() for name, t in zip(("xyz_gradient_accum", "denom", "max_radii2D"), g.stats)}
    return params, adam, stats


_NAME = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity",
         "scaling": "_scaling", "rotation": "_rotation"}


def _assert_prefix(g, opt, params, adam, stats=None):
    n = g.live_count
    assert n == int(params["xyz"].shape[0])
    for k, leaf in _NAME.items():
        assert _eq(getattr(g, leaf)[:n], params[k]), k
        if adam is not None:
            for m, want in zip(("exp_avg", "exp_avg_sq"), adam[k]):
                assert _eq(opt.state[getattr(g, leaf)][m][:n], want), (k, m)
    assert int(g.live.item()) == n
    for name, t in zip(("xyz_gradient_accum", "denom", "max_radii2D"), g.stats):
        want = torch.zeros(n, device="cuda") if stats is None else stats[name].reshape(-1)
        assert _eq(t.view(-1)[:n], want), name


def _replay_against_fresh(sr, g, opt, S, w):
    """One full step of the reserved graph against a freshly captured plain StepGraph on the live prefix (same
    parameters, moments and step counters)."""
    p = _plain(g)
    po = _opt(p)
    for k in NAMES:
        st = opt.state[getattr(g, k)]
        n = g.live_count
        po.state[p[k]] = {"step": st["step"].clone(), "exp_avg": st["exp_avg"][:n].clone(),
                          "exp_avg_sq": st["exp_avg_sq"][:n].clone()}
    sp = G.StepGraph([p], [po], views=len(S), height=H, width=W,
                     densify_stats=[tuple(t[:g.live_count].clone() for t in g.stats)], keep_means2D=False)
    flags = _flags(len(S), 1)
    a = _step(sr, S, 91, flags, w, None)
    b = _step(sp, S, 91, flags, w, None)
    for x, y in zip(a[:3], b[:3]):
        assert _eq(x, y)
    n = g.live_count
    for k in NAMES:
        assert _eq(getattr(g, k)[:n], p[k]), k
        for m in ("exp_avg", "exp_avg_sq"):
            assert _eq(opt.state[getattr(g, k)][m][:n], po.state[p[k]][m]), (k, m)


def _setup(n, cap, B=2):
    base = _groups([n], M, seed=21)[0]
    g = _reserve(base, cap)
    opt = _opt(g)
    sg = G.StepGraph([g], [opt], views=B, height=H, width=W, densify_stats=[g], keep_means2D=False)
    return g, opt, sg, _weights(B, H, W)


def _warm(sg, g, w, B=2, steps=2):
    """Steps with Adam (creating the moments) and statistics, then one densify-step backward."""
    for step in range(steps):
        _step(sg, _step_settings(B, H, W, M, step), 60 + step, _flags(B, step), w, None)
    _step(sg, _step_settings(B, H, W, M, 5), 70, _flags(B, 5), w, None, optimize=False)


def _densify_expected(g, opt, max_grad, seed):
    params, adam, _ = _snapshot(g, opt)
    n = g.live_count
    new_p, new_a, info = D.densify_and_prune(params, adam, g.xyz_gradient_accum[:n].clone(), g.denom[:n].clone(),
                                             max_grad, 0.005, 5.0, None,
                                             generator=torch.Generator(device="cuda").manual_seed(seed))
    return new_p, new_a, info


def _max_grad(g, q):
    n = g.live_count
    grads = (g.xyz_gradient_accum[:n] / g.denom[:n]).nan_to_num(0.0)
    return float(torch.quantile(grads.view(-1), q))


@DET
def test_events_rewrite_the_prefix_in_place_and_the_next_replay_does_not_capture(det_mode, monkeypatch):
    spy = _CaptureSpy(monkeypatch)
    g, opt, sg, w = _setup(1500, 4000)
    _warm(sg, g, w)
    S = _step_settings(2, H, W, M, 7)
    ptrs = [getattr(g, k).data_ptr() for k in NAMES]
    # densify_and_prune: f4 on the live rows, same z (same generator seed)
    mg = _max_grad(g, 0.7)
    new_p, new_a, info = _densify_expected(g, opt, mg, 3)
    got = g.densify_and_prune(opt, mg, 0.005, 5.0, None, generator=torch.Generator(device="cuda").manual_seed(3))
    assert got["points"] == info["points"] > 1500 and info["cloned"] > 0 and info["split_parents"] > 0
    _assert_prefix(g, opt, new_p, new_a)
    _replay_against_fresh(sg, g, opt, S, w)
    # prune
    mask = torch.rand(g.live_count, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4)) < 0.2
    params, adam, stats = _snapshot(g, opt)
    want_p, want_a, want_s = D.prune_points(params, adam, stats, mask)
    g.prune(mask, opt)
    _assert_prefix(g, opt, want_p, want_a, want_s)
    _replay_against_fresh(sg, g, opt, S, w)
    # filter: the f5 score over rows()
    cams = _settings(3, H, W, degs=[0], seed=9)
    params, adam, stats = _snapshot(g, opt)
    want_p, want_a, want_s = F.gaussian_filtering(params, adam, stats, cams, 0.1, 0.8, 0.3)
    g.filter(opt, cams, 0.1, 0.8, 0.3)
    _assert_prefix(g, opt, want_p, want_a, want_s)
    _replay_against_fresh(sg, g, opt, S, w)
    # reset_opacity: the reference's expression, opacity moments zeroed, step counter kept
    params, adam, stats = _snapshot(g, opt)
    o = params["opacity"]
    m = torch.min(torch.sigmoid(o), torch.ones_like(o) * 0.01)
    params["opacity"] = torch.log(m / (1 - m))
    adam["opacity"] = (torch.zeros_like(o), torch.zeros_like(o))
    step0 = float(opt.state[g._opacity]["step"])
    g.reset_opacity(opt)
    _assert_prefix(g, opt, params, adam, stats)
    assert float(opt.state[g._opacity]["step"]) == step0
    _replay_against_fresh(sg, g, opt, S, w)
    assert [getattr(g, k).data_ptr() for k in NAMES] == ptrs
    assert spy.of(sg) == 1
    sg.check()


@DET
def test_growth_recaptures_once_and_a_doubling_in_capacity_does_not_overflow(det_mode, monkeypatch):
    spy = _CaptureSpy(monkeypatch)
    g, opt, sg, w = _setup(1200, 3000)
    _warm(sg, g, w)
    S = _step_settings(2, H, W, M, 8)
    # an in-capacity event that roughly doubles the live count
    mg = _max_grad(g, 0.02)
    new_p, new_a, info = _densify_expected(g, opt, mg, 5)
    g.densify_and_prune(opt, mg, 0.005, 5.0, None, generator=torch.Generator(device="cuda").manual_seed(5))
    assert 1.7 * 1200 < g.live_count <= 3000
    _assert_prefix(g, opt, new_p, new_a)
    for step in range(3):
        _step(sg, _step_settings(2, H, W, M, 10 + step), 80 + step, _flags(2, step), w, None)
    sg.check()                         # no PairCapacityOverflow
    assert spy.of(sg) == 1
    # an event past the capacity: the group grows (new tensors, optimizer state moved) and re-captures once
    _step(sg, S, 88, _flags(2, 1), w, None, optimize=False)
    mg = _max_grad(g, 0.02)
    new_p, new_a, info = _densify_expected(g, opt, mg, 6)
    assert info["points"] > g.capacity
    g.densify_and_prune(opt, mg, 0.005, 5.0, None, generator=torch.Generator(device="cuda").manual_seed(6))
    assert g.capacity >= info["points"] and all(getattr(g, k).shape[0] == g.capacity for k in NAMES)
    assert [p for gr in opt.param_groups for p in gr["params"]] == [getattr(g, k) for k in NAMES]
    _assert_prefix(g, opt, new_p, new_a)
    _replay_against_fresh(sg, g, opt, S, w)
    _replay_against_fresh(sg, g, opt, S, w)
    assert spy.of(sg) == 2
    sg.check()
