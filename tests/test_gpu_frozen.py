"""Frozen parameter groups (DESIGN.md f11): render_scene(frozen=) and StepGraph(frozen=) against the unfrozen call and
the eager step.  The forward is untouched; the trainable groups' gradients are those of the unfrozen backward (bit
for bit in deterministic mode), the frozen groups get None and zero means2D rows, and the frozen kernels leave the
saved state as the default ones do."""
import ctypes as C

import pytest
import torch

from harness import regularisers_ref as ref
from tests.test_gpu_recon_step import _torch_loss
from tests.test_gpu_scene_render import NAMES, _clone, _groups, _rel, _settings
from tests.test_gpu_sds_step import _exact, _user_loss
from tests.test_gpu_step_graph import _assert_state, _flags, _optimizers, _schedule, _step_settings, det_mode  # noqa: F401

pytestmark = pytest.mark.gpu


def _render(groups, S, seed, aug, return_scales, frozen, P):
    from dreamscene_b200.scene import render_scene
    B = len(S)
    m2d = [torch.zeros(P, 3, device="cuda", requires_grad=True) for _ in range(B)]
    shs = [aug and v % 2 == 0 for v in range(B)]
    sca = [aug and v % 3 != 1 for v in range(B)]
    res = render_scene(groups, S, shs_aug=shs, scale_aug=sca, seed=seed, means2D=m2d, return_scales=return_scales,
                       frozen=frozen)
    outs, scales = res if return_scales else (res, None)
    return outs, scales, m2d


def _loss(outs, scales, w):
    loss = sum((w[0][v] * o[0]).sum() + (w[1][v] * o[2]).sum() for v, o in enumerate(outs))
    return loss if scales is None else loss + (w[2] * scales).sum()


def _weights(B, P, H, W, seed=3):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(B, 3, H, W, device="cuda", generator=g), torch.randn(B, 2, H, W, device="cuda", generator=g),
            torch.randn(B, P, 3, device="cuda", generator=g))


def _frozen_rows(sizes, frozen):
    rows = torch.zeros(sum(sizes), dtype=torch.bool, device="cuda")
    o = 0
    for n, f in zip(sizes, frozen):
        rows[o:o + n] = f
        o += n
    return rows


# sizes and frozen flags: first, middle, last, all but one; an empty, a 1-row and a non-multiple-of-128 frozen group
CASES = [
    ([1500, 700, 900], [True, False, False]),
    ([1200, 700, 900], [False, True, False]),
    ([1200, 700, 901], [False, False, True]),
    ([600, 700, 900, 300], [True, True, False, True]),
    ([1500, 0, 700, 1, 333], [False, True, False, True, True]),
    ([1, 1500, 333, 700], [True, False, True, False]),
]
CONFIGS = [(1, 4, False, False), (4, 16, True, True), (4, 4, True, False), (1, 16, False, True)]


@pytest.mark.parametrize("config", CONFIGS, ids=lambda c: "B%d-M%d-aug%d-scales%d" % c)
@pytest.mark.parametrize("case", range(len(CASES)))
def test_frozen_render_equals_the_unfrozen_one_on_the_trainable_rows(case, config):
    sizes, frozen = CASES[case]
    B, M, aug, return_scales = config
    H, W, P = 96, 80, sum(sizes)
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        S = _settings(B, H, W, degs=[3, 0, 1] if M == 16 else [1, 0])
        ge = _groups(sizes, M, seed=case)
        gf = _clone(ge)
        w = _weights(B, P, H, W)
        oe, se, me = _render(ge, S, 99, aug, return_scales, None, P)
        of, sf, mf = _render(gf, S, 99, aug, return_scales, frozen, P)
        for a, b in zip(oe, of):
            assert all(torch.equal(x, y) for x, y in zip(a, b))
        if return_scales:
            assert torch.equal(se, sf)
        _loss(oe, se, w).backward()
        _loss(of, sf, w).backward()
        for a, b, f in zip(ge, gf, frozen):
            for k in NAMES:
                if f:
                    assert b[k].grad is None, k
                else:
                    assert _exact(a[k].grad, b[k].grad), k
        rows = _frozen_rows(sizes, frozen)
        for a, b in zip(me, mf):
            assert torch.equal(a.grad[~rows], b.grad[~rows])
            assert torch.equal(b.grad[rows], torch.zeros_like(b.grad[rows]))
    finally:
        torch.use_deterministic_algorithms(old)


@pytest.mark.parametrize("case", [0, 3, 4])
def test_default_mode_trainable_gradients_within_float_atomics(case):
    sizes, frozen = CASES[case]
    B, M, H, W, P = 4, 16, 96, 80, sum(sizes)
    S = _settings(B, H, W)
    ge = _groups(sizes, M, seed=case)
    gf = _clone(ge)
    w = _weights(B, P, H, W)
    oe, se, me = _render(ge, S, 7, True, True, None, P)
    of, sf, mf = _render(gf, S, 7, True, True, frozen, P)
    _loss(oe, se, w).backward()
    _loss(of, sf, w).backward()
    for a, b, f in zip(ge, gf, frozen):
        for k in NAMES:
            if f:
                assert b[k].grad is None
            elif a[k].numel():
                assert _rel(b[k].grad, a[k].grad) < 2e-6, (k, _rel(b[k].grad, a[k].grad))
    rows = _frozen_rows(sizes, frozen)
    for a, b in zip(me, mf):
        assert _rel(b.grad[~rows], a.grad[~rows]) < 2e-6
        assert not b.grad[rows].any()


def test_two_backwards_through_one_frozen_forward_are_equal():
    sizes, frozen = CASES[4]
    B, M, H, W, P = 4, 4, 96, 80, sum(sizes)
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        g = _groups(sizes, M, seed=11)
        outs, scales, m2d = _render(g, _settings(B, H, W, degs=[1]), 5, True, True, frozen, P)
        loss = _loss(outs, scales, _weights(B, P, H, W))
        leaves = [x[k] for x, f in zip(g, frozen) if not f for k in NAMES] + m2d
        first = torch.autograd.grad(loss, leaves, retain_graph=True)
        second = torch.autograd.grad(loss, leaves)
        assert all(_exact(a, b) for a, b in zip(first, second))
    finally:
        torch.use_deterministic_algorithms(old)


def test_c_level_masked_then_unmasked_backward_and_by_value_equals_dyn():
    """One deterministic forward, then over its `saved`: the by-value frozen backward, the _dyn frozen backward (equal
    bitwise), then the plain backward, which must give render_scene's unfrozen gradients bitwise (the frozen ones
    left the saved state clean)."""
    from dreamscene_b200 import _lib, rasterizer as R
    from dreamscene_b200.scene import NOISE_COEF, _group_table, render_scene
    sizes, frozen = [1200, 1, 700, 0, 300], [False, True, True, False, False]
    B, H, W, M, seed = 4, 96, 80, 4, 4321
    mask = sum(1 << k for k, f in enumerate(frozen) if f)
    S = _step_settings(B, H, W, M, 1)
    shs, sca = [True, False, True, False], [False, True, True, False]
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        groups = _groups(sizes, M, seed=8)
        P = sum(sizes)
        m2d = [torch.zeros(P, 3, device="cuda", requires_grad=True) for _ in range(B)]
        outs, scales = render_scene(groups, S, shs_aug=shs, scale_aug=sca, seed=seed, means2D=m2d, return_scales=True)
        wc, wd, ws = _weights(B, P, H, W, seed=9)
        _loss(outs, scales, (wc, wd, ws)).backward()

        lib, ptr, dev = _lib.load(), _lib.ptr, torch.device("cuda")
        flat = [g_[k] for g_ in groups for k in NAMES]
        table = _group_table([flat[6 * k:6 * k + 6] for k in range(len(groups))])
        keep = []
        bg = torch.stack([s.bg.reshape(3) for s in S]).contiguous()
        prm = (_lib.Params * B)(*[R._make_params(s, P, M, keep, dev, bg, v) for v, s in enumerate(S)])
        rec = torch.zeros(B, 8, dtype=torch.float32)
        for v, s in enumerate(S):
            rec[v, :4] = torch.tensor([float(s.tanfovx), float(s.tanfovy), NOISE_COEF if shs[v] else 0.0,
                                       NOISE_COEF if sca[v] else 0.0], dtype=torch.float64)
            rec[v, 4:5].view(torch.int32)[0] = int(s.sh_degree)
        rec = rec.to(dev)
        seed_t = torch.tensor([seed], dtype=torch.int64, device=dev)
        c_shs = (C.c_float * B)(*[NOISE_COEF if f else 0.0 for f in shs])
        c_sca = (C.c_float * B)(*[NOISE_COEF if f else 0.0 for f in sca])
        Hs = _lib.stacked_height(B, H, W)
        cap = R._round_cap(64 * B * P)
        scratch_bytes, saved_bytes = R._layouts(B * P, Hs, W, cap, True, True)
        scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=dev)
        saved = torch.empty(saved_bytes, dtype=torch.uint8, device=dev)
        color, da = torch.empty(3, Hs, W, device=dev), torch.empty(2, Hs, W, device=dev)
        radii, sc_out = torch.empty(B, P, dtype=torch.int32, device=dev), torch.empty(B, P, 3, device=dev)
        st = _lib.stream(dev)
        _lib.check(lib.b200gsr_forward_scene(B, prm, len(groups), table, c_shs, c_sca, seed, ptr(sc_out), ptr(color),
                                             ptr(da), ptr(radii), ptr(scratch), scratch_bytes, ptr(saved),
                                             saved_bytes, cap, _lib.FWD_DETERMINISTIC, None, 0, st),
                   "b200gsr_forward_scene")
        Hp = Hs // B
        g_color, g_da = torch.zeros(3, Hs, W, device=dev), torch.zeros(2, Hs, W, device=dev)
        for v in range(B):
            g_color[:, v * Hp:v * Hp + H] = wc[v]
            g_da[:, v * Hp:v * Hp + H] = wd[v]

        def run(kind):
            grads = [{k: torch.full_like(g_[k], float("nan")) for k in NAMES} for g_ in groups]
            garr = (_lib.GroupGrad * len(groups))()
            for k, gd in enumerate(grads):
                if kind != "plain" and frozen[k]:
                    continue                              # null destinations for the frozen groups
                for name, f in zip(("xyz", "opacity", "scaling", "rotation", "f_dc", "f_rest"), NAMES):
                    setattr(garr[k], name, gd[f].data_ptr() if gd[f].numel() else None)
            d_m2d = torch.full((B, P, 3), float("nan"), device=dev)
            common = (ptr(ws), ptr(radii), ptr(da), ptr(g_color), ptr(g_da), ptr(saved), saved_bytes, cap, ptr(d_m2d),
                      _lib.BWD_DETERMINISTIC)
            if kind == "frozen":
                rc = lib.b200gsr_backward_scene_frozen(B, prm, len(groups), table, garr, c_shs, c_sca, seed, *common,
                                                       mask, st)
            elif kind == "dyn_frozen":
                rc = lib.b200gsr_backward_scene_dyn_frozen(B, prm, len(groups), table, garr, ptr(rec), ptr(seed_t),
                                                           *common, mask, st)
            else:
                rc = lib.b200gsr_backward_scene(B, prm, len(groups), table, garr, c_shs, c_sca, seed, *common, st)
            _lib.check(rc, kind)
            return grads, d_m2d

        fa, ma = run("frozen")
        fb, mb = run("dyn_frozen")
        pa, pm = run("plain")
        rows = _frozen_rows(sizes, frozen)
        want_m2d = torch.stack([m.grad for m in m2d])
        for k, f in enumerate(frozen):
            for name in NAMES:
                if f:
                    assert torch.isnan(fa[k][name]).all() and torch.isnan(fb[k][name]).all()   # never written
                else:
                    assert _exact(fa[k][name], groups[k][name].grad) and _exact(fb[k][name], fa[k][name]), (k, name)
                assert _exact(pa[k][name], groups[k][name].grad), (k, name)
        assert torch.equal(ma, mb) and torch.equal(ma[:, ~rows], want_m2d[:, ~rows])
        assert not ma[:, rows].any()
        assert torch.equal(pm, want_m2d)
    finally:
        torch.use_deterministic_algorithms(old)


# ---- StepGraph ----------------------------------------------------------------------------------------------------
def _eager_guidance(groups, opts, S, seed, shs, sca, target, wd, weights, frozen):
    from dreamscene_b200.postprocess import disparity_from_depth_alpha
    from dreamscene_b200.scene import render_scene
    B, P = len(S), sum(int(g["_xyz"].shape[0]) for g in groups)
    m2d = [torch.zeros(P, 3, device="cuda", requires_grad=True) for _ in range(B)]
    outs, scales = render_scene(groups, S, shs_aug=shs, scale_aug=sca, seed=seed, means2D=m2d, return_scales=True,
                                frozen=frozen)
    image = torch.stack([o[0] for o in outs])
    disp, _ = disparity_from_depth_alpha(torch.stack([o[2] for o in outs]), [1.0 / (2.0 * float(s.tanfovx)) for s in S])
    loss = _user_loss(image, disp, target, wd)
    for w, r in zip(weights, (ref.tv_loss(image), ref.tv_loss(disp), ref.scale_loss(scales))):
        if w:
            loss = loss + w * r
    loss.backward()
    for opt in opts:
        opt.step()
        opt.zero_grad()
    return image.detach(), torch.stack([m.grad for m in m2d])


def _snapshot(groups):
    return [{k: g[k].detach().clone() for k in NAMES} for g in groups]


@pytest.mark.parametrize("det_mode", [True], indirect=True)
@pytest.mark.parametrize("frozen", [[False, True, True, True], [True, False, True, True]], ids=["env", "floor"])
def test_frozen_step_graph_equals_the_eager_frozen_step_with_regularisers(det_mode, frozen):
    """The scene stages: one group trains, the others are frozen; regulariser weights 1 / 0 / 0.5."""
    from dreamscene_b200 import StepGraph
    sizes, M, B, H, W = [2000, 600, 333, 1], 4, 4, 96, 80
    weights = (1.0, None, 0.5)
    ge = _groups(sizes, M, seed=31)
    gg = _clone(ge)
    train = [k for k, f in enumerate(frozen) if not f]
    oe, og = _optimizers([ge[k] for k in train]), _optimizers([gg[k] for k in train])
    sg = StepGraph(gg, og, views=B, height=H, width=W, tv_weight=weights[0], tv_depth_weight=weights[1],
                   scale_weight=weights[2], frozen=frozen)
    gen = torch.Generator(device="cuda").manual_seed(31)
    target = torch.rand(B, 3, H, W, device="cuda", generator=gen)
    wd = torch.randn(B, 1, H, W, device="cuda", generator=gen) * 1e-3
    before = _snapshot(gg)
    for step in range(6):
        S = _step_settings(B, H, W, M, step, device="cpu" if step % 2 else "cuda")
        shs, sca = _flags(B, step)
        _schedule(oe, step); _schedule(og, step)
        ie, me = _eager_guidance(ge, oe, S, 600 + step, shs, sca, target, wd, weights, frozen)
        out = sg.render(S, shs_aug=shs, scale_aug=sca, seed=600 + step)
        ig = out.image.detach().clone()
        _user_loss(out.image, out.disp, target, wd).backward()
        sg.step()
        assert torch.equal(ie, ig) and torch.equal(me, sg.d_means2D), step
        assert all((sg.grads[k] is None) == f for k, f in enumerate(frozen))
        _assert_state([ge[k] for k in train], [gg[k] for k in train], oe, og, exact=True)
    for k, f in enumerate(frozen):
        if f:
            assert all(torch.equal(gg[k][n], before[k][n]) and torch.equal(ge[k][n], before[k][n]) for n in NAMES)
    sg.check()


@pytest.mark.parametrize("det_mode", [True], indirect=True)
def test_frozen_step_graph_target_mode_and_a_mask_change_recaptures(det_mode):
    from dreamscene_b200 import StepGraph
    from dreamscene_b200.scene import render_scene
    sizes, M, H, W, G = [1500, 700, 300], 16, 96, 80, 4
    ge = _groups(sizes, M, seed=41)
    gg = _clone(ge)
    gen = torch.Generator(device="cuda").manual_seed(41)
    gt = torch.rand(G, 3, H, W, device="cuda", generator=gen).half()
    oe, og = _optimizers([ge[1]]), _optimizers([gg[1]])
    frozen = [True, False, True]
    sg = StepGraph(gg, og, views=1, height=H, width=W, target=gt, target_weight=100.0, frozen=frozen)
    before = _snapshot(gg)
    for step in range(6):
        if step == 3:               # group 2 unfrozen (with its optimizer): the next render() re-captures
            frozen = [True, False, False]
            oe, og = _optimizers([ge[1], ge[2]]), _optimizers([gg[1], gg[2]])
            sg.optimizers = og
            sg.frozen = frozen
            graphs = sg._graphs
        S = _step_settings(1, H, W, M, step, device="cpu" if step % 2 else "cuda")
        i = (3 * step + 1) % G
        _schedule(oe, step); _schedule(og, step)
        P = sum(sizes)
        m2d = [torch.zeros(P, 3, device="cuda", requires_grad=True)]
        outs = render_scene(ge, S, shs_aug=False, scale_aug=False, seed=70 + step, means2D=m2d, frozen=frozen)
        _torch_loss(outs[0][0], gt[i]).backward()
        for opt in oe:
            opt.step()
            opt.zero_grad()
        out = sg.render(S, shs_aug=False, scale_aug=False, seed=70 + step, target_index=[i])
        if step == 3:
            assert sg._graphs is not graphs and sg.grads[2] is not None and sg.grads[0] is None
        assert torch.equal(out.image[0], outs[0][0].detach()), step
        sg.step()
        assert torch.equal(sg.d_means2D[0], m2d[0].grad), step
        train = [k for k, f in enumerate(frozen) if not f]
        _assert_state([ge[k] for k in train], [gg[k] for k in train], oe, og, exact=True)
    assert all(torch.equal(gg[0][n], before[0][n]) for n in NAMES)
    sg.check()
