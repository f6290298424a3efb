"""Frozen rows on the two-step scene route: assemble_scene(frozen=) + rasterize_views(frozen_rows=) against the same
calls without freezing.  The forward is untouched; the trainable leaves' gradients and means2D gradients are those of
the unfrozen backward (bit for bit in deterministic mode), frozen leaves get None, frozen rows of leaves passed
straight to rasterize_views get exact zeros, and the frozen kernels leave the saved state as the plain ones do."""
import ctypes as C

import pytest
import torch

from tests.test_gpu_frozen import CASES, _frozen_rows
from tests.test_gpu_scene_render import NAMES, _clone, _groups, _rel, _settings
from tests.test_gpu_sds_step import _exact

pytestmark = pytest.mark.gpu


def _render(groups, S, aug, noise, frozen, P, seed=1234):
    """assemble_scene + rasterize_views, with the frozen groups' rows passed explicitly.  noise="torch" draws from a
    seeded generator, so the frozen and the unfrozen call see the same draws."""
    from dreamscene_b200.multiview import rasterize_views
    from dreamscene_b200.scene import assemble_scene, frozen_rows
    B = len(S)
    gen = torch.Generator(device="cuda").manual_seed(seed) if noise == "torch" else None
    m, o, sc, r, sh = assemble_scene(groups, shs_aug=aug, scale_aug=aug, noise=noise, seed=seed, generator=gen,
                                     views=B, frozen=frozen)
    if B == 1:
        sc, sh = sc[None], sh[None]
    m2d = [torch.zeros(P, 3, device="cuda", requires_grad=True) for _ in range(B)]
    outs = rasterize_views(S, m, o, shs=list(sh.unbind(0)), scales=list(sc.unbind(0)), rotations=r, means2D=m2d,
                           frozen_rows=None if frozen is None else frozen_rows(groups, frozen))
    return outs, sc, m2d


def _loss(outs, scales, w):
    return sum((w[0][v] * o[0]).sum() + (w[1][v] * o[2]).sum() for v, o in enumerate(outs)) + (w[2] * scales).sum()


def _weights(B, P, H, W, seed=3):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(B, 3, H, W, device="cuda", generator=g), torch.randn(B, 2, H, W, device="cuda", generator=g),
            torch.randn(B, P, 3, device="cuda", generator=g))


class _Det:
    def __enter__(self):
        self.old = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(True)

    def __exit__(self, *exc):
        torch.use_deterministic_algorithms(self.old)


CONFIGS = [(1, 4, False, "torch"), (4, 16, True, "torch"), (4, 4, True, "fused"), (1, 16, True, "fused"),
           (4, 16, False, "fused")]


@pytest.mark.parametrize("config", CONFIGS, ids=lambda c: "B%d-M%d-aug%d-%s" % c)
@pytest.mark.parametrize("case", range(len(CASES)))
def test_frozen_two_op_equals_the_unfrozen_one_on_the_trainable_rows(case, config):
    sizes, frozen = CASES[case]
    B, M, aug, noise = config
    H, W, P = 96, 80, sum(sizes)
    with _Det():
        S = _settings(B, H, W, degs=[3, 0, 1] if M == 16 else [1, 0])
        ge = _groups(sizes, M, seed=case)
        gf = _clone(ge)
        w = _weights(B, P, H, W)
        oe, se, me = _render(ge, S, aug, noise, None, P)
        of, sf, mf = _render(gf, S, aug, noise, frozen, P)
        for a, b in zip(oe, of):
            assert all(torch.equal(x, y) for x, y in zip(a, b))
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


# Default mode: float atomics make two unfrozen calls differ too.  Over 60 repeated pairs of these cases (H100), two
# unfrozen calls differed by at most 3.0e-6 (relative) in _rotation - the packed gradient's atomic rounding, amplified
# by the normalisation's projection in the assemble backward - and 1.6e-6 in _scaling, 1.4e-7 in the other leaves;
# the frozen call against an unfrozen one by 3.2e-6 at most.  A wrong row would be off by O(1).
DEFAULT_MODE_REL = 1e-5


@pytest.mark.parametrize("case", [0, 3, 4])
@pytest.mark.parametrize("noise", ["torch", "fused"])
def test_default_mode_trainable_gradients_within_float_atomics(case, noise):
    sizes, frozen = CASES[case]
    B, M, H, W, P = 4, 16, 96, 80, sum(sizes)
    S = _settings(B, H, W)
    ge = _groups(sizes, M, seed=case)
    gf = _clone(ge)
    w = _weights(B, P, H, W)
    oe, se, me = _render(ge, S, True, noise, None, P, seed=7)
    of, sf, mf = _render(gf, S, True, noise, frozen, P, seed=7)
    _loss(oe, se, w).backward()
    _loss(of, sf, w).backward()
    for a, b, f in zip(ge, gf, frozen):
        for k in NAMES:
            if f:
                assert b[k].grad is None
            elif a[k].numel():
                assert _rel(b[k].grad, a[k].grad) < DEFAULT_MODE_REL, (k, _rel(b[k].grad, a[k].grad))
    rows = _frozen_rows(sizes, frozen)
    for a, b in zip(me, mf):
        assert _rel(b.grad[~rows], a.grad[~rows]) < DEFAULT_MODE_REL
        assert not b.grad[rows].any()


def _leaves(P, M, B, seed):
    """Packed rasterizer inputs as leaves: means3D / opacities / rotations shared by the views (their gradients
    accumulate in the kernel), shs and scales one tensor per view."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    shared = {"means3D": r(P, 3) * 0.6, "opacities": torch.sigmoid(r(P, 1) * 2),
              "rotations": torch.nn.functional.normalize(r(P, 4), dim=-1)}
    per_view = {"shs": [r(P, M, 3) * 0.3 for _ in range(B)], "scales": [torch.exp(r(P, 3) * 0.5 - 3.0) for _ in range(B)]}
    leaves = {k: v.contiguous().requires_grad_(True) for k, v in shared.items()}
    leaves.update({k: [t.contiguous().requires_grad_(True) for t in v] for k, v in per_view.items()})
    return leaves


def _clone_leaves(x):
    return {k: ([t.detach().clone().requires_grad_(True) for t in v] if isinstance(v, list) else
                v.detach().clone().requires_grad_(True)) for k, v in x.items()}


def _flat(x):
    return [t for v in x.values() for t in (v if isinstance(v, list) else [v])]


@pytest.mark.parametrize("B,M,ranges", [(1, 16, [(0, 1), (1, 300), (1000, 1129)]), (4, 4, [(0, 1500)]),
                                        (4, 16, [(7, 8), (129, 900), (900, 1300), (2000, 2301)])])
def test_leaves_passed_straight_to_rasterize_views_get_zero_rows(B, M, ranges):
    from dreamscene_b200.multiview import rasterize_views
    P, H, W = 2301, 96, 80
    rows = torch.zeros(P, dtype=torch.bool, device="cuda")
    for lo, hi in ranges:
        rows[lo:hi] = True
    with _Det():
        S = _settings(B, H, W, degs=[3, 1] if M == 16 else [1, 0])
        xe = _leaves(P, M, B, seed=B + M)
        xf = _clone_leaves(xe)
        w = _weights(B, P, H, W, seed=5)
        res = {}
        for name, x, fr in (("plain", xe, None), ("frozen", xf, ranges)):
            m2d = [torch.zeros(P, 3, device="cuda", requires_grad=True) for _ in range(B)]
            outs = rasterize_views(S, x["means3D"], x["opacities"], shs=x["shs"], scales=x["scales"],
                                   rotations=x["rotations"], means2D=m2d, frozen_rows=fr)
            sum((w[0][v] * o[0]).sum() + (w[1][v] * o[2]).sum() for v, o in enumerate(outs)).backward()
            res[name] = (outs, m2d)
        for a, b in zip(res["plain"][0], res["frozen"][0]):
            assert all(torch.equal(p, q) for p, q in zip(a, b))
        for a, b in zip(_flat(xe) + res["plain"][1], _flat(xf) + res["frozen"][1]):
            assert b.grad is not None
            assert torch.equal(b.grad[rows], torch.zeros_like(b.grad[rows]))
            assert not torch.signbit(b.grad[rows]).any()
            assert _exact(a.grad[~rows].contiguous(), b.grad[~rows].contiguous())


def test_frozen_backward_then_plain_backward_over_one_retained_graph():
    """One deterministic forward through rasterize_views; over its saved state the frozen C backward, then the plain
    backward of the retained graph, which must give the unfrozen gradients bit for bit (the frozen kernels left the
    saved state clean).  The frozen call's trainable rows equal them too, and its frozen rows are zeros."""
    from dreamscene_b200 import _lib
    from dreamscene_b200.multiview import rasterize_views
    B, M, P, H, W = 4, 16, 2301, 96, 80
    ranges = [(0, 1), (129, 900), (900, 1301), (2200, 2301)]
    rows = torch.zeros(P, dtype=torch.bool, device="cuda")
    for lo, hi in ranges:
        rows[lo:hi] = True
    with _Det():
        S = _settings(B, H, W)
        x = _leaves(P, M, B, seed=21)
        ref = _clone_leaves(x)
        w = _weights(B, P, H, W, seed=6)

        def fwd(leaves):
            m2d = [torch.zeros(P, 3, device="cuda", requires_grad=True) for _ in range(B)]
            outs = rasterize_views(S, leaves["means3D"], leaves["opacities"], shs=leaves["shs"], scales=leaves["scales"],
                                   rotations=leaves["rotations"], means2D=m2d)
            return outs, m2d, sum((w[0][v] * o[0]).sum() + (w[1][v] * o[2]).sum() for v, o in enumerate(outs))

        _, ref_m2d, ref_loss = fwd(ref)
        ref_loss.backward()
        want = [t.grad for t in _flat(ref) + ref_m2d]

        outs, m2d, loss = fwd(x)
        node = outs[0][0].grad_fn
        while not hasattr(node, "saved_buf"):          # the view of the stacked image -> the rasterize_views node
            node = node.next_functions[0][0]
        _spec, _B, _P, _W, Hs, cap, _wb, _nflat, det, _frozen = node.meta
        assert det and _P == P
        prm, vin = node.views
        radii, depth_alpha = node.saved_tensors[:2]
        Hp = Hs // B
        g_color, g_da = torch.zeros(3, Hs, W, device="cuda"), torch.zeros(2, Hs, W, device="cuda")
        for v in range(B):
            g_color[:, v * Hp:v * Hp + H] = w[0][v]
            g_da[:, v * Hp:v * Hp + H] = w[1][v]
        got = {"means3D": torch.full((P, 3), float("nan"), device="cuda"),
               "opacities": torch.full((P, 1), float("nan"), device="cuda"),
               "rotations": torch.full((P, 4), float("nan"), device="cuda"),
               "shs": [torch.full((P, M, 3), float("nan"), device="cuda") for _ in range(B)],
               "scales": [torch.full((P, 3), float("nan"), device="cuda") for _ in range(B)]}
        d_m2d = [torch.full((P, 3), float("nan"), device="cuda") for _ in range(B)]
        out = (_lib.ViewGrads * B)()
        for v in range(B):
            out[v] = _lib.ViewGrads(got["means3D"].data_ptr(), d_m2d[v].data_ptr(), got["shs"][v].data_ptr(), None,
                                    got["opacities"].data_ptr(), got["scales"][v].data_ptr(),
                                    got["rotations"].data_ptr(), None, 0 if v == 0 else 1 | 2 | 16)
        rr = (_lib.RowRange * len(ranges))(*[_lib.RowRange(lo, hi - lo) for lo, hi in ranges])
        lib, ptr = _lib.load(), _lib.ptr
        rc = lib.b200gsr_backward_views_frozen(B, prm, vin, ptr(radii), ptr(depth_alpha), ptr(g_color), ptr(g_da),
                                               ptr(node.saved_buf), node.saved_buf.numel(), cap, out,
                                               _lib.BWD_DETERMINISTIC, rr, len(ranges), _lib.stream(radii.device))
        _lib.check(rc, "b200gsr_backward_views_frozen")
        for a, b in zip(want, _flat(got) + d_m2d):
            assert torch.equal(b[rows], torch.zeros_like(b[rows]))
            assert _exact(a[~rows].contiguous(), b[~rows].contiguous())
        # the plain backward of the retained graph over the same saved state
        plain = torch.autograd.grad(loss, _flat(x) + m2d, retain_graph=True)
        assert all(_exact(a, b) for a, b in zip(want, plain))
        again = torch.autograd.grad(loss, _flat(x) + m2d)
        assert all(_exact(a, b) for a, b in zip(want, again))


def test_assemble_frozen_with_retain_graph_and_all_but_one_group():
    """Two backwards through one frozen forward are equal, and with every group but one frozen the trained group's
    gradients are the unfrozen ones."""
    sizes, frozen = [600, 700, 900, 300], [True, True, False, True]
    B, M, H, W, P = 4, 4, 96, 80, sum(sizes)
    with _Det():
        S = _settings(B, H, W, degs=[1])
        ge = _groups(sizes, M, seed=11)
        gf = _clone(ge)
        w = _weights(B, P, H, W)
        outs, sc, m2d = _render(gf, S, True, "torch", frozen, P)
        loss = _loss(outs, sc, w)
        leaves = [gf[2][k] for k in NAMES] + m2d
        first = torch.autograd.grad(loss, leaves, retain_graph=True)
        second = torch.autograd.grad(loss, leaves)
        assert all(_exact(a, b) for a, b in zip(first, second))
        oe, se, me = _render(ge, S, True, "torch", None, P)
        _loss(oe, se, w).backward()
        assert all(_exact(ge[2][k].grad, g) for k, g in zip(NAMES, first[:6]))
