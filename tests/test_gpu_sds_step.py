"""The guidance stages' regularisers (DESIGN.md f10): b200gsr_tv_loss / b200gsr_scale_loss and
dreamscene_b200.losses.tv_loss against torch's expressions (harness/regularisers_ref.py), bit for bit in the gradient,
and StepGraph(tv_weight=, tv_depth_weight=, scale_weight=) against the eager guidance step: render_scene +
disparity_from_depth_alpha + the user's loss + the weighted regularisers + backward + GaussianAdam.step()."""
import pytest
import torch

from harness import regularisers_ref as ref
from tests.test_gpu_scene_render import NAMES, _clone, _groups
from tests.test_gpu_step_graph import (_assert_state, _flags, _optimizers, _prune, _schedule, _step_settings,  # noqa: F401
                                       det_mode)

pytestmark = pytest.mark.gpu


def _exact(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def _close(ours, want, rel=1e-6):
    a, b = float(ours.detach()), float(want.detach())
    return abs(a - b) <= rel * abs(b)


def test_torch_forms_the_kernels_reproduce():
    """The rounding forms of csrc/loss.cu's regularisers, pinned against torch's CUDA ops: a tensor divided by a
    Python int is one multiply by the fp32 reciprocal, pow(d, 2)'s backward is g * fp32(2 d) rounded once, the two
    mean backwards are two such reciprocal multiplies, and the tv gradient's terms accumulate as the restated one."""
    g = torch.Generator(device="cuda").manual_seed(0)
    n = 1 << 22
    a = torch.randn(n, device="cuda", generator=g) * torch.exp2(torch.randint(-60, 60, (n,), device="cuda",
                                                                              generator=g).float())
    for d in (1, 2, 3, 4, 3 * 511 * 512, 3 * 512 * 511, 511 * 512, 3 * 36 * 29, 3 * 37 * 28, 2 * 2, 4 * 1200000):
        inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(d), dtype=torch.float32)
        assert torch.equal(a / d, (a.double() * inv.double().cuda()).float()), d
        assert torch.equal(a[:1].reshape(()) / d, (a[0].double() * inv.double().cuda()).float()), d   # 0-dim
    assert torch.equal(2 * a, (2.0 * a.double()).float())
    # PowBackward0: grad * (2 * d), one rounding of the product
    d = torch.randn(n, device="cuda", generator=g) * 30.0
    for go in (1.0, 0.37, 1 / 3, 2.0 ** -70):
        x = d.clone().requires_grad_(True)
        torch.pow(x, 2).sum().backward(torch.tensor(go, device="cuda"))
        assert torch.equal(x.grad, (torch.tensor(go, device="cuda").double() * (2.0 * d).double()).float()), go
    # MeanBackward0 then MeanBackward1
    for rows in (1, 7, 4097, 1200000):
        for lam in torch.rand(16, generator=torch.Generator().manual_seed(rows)).tolist() + [1.0, 0.5, 1 / 3]:
            s = torch.zeros(rows, 3, device="cuda", requires_grad=True)
            ref.scale_loss(s).backward(torch.tensor(lam, device="cuda"))
            l32 = torch.tensor(lam, dtype=torch.float32).double()
            c = ((l32 * (1.0 / torch.tensor(float(rows))).double()).float().double()
                 * (torch.tensor(1.0) / 3.0).double()).float()
            assert torch.equal(s.grad, c.expand(rows, 3).cuda()), (rows, lam)
    # the order of accumulation on CUDA (with CUDA's divisions) is the CPU-pinned one
    x = torch.randn(3, 3, 37, 29, device="cuda", generator=g)
    xg = x.clone().requires_grad_(True)
    ref.tv_loss(xg).backward(torch.tensor(1 / 3, device="cuda"))
    assert _exact(xg.grad, ref.tv_grad(x, torch.tensor(1 / 3, device="cuda")))


def _tv_input(shape, scale, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape, device="cuda", generator=g) * scale
    x.view(-1)[::13] = x.view(-1)[::13].round()           # equal neighbours: differences of zero
    x.view(-1)[5::17] = x.view(-1)[4::17][:x.view(-1)[5::17].numel()]
    return x


@pytest.mark.parametrize("shape", [(4, 3, 512, 512), (4, 1, 512, 512), (2, 3, 37, 29), (1, 1, 2, 2)])
@pytest.mark.parametrize("go", [1.0, 0.5, 0.1, 1 / 3])
@pytest.mark.parametrize("scale", [1e-3, 1.0, 1e3])
def test_tv_loss_equals_torch(shape, go, scale):
    from dreamscene_b200.losses import tv_loss
    x = _tv_input(shape, scale, seed=shape[1] * 1000 + shape[2] + int(go * 100))
    x_ref, x_ours = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    want, ours = ref.tv_loss(x_ref), tv_loss(x_ours)
    assert ours.dtype == torch.float32 and ours.shape == ()
    assert _close(ours, want), (float(ours), float(want))
    want.backward(torch.tensor(go, device="cuda"))
    ours.backward(torch.tensor(go, device="cuda"))
    assert _exact(x_ours.grad, x_ref.grad)
    assert torch.equal(tv_loss(x), ours.detach())          # the fixed-order sum is reproducible


def test_tv_loss_refuses_a_double_backward():
    from dreamscene_b200.losses import tv_loss
    x = _tv_input((1, 3, 16, 16), 1.0, seed=0).requires_grad_(True)
    with pytest.raises(RuntimeError, match="no double backward"):
        torch.autograd.grad(tv_loss(x), x, create_graph=True)
    g, = torch.autograd.grad(tv_loss(x), x)                # a first-order gradient is unaffected
    assert g.shape == x.shape and not g.requires_grad


def test_tv_entry_point_accumulates_and_takes_unaligned_rows():
    """accumulate = 1 adds each gradient with one fp32 add; a base that is not 16-byte aligned takes the scalar path."""
    from dreamscene_b200 import _lib
    lib, ptr = _lib.load(), _lib.ptr
    for shape, off in (((2, 3, 64, 96), 0), ((2, 3, 64, 96), 1), ((1, 2, 33, 40), 3)):
        n = torch.Size(shape).numel()
        buf = _tv_input((n + 4,), 2.0, seed=off)
        x = buf[off:off + n].view(shape)
        dbuf = torch.randn(n + 4, device="cuda")
        d = dbuf[off:off + n].view(shape)
        before = d.clone()
        go = torch.tensor([0.7], device="cuda")
        loss = torch.empty(1, device="cuda")
        scratch = torch.empty(lib.b200gsr_tv_loss_scratch_bytes(*shape), dtype=torch.uint8, device="cuda")
        _lib.check(lib.b200gsr_tv_loss(*shape, ptr(x), ptr(go), ptr(loss), ptr(d), 1, ptr(scratch), scratch.numel(),
                                       _lib.stream(x.device)), "b200gsr_tv_loss")
        xr = x.clone().requires_grad_(True)
        want = ref.tv_loss(xr)
        want.backward(go[0])
        assert _close(loss[0], want), (shape, off, float(loss[0]), float(want))
        assert _exact(d, before + xr.grad), (shape, off)


@pytest.mark.parametrize("lam", [1.0, 0.5, 1 / 3])
@pytest.mark.parametrize("rows,off", [(4 * 1200000, 0), (1000003, 0), (1000003, 1), (5, 3)])
def test_scale_loss_equals_torch(lam, rows, off):
    """rows = 4.8 M: the float4 path only; an odd row count: a scalar tail (3 rows is not a multiple of 4); buffers
    offset by `off` floats from a 16-byte boundary: the scalar path throughout."""
    from dreamscene_b200 import _lib
    lib, ptr = _lib.load(), _lib.ptr
    buf = torch.rand(3 * rows + off, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1)) * 0.05
    s = buf[off:].view(rows, 3)
    sr = s.clone().requires_grad_(True)
    want = ref.scale_loss(sr)
    want.backward(torch.tensor(lam, device="cuda"))
    go = torch.tensor([lam], device="cuda")
    scratch = torch.empty(lib.b200gsr_scale_loss_scratch_bytes(rows), dtype=torch.uint8, device="cuda")
    outs = []
    for acc in (0, 1):
        loss = torch.empty(1, device="cuda")
        d = (torch.randn if acc else torch.empty)(3 * rows + off, device="cuda")[off:].view(rows, 3)
        before = d.clone()
        _lib.check(lib.b200gsr_scale_loss(rows, ptr(s), ptr(go), ptr(loss), ptr(d), acc, ptr(scratch),
                                          scratch.numel(), _lib.stream(s.device)), "b200gsr_scale_loss")
        assert _close(loss[0], want), (float(loss[0]), float(want))
        assert _exact(d, before + sr.grad if acc else sr.grad), acc
        outs.append(loss.clone())
    assert torch.equal(outs[0], outs[1])


# ---- StepGraph ----------------------------------------------------------------------------------------------------
def _user_loss(image, disp, target, wd, scales=None):
    """The guidance stand-in: an L2 on the image plus a term on the disparity (and, given `scales`, one on the
    scales), each output reached by one edge."""
    loss = ((image - target) ** 2).mean() + (wd * disp).sum()
    return loss if scales is None else loss + 0.1 * scales.mean()


def _eager_step(groups, opts, S, seed, shs, sca, target, wd, weights, optimize=True, on_scales=False):
    from dreamscene_b200.postprocess import disparity_from_depth_alpha
    from dreamscene_b200.scene import render_scene
    B, P = len(S), sum(int(g["_xyz"].shape[0]) for g in groups)
    m2d = [torch.zeros(P, 3, device="cuda", requires_grad=True) for _ in range(B)]
    outs, scales = render_scene(groups, S, shs_aug=shs, scale_aug=sca, seed=seed, means2D=m2d, return_scales=True)
    image = torch.stack([o[0] for o in outs])
    disp, _ = disparity_from_depth_alpha(torch.stack([o[2] for o in outs]),
                                         [1.0 / (2.0 * float(s.tanfovx)) for s in S])
    # created before the regularisers: autograd adds its gradient last
    loss = _user_loss(image, disp, target, wd, scales if on_scales else None)
    regs = (ref.tv_loss(image), ref.tv_loss(disp), ref.scale_loss(scales))
    for w, r in zip(weights, regs):
        if w:
            loss = loss + w * r
    loss.backward()
    grads = [{k: g[k].grad.clone() for k in NAMES} for g in groups]
    for opt in opts:
        if optimize:
            opt.step()
        opt.zero_grad()
    return image.detach(), torch.stack([m.grad for m in m2d]), grads, torch.stack([r.detach() for r in regs])


def _graph_step(sg, S, seed, shs, sca, target, wd, optimize=True, on_scales=False):
    out = sg.render(S, shs_aug=shs, scale_aug=sca, seed=seed)
    image, reg = out.image.detach().clone(), sg.reg_loss.clone()
    _user_loss(out.image, out.disp, target, wd, out.scales if on_scales else None).backward()
    sg.step(optimize=optimize)
    return image, sg.d_means2D.clone(), [{k: v.clone() for k, v in d.items()} for d in sg.grads], reg


def _compare(eager, graph, ge, gg, oe, og, weights, exact, step, same_image=None):
    """exact: deterministic mode, everything bit for bit; else the image (bitwise while the parameters are still
    equal, `same_image`) and the state within the non-deterministic tolerances."""
    (ie, me, grads_e, re), (ig, mg, grads_g, rg) = eager, graph
    for k, w in enumerate(weights):
        if w:
            assert _close(rg[k], re[k]), (step, k, float(rg[k]), float(re[k]))
    if exact or same_image:
        assert torch.equal(ie, ig), step
    else:
        torch.testing.assert_close(ig, ie, rtol=1e-3, atol=1e-4)
    if exact:
        assert torch.equal(me, mg), step
        for a, b in zip(grads_e, grads_g):
            assert all(_exact(a[k], b[k]) for k in NAMES), step
    _assert_state(ge, gg, oe, og, exact=exact)


def _setup(sizes, M, B, H, W, weights, seed):
    from dreamscene_b200 import StepGraph
    ge = _groups(sizes, M, seed=seed)
    gg = _clone(ge)
    oe, og = _optimizers(ge), _optimizers(gg)
    sg = StepGraph(gg, og, views=B, height=H, width=W, tv_weight=weights[0], tv_depth_weight=weights[1],
                   scale_weight=weights[2])
    gen = torch.Generator(device="cuda").manual_seed(seed)
    target = torch.rand(B, 3, H, W, device="cuda", generator=gen)
    wd = torch.randn(B, 1, H, W, device="cuda", generator=gen) * 1e-3
    return ge, gg, oe, og, sg, target, wd


@pytest.mark.parametrize("det_mode", [True, False], indirect=True)
@pytest.mark.parametrize("M,sizes,weights", [(16, [3000], (1.0, 1.0, 1.0)), (4, [1500, 1, 700, 0], (1.0, None, 0.5))])
def test_regulariser_steps_equal_the_eager_guidance_steps(det_mode, M, sizes, weights):
    B, H, W = 3, 96, 80
    ge, gg, oe, og, sg, target, wd = _setup(sizes, M, B, H, W, weights, seed=21)
    for step in range(5):
        S = _step_settings(B, H, W, M, step, device="cpu" if step % 2 else "cuda")
        shs, sca = _flags(B, step)
        _schedule(oe, step); _schedule(og, step)
        on_scales = step % 2 == 1       # both backward graphs: adding to the scales' .grad, and writing
        eager = _eager_step(ge, oe, S, 400 + step, shs, sca, target, wd, weights, on_scales=on_scales)
        graph = _graph_step(sg, S, 400 + step, shs, sca, target, wd, on_scales=on_scales)
        _compare(eager, graph, ge, gg, oe, og, weights, exact=det_mode, step=step, same_image=step == 0)
        if not weights[1]:
            assert float(sg.reg_loss[1]) == 0.0
    sg.check()


@pytest.mark.parametrize("det_mode", [True], indirect=True)
def test_backward_only_steps_weight_changes_and_a_prune_recapture(det_mode):
    B, H, W, M = 2, 96, 80, 4
    weights = [1.0, 1.0, 0.5]
    ge, gg, oe, og, sg, target, wd = _setup([900, 400], M, B, H, W, weights, seed=8)
    for step in range(6):
        if step == 2:                                   # a weight change re-captures
            weights = [0.3, 2.0, 1.0]
            sg.tv_weight, sg.tv_depth_weight, sg.scale_weight = weights
        if step == 4:                                   # so does a prune
            mask_of = lambda gr: (gr["_opacity"].detach().reshape(-1) < -1.0)
            ge, gg = _prune(ge, oe, mask_of), _prune(gg, og, mask_of)
            sg.groups = gg
        S = _step_settings(B, H, W, M, step)
        shs, sca = _flags(B, step)
        optimize = step != 3
        on_scales = step in (1, 3, 4)
        eager = _eager_step(ge, oe, S, 60 + step, shs, sca, target, wd, weights, optimize=optimize,
                            on_scales=on_scales)
        graph = _graph_step(sg, S, 60 + step, shs, sca, target, wd, optimize=optimize, on_scales=on_scales)
        _compare(eager, graph, ge, gg, oe, og, weights, exact=True, step=step)
    assert sg.out.radii.shape[1] == sum(int(g["_xyz"].shape[0]) for g in gg) < 1300
    sg.check()
