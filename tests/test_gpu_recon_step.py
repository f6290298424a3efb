"""The reconstruction loss (dreamscene_b200.losses.recon_l2_loss, b200gsr_recon_l2) against torch's expression
`l2_loss(image.to(torch.float16), gt) * 100`, and StepGraph's target mode and step(optimize=False) against the eager
refine step of the reference: render_scene without augmentation + that loss + backward + GaussianAdam.step()."""
import math

import pytest
import torch

from tests.test_gpu_scene_render import NAMES, _clone, _groups
from tests.test_gpu_step_graph import _assert_state, _optimizers, _schedule, _step_settings, det_mode  # noqa: F401

pytestmark = pytest.mark.gpu


def _torch_loss(image, target, weight=100.0):
    return ((image.to(torch.float16) - target) ** 2).mean() * weight


def _assert_loss_close(ours, ref):
    assert ours.dtype == ref.dtype and ours.shape == ref.shape
    a, b = float(ours), float(ref)
    if ref.dtype == torch.float16:       # within one fp16 ulp of torch's
        assert abs(a - b) <= 2.0 ** (math.floor(math.log2(abs(b))) - 10), (a, b)
    else:
        assert abs(a - b) <= 1e-6 * abs(b), (a, b)


def test_torch_forms_the_kernel_reproduces():
    """The rounding forms of csrc/loss.cu, pinned against torch's CUDA ops over a few million values: a half tensor
    divided by an integer (mean's backward) is a multiply by the fp32 reciprocal, a half tensor times a Python scalar
    and half - half / half * half are computed in fp32 and rounded once."""
    g = torch.Generator(device="cuda").manual_seed(0)
    n = 1 << 22
    # halves over the whole range, subnormals included
    a = (torch.randn(n, device="cuda", generator=g) * torch.exp2(torch.randint(-26, 12, (n,), device="cuda",
                                                                               generator=g).float())).half()
    b = (torch.randn(n, device="cuda", generator=g) * torch.exp2(torch.randint(-26, 12, (n,), device="cuda",
                                                                               generator=g).float())).half()
    div_differs = []
    for N in (7, 3 * 67 * 45, 3 * 512 * 512, 3 * 1024 * 1024):
        ref = a / N
        inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(N), dtype=torch.float32)
        assert torch.equal(ref, (a.float() * inv.cuda()).half()), N
        f = a.float() * 3.7
        assert torch.equal(f / N, f * inv.cuda()), N          # the fp32 path: reciprocal multiply as well
        true_div = lambda x: x / torch.full_like(x, float(N))  # tensor / tensor: an IEEE division
        div_differs.append((int((ref != true_div(a.float()).half()).sum()), int((f / N != true_div(f)).sum())))
    print("true division differs from torch's div by a scalar (fp16, fp32) on", div_differs, "of", n, "values")
    for w in (100.0, 0.37):
        assert torch.equal(a * w, (a.float() * torch.tensor(w, dtype=torch.float32).item()).half())
    assert torch.equal(a - b, (a.float() - b.float()).half())
    assert torch.equal(a * b, (a.float() * b.float()).half())
    assert torch.equal(2.0 * a, (2.0 * a.float()).half())


def _inputs(shape, dtype, seed):
    """An image in [0,1] and a target close to it at every scale (many gradients are fp16 subnormals), with some
    image values on fp32 -> fp16 rounding ties and some differences on fp16 rounding ties."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = math.prod(shape)
    image = torch.rand(n, device="cuda", generator=g)
    scale = torch.exp2(-torch.rand(n, device="cuda", generator=g) * 20)            # 2^-20 .. 1
    target = image + (torch.rand(n, device="cuda", generator=g) - 0.5) * scale
    k = torch.arange(0, n, 7, device="cuda")
    x16 = image[k].half().float()
    image[k] = x16 + torch.where(x16 >= 1.0, 2.0 ** -11, 2.0 ** -12) * (x16 > 0.5)   # half-way between two halves
    j = torch.arange(3, n, 11, device="cuda")
    image[j] = 1.0 + torch.randint(1, 1023, (j.numel(),), device="cuda", generator=g).float() * 2.0 ** -10
    target[j] = 2.0 ** -11                 # 1 + k 2^-10 - 2^-11: a tie in fp16
    return image.reshape(shape), target.reshape(shape).to(dtype)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("shape", [(3, 67, 45), (3, 512, 512)])
@pytest.mark.parametrize("scale", [None, 0.37])
def test_recon_l2_loss_equals_torch(dtype, shape, scale):
    from dreamscene_b200.losses import recon_l2_loss
    image, target = _inputs(shape, dtype, seed=shape[1] + (dtype == torch.float16))
    x_ref = image.clone().requires_grad_(True)
    x = image.clone().requires_grad_(True)
    ref = _torch_loss(x_ref, target)
    ours = recon_l2_loss(x, target, 100.0)
    _assert_loss_close(ours.detach(), ref.detach())
    if scale is None:
        ref.backward()
        ours.backward()
    else:
        (ref * scale).backward()
        (ours * scale).backward()
    assert torch.equal(x.grad, x_ref.grad)
    nz = x_ref.grad[x_ref.grad != 0].abs()
    if dtype == torch.float16:
        assert (nz < 2.0 ** -14).float().mean() > 0.05        # the inputs do reach the fp16 subnormals
    again = recon_l2_loss(image, target, 100.0)
    assert torch.equal(again, ours.detach())                # the fixed-order sum is reproducible


def test_recon_l2_views_and_device_target_index():
    """B views in one call, the target chosen per view from device memory, against one torch expression per view;
    an unaligned view (N odd) takes the scalar path."""
    from dreamscene_b200 import _lib
    lib, ptr = _lib.load(), _lib.ptr
    for N, dtype in ((3 * 64 * 48, torch.float16), (3 * 33 * 17, torch.float32)):
        B, G = 3, 4
        image, gt = _inputs((B * N,), dtype, seed=N)
        gt = torch.cat([gt, gt.flip(0)])[:G * N].reshape(G, N).contiguous()
        idx = torch.tensor([2, 0, 2], dtype=torch.int32, device="cuda")
        go = torch.tensor([1.0, 0.37, 3.0], device="cuda").to(dtype)
        loss = torch.empty(B, dtype=dtype, device="cuda")
        d = torch.empty(B * N, device="cuda")
        scratch = torch.empty(lib.b200gsr_recon_l2_scratch_bytes(B, N), dtype=torch.uint8, device="cuda")
        _lib.check(lib.b200gsr_recon_l2(B, N, ptr(image), ptr(gt), int(dtype == torch.float16), G, ptr(idx), 100.0,
                                        ptr(go), ptr(loss), ptr(d), ptr(scratch), scratch.numel(),
                                        _lib.stream(image.device)), "b200gsr_recon_l2")
        for v in range(B):
            x = image[v * N:(v + 1) * N].clone().requires_grad_(True)
            ref = _torch_loss(x, gt[int(idx[v])])
            ref.backward(go[v])
            _assert_loss_close(loss[v], ref.detach())
            assert torch.equal(d[v * N:(v + 1) * N], x.grad), (N, v)


def _gts(G, H, W, dtype):
    g = torch.Generator(device="cuda").manual_seed(11)
    return torch.rand(G, 3, H, W, device="cuda", generator=g).to(dtype)


def _eager_refine(groups, opts, S, gt, i, seed, optimize=True):
    """The reference's refine step: render (no augmentation), l2_loss(image.half(), gt[i]) * 100, backward,
    optimizer.step()."""
    from dreamscene_b200.scene import render_scene
    P = sum(int(g["_xyz"].shape[0]) for g in groups)
    m2d = [torch.zeros(P, 3, device="cuda", requires_grad=True)]
    outs = render_scene(groups, S, shs_aug=False, scale_aug=False, seed=seed, means2D=m2d)
    image = outs[0][0]
    loss = _torch_loss(image, gt[i])
    loss.backward()
    for opt in opts:
        if optimize:
            opt.step()
        opt.zero_grad()
    return image.detach(), loss.detach(), outs[0][1], m2d[0].grad


def _graph_refine(sg, S, i, seed, optimize=True):
    out = sg.render(S, shs_aug=False, scale_aug=False, seed=seed, target_index=[i])
    res = (out.image[0].detach().clone(), sg.loss[0].clone(), out.radii[0].clone())
    sg.step(optimize=optimize)
    return res + (sg.d_means2D[0].clone(),)


@pytest.mark.parametrize("det_mode", [True, False], indirect=True)
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("M,sizes", [(16, [3000]), (4, [1500, 1, 700, 0])])
def test_target_mode_steps_equal_the_eager_refine_steps(det_mode, dtype, M, sizes):
    from dreamscene_b200 import StepGraph
    H, W, G = 96, 80, 5
    gt = _gts(G, H, W, dtype)
    ge = _groups(sizes, M, seed=3)
    gg = _clone(ge)
    oe, og = _optimizers(ge), _optimizers(gg)
    sg = StepGraph(gg, og, views=1, height=H, width=W, target=gt, target_weight=100.0)
    for step in range(6):
        S = _step_settings(1, H, W, M, step, device="cpu" if step % 2 else "cuda")   # camera, sh_degree, bg change
        i = (3 * step + 1) % G
        _schedule(oe, step); _schedule(og, step)
        ie, le, re, me = _eager_refine(ge, oe, S, gt, i, 50 + step)
        ig, lg, rg, mg = _graph_refine(sg, S, i, 50 + step)
        assert not sg.out.image.requires_grad and sg.loss.dtype == dtype and sg.loss.shape == (1,)
        if det_mode or step == 0:
            assert torch.equal(ie, ig) and torch.equal(re, rg), step
            _assert_loss_close(lg, le)
        else:
            torch.testing.assert_close(ig, ie, rtol=1e-3, atol=1e-4)
            torch.testing.assert_close(lg.float(), le.float(), rtol=1e-2, atol=0)
        if det_mode:
            assert torch.equal(me, mg), step
        _assert_state(ge, gg, oe, og, exact=det_mode)
    sg.check()


def _snapshot(groups, opts):
    return ([{k: g[k].detach().clone() for k in NAMES} for g in groups],
            [[(float(o.state[p]["step"]), o.state[p]["exp_avg"].clone(), o.state[p]["exp_avg_sq"].clone())
              for gr in o.param_groups for p in gr["params"]] for o in opts])


def _same_snapshot(a, b):
    for x, y in zip(a[0], b[0]):
        assert all(torch.equal(x[k], y[k]) for k in NAMES)
    for x, y in zip(a[1], b[1]):
        for (s1, m1, v1), (s2, m2, v2) in zip(x, y):
            assert s1 == s2 and torch.equal(m1, m2) and torch.equal(v1, v2)


@pytest.mark.parametrize("det_mode", [True], indirect=True)
@pytest.mark.parametrize("target", [False, True])
def test_backward_only_step_leaves_the_state_and_equals_a_normal_steps_gradients(det_mode, target):
    from dreamscene_b200 import StepGraph
    H, W, M, B = 96, 80, 4, (1 if target else 2)
    gt = _gts(3, H, W, torch.float16) if target else None
    w = torch.randn(B, 3, H, W, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    ga = _groups([1200, 500], M, seed=5)
    gb = _clone(ga)
    oa, ob = _optimizers(ga), _optimizers(gb)
    kw = dict(target=gt) if target else {}
    sa = StepGraph(ga, oa, views=B, height=H, width=W, **kw)
    sb = StepGraph(gb, ob, views=B, height=H, width=W, **kw)
    for step in range(3):
        S = _step_settings(B, H, W, M, step)
        res = []
        for sg, optimize in ((sa, True), (sb, False)):
            ti = dict(target_index=[step % 3]) if target else {}
            out = sg.render(S, shs_aug=False, scale_aug=False, seed=9 + step, **ti)
            if not target:
                (w * out.image).sum().backward()
            if not optimize:
                before = _snapshot(gb, ob)          # after render(): the first one creates the optimizer state
            sg.step(optimize=optimize)
            res.append((sg.d_means2D.clone(), [{k: v.clone() for k, v in d.items()} for d in sg.grads]))
        (ma, grads_a), (mb, grads_b) = res
        assert torch.equal(ma, mb), step
        for x, y in zip(grads_a, grads_b):
            assert all(torch.equal(x[k], y[k]) for k in NAMES), step
        _same_snapshot(before, _snapshot(gb, ob))
        # bring b level with a for the next step: the eager GaussianAdam.step() over the graph's gradients is
        # bitwise the Adam graph's
        for g, grads, opt in zip(gb, sb.grads, ob):
            for k in NAMES:
                g[k].grad = grads[k].clone()
            opt.step()
            opt.zero_grad()
        _assert_state(ga, gb, oa, ob, exact=True)


def _densify(groups, opts, accum, denom, seed):
    """densify.densify_and_prune on every group and its optimizer, re-wrapped as the reference's
    densification_postfix does (new leaves, moments carried over, step counters kept)."""
    from dreamscene_b200.densify import densify_and_prune
    pn = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity",
          "scaling": "_scaling", "rotation": "_rotation"}
    out, r0 = [], 0
    for gr, opt in zip(groups, opts):
        n = int(gr["_xyz"].shape[0])
        params = {k: gr[v] for k, v in pn.items()}
        adam = {k: (opt.state[gr[v]]["exp_avg"], opt.state[gr[v]]["exp_avg_sq"]) for k, v in pn.items()}
        steps = {v: opt.state[gr[v]]["step"] for v in pn.values()}
        a, d = accum[r0:r0 + n].contiguous(), denom[r0:r0 + n].contiguous()
        r0 += n
        grad = (a / d.clamp(min=1)).reshape(-1)
        new_p, new_a, _ = densify_and_prune(params, adam, a, d, float(grad.quantile(0.8)), 0.1, 1.0, None,
                                            generator=torch.Generator(device="cuda").manual_seed(seed))
        ng = {pn[k]: torch.nn.Parameter(new_p[k].contiguous()) for k in pn}
        for pg in opt.param_groups:
            k = pg["name"]
            del opt.state[pg["params"][0]]
            pg["params"] = [ng[k]]
            nk = [key for key, val in pn.items() if val == k][0]
            opt.state[ng[k]] = {"step": steps[k], "exp_avg": new_a[nk][0].contiguous(),
                                "exp_avg_sq": new_a[nk][1].contiguous()}
        out.append(ng)
    return out


@pytest.mark.parametrize("det_mode", [True], indirect=True)
def test_a_densify_step_recaptures_and_still_equals_the_eager_refine_steps(det_mode):
    """The reference's order: statistics, densify_and_prune, then an optimizer.step() that updates nothing (the new
    leaves have no gradient) - here step(optimize=False) - and later steps on the new layout."""
    from dreamscene_b200 import StepGraph
    from dreamscene_b200.densify import add_densification_stats
    H, W, M, G = 96, 80, 4, 4
    gt = _gts(G, H, W, torch.float16)
    ge = _groups([900, 400], M, seed=12)
    gg = _clone(ge)
    oe, og = _optimizers(ge), _optimizers(gg)
    sg = StepGraph(gg, og, views=1, height=H, width=W, target=gt)
    P = sum(int(g["_xyz"].shape[0]) for g in ge)
    stats = [(torch.zeros(P, 1, device="cuda"), torch.zeros(P, 1, device="cuda")) for _ in range(2)]
    for step in range(6):
        S = _step_settings(1, H, W, M, step)
        i = step % G
        densify = step == 3
        ie, le, re, me = _eager_refine(ge, oe, S, gt, i, 20 + step, optimize=not densify)
        ig, lg, rg, mg = _graph_refine(sg, S, i, 20 + step, optimize=not densify)
        assert ig.shape == ie.shape and torch.equal(ie, ig) and torch.equal(re, rg) and torch.equal(me, mg), step
        _assert_loss_close(lg, le)
        if step <= 3:
            add_densification_stats(me, re, *stats[0])
            add_densification_stats(sg.d_means2D[0], sg.out.radii[0], *stats[1])
        if densify:
            assert torch.equal(stats[0][0], stats[1][0]) and torch.equal(stats[0][1], stats[1][1])
            ge, gg = _densify(ge, oe, *stats[0], seed=4), _densify(gg, og, *stats[1], seed=4)
            sg.groups = gg
            assert sum(int(g["_xyz"].shape[0]) for g in gg) != P
        _assert_state(ge, gg, oe, og, exact=True)
    assert sg.out.radii.shape[1] == sum(int(g["_xyz"].shape[0]) for g in gg)
    sg.check()
