"""StepGraph (dreamscene_b200.graph): a training step replayed from two CUDA graphs against the eager step it replaces,
render_scene + disparity_from_depth_alpha + the same loss + backward + GaussianAdam.step(), with every per-step value
(cameras, FoV, augmentation flags, sh_degree, bg, seed, lr) changing between steps."""
import ctypes as C

import pytest
import torch

from harness import cameras
from tests import util_scene as U
from tests.test_gpu_scene_render import NAMES, _clone, _groups

pytestmark = pytest.mark.gpu


@pytest.fixture
def det_mode(request):
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(request.param)
    yield request.param
    torch.use_deterministic_algorithms(old)


def _step_settings(B, H, W, M, step, device="cuda"):
    """Per-step cameras: orbit position, two alternating FoVs, a degree-0 view and per-view bg (camera tensors on
    `device`)."""
    g = torch.Generator().manual_seed(100 + step)
    degs = [d for d in range(4) if (d + 1) ** 2 <= M]
    out = []
    for v in range(B):
        cam = cameras.orbit_camera(radius=3.5, theta_deg=50.0 + 7 * v + 3 * step, phi_deg=37.0 * v + 11 * step,
                                   fovx=0.5 if (v + step) % 2 else 0.7, height=H, width=W)
        deg = 0 if v == 1 else degs[(v + step) % len(degs)]
        bg = tuple(float(x) for x in torch.rand(3, generator=g))
        out.append(U.cuda_settings(cam, deg, bg=bg, device=device))
    return out


def _optimizers(groups):
    from dreamscene_b200 import GaussianAdam
    lrs = {"_xyz": 1.6e-4, "_opacity": 0.05, "_scaling": 0.005, "_rotation": 0.001, "_features_dc": 0.0025,
           "_features_rest": 0.000125}
    return [GaussianAdam([{"params": [g[k]], "lr": lrs[k], "name": k} for k in NAMES], lr=0.0, eps=1e-15)
            for g in groups]


def _schedule(opts, step):
    for opt in opts:                      # update_learning_rate: the xyz lr changes every step
        opt.param_groups[0]["lr"] = 1.6e-4 * (0.9 ** step)


def _weights(B, H, W):
    g = torch.Generator(device="cuda").manual_seed(7)
    return (torch.randn(B, 3, H, W, device="cuda", generator=g), torch.randn(B, 1, H, W, device="cuda", generator=g))


def _loss(image, disp, alpha, scales, w):
    tv = (image[..., 1:, :] - image[..., :-1, :]).abs().mean() + (image[..., :, 1:] - image[..., :, :-1]).abs().mean()
    return (w[0] * image).sum() + (w[1] * disp).sum() + 0.3 * alpha.mean() + 0.1 * tv + 3.0 * scales.mean()


def _flags(B, step):
    return [(v + step) % 3 != 0 for v in range(B)], [(v + step) % 2 == 0 for v in range(B)]


def _eager_step(groups, opts, S, seed, shs, sca, w):
    from dreamscene_b200.postprocess import disparity_from_depth_alpha
    from dreamscene_b200.scene import render_scene
    B, P = len(S), sum(int(g["_xyz"].shape[0]) for g in groups)
    m2d = [torch.zeros(P, 3, device="cuda", requires_grad=True) for _ in range(B)]
    outs, scales = render_scene(groups, S, shs_aug=shs, scale_aug=sca, seed=seed, means2D=m2d, return_scales=True)
    image = torch.stack([o[0] for o in outs])
    radii = torch.stack([o[1] for o in outs])
    disp, alpha = disparity_from_depth_alpha(torch.stack([o[2] for o in outs]),
                                             [1.0 / (2.0 * float(s.tanfovx)) for s in S])
    _loss(image, disp, alpha, scales, w).backward()
    for opt in opts:
        opt.step()
        opt.zero_grad()
    return image.detach(), disp.detach(), radii, torch.stack([m.grad for m in m2d])


def _graph_step(sg, S, seed, shs, sca, w):
    out = sg.render(S, shs_aug=shs, scale_aug=sca, seed=seed)
    res = (out.image.detach().clone(), out.disp.detach().clone(), out.radii.clone())
    _loss(out.image, out.disp, out.alpha, out.scales, w).backward()
    sg.step()
    return res + (sg.d_means2D.clone(),)


def _assert_state(ge, gg, oe, og, exact):
    for a, b in zip(ge, gg):
        for k in NAMES:
            if exact:
                assert torch.equal(a[k], b[k]), k
            else:
                torch.testing.assert_close(b[k], a[k], rtol=1e-3, atol=1e-5)
    for x, y in zip(oe, og):
        for p, q in zip([p for gr in x.param_groups for p in gr["params"]], [q for gr in y.param_groups for q in gr["params"]]):
            se, sg_ = x.state[p], y.state[q]
            assert float(se["step"]) == float(sg_["step"])
            if exact:
                assert torch.equal(se["exp_avg"], sg_["exp_avg"]) and torch.equal(se["exp_avg_sq"], sg_["exp_avg_sq"])


@pytest.mark.parametrize("det_mode", [True, False], indirect=True)
@pytest.mark.parametrize("M,sizes", [(16, [3000]), (4, [1500, 1, 700, 0])])
def test_replayed_steps_equal_the_eager_steps(det_mode, M, sizes):
    from dreamscene_b200 import StepGraph
    B, H, W = 4, 96, 80
    ge, gg = _groups(sizes, M, seed=1), None
    gg = _clone(ge)
    oe, og = _optimizers(ge), _optimizers(gg)
    sg = StepGraph(gg, og, views=B, height=H, width=W)
    w = _weights(B, H, W)
    for step in range(6):
        S = _step_settings(B, H, W, M, step, device="cpu" if step % 2 else "cuda")   # both upload paths
        shs, sca = _flags(B, step)
        _schedule(oe, step); _schedule(og, step)
        ie, de, re, me = _eager_step(ge, oe, S, 1234 + step, shs, sca, w)
        ig, dg, rg, mg = _graph_step(sg, S, 1234 + step, shs, sca, w)
        if det_mode or step == 0:          # default mode: the parameters differ within tolerance after one backward
            assert torch.equal(ie, ig) and torch.equal(re, rg), step
        else:
            torch.testing.assert_close(ig, ie, rtol=1e-3, atol=1e-4)
        if det_mode:
            assert torch.equal(de, dg) and torch.equal(me, mg), step
        _assert_state(ge, gg, oe, og, exact=det_mode)
    sg.check()


@pytest.mark.parametrize("M,sizes", [(16, [2500]), (4, [1200, 1, 600, 0, 300])])
def test_dyn_entry_points_equal_the_by_value_ones(M, sizes):
    """b200gsr_forward_scene_dyn / b200gsr_backward_scene_dyn called directly, with host tanfov / sh_degree set to
    values they must ignore, against render_scene (b200gsr_forward_scene / _backward_scene) for the same per-view
    values: images, depth_alpha, radii and scales bitwise; in deterministic mode the leaf gradients and d_means2D too.
    Mixed per-view flags, a degree-0 view and two FoVs."""
    from dreamscene_b200 import _lib, rasterizer as R
    from dreamscene_b200.scene import NOISE_COEF, _group_table, render_scene
    B, H, W, seed = 4, 96, 80, 4321
    S = _step_settings(B, H, W, M, 1)
    assert len({round(float(s.tanfovx), 6) for s in S}) == 2 and any(int(s.sh_degree) == 0 for s in S)
    shs, sca = [True, False, True, False], [False, True, True, False]
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        groups = _groups(sizes, M, seed=8)
        P = sum(sizes)
        m2d = [torch.zeros(P, 3, device="cuda", requires_grad=True) for _ in range(B)]
        outs, scales = render_scene(groups, S, shs_aug=shs, scale_aug=sca, seed=seed, means2D=m2d, return_scales=True)
        g = torch.Generator(device="cuda").manual_seed(9)
        wc, wd, ws = (torch.randn(B, 3, H, W, device="cuda", generator=g), torch.randn(B, 2, H, W, device="cuda", generator=g),
                      torch.randn(B, P, 3, device="cuda", generator=g))
        (sum((wc[v] * o[0]).sum() + (wd[v] * o[2]).sum() for v, o in enumerate(outs)) + (ws * scales).sum()).backward()

        lib, ptr, dev = _lib.load(), _lib.ptr, torch.device("cuda")
        flat = [g_[k] for g_ in groups for k in NAMES]
        table = _group_table([flat[6 * k:6 * k + 6] for k in range(len(groups))])
        keep = []
        bg = torch.stack([s.bg.reshape(3) for s in S]).contiguous()
        prm = (_lib.Params * B)(*[R._make_params(s._replace(tanfovx=9.0, tanfovy=9.0, sh_degree=3), P, M, keep, dev,
                                                 bg, v) for v, s in enumerate(S)])
        rec = torch.zeros(B, 8, dtype=torch.float32, device="cpu")
        for v, s in enumerate(S):
            rec[v, :4] = torch.tensor([float(s.tanfovx), float(s.tanfovy), NOISE_COEF if shs[v] else 0.0,
                                       NOISE_COEF if sca[v] else 0.0], dtype=torch.float64)
            rec[v, 4:5].view(torch.int32)[0] = int(s.sh_degree)
        rec = rec.to(dev)
        seed_t = torch.tensor([seed], dtype=torch.int64, device=dev)
        Hs = _lib.stacked_height(B, H, W)
        cap = R._round_cap(64 * B * P)
        scratch_bytes, saved_bytes = R._layouts(B * P, Hs, W, cap, True, True)
        scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=dev)
        saved = torch.empty(saved_bytes, dtype=torch.uint8, device=dev)
        color, da = torch.empty(3, Hs, W, device=dev), torch.empty(2, Hs, W, device=dev)
        radii, sc_out = torch.empty(B, P, dtype=torch.int32, device=dev), torch.empty(B, P, 3, device=dev)
        st = _lib.stream(dev)
        _lib.check(lib.b200gsr_forward_scene_dyn(B, prm, len(groups), table, ptr(rec), ptr(seed_t), ptr(sc_out),
                                                 ptr(color), ptr(da), ptr(radii), ptr(scratch), scratch_bytes,
                                                 ptr(saved), saved_bytes, cap, _lib.FWD_DETERMINISTIC, None, 0, st),
                   "b200gsr_forward_scene_dyn")
        Hp = Hs // B
        for v, o in enumerate(outs):
            assert torch.equal(o[0], color[:, v * Hp:v * Hp + H]) and torch.equal(o[2], da[:, v * Hp:v * Hp + H]), v
            assert torch.equal(o[1], radii[v]), v
        assert torch.equal(scales, sc_out)
        g_color, g_da = torch.zeros(3, Hs, W, device=dev), torch.zeros(2, Hs, W, device=dev)
        for v in range(B):
            g_color[:, v * Hp:v * Hp + H] = wc[v]
            g_da[:, v * Hp:v * Hp + H] = wd[v]
        grads = [{k: torch.empty_like(g_[k]) for k in NAMES} for g_ in groups]
        garr = (_lib.GroupGrad * len(groups))()
        for k, gd in enumerate(grads):
            for name, f in zip(("xyz", "opacity", "scaling", "rotation", "f_dc", "f_rest"), NAMES):
                setattr(garr[k], name, gd[f].data_ptr() if gd[f].numel() else None)
        d_m2d = torch.empty(B, P, 3, device=dev)
        _lib.check(lib.b200gsr_backward_scene_dyn(B, prm, len(groups), table, garr, ptr(rec), ptr(seed_t),
                                                  ptr(ws), ptr(radii), ptr(da), ptr(g_color), ptr(g_da),
                                                  ptr(saved), saved_bytes, cap, ptr(d_m2d), _lib.BWD_DETERMINISTIC, st),
                   "b200gsr_backward_scene_dyn")
        for gd, gr in zip(grads, groups):
            for k in NAMES:
                assert torch.equal(gd[k], gr[k].grad), k
        assert torch.equal(d_m2d, torch.stack([m.grad for m in m2d]))
    finally:
        torch.use_deterministic_algorithms(old)


def test_adam_dyn_kernel_equals_torch_adam_over_steps_with_changing_lr():
    from dreamscene_b200 import _lib
    from dreamscene_b200.optim import adam_scalars
    g = torch.Generator(device="cuda").manual_seed(5)
    sizes = [1, 3, 4096, 4097, 0, 70001] + [17 * k + 5 for k in range(30)]           # 36 tensors, two launches
    base = torch.randn(sum(sizes) + 1, device="cuda", generator=g)
    ps, o = [], 0
    for k, n in enumerate(sizes):
        off = 1 if k == 2 else 0                     # one tensor 4-byte aligned only: the scalar path
        ps.append(base[o + off:o + off + n].clone() if k != 2 else torch.empty(n + 1, device="cuda")[1:].copy_(base[o:o + n]))
        o += n
    assert sizes[4] == 0 and all(n > 0 for n in sizes[5:])    # an empty tensor before non-empty ones: rows != entries
    ref = [torch.nn.Parameter(p.clone()) for p in ps]
    # one param group per tensor, each with its own lr and beta2: every row of the scalar array differs, so a kernel
    # that read entry k's row instead of row i (the empty tensor shifts the two apart) would fail
    opt = torch.optim.Adam([{"params": [q], "betas": (0.9, 0.999 - 1e-4 * k)} for k, q in enumerate(ref)], lr=1e-2,
                           eps=1e-15)
    m = [torch.zeros_like(p) for p in ps]
    v = [torch.zeros_like(p) for p in ps]
    lib = _lib.load()
    for step in range(1, 6):
        lrs = [1e-2 * 0.7 ** step * (1.0 + 0.05 * k) for k in range(len(ps))]
        grads = [torch.randn(p.shape, device="cuda", generator=g) for p in ps]
        for q, gr in zip(ref, grads):
            q.grad = gr.clone()
        for k, pg in enumerate(opt.param_groups):
            pg["lr"] = lrs[k]
        opt.step()
        sc = torch.tensor([adam_scalars(lrs[k], 0.9, 0.999 - 1e-4 * k, 1e-15, float(step)) for k in range(len(ps))],
                          dtype=torch.float32, device="cuda")
        for i0 in range(0, len(ps), _lib.ADAM_MAX_TENSORS):
            idx = range(i0, min(i0 + _lib.ADAM_MAX_TENSORS, len(ps)))
            arr = (_lib.AdamTensor * len(idx))(*[_lib.AdamTensor(ps[i].data_ptr(), grads[i].data_ptr(), m[i].data_ptr(),
                                                                 v[i].data_ptr(), ps[i].numel()) for i in idx])
            _lib.check(lib.b200gsr_adam_step_dyn(len(idx), arr, C.c_void_p(sc.data_ptr() + 24 * i0), _lib.stream(sc.device)),
                       "b200gsr_adam_step_dyn")
    for k, (p, q) in enumerate(zip(ps, ref)):
        st = opt.state[q]
        assert torch.equal(p, q.detach()) and torch.equal(m[k], st["exp_avg"]) and torch.equal(v[k], st["exp_avg_sq"]), k


def _prune(groups, opts, mask_of):
    """densify.prune_points on every group and its optimizer (the reference's _prune_optimizer surgery)."""
    from dreamscene_b200.densify import prune_points
    new_groups = []
    for gr, opt in zip(groups, opts):
        mask = mask_of(gr)
        adam = {k: (opt.state[gr[k]]["exp_avg"], opt.state[gr[k]]["exp_avg_sq"]) for k in NAMES}
        steps = {k: opt.state[gr[k]]["step"] for k in NAMES}
        new_p, new_a, _ = prune_points({k: gr[k] for k in NAMES}, adam, None, mask)
        ng = {k: torch.nn.Parameter(new_p[k].contiguous()) for k in NAMES}
        for pg in opt.param_groups:
            k = pg["name"]
            del opt.state[pg["params"][0]]
            pg["params"] = [ng[k]]
            opt.state[ng[k]] = {"step": steps[k], "exp_avg": new_a[k][0].contiguous(), "exp_avg_sq": new_a[k][1].contiguous()}
        new_groups.append(ng)
    return new_groups


@pytest.mark.parametrize("det_mode", [True], indirect=True)
def test_a_prune_between_steps_recaptures_and_still_equals_the_eager_path(det_mode):
    from dreamscene_b200 import StepGraph
    B, H, W, M = 2, 96, 80, 4
    ge = _groups([900, 400], M, seed=2)
    gg = _clone(ge)
    oe, og = _optimizers(ge), _optimizers(gg)
    sg = StepGraph(gg, og, views=B, height=H, width=W)
    w = _weights(B, H, W)
    for step in range(4):
        if step == 2:
            mask_of = lambda gr: (gr["_opacity"].detach().reshape(-1) < -1.0)
            ge, gg = _prune(ge, oe, mask_of), _prune(gg, og, mask_of)
            sg.groups = gg
        S = _step_settings(B, H, W, M, step)
        shs, sca = _flags(B, step)
        ie, _, re, me = _eager_step(ge, oe, S, 77 + step, shs, sca, w)
        ig, _, rg, mg = _graph_step(sg, S, 77 + step, shs, sca, w)
        assert ig.shape == ie.shape and torch.equal(ie, ig) and torch.equal(re, rg) and torch.equal(me, mg), step
        _assert_state(ge, gg, oe, og, exact=True)
    assert sg.out.radii.shape[1] == sum(int(g["_xyz"].shape[0]) for g in gg) < 1300


def test_a_replay_that_overflows_its_key_buffer_is_reported():
    from dreamscene_b200 import PairCapacityOverflow, StepGraph, rasterizer as R
    d = R._device_state(torch.device("cuda", torch.cuda.current_device()))
    saved = (d.capacity, d.user_capacity, dict(d.caps))
    try:
        R.set_workspace_capacity(1 << 20)
        B, H, W, M = 1, 512, 512, 1
        groups = _groups([20000], M, seed=4)
        with torch.no_grad():
            groups[0]["_scaling"].fill_(-6.0)          # tiny splats: about one tile each
        opts = _optimizers(groups)
        sg = StepGraph(groups, opts, views=B, height=H, width=W)
        S = [U.cuda_settings(cameras.orbit_camera(radius=3.5, fovx=0.6, height=H, width=W), 0)]
        sg.render(S, shs_aug=False, scale_aug=False, seed=1)
        sg.step()
        sg.check()                                      # fits
        with torch.no_grad():
            groups[0]["_scaling"].fill_(0.5)            # same tensors, screen-filling splats: > 1M pairs
        sg.render(S, shs_aug=False, scale_aug=False, seed=2)
        with pytest.raises(PairCapacityOverflow):
            sg.check()
        sg.render(S, shs_aug=False, scale_aug=False, seed=3)     # re-captured with room for the count
        sg.step()
        sg.check()
    finally:
        d.capacity, d.user_capacity, d.caps = saved[0], saved[1], saved[2]


def test_an_overflow_before_a_recapture_is_still_reported():
    """Overflowing replay, then a prune (new layout), then a render that re-captures: check() still raises."""
    from dreamscene_b200 import PairCapacityOverflow, StepGraph, rasterizer as R
    d = R._device_state(torch.device("cuda", torch.cuda.current_device()))
    saved = (d.capacity, d.user_capacity, dict(d.caps))
    try:
        R.set_workspace_capacity(1 << 20)
        B, H, W, M = 1, 512, 512, 1
        groups = _groups([20000], M, seed=4)
        with torch.no_grad():
            groups[0]["_scaling"].fill_(-6.0)
        opts = _optimizers(groups)
        sg = StepGraph(groups, opts, views=B, height=H, width=W)
        S = [U.cuda_settings(cameras.orbit_camera(radius=3.5, fovx=0.6, height=H, width=W), 0)]
        sg.render(S, shs_aug=False, scale_aug=False, seed=1)
        sg.step()
        with torch.no_grad():
            groups[0]["_scaling"].fill_(0.5)
        sg.render(S, shs_aug=False, scale_aug=False, seed=2)     # overflows; not checked yet
        sg.step()
        with torch.no_grad():
            groups[0]["_scaling"].fill_(-6.0)
        sg.groups = _prune(groups, opts, lambda gr: torch.arange(gr["_xyz"].shape[0], device="cuda") % 4 == 0)
        sg.render(S, shs_aug=False, scale_aug=False, seed=3)     # new layout: re-captures, fits
        assert sg.out.radii.shape[1] == 15000
        with pytest.raises(PairCapacityOverflow):
            sg.check()
    finally:
        d.capacity, d.user_capacity, d.caps = saved[0], saved[1], saved[2]


def test_refuses_leaf_gradients_it_would_discard_and_parameters_adam_would_skip():
    from dreamscene_b200 import StepGraph
    B, H, W, M = 1, 64, 64, 4
    groups = _groups([300], M, seed=6)
    opts = _optimizers(groups)
    sg = StepGraph(groups, opts, views=B, height=H, width=W)
    S = _step_settings(B, H, W, M, 0)[:1]
    out = sg.render(S, seed=1)
    (out.image.sum() + groups[0]["_xyz"].sum()).backward()       # a loss term straight on a leaf
    with pytest.raises(RuntimeError, match="has a .grad of its own"):
        sg.step()
    groups[0]["_xyz"].grad = None
    sg.step()
    assert set(sg.grads[0]) == set(NAMES) and sg.grads[0]["_xyz"].shape == groups[0]["_xyz"].shape
    frozen = _groups([300], M, seed=7)
    frozen[0]["_opacity"].requires_grad_(False)
    sg2 = StepGraph(frozen, _optimizers(frozen), views=B, height=H, width=W)
    with pytest.raises(ValueError, match="does not require grad"):
        sg2.render(S, seed=1)
