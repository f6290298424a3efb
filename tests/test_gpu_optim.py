"""GaussianAdam on the GPU against torch.optim.Adam's default path, bitwise (int32 views): the reference's seven
groups over 30 steps with hostile gradients and a new lr every step, skipped parameters, the reference's optimizer
surgery mid-run, state_dict round trips, edge cases, one launch per step without host syncs, and 10 end-to-end
training steps through the rasterizer in deterministic mode."""
import copy
import math

import pytest
import torch
from torch import nn

from dreamscene_b200 import GaussianAdam
from harness import adam_ref as S
from harness.adam_ref import LRS, NAMES, reference_adam

pytestmark = pytest.mark.gpu


def layout(P, M, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    shapes = dict(xyz=(P, 3), f_dc=(P, 1, 3), f_rest=(P, M - 1, 3), opacity=(P, 1), scaling=(P, 3), rotation=(P, 4),
                  background=(3, 1, 1))
    return {k: torch.randn(s, device="cuda", generator=g) for k, s in shapes.items()}


def make_pair(tensors, cls_b=GaussianAdam):
    """Two optimizers over identical copies, built as the reference builds its optimizer."""
    out = []
    for cls in (torch.optim.Adam, cls_b):
        params = {k: nn.Parameter(v.clone()) for k, v in tensors.items()}
        out.append((params, reference_adam(params, cls)))
    return out


def hostile_grad(shape, gen):
    x = torch.randn(shape, device="cuda", generator=gen) * torch.exp2(
        torch.randint(-30, 30, shape, device="cuda", generator=gen).float())
    r = torch.rand(shape, device="cuda", generator=gen)
    specials = [(0.05, 0.0), (0.07, 1e-41), (0.08, -3e-39), (0.09, 3e38), (0.095, -1e30), (0.097, float("nan")),
                (0.098, float("inf")), (0.099, float("-inf"))]
    lo = 0.0
    for hi, val in specials:
        x = torch.where((r >= lo) & (r < hi), torch.full_like(x, val), x)
        lo = hi
    return x


def set_grads(pairs, gen, skip=()):
    p0 = pairs[0][0]
    for k, p in p0.items():
        g = None if k in skip else hostile_grad(p.shape, gen)
        for params, _ in pairs:
            params[k].grad = None if g is None else g.clone()


def assert_same(pairs, what=""):
    (pa, oa), (pb, ob) = pairs
    for k in pa:
        a, b = pa[k].detach(), pb[k].detach()
        assert a.shape == b.shape, (what, k)
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), (what, k, "param")
        sa, sb = oa.state.get(pa[k], {}), ob.state.get(pb[k], {})
        assert set(sa) == set(sb), (what, k)
        for key in sa:
            if key == "step":
                assert sa[key].item() == sb[key].item() and sa[key].dtype == sb[key].dtype, (what, k, "step")
                assert sb[key].device.type == "cpu"
            else:
                assert torch.equal(sa[key].view(torch.int32), sb[key].view(torch.int32)), (what, k, key)


def run(pairs, steps, gen, skip_fn=lambda it: (), it0=0):
    for it in range(it0, it0 + steps):
        set_grads(pairs, gen, skip_fn(it))
        for _, opt in pairs:
            for grp in opt.param_groups:          # update_learning_rate: a new lr every step
                grp["lr"] = LRS[grp["name"]] * (0.5 + 0.5 * math.cos(0.3 * it))
            opt.step()
        assert_same(pairs, f"step {it}")


@pytest.mark.parametrize("P,M", [(10007, 16), (4099, 4)])
def test_thirty_steps_of_the_reference_groups_are_bitwise_equal(P, M):
    pairs = make_pair(layout(P, M))
    gen = torch.Generator(device="cuda").manual_seed(1)
    run(pairs, 30, gen)
    # the moments really went through the special values
    v = pairs[1][1].state[pairs[1][0]["xyz"]]["exp_avg_sq"]
    assert torch.isnan(v).any() and torch.isinf(v).any()


def test_a_large_lerp_weight_and_beta2_zero_follow_torch():
    """beta1 <= 0.5 takes lerp's other branch; beta2 = 0 makes addcmul's value exactly 1."""
    for betas in ((0.3, 0.999), (0.9, 0.0), (0.0, 0.5)):
        t = layout(1001, 4, seed=3)
        pairs = []
        for cls in (torch.optim.Adam, GaussianAdam):
            params = {k: nn.Parameter(v.clone()) for k, v in t.items()}
            pairs.append((params, reference_adam(params, cls, betas=betas)))
        gen = torch.Generator(device="cuda").manual_seed(2)
        run(pairs, 5, gen)


def test_skipped_parameters_keep_their_step_counter():
    pairs = make_pair(layout(3001, 16))
    gen = torch.Generator(device="cuda").manual_seed(4)
    skip = lambda it: ("background",) + tuple(NAMES[j] for j in range(6) if it % (j + 2) == 0)
    run(pairs, 12, gen, skip)
    steps = {k: pairs[1][1].state[p]["step"].item() for k, p in pairs[1][0].items() if p in pairs[1][1].state}
    assert "background" not in steps and len(set(steps.values())) > 1


def test_reference_optimizer_surgery_mid_run():
    pairs = make_pair(layout(5003, 16))
    gen = torch.Generator(device="cuda").manual_seed(5)
    run(pairs, 8, gen, lambda it: ("background",))
    keep = torch.rand(5003, device="cuda", generator=gen) > 0.3
    new_rows = {k: torch.randn((777,) + tuple(v.shape[1:]), device="cuda", generator=gen)
                for k, v in pairs[0][0].items() if k != "background"}
    for params, opt in pairs:
        params.update(S.prune(opt, keep))
        params.update(S.cat_tensors(opt, new_rows))
        op = torch.sigmoid(params["opacity"].detach())
        params.update(S.replace_tensor(opt, torch.logit(torch.min(op, torch.ones_like(op) * 0.01)), "opacity"))
    assert_same(pairs, "after surgery")
    run(pairs, 8, gen, lambda it: ("background",), it0=8)


def test_state_dict_round_trips_torch_native_torch():
    t = layout(2003, 16, seed=6)
    gen_a = torch.Generator(device="cuda").manual_seed(7)
    ref = make_pair(t, cls_b=torch.optim.Adam)[0]                  # one uninterrupted torch run
    params = {k: nn.Parameter(v.clone()) for k, v in t.items()}
    opt = reference_adam(params)
    grads = []
    for it in range(15):
        gen_a.manual_seed(100 + it)
        grads.append({k: hostile_grad(p.shape, gen_a) for k, p in params.items()})
    for it in range(15):
        if it == 5:
            sd = copy.deepcopy(opt.state_dict())
            opt = reference_adam(params, GaussianAdam)
            opt.load_state_dict(sd)
        if it == 10:
            sd = copy.deepcopy(opt.state_dict())
            native_sd = opt.state_dict()
            opt = reference_adam(params)
            opt.load_state_dict(sd)
            torch_sd = ref[1].state_dict()
            assert native_sd["param_groups"] == torch_sd["param_groups"]
            for i in torch_sd["state"]:
                a, b = torch_sd["state"][i], native_sd["state"][i]
                assert set(a) == set(b)
                for key in a:
                    assert (a[key].dtype, a[key].device, a[key].shape) == (b[key].dtype, b[key].device, b[key].shape)
        for k in params:
            params[k].grad = grads[it][k].clone()
            ref[0][k].grad = grads[it][k].clone()
        opt.step()
        ref[1].step()
        assert_same([ref, (params, opt)], f"step {it}")


def test_edge_cases_empty_one_element_unaligned_and_non_contiguous_grad():
    gen = torch.Generator(device="cuda").manual_seed(8)
    base = torch.randn(4099, device="cuda", generator=gen)
    t = dict(empty=torch.zeros(0, 3, device="cuda"), one=torch.randn(1, device="cuda", generator=gen),
             five=torch.randn(5, device="cuda", generator=gen), big=torch.randn(700, 9, device="cuda", generator=gen))
    pairs = []
    for cls in (torch.optim.Adam, GaussianAdam):
        params = {k: nn.Parameter(v.clone()) for k, v in t.items()}
        params["unaligned"] = nn.Parameter(base.clone()[1:])                 # storage offset 4 bytes
        pairs.append((params, cls([{"params": [params[k]], "lr": 0.01 * (1 + i), "name": k}
                                   for i, k in enumerate(params)], lr=0.0, eps=1e-15)))
    assert pairs[1][0]["unaligned"].data_ptr() % 16 != 0
    for it in range(6):
        gsrc = {k: hostile_grad(p.shape, gen) for k, p in pairs[0][0].items()}
        nc = hostile_grad((9, 700), gen)                                     # transposed: a non-contiguous grad
        gu = hostile_grad((4099,), gen)
        for params, _ in pairs:
            for k in ("empty", "one", "five"):
                params[k].grad = gsrc[k].clone()
            params["big"].grad = nc.clone().t()
            params["unaligned"].grad = gu.clone()[1:]
            assert not params["big"].grad.is_contiguous()
        for _, opt in pairs:
            opt.step()
        assert_same(pairs, f"step {it}")
    assert pairs[1][1].state[pairs[1][0]["empty"]]["step"].item() == 6


def test_second_step_is_one_kernel_without_host_sync_and_runs_on_a_side_stream():
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    pairs = make_pair(layout(20011, 16, seed=9))
    gen = torch.Generator(device="cuda").manual_seed(10)
    run(pairs, 1, gen, lambda it: ("background",))                 # lazy state creation happens here
    set_grads(pairs, gen, ("background",))
    native = pairs[1][1]
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.cuda.set_sync_debug_mode("error")
        try:
            native.step()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        torch.cuda.synchronize()
    kernels = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]
    assert len(kernels) == 1 and "adam_step_kernel" in kernels[0], kernels
    pairs[0][1].step()
    assert_same(pairs, "profiled step")
    side = torch.cuda.Stream()
    for it in range(3):
        set_grads(pairs, gen, ("background",))
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _, opt in pairs:
                opt.step()
        torch.cuda.current_stream().wait_stream(side)
        assert_same(pairs, f"side stream step {it}")


def _render_loss(leaves, cam_settings, target):
    from dreamscene_b200 import GaussianRasterizer
    means2D = torch.zeros_like(leaves["xyz"], requires_grad=True)
    shs = torch.cat((leaves["f_dc"], leaves["f_rest"]), dim=1)
    img, radii, _ = GaussianRasterizer(cam_settings)(
        means3D=leaves["xyz"], means2D=means2D, opacities=torch.sigmoid(leaves["opacity"]), shs=shs,
        colors_precomp=None, scales=torch.exp(leaves["scaling"]),
        rotations=torch.nn.functional.normalize(leaves["rotation"]), cov3D_precomp=None)
    return ((img - target) ** 2).mean()


def test_ten_training_steps_through_the_rasterizer_are_bitwise_equal():
    from harness import cameras, synthetic
    from tests import util_scene as U
    P, H, W = 4000, 96, 96
    sc = synthetic.ball_scene(P, radius=0.5, sh_degree_max=3, seed=11, opacity="sigmoid_normal", exact_knn=False)
    t = {"xyz": sc["means3D"], "f_dc": sc["shs"][:, :1], "f_rest": sc["shs"][:, 1:],
         "opacity": torch.logit(sc["opacities"].clamp(1e-4, 1 - 1e-4)), "scaling": sc["scales"].log(),
         "rotation": sc["rotations"]}
    t = {k: v.contiguous().float().cuda() for k, v in t.items()}
    t["background"] = torch.zeros(3, 1, 1, device="cuda")
    pairs = make_pair(t)
    target = torch.linspace(0, 1, 3 * H * W, device="cuda").reshape(3, H, W)
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for it in range(10):
            cam = cameras.orbit_camera(radius=3.5, phi_deg=36.0 * it, fovx=0.7, height=H, width=W)
            settings = U.cuda_settings(cam, 3)
            for params, opt in pairs:
                opt.zero_grad(set_to_none=True)
                _render_loss(params, settings, target).backward()
                for grp in opt.param_groups:
                    grp["lr"] = LRS[grp["name"]] * (1.0 - 0.05 * it)
                opt.step()
            assert pairs[0][0]["xyz"].grad is not None and pairs[0][0]["background"].grad is None
            assert_same(pairs, f"training step {it}")
    finally:
        torch.use_deterministic_algorithms(old)
    assert not torch.equal(pairs[1][0]["xyz"].detach(), t["xyz"])
