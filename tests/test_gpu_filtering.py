"""3D Gaussian filtering on the GPU: the fused important score over a camera set (b200gsr_score_views) against
per-view score_flag renders and the oracle, its deterministic mode, edge cases and overflow re-issue, and
gaussian_filtering against a torch restatement of the reference's calculate_v_imp_score + prune_gaussians."""
import contextlib

import pytest
import torch

from harness import cameras
from tests import util_scene as U

pytestmark = pytest.mark.gpu


@contextlib.contextmanager
def deterministic(on=True):
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(old)


def sphere_settings(n, H=512, W=512, seed=0, fovx=0.55, radius=3.5):
    cams = cameras.sphere_cameras(n, radius=radius, fovx=fovx, H=H, W=W, generator=torch.Generator().manual_seed(seed))
    return [U.cuda_settings(c, 3, score=True) for c in cams]


def to_dev(sc):
    return {k: v.to("cuda") for k, v in sc.items()}


def per_view_scores(settings, t, use_cov=False):
    """[views, P]: the score of GaussianRasterizer(score_flag=True) for every view, as the reference's prune_list
    renders them (a grad-requiring means2D)."""
    from dreamscene_b200 import GaussianRasterizer
    out = []
    for S in settings:
        m2d = torch.zeros_like(t["means3D"], requires_grad=True)
        kw = dict(cov3D_precomp=t["cov3D_precomp"]) if use_cov else dict(scales=t["scales"], rotations=t["rotations"])
        score, _, _, _ = GaussianRasterizer(S)(means3D=t["means3D"], means2D=m2d, opacities=t["opacities"],
                                               shs=t["shs"], **kw)
        out.append(score.detach())
    return torch.stack(out)


def fused(settings, t, vpp=16, use_cov=False):
    from dreamscene_b200.filtering import important_score
    kw = dict(cov3D_precomp=t["cov3D_precomp"]) if use_cov else dict(scales=t["scales"], rotations=t["rotations"])
    s = important_score(settings, t["means3D"], t["opacities"], views_per_pass=vpp, **kw)
    torch.cuda.synchronize()
    return s


def view_order_sum(scores):
    acc = scores[0].clone()
    for s in scores[1:]:
        acc += s
    return acc


@pytest.fixture(scope="module")
def ball100k():
    sc, _, _ = U.make_inputs(100_000, 16, 16, seed=3)
    return to_dev(sc)


@pytest.mark.parametrize("vpp", [1, 7, 16])
def test_fused_score_equals_the_sum_of_per_view_renders(ball100k, vpp):
    S = sphere_settings(48)
    ref = view_order_sum(per_view_scores(S, ball100k))
    got = fused(S, ball100k, vpp)
    assert got.dtype == torch.float32 and got.shape == ref.shape
    assert float(ref.max()) > 0 and int((ref > 0).sum()) > 1000
    assert float((got - ref).abs().max()) <= 1e-5 * float(ref.max())


def test_fused_score_matches_the_oracle_on_cfg1():
    from tests.test_gpu_parity import run_oracle
    sc, _, deg = U.make_inputs(10000, 256, 256)
    cams = cameras.sphere_cameras(3, H=256, W=256, generator=torch.Generator().manual_seed(5))
    ref = sum(run_oracle(sc, c, deg, score=True)["score"] for c in cams)
    got = fused([U.cuda_settings(c, deg, score=True) for c in cams], to_dev(sc))
    assert float(ref.abs().max()) > 0
    assert U.rel_err(got, ref) < 1e-4


def test_deterministic_single_view_equals_the_deterministic_render(ball100k):
    S = sphere_settings(1, seed=2)
    with deterministic():
        ref = per_view_scores(S, ball100k)[0]
        got = fused(S, ball100k)
    assert float(ref.max()) > 0
    assert torch.equal(got, ref)


def test_deterministic_score_is_bitwise_repeatable_and_independent_of_batching(ball100k):
    S = sphere_settings(48)
    with deterministic():
        runs = [fused(S, ball100k, vpp) for vpp in (1, 5, 16, 16)]
        ref = view_order_sum(per_view_scores(S[:8], ball100k))
    for r in runs[1:]:
        assert torch.equal(r, runs[0])
    assert float(runs[0].max()) > 0
    with deterministic():
        got8 = fused(S[:8], ball100k, 3)
    assert float((got8 - ref).abs().max()) <= 1e-5 * float(ref.max())    # fixed point vs fp32 sum of 8 views


def _cov3d(scales, rots):
    r, x, y, z = rots.unbind(1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).view(-1, 3, 3)
    L = R * scales[:, None, :]
    S = L @ L.transpose(1, 2)
    return torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1).contiguous()


def test_cov3d_precomp_input(ball100k):
    t = dict(ball100k)
    t["cov3D_precomp"] = _cov3d(t["scales"], t["rotations"])
    S = sphere_settings(6, H=256, W=256, seed=4)
    ref = view_order_sum(per_view_scores(S, t, use_cov=True))
    got = fused(S, t, 4, use_cov=True)
    assert float(ref.max()) > 0
    assert float((got - ref).abs().max()) <= 1e-5 * float(ref.max())
    with deterministic():
        one = fused(S[:1], t, use_cov=True)
        assert torch.equal(one, per_view_scores(S[:1], t, use_cov=True)[0])


def test_empty_and_culled_inputs_give_zeros():
    from dreamscene_b200.filtering import important_score
    S = sphere_settings(3, H=64, W=64)
    e = lambda *s: torch.zeros(*s, device="cuda")
    for det in (False, True):
        with deterministic(det):
            z = important_score(S, e(0, 3), e(0, 1), e(0, 3), e(0, 4))
            assert z.shape == (0,) and z.dtype == torch.float32
            assert important_score([], e(5, 3), e(5, 1), e(5, 3), e(5, 4)).eq(0).all()
    sc, _, _ = U.make_inputs(2000, 64, 64, seed=1)
    t = to_dev(sc)
    away = [_looking_away(64, 64)] * 3                       # the whole scene is behind every camera
    for det in (False, True):
        with deterministic(det):
            s = important_score(away, t["means3D"], t["opacities"], t["scales"], t["rotations"], views_per_pass=2)
            torch.cuda.synchronize()
            assert s.shape == (2000,) and float(s.abs().max()) == 0.0


def _looking_away(H, W):
    pose = cameras.orbit_pose(3.5, 60.0, 30.0)
    pose[:3, 0] *= -1
    pose[:3, 2] *= -1                          # forward axis flipped: the scene is behind the camera
    return U.cuda_settings(cameras.camera_from_pose(pose, 0.55, H, W), 3, score=True)


@pytest.mark.parametrize("H,W", [(150, 200), (67, 33)])
def test_non_square_partial_tiles_and_a_view_with_zero_pairs(H, W):
    sc, _, _ = U.make_inputs(20000, H, W, seed=9)
    t = to_dev(sc)
    away = _looking_away(H, W)
    S = sphere_settings(5, H=H, W=W, seed=6)
    S = S[:2] + [away] + S[2:]
    per = per_view_scores(S, t)
    assert float(per[2].abs().max()) == 0.0 and float(per[0].max()) > 0
    ref = view_order_sum(per)
    for vpp in (1, 3, 6):
        got = fused(S, t, vpp)
        assert float((got - ref).abs().max()) <= 1e-5 * float(ref.max())
    assert float(fused([away], t).abs().max()) == 0.0
    with deterministic():
        a, b = fused(S, t, 1), fused(S, t, 6)
    assert torch.equal(a, b)


def test_tiny_capacity_is_reissued_and_the_score_stays_exact():
    """Every pass starts from a capacity far below its pair count: it overflows, adds nothing, and is issued again
    with room for its count; the result is the exact score (bitwise in deterministic mode)."""
    from dreamscene_b200 import rasterizer as R
    P, H, W = 40000, 48, 48
    sc, _, _ = U.make_inputs(P, H, W, seed=17, radius=0.3, exact_knn=False, scale_mul=0.5)
    t = to_dev(sc)
    S = sphere_settings(12, H=H, W=W, seed=8, radius=6.0)
    with deterministic():
        ref_det = fused(S, t, 6)
    ref = view_order_sum(per_view_scores(S, t))
    dstate = R._device_state(torch.device("cuda", torch.cuda.current_device()))
    R.flush_checks()
    old = (R._pair_mode, R._MIN_CAPACITY, R._MIN_PAIRS_PER_GAUSSIAN, dstate.capacity, dstate.user_capacity, dict(dstate.caps))
    try:
        for det in (False, True):
            R._MIN_CAPACITY, R._MIN_PAIRS_PER_GAUSSIAN = 1024, 0
            R.set_workspace_capacity(1024)
            first = R._round_cap(1024)                                # 2^18 pairs; 12 views of 40k visible Gaussians exceed it
            with deterministic(det):
                got = fused(S, t, 12)
            assert dstate.capacity > first                            # the passes did overflow and were re-issued
            if det:
                assert torch.equal(got, ref_det)
            else:
                assert float((got - ref).abs().max()) <= 1e-5 * float(ref.max())
    finally:
        R._pair_mode, R._MIN_CAPACITY, R._MIN_PAIRS_PER_GAUSSIAN, dstate.capacity, dstate.user_capacity, caps = old
        dstate.caps.clear(); dstate.caps.update(caps)


def _raw_params(P, seed):
    g = torch.Generator().manual_seed(seed)
    sc, _, _ = U.make_inputs(P, 16, 16, seed=seed)
    params = {"xyz": sc["means3D"], "f_dc": sc["shs"][:, :1].contiguous(), "f_rest": sc["shs"][:, 1:].contiguous(),
              "opacity": torch.logit(sc["opacities"].clamp(1e-4, 1 - 1e-4)), "scaling": torch.log(sc["scales"]),
              "rotation": sc["rotations"] * 2.0}
    adam = {k: (torch.randn(v.shape, generator=g), torch.rand(v.shape, generator=g)) for k, v in params.items()}
    stats = {"xyz_gradient_accum": torch.rand(P, 1, generator=g), "denom": torch.rand(P, 1, generator=g),
             "max_radii2D": torch.rand(P, generator=g)}
    c = lambda d: {k: (tuple(x.cuda() for x in v) if isinstance(v, tuple) else v.cuda()) for k, v in d.items()}
    return c(params), c(adam), c(stats)


def test_gaussian_filtering_keeps_the_reference_index_set():
    from dreamscene_b200.filtering import gaussian_filtering, volume_weighted_score
    P = 30000
    params, adam, stats = _raw_params(P, 21)
    score = torch.rand(P, device="cuda") * 50
    score[::7] = 0.0                                       # culled in every view: ties at zero, as in practice
    v_pow, prune_decay, prune_percent = 0.1, 0.6, 0.5      # the object trainer's defaults
    # torch restatement of calculate_v_imp_score + prune_gaussians (scene_gaussian.py:1046-1060, gs_renderer.py:1082-1087)
    volume = torch.prod(torch.exp(params["scaling"]), dim=1)
    sorted_volume, _ = torch.sort(volume, descending=True)
    v_list = torch.pow(volume / sorted_volume[int(len(volume) * 0.9)], 0.1) * score
    assert torch.equal(volume_weighted_score(score, params["scaling"], v_pow), v_list)
    sorted_t, _ = torch.sort(v_list, dim=0)
    thr = sorted_t[int((prune_decay ** 1) * prune_percent * (sorted_t.shape[0] - 1))]
    keep = ~(v_list <= thr).squeeze()
    new_p, new_a, new_s = gaussian_filtering(params, adam, stats, [], v_pow, prune_decay, prune_percent, score=score)
    assert new_p["xyz"].shape[0] == int(keep.sum()) < P
    for k in params:
        assert torch.equal(new_p[k], params[k][keep]), k
        assert torch.equal(new_a[k][0], adam[k][0][keep]) and torch.equal(new_a[k][1], adam[k][1][keep]), k
    for k in stats:
        assert torch.equal(new_s[k], stats[k][keep]), k


def test_gaussian_filtering_renders_the_activated_gaussians():
    from dreamscene_b200.filtering import gaussian_filtering, important_score
    P = 20000
    params, adam, stats = _raw_params(P, 22)
    S = sphere_settings(4, H=128, W=128, seed=3)
    with deterministic():
        score = important_score(S, params["xyz"], torch.sigmoid(params["opacity"]), torch.exp(params["scaling"]),
                                torch.nn.functional.normalize(params["rotation"]))
        a = gaussian_filtering(params, adam, stats, S, 0.1, 0.6, 0.5)
        b = gaussian_filtering(params, adam, stats, S, 0.1, 0.6, 0.5, score=score)
    assert float(score.max()) > 0
    for k in params:
        assert torch.equal(a[0][k], b[0][k]), k
