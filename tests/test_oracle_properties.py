"""CPU-only property tests of the oracle (hypothesis): invariants any correct restatement of the
rasterizer must satisfy, on small random scenes.  They guard the checker itself."""
import numpy as np
import torch
from hypothesis import given, settings, strategies as st

from oracle import splat_ref as O
from tests import util_scene as U


def _render(P, H, W, seed, deg, bg=(1.0, 1.0, 1.0), score=False, **kw):
    sc, cam, _ = U.make_inputs(P, H, W, seed=seed, exact_knn=False, **kw)
    S = U.oracle_settings(cam, deg, bg, score)
    with torch.no_grad():
        r = O.rasterize(S, sc["means3D"], sc["opacities"], shs=sc["shs"], scales=sc["scales"],
                        rotations=sc["rotations"])
    return sc, cam, r


@settings(max_examples=8, deadline=None)
@given(seed=st.integers(0, 10_000), P=st.integers(1, 400), H=st.integers(8, 70), W=st.integers(8, 70),
       deg=st.integers(0, 3))
def test_lists_sorted_ranges_partition_and_outputs_bounded(seed, P, H, W, deg):
    sc, cam, r = _render(P, H, W, seed, deg)
    keys, pl, ranges = r["keys"], r["point_list"], r["ranges"]
    D = len(pl)
    assert D == int(r["pre"]["touched"].sum())
    if D:
        assert np.all(keys[1:] >= keys[:-1])                       # tile-major, depth-sorted
        same = keys[1:] == keys[:-1]
        assert np.all(pl[1:][same] > pl[:-1][same])                # equal keys keep index order (stable)
    assert ranges[0, 0] == 0 and ranges[-1, 1] == D
    assert np.all(ranges[1:, 0] == ranges[:-1, 1])                 # ranges partition the list
    T = r["depth_alpha"][1]
    assert float(T.min()) >= 0.0 and float(T.max()) <= 1.0
    assert float(r["depth_alpha"][0].min()) >= 0.0                  # depths are > 0.2, weights >= 0
    assert torch.isfinite(r["color"]).all()
    vis = r["radii"] > 0
    assert torch.equal(vis, r["pre"]["visible"])
    n = ranges[:, 1] - ranges[:, 0]
    gx = (W + 15) // 16
    nc = r["n_contrib"].numpy()
    for t in np.nonzero(n)[0][:6]:
        ty, tx = divmod(int(t), gx)
        assert nc[ty * 16:(ty + 1) * 16, tx * 16:(tx + 1) * 16].max() <= n[t]


@settings(max_examples=5, deadline=None)
@given(seed=st.integers(0, 10_000), P=st.integers(5, 300))
def test_background_enters_linearly_and_score_is_total_blend_weight(seed, P):
    _, _, r1 = _render(P, 40, 48, seed, 2, bg=(1.0, 1.0, 1.0), score=True)
    _, _, r0 = _render(P, 40, 48, seed, 2, bg=(0.0, 0.0, 0.0))
    T = r1["depth_alpha"][1]
    for c in range(3):
        assert torch.allclose(r1["color"][c] - r0["color"][c], T, atol=1e-6)
    # sum of importance scores == sum over pixels of (1 - T) when every weight is counted once
    assert abs(float(r1["score"].sum()) - float((1.0 - T).sum())) < 1e-3 * max(1.0, float((1.0 - T).sum()))


def test_culled_gaussians_get_exactly_zero_gradients():
    sc, cam, deg = U.make_inputs(200, 32, 32, seed=3)
    sc["means3D"][::2] += cam.camera_center * 2.0            # every other Gaussian behind the camera
    S = U.oracle_settings(cam, deg)
    t = {k: v.clone().requires_grad_(True) for k, v in sc.items()}
    r = O.rasterize(S, t["means3D"], t["opacities"], shs=t["shs"], scales=t["scales"], rotations=t["rotations"])
    (r["color"].sum() + r["depth_alpha"].sum()).backward()
    culled = r["radii"] == 0
    assert culled[::2].all()
    for k, v in t.items():
        assert float(v.grad[culled].abs().max()) == 0.0, k


def test_fp64_run_on_fp32_decisions_agrees_with_fp32_run():
    sc, cam, deg = U.make_inputs(300, 48, 48, seed=9)
    S = U.oracle_settings(cam, deg)
    kw = dict(shs=sc["shs"], scales=sc["scales"], rotations=sc["rotations"])
    with torch.no_grad():
        r32 = O.rasterize(S, sc["means3D"], sc["opacities"], **kw)
        r64 = O.rasterize(S, sc["means3D"], sc["opacities"], dtype=torch.float64, decisions=r32["decisions"], **kw)
    assert (r64["color"].float() - r32["color"]).abs().max() < 5e-3
    assert ((r64["color"].float() - r32["color"]).abs() > 1e-4).float().mean() < 1e-3


def test_fp64_run_replays_the_fp32_branch_flags():
    """The EWA clamp (in_x / in_y) and the colour clamp are branch decisions: an fp64 run recomputing them can take
    the other gradient branch (identity vs zero) than the fp32 run it checks, for a Gaussian whose t.x/t.z sits within
    an ulp of the limit or whose colour sits within an ulp of 0.  Given the fp32 run's flags it takes the fp32 branch
    on every Gaussian; without them at least one of these constructed Gaussians flips."""
    from tests import room_edges as E
    cam = E.axis_camera(64)
    sc = E.as_inputs(E.boundary_rows(cam, np.random.RandomState(0), colour_flip=True), M=4)
    S = U.oracle_settings(cam, 1)
    limx, limy = E.limits(cam)
    tx, ty, tz = E.view_f32(cam.world_view_transform.numpy(), sc["means3D"].numpy())
    q = np.concatenate([tx[:6] / tz[:6], ty[6:12] / tz[6:12]])
    want = np.array([s * lim for lim in (limx, limy) for s in (1, -1) for _ in range(3)], np.float32)
    want = np.array([np.nextafter(w, np.float32(d * np.inf)) if d else w
                     for w, d in zip(want, [-1, 0, 1] * 4)], np.float32)
    np.testing.assert_array_equal(q, want)                       # t/t.z exactly at +-limit and one ulp either side

    def run(dtype, dec=None):
        t = {k: v.clone().to(dtype).requires_grad_(True) for k, v in sc.items()}
        pre = O.preprocess(S, t["means3D"], t["opacities"], shs=t["shs"], scales=t["scales"],
                           rotations=t["rotations"], dtype=dtype, decisions=dec)
        (sum(c.sum() for c in pre["conic"]) + pre["rgb"].sum()).backward()
        return pre, t["means3D"].grad, t["shs"].grad

    pre32, gm32, gs32 = run(torch.float32)
    raw0 = pre32["rgb"][12:15].detach()
    assert bool(pre32["clamped"][12].all()) and not bool(pre32["clamped"][13:15].any())
    assert bool((raw0[1] == 0).all()) and bool((raw0[2] > 0).all())   # the fp32 colour is exactly 0, then one ulp up
    np.testing.assert_array_equal(pre32["in_x"][:6].numpy(), [True, True, False, False, True, True])
    np.testing.assert_array_equal(pre32["in_y"][6:12].numpy(), [True, True, False, False, True, True])
    dec = dict(visible=pre32["visible"], radii=pre32["radii"], rect=pre32["rect"], touched=pre32["touched"],
               in_x=pre32["in_x"], in_y=pre32["in_y"], clamped=pre32["clamped"])
    pre64, gm64, gs64 = run(torch.float64, dec)
    for k in ("in_x", "in_y", "clamped"):
        assert torch.equal(pre64[k], pre32[k]), k
    # the branch shows in the gradients: the fp64 rows agree with the fp32 rows Gaussian by Gaussian
    rel = ((gm64 - gm32.double()).norm(dim=1) / gm64.norm(dim=1)).max()
    assert float(rel) < 1e-3, float(rel)
    assert torch.equal(gs64 == 0, gs32 == 0)
    # without the flags fp64 recomputes them and at least one Gaussian takes the other branch
    # (row 15 is built so that its colour clamp flips)
    pre_own, gm_own, gs_own = run(torch.float64, {k: dec[k] for k in ("visible", "radii", "rect", "touched")})
    assert bool((pre_own["in_x"] != pre32["in_x"]).any() | (pre_own["in_y"] != pre32["in_y"]).any())
    assert bool((pre_own["clamped"][15] != pre32["clamped"][15]).all())
    rel_own = ((gm_own - gm32.double()).norm(dim=1) / gm_own.norm(dim=1)).max()
    assert float(rel_own) > 1e-2
    assert not torch.equal(gs_own[15] == 0, gs32[15] == 0)
