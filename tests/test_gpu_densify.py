"""SURVEY 8(f4): densify/prune kernels vs the reference logic restated in PyTorch (harness/densify_ref.py)."""
import pytest
import torch

from harness import densify_ref as REF

pytestmark = pytest.mark.gpu


def _model(P, M=4, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    params = {"xyz": r(P, 3), "f_dc": r(P, 1, 3), "f_rest": r(P, M - 1, 3) * 0.1, "opacity": r(P, 1) * 2.5,
              "scaling": r(P, 3) * 0.8 - 3.5, "rotation": r(P, 4)}
    adam = {k: (r(*v.shape), r(*v.shape).abs()) for k, v in params.items()}
    accum = r(P, 1).abs() * 2e-3
    denom = torch.randint(0, 6, (P, 1), device="cuda", generator=g).float()      # zeros -> NaN grads -> 0
    return params, adam, accum, denom


@pytest.mark.parametrize("P,max_screen,N", [(20000, 20, 2), (5000, None, 2), (4097, 20, 3), (1, 20, 2)])
def test_densify_and_prune_matches_reference_logic(P, max_screen, N):
    from dreamscene_b200 import densify as D
    params, adam, accum, denom = _model(P, seed=P)
    extent, pd, max_grad, min_op = 5.0, 0.01, 1e-3, 0.05
    z = torch.randn(N * P, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    want_p, want_a = REF.densify_and_prune(params, adam, accum.clone(), denom, max_grad, min_op, extent, max_screen, pd, N, z)
    got_p, got_a, info = D.densify_and_prune(params, adam, accum.clone(), denom, max_grad, min_op, extent, max_screen,
                                             percent_dense=pd, N=N, z=z)
    n = want_p["xyz"].shape[0]
    assert info["points"] == n and got_p["xyz"].shape[0] == n
    if P > 100:
        assert info["cloned"] > 0 and info["split_parents"] > 0 and info["kept"] < P      # every path exercised
    first_child = info["kept"] + info["cloned"]
    for k in REF.NAMES:
        if k == "xyz":           # the reference forms the children's positions with torch.bmm
            assert torch.equal(got_p[k][:first_child], want_p[k][:first_child]), k
            assert torch.allclose(got_p[k][first_child:], want_p[k][first_child:], rtol=2e-6, atol=2e-6), k
        else:
            assert torch.equal(got_p[k], want_p[k]), k
        for a, b in zip(got_a[k], want_a[k]):
            assert torch.equal(a, b), k
    assert info["xyz_gradient_accum"].shape == (n, 1) and float(info["max_radii2D"].abs().max() if n else 0.0) == 0.0


def test_densification_stats_prune_points_and_score_percentile():
    from dreamscene_b200 import densify as D
    P = 30000
    params, adam, accum, denom = _model(P, seed=3)
    g = torch.Generator(device="cuda").manual_seed(5)
    grad = torch.randn(P, 3, device="cuda", generator=g)
    radii = torch.randint(-1, 40, (P,), device="cuda", generator=g, dtype=torch.int32)
    max_r = torch.rand(P, device="cuda", generator=g) * 30
    a2, d2, m2 = accum.clone(), denom.clone(), max_r.clone()
    vis = radii > 0
    a2[vis] += torch.norm(grad[vis, :2], dim=-1, keepdim=True)
    d2[vis] += 1
    m2[vis] = torch.max(m2[vis], radii[vis].float())
    D.add_densification_stats(grad, radii, accum, denom, max_r)
    assert torch.allclose(accum, a2, rtol=1e-6, atol=0) and torch.equal(denom, d2) and torch.equal(max_r, m2)
    # prune_points with an arbitrary mask, incl. Adam moments and statistics
    mask = torch.rand(P, device="cuda", generator=g) < 0.37
    stats = {"xyz_gradient_accum": accum, "denom": denom, "max_radii2D": max_r}
    p2, ad2, s2 = D.prune_points(params, adam, stats, mask)
    for k in params:
        assert torch.equal(p2[k], params[k][~mask])
        assert torch.equal(ad2[k][0], adam[k][0][~mask]) and torch.equal(ad2[k][1], adam[k][1][~mask])
    assert torch.equal(s2["max_radii2D"], max_r[~mask]) and torch.equal(s2["denom"], denom[~mask])
    # percentile threshold == sorted[int(percent * (n - 1))] (gs_renderer.py:1076-1081), incl. negatives / ties
    score = torch.randn(P, device="cuda", generator=g)
    score[::7] = score[3]
    for percent in (0.0, 0.1, 0.5, 0.93, 1.0):
        want = torch.sort(score)[0][int(percent * (P - 1))]
        got = D.percentile_threshold(score, percent)
        assert float(got) == float(want), percent
    p3, _, _ = D.prune_by_score(params, None, None, score, 0.3)
    thr = torch.sort(score)[0][int(0.3 * (P - 1))]
    assert torch.equal(p3["xyz"], params["xyz"][~(score <= thr)])
