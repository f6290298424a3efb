"""DESIGN.md f4 at its edges: densify_and_prune, prune_points and the radix select against the reference's statements
(harness/densify_ref.py) and torch.sort, bit for bit on the same GPU.

  * Split children: log-scales equal to the reference's for N = 1..4 with thousands of split parents; positions against
    an fp64 evaluation, because the reference forms them with torch.bmm.
  * Inputs built to sit on each decision threshold as the reference's own torch ops see it (gradient, dense extent with
    each scale component in turn, opacity, the children's world-size prune), with the nearest values either side.
  * Production sizes, where the two-level scan takes its carry loop: densify at 1.1 M rows, prune at 4.2 M rows.
  * kth_smallest / percentile_threshold on ties at radix-digit boundaries, signed zeros, infinities, subnormals and
    NaNs, in one block and in the multi-block grid.
"""
import math

import pytest
import torch

from dreamscene_b200 import densify as D
from harness import densify_ref as REF

pytestmark = pytest.mark.gpu

F32 = torch.float32
INF = float("inf")
U = 2.0 ** -24                       # fp32 unit roundoff
KIND = (0, 1 << 30, -(1 << 31))      # src_map bits 30..31: original, clone, split child (as int32)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _f32(x):
    """x rounded to fp32, as torch rounds a Python scalar that a float tensor is compared with."""
    return float(torch.tensor(x, dtype=F32))


def _window(x, k):
    """The values of x stepped -k..k ulps with torch.nextafter, concatenated along dim 0 (x itself in the middle)."""
    lo, hi, out = x, x, [x]
    for _ in range(k):
        lo = torch.nextafter(lo, torch.full_like(lo, -INF))
        hi = torch.nextafter(hi, torch.full_like(hi, INF))
        out = [lo] + out + [hi]
    return torch.cat(out)


def _sides(v, t):
    """(some below, some on, some above) of v against the threshold t."""
    return bool((v < t).any()), bool((v == t).any()), bool((v > t).any())


def _child_act(e, N):
    """The reference's view of a split child's scale component: exp(log(exp(s) / (0.8 N))), the divide by the Python
    scalar as torch does it (a multiply by the fp32 reciprocal)."""
    return torch.exp(torch.log(e / (0.8 * N)))


def _model(P, M=4, seed=0, adam=True):
    g = _gen(seed)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)  # noqa: E731
    params = {"xyz": r(P, 3), "f_dc": r(P, 1, 3), "f_rest": r(P, M - 1, 3) * 0.1, "opacity": r(P, 1) * 2.5,
              "scaling": r(P, 3) * 0.8 - 3.5, "rotation": r(P, 4)}
    moments = {k: (r(*v.shape), r(*v.shape).abs()) for k, v in params.items()} if adam else None
    accum = r(P, 1).abs() * 2e-3
    denom = torch.randint(0, 6, (P, 1), device="cuda", generator=g).float()      # zeros -> NaN grads -> 0
    return params, moments, accum, denom


def _plan(params, accum, denom, max_grad, min_opacity, extent, max_screen_size, percent_dense, N):
    """The reference's decisions (harness/densify_ref.py, statement for statement) on row indices.  -> the expected
    src_map [kept originals | clones | N blocks of surviving children] with the kind in bits 30..31, and the clone,
    split and surviving-child masks (the last over the split parents)."""
    assert max_grad > 0                    # then the clones' zero-padded gradients never split
    s = params["scaling"]
    grads = accum / denom
    grads[grads.isnan()] = 0.0
    emax = torch.max(torch.exp(s), dim=1).values
    clone = (torch.norm(grads, dim=-1) >= max_grad) & (emax <= percent_dense * extent)
    split = (grads.squeeze(-1) >= max_grad) & (emax > percent_dense * extent)
    child_s = torch.log(torch.exp(s)[split] / (0.8 * N))

    def big(x):
        if not max_screen_size:
            return torch.zeros(x.shape[0], dtype=torch.bool, device=x.device)
        return torch.exp(x).max(dim=1).values > 0.1 * extent

    low = (torch.sigmoid(params["opacity"]) < min_opacity).squeeze(-1)
    pruned = low | big(s)
    child_keep = ~(low[split] | big(child_s))
    rows = torch.arange(s.shape[0], dtype=torch.int32, device=s.device)
    src = torch.cat((rows[~split & ~pruned], rows[clone & ~pruned] | KIND[1], (rows[split][child_keep] | KIND[2]).repeat(N)))
    return src, clone, split, child_keep


def _rotation64(q):
    q = q / q.norm(dim=1, keepdim=True)
    r, x, y, z = q.unbind(1)
    return torch.stack((1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)), 1).view(-1, 3, 3)


def _check_children(got_p, first_child, params, z, split, child_keep, N):
    """The children rows: log-scales as the reference's expression on the parents' rows (bitwise); positions against
    R(q) (z * exp(s)) + xyz in fp64 with the reference's draw order (child block k of the r-th split parent takes
    z[k * n_split + r]).  R's entries are built from unit-quaternion products, so they carry absolute rounding errors
    of a few ulp of 1: the bound is 16 u of sum_j |z_j exp(s_j)| + |xyz|, which is at least |R| |z exp(s)| + |xyz|."""
    sel = split.nonzero().squeeze(1)
    n_sel = sel.numel()
    par = sel[child_keep].repeat(N)
    zrow = (torch.arange(N, device="cuda")[:, None] * n_sel + torch.arange(n_sel, device="cuda")[None, :])[:, child_keep]
    e = torch.exp(params["scaling"][par])
    assert torch.equal(got_p["scaling"][first_child:], torch.log(e / (0.8 * N)))
    sm = z[zrow.reshape(-1)].double() * e.double()
    xyz = params["xyz"][par].double()
    want = (_rotation64(params["rotation"][par].double()) @ sm.unsqueeze(-1)).squeeze(-1) + xyz
    err = (got_p["xyz"][first_child:].double() - want).abs()
    scale = sm.abs().sum(1, keepdim=True) + xyz.abs()
    worst = float((err / scale).max()) if err.numel() else 0.0
    assert worst <= 16 * U, f"children xyz: {worst / U:.2f} u"
    return worst


def _compare(got_p, got_a, info, want_p, want_a, plan, params, z, N):
    src, _, split, child_keep = plan
    first_child = info["kept"] + info["cloned"]
    assert info["points"] == want_p["xyz"].shape[0] == src.numel()
    assert info["split_parents"] == int(split.sum()) and info["split_parents_surviving"] == int(child_keep.sum())
    assert info["kept"] == int(((src >= 0) & (src < KIND[1])).sum())
    assert torch.equal(info["src_map"], src)
    for k in REF.NAMES:
        if k == "xyz":
            assert torch.equal(got_p[k][:first_child], want_p[k][:first_child]), k
        else:
            assert torch.equal(got_p[k], want_p[k]), k
        for a, b in zip(got_a[k], want_a[k]):
            assert torch.equal(a, b), k
    return _check_children(got_p, first_child, params, z, split, child_keep, N)


# ---- 1. split children bit for bit ------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 2, 3, 4])
def test_split_children_log_scales_equal_the_reference(N):
    P = 20000
    params, adam, accum, denom = _model(P, seed=10 + N)
    kw = dict(max_grad=1e-3, min_opacity=0.05, extent=5.0, max_screen_size=20, percent_dense=0.01, N=N)
    z = torch.randn(N * P, 3, device="cuda", generator=_gen(N))
    want_p, want_a = REF.densify_and_prune(params, adam, accum.clone(), denom, z=z, **kw)
    got_p, got_a, info = D.densify_and_prune(params, adam, accum.clone(), denom, z=z, **kw)
    plan = _plan(params, accum, denom, **kw)
    assert info["split_parents_surviving"] > 2000
    # the inputs tell the reference's reciprocal multiply from a true division by fp32(0.8 N)
    e = torch.exp(params["scaling"][plan[2]])
    assert not torch.equal(torch.log(e / (0.8 * N)), torch.log(e / torch.tensor(0.8 * N, device="cuda")))
    _compare(got_p, got_a, info, want_p, want_a, plan, params, z, N)


def test_densify_and_prune_on_zero_rows():
    params, adam, accum, denom = _model(0)
    kw = dict(max_grad=1e-3, min_opacity=0.05, extent=5.0, max_screen_size=20, percent_dense=0.01, N=2)
    z = torch.randn(2, 3, device="cuda", generator=_gen(0))
    want_p, want_a = REF.densify_and_prune(params, adam, accum.clone(), denom, z=z, **kw)
    got_p, got_a, info = D.densify_and_prune(params, adam, accum.clone(), denom, z=z, **kw)
    assert info["points"] == 0 and info["src_map"].numel() == 0
    for k in REF.NAMES:
        assert got_p[k].shape == want_p[k].shape and all(a.shape == b.shape for a, b in zip(got_a[k], want_a[k]))


# ---- 2. decision boundaries -------------------------------------------------------------------------------------------
def _boundary_case(N, M=4, seed=0):
    """A model whose rows are every combination of a gradient row, a scale row and an opacity row, each built around a
    threshold with torch's own ops, so that the reference's view of the threshold decides:
      gradient  accum / denom == max_grad and the nearest quotients either side (a 9-ulp window of accum, denom 1, 3,
                7); denom 0 with accum 0 (NaN -> 0), > 0 (inf) and < 0 (-inf); accum < 0 with |g| == max_grad (clones,
                never splits) and below it; one clearly above
      scale     max(exp(s)) == fp32(percent_dense * extent) and the nearest values either side; a split parent whose
                children's max_k exp(log(exp(s_k) / (0.8 N))) lands on, below and above fp32(0.1 * extent); both with
                the max carried by each component in turn; one clearly small, one mid and one huge parent
      opacity   sigmoid(opacity) == min_opacity and the nearest values either side; one clearly opaque
    fp32(0.1 * extent) is what a true division by fp32(0.8 N) gives at a parent log-scale s* where the reference's
    reciprocal multiply gives more (so a kernel that divides keeps a child the reference prunes), and what the
    reference gives at a log-scale a few ulp below s*.
    -> params, adam, accum, denom and the keyword arguments of densify_and_prune."""
    dev = "cuda"
    g = _gen(seed)
    cand = math.log(0.4 * N) + (torch.rand(1 << 16, device=dev, generator=g) - 0.5) * 0.1
    e = torch.exp(cand)
    c_div = torch.exp(torch.log(e / torch.tensor(0.8 * N, device=dev)))
    hit = (c_div < _child_act(e, N)).nonzero().view(-1)[:256]
    on = (_child_act(torch.exp(_window(cand[hit], 64)), N).view(129, -1) == c_div[hit]).any(0)
    assert on.any(), "no parent scale where a true division and the reciprocal multiply disagree on the threshold"
    j = int(hit[on][0])
    s_star = cand[j:j + 1]
    t_big = float(c_div[j])
    extent = t_big / 0.1
    s_d = torch.tensor([-3.0], device=dev)
    t_dense = float(torch.exp(s_d))
    percent_dense = t_dense / extent
    max_grad = _f32(2e-4)
    o0 = torch.tensor([-3.0], device=dev)
    min_opacity = float(torch.sigmoid(o0))
    assert _f32(0.1 * extent) == t_big and _f32(percent_dense * extent) == t_dense
    assert 4 * t_dense < t_big          # children of the dense window stay small, parents of the children window split

    grad_rows = []
    for d in (1.0, 3.0, 7.0):
        a = _window(torch.tensor([max_grad * d], device=dev), 4)
        grad_rows.append(torch.stack((a, torch.full_like(a, d)), 1))
    grad_rows.append(torch.tensor([[0.0, 0.0], [5 * max_grad, 0.0], [-5 * max_grad, 0.0], [-2 * max_grad, 2.0],
                                   [-0.5 * max_grad, 1.0], [5 * max_grad, 1.0]], device=dev))
    grad_rows = torch.cat(grad_rows)
    win_d, win_c = _window(s_d, 4), _window(s_star, 64)
    scale_rows = []
    for k in range(3):
        for w, other in ((win_d, -3.5), (win_c, float(s_star) - 0.5)):
            r = torch.full((w.numel(), 3), other, device=dev)
            r[:, k] = w
            scale_rows.append(r)
    scale_rows.append(torch.tensor([[-5.0, -4.5, -4.0], [-2.0, -1.6, -2.2], [-1.0, -0.5, 1.5]], device=dev))
    scale_rows = torch.cat(scale_rows)
    op_rows = torch.cat((_window(o0, 4), torch.tensor([3.0], device=dev)))

    # the reference's view of each window: on, below and above its threshold
    assert _sides(grad_rows[:9, 0] / grad_rows[:9, 1], max_grad) == (True, True, True)
    assert _sides(torch.exp(win_d), t_dense) == (True, True, True)
    assert _sides(_child_act(torch.exp(win_c), N), t_big) == (True, True, True)
    assert _sides(torch.sigmoid(op_rows[:9]), min_opacity) == (True, True, True)

    gi, si, oi = (t.reshape(-1) for t in torch.meshgrid(torch.arange(grad_rows.shape[0], device=dev),
                                                         torch.arange(scale_rows.shape[0], device=dev),
                                                         torch.arange(op_rows.shape[0], device=dev), indexing="ij"))
    P = gi.numel()
    r = lambda *s: torch.randn(*s, device=dev, generator=g)  # noqa: E731
    params = {"xyz": r(P, 3), "f_dc": r(P, 1, 3), "f_rest": r(P, M - 1, 3) * 0.1, "opacity": op_rows[oi][:, None].clone(),
              "scaling": scale_rows[si].contiguous(), "rotation": r(P, 4)}
    adam = {k: (r(*v.shape), r(*v.shape).abs()) for k, v in params.items()}
    accum, denom = grad_rows[gi, 0:1].contiguous(), grad_rows[gi, 1:2].contiguous()
    kw = dict(max_grad=max_grad, min_opacity=min_opacity, extent=extent, percent_dense=percent_dense, N=N)
    return params, adam, accum, denom, kw


@pytest.mark.parametrize("max_screen", [20, None])
@pytest.mark.parametrize("N", [1, 2, 3])
def test_decisions_on_their_boundaries_equal_the_reference(N, max_screen):
    params, adam, accum, denom, kw = _boundary_case(N)
    kw["max_screen_size"] = max_screen
    P = params["xyz"].shape[0]
    z = torch.randn(N * P, 3, device="cuda", generator=_gen(7))
    want_p, want_a = REF.densify_and_prune(params, adam, accum.clone(), denom, z=z, **kw)
    got_p, got_a, info = D.densify_and_prune(params, adam, accum.clone(), denom, z=z, **kw)
    plan = _plan(params, accum, denom, **kw)
    _, clone, split, child_keep = plan
    neg = (accum.squeeze(-1) < 0)
    assert clone[neg].any() and not split[neg].any()          # |g| clones, g never splits
    assert clone.any() and split.any() and 0 < int(child_keep.sum()) < int(split.sum())
    if max_screen:
        # children on the world-size threshold, and one the reference prunes where a true division would keep it
        e = torch.exp(params["scaling"][split])
        t_big = _f32(0.1 * kw["extent"])
        assert (_child_act(e, N).max(dim=1).values == t_big).any()
        c_div = torch.exp(torch.log(e / torch.tensor(0.8 * N, device="cuda"))).max(dim=1).values
        opaque = (torch.sigmoid(params["opacity"][split]) >= kw["min_opacity"]).squeeze(-1)
        assert (~child_keep & opaque & (c_div <= t_big)).any()
    _compare(got_p, got_a, info, want_p, want_a, plan, params, z, N)


# ---- 3. production sizes ---------------------------------------------------------------------------------------------
def test_densify_and_prune_at_1_1M_rows_through_the_scan_carry_loop():
    P, N, M = 1_100_000, 2, 16
    assert (4 * P + 4095) // 4096 > 1024                    # the 4P-flag scan has more than 1024 block sums
    params, adam, accum, denom = _model(P, M=M, seed=21)
    kw = dict(max_grad=1e-3, min_opacity=0.05, extent=5.0, max_screen_size=20, percent_dense=0.01, N=N)
    z = torch.randn(N * P, 3, device="cuda", generator=_gen(22))
    got_p, got_a, info = D.densify_and_prune(params, adam, accum, denom, z=z, **kw)
    src, clone, split, child_keep = _plan(params, accum, denom, **kw)
    assert torch.equal(info["src_map"], src)
    n_keep, n_clone = info["kept"], info["cloned"]
    assert (n_clone, info["split_parents"], info["split_parents_surviving"]) == \
        (int((src >= KIND[1]).sum()), int(split.sum()), int(child_keep.sum()))
    assert info["points"] == n_keep + n_clone + N * info["split_parents_surviving"] == src.numel()
    rows = (src & ((1 << 30) - 1)).long()
    first_child = n_keep + n_clone
    for k in REF.NAMES:
        if k in ("xyz", "scaling"):
            assert torch.equal(got_p[k][:first_child], params[k][rows[:first_child]]), k
        else:
            assert torch.equal(got_p[k], params[k][rows]), k
        for got, m in zip(got_a[k], adam[k]):
            assert torch.equal(got[:n_keep], m[rows[:n_keep]]) and not got[n_keep:].any(), k
    _check_children(got_p, first_child, params, z, split, child_keep, N)


def test_prune_points_at_4_2M_rows_through_the_scan_carry_loop():
    P, M = 4_200_001, 16
    assert (P + 4095) // 4096 > 1024 and P % 4 and P % 4096
    params, _, _, _ = _model(P, M=M, seed=31, adam=False)
    g = _gen(32)
    adam = {k: tuple(torch.randn(P, *params[k].shape[1:], device="cuda", generator=g) for _ in range(2))
            for k in ("xyz", "opacity")}
    stats = {"row": torch.arange(P, device="cuda", dtype=F32), "denom": torch.rand(P, 1, device="cuda", generator=g)}
    mask = torch.rand(P, device="cuda", generator=g) < 0.37
    new_p, new_a, new_s = D.prune_points(params, adam, stats, mask)
    keep = (~mask).nonzero().squeeze(1)
    assert torch.equal(new_s["row"], keep.float())          # the index set (rows are exact in fp32 below 2^24)
    assert torch.equal(new_s["denom"], stats["denom"][keep])
    for k in params:
        assert torch.equal(new_p[k], params[k][keep]), k
    for k in adam:
        assert torch.equal(new_a[k][0], adam[k][0][keep]) and torch.equal(new_a[k][1], adam[k][1][keep]), k


@pytest.mark.parametrize("P", [0, 1, 4097])
@pytest.mark.parametrize("mask_kind", ["all", "none", "random"])
def test_prune_points_with_all_no_and_some_rows(P, mask_kind):
    params, adam, accum, denom = _model(P, seed=40 + P)
    mask = {"all": torch.ones(P, dtype=torch.bool, device="cuda"), "none": torch.zeros(P, dtype=torch.bool, device="cuda"),
            "random": torch.rand(P, device="cuda", generator=_gen(41)) < 0.5}[mask_kind]
    stats = {"xyz_gradient_accum": accum, "denom": denom}
    new_p, new_a, new_s = D.prune_points(params, adam, stats, mask)
    for k in params:
        assert torch.equal(new_p[k], params[k][~mask]), k
        assert torch.equal(new_a[k][0], adam[k][0][~mask]) and torch.equal(new_a[k][1], adam[k][1][~mask]), k
    for k in stats:
        assert torch.equal(new_s[k], stats[k][~mask]), k


# ---- 4. radix select against torch.sort ------------------------------------------------------------------------------
def _bits(b):
    """float32 values from their bit patterns (int64 in [0, 2^32))."""
    return torch.where(b >= 1 << 31, b - (1 << 32), b).to(torch.int32).view(F32)


_SPECIALS = [0xFF800000, 0x7F800000, 0x80000000, 0x00000000, 0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF,
             0x00800000, 0x80800000, 0x7F7FFFFF, 0xFF7FFFFF, 0xBFC00000, 0x40400000]
_DIGIT_EDGES = [0x3F80FFFE, 0x3F80FFFF, 0x3F810000, 0x3F810001, 0x3FFFFFFF, 0x40000000, 0xBF80FFFF, 0xBF810000]


def _values(n, dist, g):
    """Test vectors of the radix select (the keys are the float bits, one 8-bit digit per pass)."""
    dev = "cuda"
    ri = lambda hi: torch.randint(0, hi, (n,), device=dev, generator=g)  # noqa: E731
    if dist == "normal":
        return torch.randn(n, device=dev, generator=g)
    if dist == "all_equal":
        return torch.full((n,), -0.37, device=dev)
    if dist == "low_byte":                              # negatives (reversed keys) that differ in the last digit only
        return _bits(0xC0490F00 + ri(256))
    if dist == "high_byte":                             # both signs, normal and subnormal: only the first digit varies
        return _bits(ri(256) * (1 << 24) + 0x2B5A3C)
    if dist == "digit_runs":                            # runs of equal values ending on a digit boundary
        return _bits(torch.tensor(_DIGIT_EDGES, device=dev)[ri(len(_DIGIT_EDGES))])
    if dist == "specials":                              # +-inf, +-0, subnormals, min normals, +-max
        return _bits(torch.tensor(_SPECIALS, device=dev)[ri(len(_SPECIALS))])
    v = torch.randn(n, device=dev, generator=g)
    nans = [0x7FC00000, 0x7F800001] + ([0xFFC00000, 0xFFFFFFFF] if dist == "signed_nan" else [])
    pick = ri(5 * len(nans))                            # about a fifth NaNs
    return torch.where(pick < len(nans), _bits(torch.tensor(nans, device=dev)[pick.clamp(max=len(nans) - 1)]), v)


def _same(got, want):
    return (math.isnan(got) and math.isnan(want)) or got == want


@pytest.mark.parametrize("dist", ["normal", "all_equal", "low_byte", "high_byte", "digit_runs", "specials", "pos_nan",
                                  "signed_nan"])
@pytest.mark.parametrize("n", [1, 2, 255, 256, 257, 4097, (1 << 20) + 3])
def test_kth_smallest_equals_torch_sort(n, dist):
    v = _values(n, dist, _gen(n))
    # every NaN sorts last, whatever its sign bit (torch.sort's order of positive NaNs; kth_smallest maps all NaNs there)
    want = torch.sort(torch.where(v.isnan(), torch.full_like(v, float("nan")), v))[0]
    if dist != "signed_nan":
        want = torch.sort(v)[0]
    ks = sorted({k for k in (0, 1, n // 2, n - 2, n - 1, n - 1 - int(0.9 * n)) if 0 <= k < n})
    for k in ks:
        got, w = float(D.kth_smallest(v, k)), float(want[k])
        assert _same(got, w), (k, got, w)
    for percent in (0.0, 0.1, 0.5, 1.0):
        got, w = float(D.percentile_threshold(v, percent)), float(want[int(percent * (n - 1))])
        assert _same(got, w), (percent, got, w)


# ---- 5. the in-place event on the boundary rows ----------------------------------------------------------------------
def test_reserved_group_densify_on_the_boundary_rows_equals_the_functional_call():
    from dreamscene_b200 import GaussianAdam
    from dreamscene_b200.reserve import ReservedGroup
    N = 2
    params, adam, accum, denom, kw = _boundary_case(N, M=16)
    kw["max_screen_size"] = 20
    P = params["xyz"].shape[0]
    z = torch.randn(N * P, 3, device="cuda", generator=_gen(51))
    want_p, want_a, info = D.densify_and_prune(params, adam, accum, denom, z=z, **kw)
    leaf = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity",
            "scaling": "_scaling", "rotation": "_rotation"}
    cap = max(P, info["points"]) + 777
    g = ReservedGroup.from_tensors(params["xyz"], params["f_dc"], params["f_rest"], params["opacity"], params["scaling"],
                                   params["rotation"], capacity=cap, stats=(accum, denom, torch.rand(P, device="cuda")))
    opt = GaussianAdam(g.param_groups({k: 1e-3 for k in leaf}), lr=0.0, eps=1e-15)
    for k, name in leaf.items():
        st = {"step": torch.tensor(3.0)}
        for m, src in zip(("exp_avg", "exp_avg_sq"), adam[k]):
            st[m] = torch.zeros_like(getattr(g, name))
            st[m][:P] = src
        opt.state[getattr(g, name)] = st
    ptrs = [getattr(g, name).data_ptr() for name in leaf.values()]
    got = g.densify_and_prune(opt, z=z, **kw)
    n = g.live_count
    assert got["points"] == n == info["points"] and int(g.live.item()) == n and g.capacity == cap
    assert torch.equal(got["src_map"], info["src_map"])
    assert [getattr(g, name).data_ptr() for name in leaf.values()] == ptrs
    for k, name in leaf.items():
        t = getattr(g, name)
        assert torch.equal(t[:n], want_p[k]), k
        for m, want in zip(("exp_avg", "exp_avg_sq"), want_a[k]):
            assert torch.equal(opt.state[t][m][:n], want), (k, m)
    for t in g.stats:
        assert not t.view(-1)[:n].any()
