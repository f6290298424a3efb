"""The fused disparity (dreamscene_b200.postprocess, csrc/postprocess.cu) bit for bit against torch's own evaluation of
the reference expression (DreamScene's scene_gaussian.py:871-881, restated as tests.test_gpu_postprocess.
reference_disparity) on CUDA, in default and deterministic mode:

* the forward, NaN in the same places (a view whose max equals min_d divides 0 by 0), and the alpha it returns;
* the gradient outside the min / max tie sets, which is a purely elementwise fp32 chain;
* the tie sets themselves, found from where the gradient is non-zero when g_disp is non-zero on a few probe pixels;
* on the tie sets, where the kernel sums over the view in its own order, the distance to an fp64 evaluation that uses
  the fp32 decisions (mask, ties, clamp gate), within the fp32 summation bound N eps sum|terms|.

Inputs: 512^2 renders of the small room from inside it, of an object with background and of a faint object no pixel of
which is opaque (the fallback min_d, tied over the whole background); constructed views on the 0.1 mask boundary, with
ties of 2..64 pixels, with pixel pairs whose x differ but whose rcp(x) * focal coincide, the two views whose max equals
min_d, N = 1, 255, 257, 221, one 1024^2 view and a batch of B200GSR_MAX_VIEWS views.  Then two routes end to end:
StepGraph.render against the expression on render_scene's depth_alpha, and render_frames against the reference's
video loop over the expression."""
import contextlib
import math

import numpy as np
import pytest
import torch

from dreamscene_b200 import _lib
from dreamscene_b200.postprocess import disparity_from_depth_alpha
from harness import cameras, video_ref
from tests import util_scene as U
from tests.test_gpu_postprocess import reference_disparity

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -23
F32 = np.float32
MODES = pytest.mark.parametrize("det", [False, True], ids=["default", "deterministic"])


@contextlib.contextmanager
def _mode(det):
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(old)


def _focal(fovx):
    return 1.0 / (2.0 * math.tan(fovx / 2.0))


def _same(a, b):
    """Bitwise equal as torch.equal sees it (-0 == 0), NaN in the same places."""
    na, nb = a.isnan(), b.isnan()
    return torch.equal(na, nb) and torch.equal(a[~na], b[~nb])


# ---- torch's forms, pinned on the GPU ----------------------------------------------------------------------------

def test_torch_forms_the_kernel_reproduces():
    """The rounding forms csrc/postprocess.cu reproduces, pinned against torch's CUDA ops: focal / x is
    x.reciprocal() * focal and reciprocal is the correctly rounded 1 / x; a tensor over a 0-dim CUDA tensor is a true
    division; alpha <= 0.1 compares with 0.1f; clamp keeps NaN; the autograd of the expression, outside the tie sets,
    is the fp32 chain Clamp-, Div-, Mul-, ReciprocalBackward (and * 10 + g_alpha on the alpha channel)."""
    g = torch.Generator(device="cuda").manual_seed(0)
    n = 1 << 22
    x = torch.exp2(torch.rand(n, device="cuda", generator=g) * 24 - 17) * (1 + torch.rand(n, device="cuda", generator=g))
    for f in (_focal(0.96), _focal(0.55), _focal(0.7), 1.0 / 3.0):
        assert torch.equal(f / x, x.reciprocal() * f), f
        ff = float(F32(f))
        assert torch.equal(f / x, x.reciprocal() * ff), f          # the scalar enters as its float32 value
        print("focal / x differs from the correctly rounded quotient on", int((f / x != (ff / x.double()).float())
                                                                             .sum()), "of", n)
    # correctly rounded: double rounding through fp64 is exact for a quotient of floats (53 >= 2 * 24 + 2)
    assert torch.equal(x.reciprocal(), (1.0 / x.double()).float())
    t = torch.rand(n, device="cuda", generator=g)
    for den in (0.37, 3.0, 1e-3, 0.7431):
        den_t = torch.tensor(den, device="cuda")
        assert den_t.dim() == 0
        assert torch.equal(t / den_t, (t.double() / den_t.double()).float()), den
    # the mask's constant is 0.1f
    b = torch.tensor([float(np.nextafter(F32(0.1), F32(0))), float(F32(0.1)), float(np.nextafter(F32(0.1), F32(1)))],
                     device="cuda")
    assert (b <= 0.1).tolist() == [True, True, False]
    c = torch.tensor([float("nan"), -float("inf"), float("inf"), 0.5, -0.0, 1.0], device="cuda")
    out = torch.clamp(c, 0.0, 1.0)
    assert bool(out[0].isnan()) and out[1:].tolist() == [0.0, 1.0, 0.5, 0.0, 1.0]
    # autograd of the expression against the explicit fp32 composition, outside the tie sets
    H, W = 256, 192
    f = _focal(0.96)
    da = _constructed(H, W, np.random.RandomState(1), opaque=0.5, background=0.2)
    gd = torch.randn(1, H, W, device="cuda", generator=g)
    ga = torch.randn(1, H, W, device="cuda", generator=g)
    _, _, tg = _torch(da, f, gd, ga)
    dec = _decisions(da, f)
    gq = torch.where(dec["gate"], gd, torch.zeros_like(gd)) / dec["den"]
    gx = -((gq * float(F32(f))) * (dec["r"] * dec["r"]))
    want = torch.cat([gx, gx * 10 + ga])
    keep = ~(dec["tmin"] | dec["tmax"])
    assert int(keep.sum()) > H * W // 2 and int((~dec["gate"]).sum()) > 0
    assert torch.equal(tg[:, keep[0]], want[:, keep[0]])


# ---- the oracle and the checks -----------------------------------------------------------------------------------

def _torch(da, focal, g_disp, g_alpha):
    """reference_disparity evaluated and differentiated by torch on CUDA, for one view [2,H,W]."""
    x = da.clone().requires_grad_(True)
    with _mode(False):
        d, a = reference_disparity(x, focal)
        outs, grads = [d], [g_disp]
        if g_alpha is not None:
            outs.append(a)
            grads.append(g_alpha)
        torch.autograd.backward(outs, grads)
    return d.detach(), a.detach(), x.grad


def _kernel(da, focals, g_disp, g_alpha, det):
    x = da.clone().requires_grad_(True)
    with _mode(det):
        d, a = disparity_from_depth_alpha(x, focals)
        outs, grads = [d], [g_disp]
        if g_alpha is not None:
            outs.append(a)
            grads.append(g_alpha)
        torch.autograd.backward(outs, grads)
    return d.detach(), a.detach(), x.grad


def _decisions(da, focal):
    """The fp32 values and decisions of the expression for one view, in torch's forms (pinned above)."""
    depth, alpha = da[0:1], da[1:2]
    r = (depth + alpha * 10 + 1e-5).reciprocal()
    d = r * focal
    mask = alpha <= 0.1
    masked = bool(mask.any())
    m = d[mask].min() if masked else d.min()
    M = d.max()
    den = M - m
    q = (d - m) / den
    return {"r": r, "d": d, "mask": mask, "masked": masked, "m": m, "M": M, "den": den, "gate": (q >= 0) & (q <= 1),
            "tmin": (d == m) & mask if masked else d == m, "tmax": d == M}


def _tie_reference(dec, focal, g_disp, g_alpha):
    """fp64 gradient on the tie pixels from the fp32 decisions, and two error bounds on it: the sums through min_d and
    disp.max() are sum_j gq_j (d_j - M) / den^2 and -sum_j gq_j (d_j - m) / den^2, and a bound is
    (N + 16) eps (|gq / den| + sum|terms| / ties) focal r^2 per pixel: the fp32 summation bound plus the chain's few
    roundings.  The kernel sums those terms; torch sums gq / den and gq q / den separately (q = (d - m) / den, the
    backwards of the subtraction and of the division by den), so its terms are those two."""
    d, r = dec["d"].double(), dec["r"].double()
    m, M, den = float(dec["m"]), float(dec["M"]), float(dec["den"])
    f = float(F32(focal))
    N = d.numel()
    gq = torch.where(dec["gate"], g_disp.double(), torch.zeros_like(d))
    tmin, tmax = dec["tmin"].double(), dec["tmax"].double()
    s_min, s_max = gq * (d - M) / den ** 2, -gq * (d - m) / den ** 2
    cmin, cmax = tmin.sum(), tmax.sum()
    gd = gq / den + tmin * s_min.sum() / cmin + tmax * s_max.sum() / cmax
    fr2 = f * r * r
    gx = -gd * fr2
    ga = 10 * gx + (g_alpha.double() if g_alpha is not None else 0.0)
    s_y, s_q = (gq / den).abs().sum(), (gq * (d - m) / den ** 2).abs().sum()
    bounds = []
    for sum_min, sum_max in ((s_min.abs().sum(), s_max.abs().sum()), (s_y + s_q, s_q)):
        mag = (gq / den).abs() + tmin * sum_min / cmin + tmax * sum_max / cmax
        bx = (N + 16) * EPS * mag * fr2
        ba = 10 * bx + 4 * EPS * (10 * mag * fr2 + (g_alpha.double().abs() if g_alpha is not None else 0.0))
        bounds.append(torch.cat([bx, ba]))
    return torch.cat([gx, ga]), bounds


def _check(da, focals, det, seed=0, probes=4):
    """Every check of this file on a batch da [B,2,H,W] with Python-float focals; the kernel's departures from torch
    are collected and reported together (NaN placement, forward values, alpha, the gradient outside the ties, the tie
    values, the tie sets, deterministic repeats).  -> the per-view decisions."""
    B, _, H, W = da.shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    gd = torch.randn(B, 1, H, W, device="cuda", generator=g)
    ga = torch.randn(B, 1, H, W, device="cuda", generator=g)
    d, a, grad = _kernel(da, focals, gd, ga, det)
    bad = []
    if det:
        d2, _, grad2 = _kernel(da, focals, gd, ga, det)
        if not (torch.equal(d.view(torch.int32), d2.view(torch.int32))
                and torch.equal(grad.view(torch.int32), grad2.view(torch.int32))):
            bad.append(("deterministic repeat",))
    decs = []
    gp = torch.zeros(B, 1, H, W, device="cuda")
    for v in range(B):
        td, ta, tg = _torch(da[v], focals[v], gd[v], ga[v])
        if not torch.equal(d[v].isnan(), td.isnan()):
            bad.append(("NaN forward", v, int((d[v].isnan() != td.isnan()).sum())))
        elif not _same(d[v], td):
            bad.append(("forward", v, int((d[v] != td).sum())))
        if not torch.equal(a[v], ta):
            bad.append(("alpha", v))
        dec = _decisions(da[v], focals[v])
        decs.append(dec)
        ties = (dec["tmin"] | dec["tmax"])[0]
        if float(dec["den"]) == 0.0:          # max == min_d: torch's gradient is NaN everywhere, and so must ours be
            assert bool(tg.isnan().all()), v
            if not bool(grad[v].isnan().all()):
                bad.append(("NaN gradient", v, int((~grad[v].isnan()).sum())))
            continue
        if not _same(grad[v][:, ~ties], tg[:, ~ties]):
            bad.append(("gradient outside the ties", v, int((grad[v][:, ~ties] != tg[:, ~ties]).sum())))
        want, bounds = _tie_reference(dec, focals[v], gd[v], ga[v])
        for who, got, bound in (("kernel", grad[v], bounds[0]), ("torch", tg, bounds[1])):
            err = (got[:, ties].double() - want[:, ties]).abs()
            if not bool((err <= bound[:, ties]).all()):
                assert who == "kernel", ("torch's ties against fp64", v, float((err / bound[:, ties]).max()))
                bad.append(("tie values", v, float((err / bound[:, ties]).max())))
        cand = dec["gate"] & ~dec["tmin"] & ~dec["tmax"] & (dec["d"] > dec["m"]) & (dec["d"] < dec["M"])
        idx = cand.reshape(-1).nonzero()[:, 0]
        if idx.numel():
            pick = idx[torch.randperm(idx.numel(), device="cuda", generator=g)[:probes]]
            gp[v].view(-1)[pick] = torch.randn(pick.numel(), device="cuda", generator=g)
    # the tie sets: with g_disp non-zero on a few probe pixels only, the gradient is non-zero on exactly the probes and
    # the two tie sets, in torch and in the kernel
    _, _, pgrad = _kernel(da, focals, gp, None, det)
    for v in range(B):
        if not bool(gp[v].any()):
            continue
        _, _, tg = _torch(da[v], focals[v], gp[v], None)
        want = ((gp[v] != 0) | decs[v]["tmin"] | decs[v]["tmax"])[0]
        assert torch.equal(tg[0] != 0, want) and torch.equal(tg[1] != 0, want), ("torch's tie sets", v)
        if not (torch.equal(pgrad[v][0] != 0, want) and torch.equal(pgrad[v][1] != 0, want)):
            bad.append(("tie sets", v, int(((pgrad[v][0] != 0) != want).sum())))
    assert not bad, bad
    return decs


# ---- constructed views -------------------------------------------------------------------------------------------

def _constructed(H, W, rs, opaque=0.5, background=0.0, fallback=False):
    """A synthetic depth_alpha [2,H,W] (channel 1 the transmittance T): a fraction `opaque` of the pixels with
    T <= 0.05 and depth in (1.9, 4.85), the rest T in (0.2, 1); a fraction `background` at depth 0 and T 1.
    fallback: no pixel has T <= 0.1."""
    T = rs.uniform(0.2, 1.0, (H, W)).astype(F32)
    if not fallback:
        op = rs.uniform(size=(H, W)) < opaque
        T[op] = (T[op] * F32(0.05)).astype(F32)
    depth = ((F32(1) - T) * rs.uniform(2.0, 5.0, (H, W)).astype(F32)).astype(F32)
    bg = rs.uniform(size=(H, W)) < background
    depth[bg], T[bg] = 0.0, 1.0
    return torch.from_numpy(np.stack([depth, T])).cuda()


def _x_np(depth, T):
    return ((depth + T * F32(10)) + F32(1e-5)).astype(F32)


def _coincident_depths(lo, hi, focal, rs, n=1):
    """n pairs of depths (at T = 0) in [lo, hi) whose x differ and whose torch disparity rcp(x) * focal is the same,
    while the correctly rounded focal / x is not: ties that only torch's two roundings make."""
    f = F32(focal)
    d1 = rs.uniform(lo, hi, 200_000).astype(F32)
    d2 = np.nextafter(d1, F32(hi + 1))
    x1, x2 = _x_np(d1, F32(0)), _x_np(d2, F32(0))
    same = (x1 != x2) & ((F32(1) / x1) * f == (F32(1) / x2) * f) & (f / x1 != f / x2)
    k = np.flatnonzero(same)
    assert k.size >= n, (lo, hi, focal)
    k = k[:n]
    return list(zip(d1[k], d2[k]))


@MODES
def test_mask_boundary_on_the_minimum(det):
    """The pixel that would be the masked minimum at T = 0.1f and one ulp either side: in the mask (and min_d) at and
    below 0.1f, out of it one ulp above."""
    H, W = 64, 72
    rs = np.random.RandomState(2)
    ts = [np.nextafter(F32(0.1), F32(0)), F32(0.1), np.nextafter(F32(0.1), F32(1))]
    views = []
    for t in ts:
        da = _constructed(H, W, rs)
        da[0, 20, 30], da[1, 20, 30] = 6.0, float(t)            # x ~ 7: past every other opaque pixel's 5.4
        views.append(da)
    f = _focal(0.96)
    decs = _check(torch.stack(views), [f] * 3, det, seed=2)
    for dec, inside in zip(decs, (True, True, False)):
        assert bool(dec["mask"][0, 20, 30]) == inside
        assert bool(dec["tmin"][0, 20, 30]) == inside and (int(dec["tmin"].sum()) == 1 or not inside)


@MODES
def test_ties_of_several_pixels(det):
    """Min ties (masked) and max ties of k = 2, 3, 7, 64 pixels with the same depth and T."""
    H, W = 80, 96
    rs = np.random.RandomState(3)
    views, ks = [], (2, 3, 7, 64)
    for k in ks:
        da = _constructed(H, W, rs, background=0.1)
        pix = rs.permutation(H * W)[:2 * k]
        dv, tv = da[0].view(-1), da[1].view(-1)
        dv[pix[:k]], tv[pix[:k]] = 6.0, 0.05                    # the masked minimum, k times
        dv[pix[k:]], tv[pix[k:]] = 0.01, 0.0                    # the maximum, k times
        views.append(da)
    focals = [_focal(fx) for fx in (0.96, 0.55, 0.7, 1.1)]
    decs = _check(torch.stack(views), focals, det, seed=3)
    for k, dec in zip(ks, decs):
        assert int(dec["tmin"].sum()) == k and int(dec["tmax"].sum()) == k


@MODES
def test_ties_of_different_x_with_the_same_disparity(det):
    """Pairs of pixels whose x differ by one ulp but whose rcp(x) * focal coincide (and whose correctly rounded
    focal / x do not), placed on the masked minimum and on the maximum: each tie set is the pair."""
    H, W = 64, 64
    rs = np.random.RandomState(4)
    views, focals = [], [_focal(fx) for fx in (0.96, 0.55, 0.8)]
    for f in focals:
        da = _constructed(H, W, rs)
        (lo1, lo2), = _coincident_depths(6.0, 7.0, f, rs)
        (hi1, hi2), = _coincident_depths(0.005, 0.02, f, rs)
        mids = _coincident_depths(1.0, 4.0, f, rs, n=8)         # pairs inside the range as well
        for (p, q), (a, b) in zip([((3, 5), (40, 41)), ((10, 60), (63, 0))], [(lo1, lo2), (hi1, hi2)]):
            da[0][p], da[1][p], da[0][q], da[1][q] = float(a), 0.0, float(b), 0.0
        for j, (a, b) in enumerate(mids):
            da[0, 30, 2 * j], da[1, 30, 2 * j], da[0, 31, 2 * j], da[1, 31, 2 * j] = float(a), 0.0, float(b), 0.0
        views.append(da)
    decs = _check(torch.stack(views), focals, det, seed=4)
    for dec in decs:
        assert int(dec["tmin"].sum()) == 2 and int(dec["tmax"].sum()) == 2
        assert bool(dec["tmin"][0, 3, 5] & dec["tmin"][0, 40, 41] & dec["tmax"][0, 10, 60] & dec["tmax"][0, 63, 0])


@MODES
def test_views_whose_max_equals_min_d(det):
    """An all-background view (the fallback min_d over equal values) and a view whose only pixel with T <= 0.1 is its
    maximum: max - min_d = 0, and torch gives 0 / 0 = NaN at the pixels equal to min_d and NaN gradients everywhere.
    With an ordinary view beside them, which they must not disturb."""
    H, W = 48, 40
    rs = np.random.RandomState(5)
    empty = torch.zeros(2, H, W, device="cuda")
    empty[1] = 1.0
    single = _constructed(H, W, rs, fallback=True)
    single[0, 7, 9], single[1, 7, 9] = 0.01, 0.05
    ordinary = _constructed(H, W, rs, background=0.3)
    focals = [_focal(0.96), _focal(0.7), _focal(0.55)]
    decs = _check(torch.stack([empty, single, ordinary]), focals, det, seed=5)
    assert float(decs[0]["den"]) == 0.0 and not decs[0]["masked"]
    assert float(decs[1]["den"]) == 0.0 and decs[1]["masked"] and int(decs[1]["mask"].sum()) == 1
    d, _ = disparity_from_depth_alpha(torch.stack([empty, single, ordinary]), focals)
    assert bool(d[0].isnan().all()) and int(d[1].isnan().sum()) == 1 and bool(d[1][0, 7, 9].isnan())
    assert not bool(d[2].isnan().any()) and float(d[2].max()) == 1.0


@MODES
@pytest.mark.parametrize("H,W", [(1, 1), (15, 17), (1, 257), (13, 17), (1024, 1024)])
def test_view_sizes(det, H, W):
    """N = 1 (max == min_d), 255, 257, 221 (not a multiple of 4), and 1024^2 (the grid-stride loop goes round more
    than once); one view with opaque pixels and one on the fallback min_d."""
    rs = np.random.RandomState(H * W)
    da = torch.stack([_constructed(H, W, rs, background=0.2), _constructed(H, W, rs, fallback=True, background=0.2)])
    decs = _check(da, [_focal(0.96), _focal(0.6)], det, seed=H + W)
    if H * W > 1:
        assert decs[0]["masked"] and not decs[1]["masked"]


@MODES
def test_max_views_with_different_focals(det):
    """B200GSR_MAX_VIEWS views, each with its own focal, alternating fallback and masked views."""
    B, H, W = _lib.MAX_VIEWS, 96, 80
    rs = np.random.RandomState(6)
    da = torch.stack([_constructed(H, W, rs, background=0.15 * (v % 3), fallback=v % 2 == 1) for v in range(B)])
    focals = [_focal(0.4 + 0.05 * v) for v in range(B)]
    decs = _check(da, focals, det, seed=6)
    assert [dec["masked"] for dec in decs] == [v % 2 == 0 for v in range(B)]


# ---- real renders ------------------------------------------------------------------------------------------------

def _object_groups(n, opacity=None, seed=1, M=4):
    """A compact ball of small Gaussians, which leaves most of an orbit view's frame untouched (depth 0, T 1)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    op = r(n, 1) * 2 if opacity is None else torch.full((n, 1), math.log(opacity / (1 - opacity)), device="cuda")
    return [{"_xyz": r(n, 3) * 0.3, "_opacity": op, "_scaling": r(n, 3) * 0.3 - 4.0, "_rotation": r(n, 4),
             "_features_dc": r(n, 1, 3), "_features_rest": r(n, M - 1, 3) * 0.3}]


def _render(groups, cams, deg):
    from dreamscene_b200.scene import render_scene
    S = [U.cuda_settings(c, deg, bg=(0.2, 0.3, 0.4)) for c in cams]
    with torch.no_grad():
        outs = render_scene(groups, S, shs_aug=False, scale_aug=False)
    return torch.stack([o[2] for o in outs]).contiguous(), [_focal(c.FoVx) for c in cams]


def _orbit(size, n=4):
    return [cameras.orbit_camera(radius=3.5, theta_deg=50.0 + 9 * v, phi_deg=80.0 * v, fovx=0.7, height=size,
                                 width=size) for v in range(n)]


_renders: dict = {}


def _scene(kind):
    if kind not in _renders:
        if kind == "room":
            from harness import room
            from tests.test_gpu_room import DEG, M, SMALL, views
            groups = room.named_groups(room.build_scene(torch.device("cuda"), M=M, **SMALL))
            _renders[kind] = _render(groups, views(512), DEG)
        elif kind == "object":
            _renders[kind] = _render(_object_groups(3000), _orbit(512), 1)
        else:
            _renders[kind] = _render(_object_groups(800, opacity=0.1, seed=2), _orbit(512), 1)
    return _renders[kind]


@MODES
@pytest.mark.parametrize("kind", ["room", "object", "faint_object"])
def test_renders(det, kind):
    """Four 512^2 views each: the small room from cameras inside it (almost every pixel opaque, no background), an
    object with background, and an early-training object at opacity 0.1 that no pixel sees opaquely (the fallback
    min_d, whose tie set is every background pixel)."""
    da, focals = _scene(kind)
    decs = _check(da, focals, det, seed=7)
    T = da[:, 1:2]
    if kind == "room":
        assert all(float(dec["mask"].float().mean()) > 0.5 for dec in decs)
    elif kind == "object":
        assert all(dec["masked"] for dec in decs) and all(int((T[v] == 1).sum()) > 1000 for v in range(len(decs)))
    else:
        for v, dec in enumerate(decs):
            background = (da[v, 0:1] == 0) & (T[v] == 1)
            assert not dec["masked"], v                    # no pixel with T <= 0.1: the reference's except branch
            assert int(background.sum()) > 1000 and torch.equal(dec["tmin"], background), v


# ---- two routes end to end ---------------------------------------------------------------------------------------

def test_step_graph_disparity_equals_the_expression():
    """StepGraph.render's disparity against the expression on the depth_alpha of the eager render_scene with the
    same seed and augmentation, one of the four views seeing nothing (its disparity NaN where torch's is)."""
    from dreamscene_b200 import StepGraph
    from dreamscene_b200.scene import render_scene
    from tests.test_gpu_frames import _away
    from tests.test_gpu_scene_render import _clone, _groups
    from tests.test_gpu_step_graph import _optimizers, _step_settings
    B, H, W, M = 4, 96, 80, 16
    ge = _groups([3000], M, seed=1)
    gg = _clone(ge)
    sg = StepGraph(gg, _optimizers(gg), views=B, height=H, width=W)
    S = _step_settings(B, H, W, M, 0)
    S[3] = U.cuda_settings(_away(H, W), 1, bg=(0.5, 0.5, 0.5))
    for seed in (11, 12):
        out = sg.render(S, shs_aug=True, scale_aug=True, seed=seed)
        with torch.no_grad():
            outs = render_scene(ge, S, shs_aug=True, scale_aug=True, seed=seed)
        nan_views = 0
        for v in range(B):
            ref, _ = reference_disparity(outs[v][2], 1.0 / (2.0 * float(S[v].tanfovx)))
            assert _same(out.disp[v].detach(), ref), (seed, v)
            nan_views += bool(ref.isnan().any())
        assert nan_views == 1


def test_render_frames_depth_equals_the_loop_over_the_expression(monkeypatch):
    """render_frames against the reference's video loop whose render callable returns the torch expression (not the
    native disparity): every rgb and depth frame bit for bit, the view that sees nothing included."""
    from dreamscene_b200 import rasterizer as R
    from dreamscene_b200.scene import render_scene
    from dreamscene_b200.video import render_frames
    from tests.test_gpu_frames import _groups, _views
    groups = _groups([3000], 16, seed=1)
    S = _views(9, 16, H=96, W=104, seed=2)

    def render(s):
        color, _, depth_alpha = render_scene(groups, [s], shs_aug=False, scale_aug=False)[0]
        disp, _ = reference_disparity(depth_alpha, 1.0 / (2.0 * float(s.tanfovx)))
        return color, disp

    monkeypatch.setattr(R, "_pair_mode", "sync")
    with torch.no_grad():
        img, dep = video_ref.frames(render, S)
    monkeypatch.undo()
    rgb, depth = render_frames(groups, S, views_per_pass=4)
    np.testing.assert_array_equal(rgb.numpy(), np.stack(img))
    np.testing.assert_array_equal(depth.numpy(), np.stack(dep))
    assert not depth[7].any() and depth[0].max() == 255
