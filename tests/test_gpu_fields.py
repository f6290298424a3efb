"""dreamscene_b200.fields.extract_fields on the GPU against the restatement of the reference (harness/fields_ref.py),
evaluated by torch on the same device.

The filter, the normalisation and the block memberships are compared bit for bit (centre, scale, per-block member
counts).  The field itself is a sum in a different order from the reference's 1024-wide batches, so it is held to

    |occ - occ64| <= RTOL * occ64 + ATOL,   RTOL = 1e-4, ATOL = 1e-5,

against the float64 restatement (the same members, every weight and sum in float64).  On these objects torch's own
float32 evaluation of the reference stays about ten times inside that bound (relative error ~1e-5, absolute ~2e-6 at
fields up to ~5), which the tests assert as well: the bound is what float32 reordering gives, with room for the
native path's own rounding of the covariance inverse and exp2, and nothing larger.
"""
import math

import pytest
import torch

from dreamscene_b200 import fields as Fd
from dreamscene_b200.reserve import ReservedGroup
from harness import fields_ref

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-4, 1e-5
DEV = "cuda"


def _group(P, seed=0, std=0.02, device=DEV):
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(P, 3, generator=g)
    d /= d.norm(dim=1, keepdim=True)
    xyz = 0.5 * torch.rand(P, 1, generator=g) ** (1 / 3) * d
    leaves = dict(_xyz=xyz, _opacity=1.5 * torch.randn(P, 1, generator=g),
                  _scaling=math.log(std) + 0.3 * torch.randn(P, 3, generator=g), _rotation=torch.randn(P, 4, generator=g))
    return {k: v.to(device) for k, v in leaves.items()}


def _within(occ, ref64, rtol=RTOL, atol=ATOL):
    err = (occ.double() - ref64).abs()
    bound = rtol * ref64.abs() + atol
    return bool((err <= bound).all()), float((err / bound).max())


def _native_counts(group, R, nb, rr):
    """Per-block member counts of the native binning, read back from a field in which every member weighs 1 at every
    point: the kept rows get opacity logit 20 (sigmoid 1.0 in float32) and scales so large (~2000 after
    normalisation) that every weight is 1 - O(1e-6), so the first point of a block sums to its member count.  The
    filtered rows keep their opacity, so the kept set, the normalisation and the memberships are unchanged."""
    keep = torch.sigmoid(group["_opacity"]) > 0.005
    flat = dict(group, _opacity=torch.where(keep, torch.full_like(group["_opacity"], 20.0), group["_opacity"]),
                _scaling=torch.full_like(group["_scaling"], 7.0))
    occ, _, _ = Fd.extract_fields(flat, R, nb, rr)
    split = R // nb
    return occ[::split, ::split, ::split].round().long().cpu()


@pytest.mark.parametrize("P,R,nb", [(1000, 64, 8), (10_000, 64, 8), (100_000, 64, 8), (20_000, 128, 16),
                                    (3000, 50, 8)])
def test_field_matches_the_reference(P, R, nb):
    g = _group(P, seed=P + R)
    occ, center, scale = Fd.extract_fields(g, R, nb)
    ref32, c32, s32 = fields_ref.extract_fields(g, R, nb)
    ref64, _, _ = fields_ref.extract_fields(g, R, nb, dtype=torch.float64)
    assert torch.equal(center, c32) and scale == s32
    assert occ.shape == (R, R, R) and occ.dtype == torch.float32 and occ.is_cuda
    ok, worst = _within(occ, ref64)
    assert ok, worst
    ok32, worst32 = _within(ref32, ref64, RTOL / 4, ATOL / 4)    # torch's float32 evaluation, well inside the bound
    assert ok32, worst32
    assert ((occ.double() - ref32.double()).abs() <= 2 * (RTOL * ref64 + ATOL)).all()
    assert float(ref64.max()) > 0.5


def test_memberships_and_centres_are_the_reference_bits():
    """Rows moved onto the relaxed-box boundaries: a normalised coordinate exactly on a chunk's lo or hi, or one float
    step below or above it, each on its own row and axis."""
    g = _group(4000, seed=7)
    R, nb, rr = 64, 8, 1.5
    n = fields_ref.normalise(g)
    center, scale = n["center"], n["scale"]
    coords = torch.linspace(-1, 1, R).to(DEV)
    r = (2 / nb) * rr
    edges = []
    for c in range(0, R, R // nb):
        xs = coords[c:c + R // nb]
        edges += [xs.amin() - r, xs.amax() + r]
    edges = [e for e in edges if -0.7 < float(e) < 0.7]          # inside the extent: the normalisation stays put
    targets = [t for e in edges for t in (e, torch.nextafter(e, e + 1), torch.nextafter(e, e - 1))]
    inner = torch.nonzero(n["mask"] & (((g["_xyz"] - center) * scale).abs() < 0.6).all(1)).squeeze(1)
    xyz = g["_xyz"].clone()
    placed = []
    for k, target in enumerate(targets):
        row, axis = int(inner[k]), k % 3
        x = target / scale + center[axis]                       # then walk to the float32 that normalises to target
        for _ in range(64):
            y = (x - center[axis]) * scale
            if y == target:
                xyz[row, axis] = x
                placed.append(k)
                break
            x = torch.nextafter(x, x + (1 if y < target else -1))
    assert len(placed) > len(targets) // 2
    g = dict(g, _xyz=xyz)
    n = fields_ref.normalise(g)
    assert torch.equal(n["center"], center) and n["scale"] == scale
    on = torch.stack(targets).view(1, 1, -1)
    assert int((n["xyz"].unsqueeze(-1) == on).any(-1).any(-1).sum()) >= len(placed)
    occ, c_native, s_native = Fd.extract_fields(g, R, nb, rr)
    assert torch.equal(c_native, n["center"]) and s_native == n["scale"]
    assert torch.equal(_native_counts(g, R, nb, rr), fields_ref.member_counts(g, R, nb, rr))


def test_member_counts_on_the_default_grid():
    g = _group(30_000, seed=11)
    assert torch.equal(_native_counts(g, 128, 16, 1.5), fields_ref.member_counts(g, 128, 16, 1.5))


def test_object_layout_against_float64_on_a_subset_of_blocks():
    """1.2 M rows (the object layout of benchmarks/), R = 128: every block of a line through the centre of the grid
    and a few off it, against the float64 restatement."""
    g = _group(1_200_000, seed=0, std=0.004)
    occ, center, scale = Fd.extract_fields(g, 128, 16)
    blocks = [(i, 7, 8) for i in range(16)] + [(8, 8, 8), (3, 12, 5), (0, 0, 0)]
    ref64, c32, s32 = fields_ref.extract_fields(g, 128, 16, dtype=torch.float64, blocks=blocks)
    assert torch.equal(center, c32) and scale == s32
    for (i, j, k) in blocks:
        sl = (slice(8 * i, 8 * i + 8), slice(8 * j, 8 * j + 8), slice(8 * k, 8 * k + 8))
        ok, worst = _within(occ[sl], ref64[sl])
        assert ok, ((i, j, k), worst)
    assert float(ref64.max()) > 1.0


def test_degenerate_covariances_weigh_zero():
    """Flat Gaussians (one scale e^-40): their float32 determinant is rounding noise, negative for some of them, and
    there the reference's power is > 0 and its weight 0; where it is positive the inverse is ~1e8 along the flat
    direction and the weight is 0 too, except within ~1e-4 of the Gaussian's plane.  Grid points that close to a plane
    depend on the sign of that noise in either evaluation and are left out of the comparison."""
    g = _group(2000, seed=5)
    flat = _group(64, seed=6, std=0.3)
    flat["_scaling"][:, 2] = -40.0
    flat["_opacity"][:] = 3.0
    both = {k: torch.cat([g[k], flat[k]]) for k in g}
    n = fields_ref.normalise(both)
    mu = (flat["_xyz"] - n["center"]) * n["scale"]
    covs = fields_ref.covariance(torch.exp(flat["_scaling"]) * n["scale"], flat["_rotation"])
    R = 64
    X = torch.linspace(-1, 1, R).to(DEV)
    pts = torch.stack(torch.meshgrid(X, X, X, indexing="ij"), -1).reshape(-1, 3)
    d = (pts[::97].unsqueeze(1) - mu.unsqueeze(0)).reshape(-1, 3)
    _, power = fields_ref.gaussian_3d_coeff(d, covs.repeat(len(pts[::97]), 1), return_power=True)
    assert int((power > 0).sum()) > 100
    normal = fields_ref.build_rotation(flat["_rotation"])[:, :, 2]
    near = torch.zeros(len(pts), dtype=torch.bool, device=DEV)
    for k in range(len(mu)):
        near |= ((pts - mu[k]) @ normal[k]).abs() < 1e-3
    far = ~near.view(R, R, R)
    occ, _, _ = Fd.extract_fields(both, R, 8)
    ref32, _, _ = fields_ref.extract_fields(both, R, 8)
    assert torch.isfinite(occ).all() and float(far.float().mean()) > 0.5
    ok, worst = _within(occ[far], ref32[far].double(), 2 * RTOL, 2 * ATOL)
    assert ok, worst


def test_rows_below_the_opacity_cut_are_left_out():
    g = _group(5000, seed=9)
    low = _group(300, seed=10, std=0.2)
    low["_xyz"] = low["_xyz"] * 4.0                          # far outside: they would move the normalisation
    low["_opacity"][:] = -6.0                                # sigmoid 0.00247 < 0.005
    both = {k: torch.cat([g[k][:2500], low[k], g[k][2500:]]) for k in g}
    a = Fd.extract_fields(g, 64, 8)
    b = Fd.extract_fields(both, 64, 8)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and a[2] == b[2]


def test_reserved_rows_give_the_plain_group_result():
    g = _group(6000, seed=12)
    rg = ReservedGroup.from_tensors(g["_xyz"], torch.zeros(6000, 1, 3, device=DEV), torch.zeros(6000, 15, 3, device=DEV),
                                    g["_opacity"], g["_scaling"], g["_rotation"], capacity=8000)
    with pytest.raises(TypeError, match="ReservedGroup"):
        Fd.extract_fields(rg, 64, 8)
    a = Fd.extract_fields(g, 64, 8)
    b = Fd.extract_fields(rg.rows(), 64, 8)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and a[2] == b[2]


def test_two_calls_are_bitwise_equal():
    g = _group(50_000, seed=13)
    a = Fd.extract_fields(g, 128, 16)
    b = Fd.extract_fields(g, 128, 16)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and a[2] == b[2]


def test_refused_inputs():
    g = _group(100, seed=14)
    with pytest.raises(ValueError, match="opacity above 0.005"):
        Fd.extract_fields(dict(g, _opacity=torch.full_like(g["_opacity"], -10.0)), 32, 4)
    with pytest.raises(ValueError, match="same centre"):
        Fd.extract_fields(dict(g, _xyz=torch.full_like(g["_xyz"], 0.25)), 32, 4)
    with pytest.raises(ValueError, match="CUDA tensors"):
        Fd.extract_fields({k: v.cpu() for k, v in g.items()}, 32, 4)
    with pytest.raises(ValueError, match="multiple of the block size"):
        Fd.extract_fields(g, 4, 3)
    # a group that keeps one row passes: a single centre has no extent either
    one = {k: v[:1] for k, v in g.items()}
    with pytest.raises(ValueError, match="same centre"):
        Fd.extract_fields(dict(one, _opacity=torch.full_like(one["_opacity"], 2.0)), 32, 4)
