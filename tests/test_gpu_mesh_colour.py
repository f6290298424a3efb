"""The mesh colour on the GPU (include/b200gsr_mesh_colour.h): dreamscene_b200.fields.extract_fields_rgb,
marching_cubes(..., attributes=) and extract_coloured_mesh, against the existing opacity field and mesh, the
restatements (harness/fields_ref.py, harness/mesh_ref.py), and the colour's own meaning.

Exact: extract_fields_rgb's occ is extract_fields' occ bit for bit, extract_coloured_mesh's vertices and faces are
extract_mesh's, and the vertex attributes are the numpy restatement's bits (each is three float32 operations with the
vertex's own t; NaN compared as NaN).

The colour field is a ratio of two float32 sums in row order, against the float64 restatement (the same members and
float32 colours, every weight, product and sum in float64):

    |rgb - rgb64| <= RTOL * |rgb64| + ATOL,   RTOL = ATOL = 1e-4,   where occ64 >= OCC_MIN = 1e-3.

Both sums have all terms >= 0 (colours are clamped at 0), so each is within test_gpu_fields.py's 1e-4 relative bound
of its float64 value, and the ratio, a weighted mean of colours of size ~1, moves by about that much.  Below OCC_MIN
the field is made of far tails whose float32 weights carry large relative errors (occ itself is only held to an
absolute 1e-5 there); those points are held to the weighted-mean property instead: within the members' colour range.
That property needs occ in float32's normal range: below it the two sums keep few bits, each rounded in its own
places, so their ratio is only held to be finite and >= 0 where occ < NORMAL = 2^-100.
"""
import math

import numpy as np
import pytest
import torch

from dreamscene_b200 import fields as Fd
from dreamscene_b200 import mesh as Mh
from dreamscene_b200.reserve import ReservedGroup
from harness import fields_ref, mesh_ref

pytestmark = pytest.mark.gpu
RTOL, ATOL, OCC_MIN = 1e-4, 1e-4, 1e-3
NORMAL = 2.0 ** -100
DEV = "cuda"


def _group(P, seed=0, std=0.02, device=DEV):
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(P, 3, generator=g)
    d /= d.norm(dim=1, keepdim=True)
    xyz = 0.5 * torch.rand(P, 1, generator=g) ** (1 / 3) * d
    leaves = dict(_xyz=xyz, _opacity=1.5 * torch.randn(P, 1, generator=g),
                  _scaling=math.log(std) + 0.3 * torch.randn(P, 3, generator=g), _rotation=torch.randn(P, 4, generator=g),
                  _features_dc=1.2 * torch.randn(P, 1, 3, generator=g))
    return {k: v.to(device) for k, v in leaves.items()}


def _check_colour(occ, rgb, group, occ64, rgb64, where=None):
    """The colour field against the float64 restatement where occ64 >= OCC_MIN; in the member colour range wherever
    occ >= NORMAL; finite and >= 0 below; 0 where occ == 0.  where: a boolean [R,R,R] mask of the points to compare
    (all when None)."""
    keep = torch.sigmoid(group["_opacity"][:, 0]) > 0.005
    cols = fields_ref.sh2rgb(group["_features_dc"])[keep]
    lo, hi = cols.amin(0).double(), cols.amax(0).double()
    mask = torch.ones_like(occ, dtype=torch.bool) if where is None else where
    near = mask & (occ64 >= OCC_MIN)
    err = (rgb.double() - rgb64)[near].abs()
    bound = RTOL * rgb64[near].abs() + ATOL
    assert int(near.sum()) > 50 and bool((err <= bound).all()), float((err / bound).max())
    r = rgb.double()[mask & (occ >= NORMAL)]
    slack = 1e-6 * (1 + hi.abs())
    assert bool(((r >= lo - slack) & (r <= hi + slack)).all())
    tiny = rgb[mask & (occ > 0) & (occ < NORMAL)]
    assert bool((torch.isfinite(tiny) & (tiny >= 0)).all())
    assert bool((rgb[mask & (occ == 0)] == 0).all())


@pytest.mark.parametrize("P,R,nb", [(1000, 64, 8), (20_000, 64, 8), (20_000, 128, 16), (3000, 50, 8), (500, 9, 2)])
def test_occ_is_extract_fields_bits_and_rgb_matches_float64(P, R, nb):
    g = _group(P, seed=P + R, std=0.05 if P < 5000 else 0.02)
    occ, rgb, center, scale = Fd.extract_fields_rgb(g, R, nb)
    occ0, center0, scale0 = Fd.extract_fields(g, R, nb)
    assert torch.equal(occ, occ0) and torch.equal(center, center0) and scale == scale0
    assert rgb.shape == (R, R, R, 3) and rgb.dtype == torch.float32 and rgb.is_cuda
    occ64, rgb64, _, _ = fields_ref.extract_fields_rgb(g, R, nb, dtype=torch.float64)
    _check_colour(occ, rgb, g, occ64, rgb64)
    # torch's float32 restatement is held to the same bound
    occ32, rgb32, _, _ = fields_ref.extract_fields_rgb(g, R, nb)
    near = occ64 >= OCC_MIN
    assert bool(((rgb32.double() - rgb64)[near].abs() <= RTOL * rgb64[near].abs() + ATOL).all())


def test_object_layout_occ_bits_and_colour_on_a_subset_of_blocks():
    """1.2 M rows (the object layout of benchmarks/), R = 128: occ bit for bit extract_fields', and the colour on a
    line of blocks through the centre and a few off it against float64."""
    g = _group(1_200_000, seed=0, std=0.004)
    occ, rgb, center, scale = Fd.extract_fields_rgb(g, 128, 16)
    occ0, center0, scale0 = Fd.extract_fields(g, 128, 16)
    assert torch.equal(occ, occ0) and torch.equal(center, center0) and scale == scale0
    del occ0
    blocks = [(i, 7, 8) for i in range(16)] + [(8, 8, 8), (3, 12, 5), (0, 0, 0)]
    occ64, rgb64, _, _ = fields_ref.extract_fields_rgb(g, 128, 16, dtype=torch.float64, blocks=blocks)
    where = torch.zeros_like(occ, dtype=torch.bool)
    for (i, j, k) in blocks:
        where[8 * i:8 * i + 8, 8 * j:8 * j + 8, 8 * k:8 * k + 8] = True
    _check_colour(occ, rgb, g, occ64, rgb64, where)
    assert bool(torch.isfinite(rgb).all())


def _same_attributes(volume, iso, attributes):
    """marching_cubes with attributes: the same vertices and faces as without, and the restatement's attribute bits."""
    vol, attr = volume.to(DEV), attributes.to(DEV)
    v0, f0 = Mh.marching_cubes(vol, iso)
    v, f, a = Mh.marching_cubes(vol, iso, attr)
    assert torch.equal(f, f0) and np.array_equal(v.cpu().numpy().view(np.uint32), v0.cpu().numpy().view(np.uint32))
    ra = mesh_ref.vertex_attributes(volume.cpu().numpy(), np.float32(iso), attributes.cpu().numpy())
    assert a.dtype == torch.float32 and a.is_cuda and a.shape == (len(v), 3) and ra.shape == (len(v), 3)
    x = a.cpu().numpy()
    nan = np.isnan(x)
    assert np.array_equal(nan, np.isnan(ra))
    assert np.array_equal(x[~nan].view(np.uint32), ra[~nan].view(np.uint32))
    return v, f, a


@pytest.mark.parametrize("shape", [(7, 9, 11), (2, 2, 2), (1, 5, 5), (5, 1, 7), (3, 17, 2), (33, 40, 29)])
def test_attributes_on_random_volumes(shape):
    g = torch.Generator().manual_seed(sum(shape))
    vol = torch.randn(shape, generator=g)
    v, f, a = _same_attributes(vol, 0.1, torch.rand(shape + (3,), generator=g) * 4 - 1)
    if min(shape) < 2:
        assert len(v) == 0 and len(a) == 0


def test_attributes_at_values_equal_to_iso_and_a_nan_voxel():
    g = torch.Generator().manual_seed(1)
    vol = torch.randint(-2, 3, (12, 10, 14), generator=g).float()
    attr = torch.randn(12, 10, 14, 3, generator=g)
    _same_attributes(vol, 0.0, attr)              # t = 0 and t = 1 at points equal to iso
    _same_attributes(vol, 1.0, attr)
    vol = torch.randn(9, 8, 7, generator=g)
    vol[4, 3, 2] = math.nan
    v, _, a = _same_attributes(vol, 0.0, torch.randn(9, 8, 7, 3, generator=g))
    assert bool(torch.isnan(a).any()) and torch.equal(torch.isnan(a).any(1), torch.isnan(v).any(1))


def _positive_ends(occ, iso, vertices):
    """Vertices whose two edge ends both have occ > 0, from the restatement: an indicator interpolates to exactly 1
    there (the colour field is 0 where occ is 0, so other vertices mix in black)."""
    pos = (occ > 0).float().unsqueeze(-1).expand(*occ.shape, 3).contiguous()
    ind = mesh_ref.vertex_attributes(occ.cpu().numpy(), np.float32(iso), pos.cpu().numpy())[:, 0]
    assert len(ind) == len(vertices)
    return torch.from_numpy(ind == 1).to(DEV)


def test_a_single_colour_group_colours_every_vertex_that_colour():
    g = _group(200_000, seed=3, std=0.01)
    R = 96
    for colour, exact in (((0.5, 0.5, 0.5), True), ((0.2, 0.7, 0.9), False)):
        c = torch.tensor(colour, device=DEV)
        g["_features_dc"] = ((c - 0.5) / fields_ref.SH_C0).view(1, 1, 3).expand(len(g["_xyz"]), 1, 3).contiguous()
        c32 = fields_ref.sh2rgb(g["_features_dc"][:1])[0]                   # the colour as float32 makes it
        occ, rgb, _, _ = Fd.extract_fields_rgb(g, R, 16)
        iso = 0.5 * float(occ.max())
        v, f, cols = Mh.extract_coloured_mesh(g, R, iso, 16)
        _, _, vi = Mh.marching_cubes(occ, iso, rgb)
        assert torch.equal(cols, vi) and len(f) > 1000
        both = _positive_ends(occ, iso, v)
        assert float(both.float().mean()) > 0.99
        if exact:
            # dc = 0 gives 0.5: op * 0.5 is exact and scales every rounding of the two sums alike
            # (above the subnormal range, where halving a partial sum can round)
            assert bool((cols[both] == 0.5).all()) and bool((rgb[occ >= 2.0 ** -100] == 0.5).all())
        else:
            assert float((cols[both] - c32).abs().max()) <= 2.0 ** -14 * float(c32.max())
        assert bool(((cols >= 0) & (cols <= c32 * (1 + 2.0 ** -14))).all())


def test_two_separate_gaussians_colour_their_own_spheres():
    red, blue = (0.9, 0.15, 0.1), (0.1, 0.2, 0.95)
    g = dict(_xyz=torch.tensor([[-0.5, 0.0, 0.0], [0.5, 0.0, 0.0]]), _opacity=torch.full((2, 1), 4.0),
             _scaling=torch.full((2, 3), math.log(0.03)), _rotation=torch.tensor([[1.0, 0, 0, 0], [1.0, 0, 0, 0]]),
             _features_dc=((torch.tensor([red, blue]) - 0.5) / fields_ref.SH_C0).view(2, 1, 3))
    g = {k: v.to(DEV) for k, v in g.items()}
    R = 128                                     # spheres of radius ~4 grid steps, inside the grid
    occ, _, _ = Fd.extract_fields(g, R, 16)
    iso = 0.5 * float(occ.max())
    v, f, cols = Mh.extract_coloured_mesh(g, R, iso, 16)
    vm, fm = Mh.extract_mesh(g, R, iso, 16)
    assert torch.equal(v, vm) and torch.equal(f, fm)
    c = fields_ref.sh2rgb(g["_features_dc"])
    left = v[:, 0] < 0
    assert 100 < int(left.sum()) < len(v) - 100
    for side, col in ((left, c[0]), (~left, c[1])):
        assert float((cols[side] - col).abs().max()) <= 1e-6, float((cols[side] - col).abs().max())


def test_extract_coloured_mesh_is_extract_mesh_with_colours():
    g = _group(200_000, seed=4, std=0.01)
    R = 96
    occ, rgb, _, _ = Fd.extract_fields_rgb(g, R, 16)
    iso = 0.5 * float(occ.max())
    v, f, cols = Mh.extract_coloured_mesh(g, R, iso, 16)
    vm, fm = Mh.extract_mesh(g, R, iso, 16)
    assert torch.equal(v, vm) and torch.equal(f, fm) and cols.dtype == torch.float32 and cols.shape == v.shape
    _, _, vi = _same_attributes(occ, iso, rgb)
    assert torch.equal(cols, vi)
    # reserved rows: the plain group's result, bit for bit
    P = len(g["_xyz"])
    rg = ReservedGroup.from_tensors(g["_xyz"], g["_features_dc"], torch.zeros(P, 15, 3, device=DEV), g["_opacity"],
                                    g["_scaling"], g["_rotation"], capacity=P + 50_000)
    a = Fd.extract_fields_rgb(g, 64, 8)
    b = Fd.extract_fields_rgb(rg.rows(), 64, 8)
    assert all(torch.equal(x, y) for x, y in zip(a[:3], b[:3])) and a[3] == b[3]
    vr, fr, cr = Mh.extract_coloured_mesh(rg.rows(), R, iso, 16)
    assert torch.equal(vr, v) and torch.equal(fr, f) and torch.equal(cr, cols)
    with pytest.raises(TypeError, match="ReservedGroup"):
        Mh.extract_coloured_mesh(rg, R, iso, 16)


def test_two_calls_are_bitwise_equal():
    g = _group(50_000, seed=13)
    a = Fd.extract_fields_rgb(g, 128, 16)
    b = Fd.extract_fields_rgb(g, 128, 16)
    assert all(torch.equal(x, y) for x, y in zip(a[:3], b[:3])) and a[3] == b[3]
    iso = 0.3 * float(a[0].max())
    m1 = Mh.marching_cubes(a[0], iso, a[1])
    m2 = Mh.marching_cubes(b[0], iso, b[1])
    assert all(torch.equal(x, y) for x, y in zip(m1, m2)) and len(m1[2]) > 1000


def test_refused_inputs():
    g = _group(100, seed=14)
    for bad, msg in ((dict(g, _features_dc=g["_features_dc"][:, :, :2]), "_features_dc has shape"),
                     (dict(g, _features_dc=g["_features_dc"].view(100, 3)), "_features_dc has shape"),
                     (dict(g, _features_dc=g["_features_dc"][:50]), "_features_dc has shape"),
                     ({k: v for k, v in g.items() if k != "_features_dc"}, "no _features_dc"),
                     (dict(g, _features_dc=g["_features_dc"].cpu()), "device"),
                     (dict(g, _opacity=torch.full_like(g["_opacity"], -10.0)), "opacity above 0.005"),
                     (dict(g, _xyz=torch.full_like(g["_xyz"], 0.25)), "same centre")):
        with pytest.raises(ValueError, match=msg):
            Fd.extract_fields_rgb(bad, 32, 4)
    with pytest.raises(ValueError, match="no _features_dc"):
        Mh.extract_coloured_mesh({k: v for k, v in g.items() if k != "_features_dc"}, 32, 0.5, 4)
    with pytest.raises(ValueError, match="3 R"):
        Fd.extract_fields_rgb(g, 895, 2)
    vol = torch.rand(8, 9, 10, device=DEV)
    for attr, msg in ((torch.rand(8, 9, 10, device=DEV), "shape"), (torch.rand(8, 9, 10, 4, device=DEV), "shape"),
                      (torch.rand(9, 8, 10, 3, device=DEV), "shape"),
                      (torch.rand(8, 9, 10, 3, device=DEV, dtype=torch.float64), "float32"),
                      (torch.rand(8, 9, 10, 3), "CUDA tensor"), (np.zeros((8, 9, 10, 3), np.float32), "torch tensor")):
        with pytest.raises(ValueError, match=msg):
            Mh.marching_cubes(vol, 0.5, attr)
    attr = torch.rand(8, 9, 10, 3, device=DEV)
    Mh.marching_cubes(vol, 0.5, attr)              # warm: nothing left to initialise during the capture
    torch.cuda.synchronize()
    graph, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    with torch.cuda.stream(s):
        graph.capture_begin()
        try:
            with pytest.raises(RuntimeError, match="CUDA graph"):
                Mh.marching_cubes(vol, 0.5, attr)
        finally:
            graph.capture_end()
    torch.cuda.synchronize()
