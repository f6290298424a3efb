"""dreamscene_b200.mesh on the GPU against the numpy restatement of include/b200gsr_mesh.h (harness/mesh_ref.py).

The faces must be identical and the vertices the same bits: every vertex is three float32 operations the header
defines, with nothing reordered.  A NaN vertex coordinate (an edge from a NaN point) is compared as NaN, whatever its
payload.  The geometry is then checked on its own: a single Gaussian's surface is a sphere (V - E + F = 2) turned
outwards, enclosing the analytic ellipsoid's volume, with every vertex on the iso-surface.
"""
import math

import numpy as np
import pytest
import torch

from dreamscene_b200 import mesh as Mh
from dreamscene_b200.fields import extract_fields
from dreamscene_b200.reserve import ReservedGroup
from harness import mesh_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _same(volume, iso):
    """March `volume` natively and in the restatement; assert the same faces and the same vertex bits."""
    v, f = Mh.marching_cubes(volume.to(DEV), iso)
    rv, rf = mesh_ref.marching_cubes(volume.cpu().numpy(), np.float32(iso))
    assert v.dtype == torch.float32 and f.dtype == torch.int32 and v.is_cuda and f.is_cuda
    assert v.shape == (len(rv), 3) and f.shape == (len(rf), 3)
    assert np.array_equal(f.cpu().numpy(), rf)
    a, b = v.cpu().numpy(), rv
    nan = np.isnan(a)
    assert np.array_equal(nan, np.isnan(b))
    assert np.array_equal(a[~nan].view(np.uint32), b[~nan].view(np.uint32))
    return v, f


def _topology(v, f):
    f = f.cpu().long()
    e = torch.cat([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    key = e[:, 0] * len(v) + e[:, 1]
    rev = e[:, 1] * len(v) + e[:, 0]
    once = len(torch.unique(key)) == len(key)
    paired = bool(torch.isin(rev, key).all())
    faces_unique = len(torch.unique(torch.sort(f, 1).values, dim=0)) == len(f)
    return once and paired and faces_unique, len(v) - len(key) // 2 + len(f)


def test_every_single_cell_case():
    g = torch.Generator().manual_seed(0)
    for case in range(256):
        inside = torch.tensor([(case >> c) & 1 for c in range(8)], dtype=torch.bool)
        vals = torch.where(inside, 0.5 + torch.rand(8, generator=g), 0.5 - torch.rand(8, generator=g))
        vol = torch.empty(2, 2, 2)
        for c in range(8):
            vol[c & 1, (c >> 1) & 1, (c >> 2) & 1] = vals[c]
        v, f = _same(vol, 0.5)
        assert len(f) == int(mesh_ref.COUNTS[case]), case


@pytest.mark.parametrize("shape", [(7, 9, 11), (2, 2, 2), (1, 5, 5), (5, 1, 7), (3, 17, 2), (33, 40, 29)])
def test_random_volumes(shape):
    g = torch.Generator().manual_seed(sum(shape))
    vol = torch.randn(shape, generator=g)
    v, f = _same(vol, 0.1)
    if min(shape) < 2:
        assert len(v) == 0 and len(f) == 0


def test_values_equal_to_iso_and_a_nan_voxel():
    g = torch.Generator().manual_seed(1)
    vol = torch.randint(-2, 3, (12, 10, 14), generator=g).float()
    _same(vol, 0.0)                              # a point equal to iso is outside: vertices at t = 0 and t = 1
    _same(vol, 1.0)
    vol = torch.randn(9, 8, 7, generator=g)
    vol[4, 3, 2] = math.nan
    v, f = _same(vol, 0.0)
    assert bool(torch.isnan(v).any())            # the edges from the NaN point into inside points


def test_iso_that_nothing_crosses():
    vol = torch.rand(20, 21, 22)
    for iso in (1.0, 5.0, -1e30):
        v, f = Mh.marching_cubes(vol.to(DEV), iso)
        assert v.shape == (0, 3) and f.shape == (0, 3)


def _object_group(P=1_200_000, seed=0, std=0.004):
    """The 1.2 M-row object layout of tests/test_gpu_fields.py: a ball of small Gaussians."""
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(P, 3, generator=g)
    d /= d.norm(dim=1, keepdim=True)
    xyz = 0.5 * torch.rand(P, 1, generator=g) ** (1 / 3) * d
    leaves = dict(_xyz=xyz, _opacity=1.5 * torch.randn(P, 1, generator=g),
                  _scaling=math.log(std) + 0.3 * torch.randn(P, 3, generator=g), _rotation=torch.randn(P, 4, generator=g))
    return {k: v.to(DEV) for k, v in leaves.items()}


def test_object_field_at_128_and_two_calls_agree():
    occ, _, _ = extract_fields(_object_group(), 128, 16)
    top = float(occ.max())
    for iso in (0.5 * top, 0.1 * top):
        v, f = _same(occ, iso)
        assert len(f) > 10_000
        v2, f2 = Mh.marching_cubes(occ, iso)
        assert torch.equal(v, v2) and torch.equal(f, f2)


def _gaussian(R, centre, sigma, rot):
    """opacity 0.9 * exp(-1/2 d^T Sigma^-1 d) on an R^3 index grid, Sigma = rot diag(sigma^2) rot^T, in float64."""
    ax = torch.arange(R, dtype=torch.float64, device=DEV)
    p = torch.stack(torch.meshgrid(ax, ax, ax, indexing="ij"), -1) - torch.tensor(centre, dtype=torch.float64,
                                                                                  device=DEV)
    local = p @ rot
    q = ((local / torch.tensor(sigma, dtype=torch.float64, device=DEV)) ** 2).sum(-1)
    return 0.9 * torch.exp(-0.5 * q)


def test_single_gaussian_is_a_closed_sphere_around_the_ellipsoid():
    R, centre, sigma, iso = 64, (31.3, 30.6, 32.2), (9.0, 6.0, 7.5), 0.3
    rot = torch.linalg.qr(torch.randn(3, 3, generator=torch.Generator().manual_seed(2), dtype=torch.float64))[0].to(DEV)
    field = _gaussian(R, centre, sigma, rot)
    v, f = _same(field.float(), iso)
    ok, chi = _topology(v, f)
    assert ok and chi == 2
    a, b, c = (v[f[:, k].long()].double() for k in range(3))
    signed = float((a * torch.cross(b, c, dim=1)).sum()) / 6
    r = math.sqrt(2 * math.log(0.9 / iso))
    exact = 4 / 3 * math.pi * sigma[0] * sigma[1] * sigma[2] * r ** 3
    assert 0.98 * exact < signed < 1.01 * exact, (signed, exact)
    # every vertex on the surface: the analytic field there is iso to within the linear interpolation's error
    local = (v.double() - torch.tensor(centre, dtype=torch.float64, device=DEV)) @ rot
    at = 0.9 * torch.exp(-0.5 * ((local / torch.tensor(sigma, dtype=torch.float64, device=DEV)) ** 2).sum(-1))
    assert float((at - iso).abs().max()) < 0.01


def _world(v, center, scale, R):
    return (v.double() / (R - 1) * 2 - 1) / scale + center.double()


def test_extract_mesh_maps_the_index_space_vertices():
    g = _object_group(200_000, seed=3, std=0.01)
    R = 96
    occ, center, scale = extract_fields(g, R, 16)
    iso = 0.5 * float(occ.max())
    vi, fi = Mh.marching_cubes(occ, iso)
    vw, fw = Mh.extract_mesh(g, R, iso, 16)
    assert len(fw) > 1000 and torch.equal(fw, fi) and vw.dtype == torch.float32 and vw.is_cuda
    expect = _world(vi, center, scale, R)
    # a few float32 roundings of coordinates below ~1 in magnitude
    assert float((vw.double() - expect).abs().max()) <= 1e-6 * (1 + float(expect.abs().max()))
    # reserved rows: the live rows' mesh, the same bits as the plain group's
    rg = ReservedGroup.from_tensors(g["_xyz"], torch.zeros(200_000, 1, 3, device=DEV),
                                    torch.zeros(200_000, 15, 3, device=DEV), g["_opacity"], g["_scaling"],
                                    g["_rotation"], capacity=260_000)
    vr, fr = Mh.extract_mesh(rg.rows(), R, iso, 16)
    assert torch.equal(vr, vw) and torch.equal(fr, fw)
    with pytest.raises(TypeError, match="ReservedGroup"):
        Mh.extract_mesh(rg, R, iso, 16)


def test_refusals_on_the_device():
    with pytest.raises(ValueError, match="finite"):
        Mh.marching_cubes(torch.rand(4, 4, 4, device=DEV), math.inf)
    with pytest.raises(ValueError, match="dimension"):
        Mh.marching_cubes(torch.rand(1025, 2, 2, device=DEV), 0.5)
    vol = torch.rand(8, 8, 8, device=DEV)
    Mh.marching_cubes(vol, 0.5)                  # warm: nothing left to initialise during the capture
    torch.cuda.synchronize()
    graph, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    with torch.cuda.stream(s):
        graph.capture_begin()
        try:
            with pytest.raises(RuntimeError, match="CUDA graph"):
                Mh.marching_cubes(vol, 0.5)
        finally:
            graph.capture_end()
    torch.cuda.synchronize()
