"""dreamscene_b200.mesh.mesh_components and clean_mesh on the GPU against the numpy / scipy restatement of
include/b200gsr_mesh_clean.h (harness/mesh_ref.py).

Labels must be identical, and the cleaned mesh the same bits: vertices are copies of the input's bits, faces and kept
indices integers, and the decision uses integer counts and one float64 expression the header fixes operation by
operation.  Then properties on their own: the defaults give a marching-cubes mesh back unchanged, an ellipsoid among
small blobs cleans to exactly the ellipsoid's own mesh, a closed sphere, and two calls agree.
"""
import math

import numpy as np
import pytest
import torch

from dreamscene_b200 import mesh as Mh
from dreamscene_b200.fields import extract_fields
from harness import mesh_ref
from tests.test_gpu_mesh import _object_group, _topology

pytestmark = pytest.mark.gpu
DEV = "cuda"
GRID = [dict(), dict(min_faces=0), dict(min_faces=8), dict(min_faces=64), dict(min_diameter=0.05),
        dict(min_diameter=0.1), dict(min_faces=64, min_diameter=0.1), dict(keep_largest=True),
        dict(keep_largest=True, min_diameter=0.1), dict(keep_largest=True, min_faces=10**9)]


def _same_labels(faces, V):
    lab = Mh.mesh_components(faces, V)
    assert lab.dtype == torch.int32 and lab.is_cuda and lab.shape == (V,)
    ref = mesh_ref.components(faces.cpu().numpy(), V)
    assert np.array_equal(lab.cpu().numpy(), ref)
    return lab


def _same_clean(v, f, **kw):
    ov, of, kept = Mh.clean_mesh(v, f, **kw)
    rv, rf, rk = mesh_ref.clean_mesh(v.cpu().numpy(), f.cpu().numpy(), **kw)
    assert ov.dtype == torch.float32 and of.dtype == torch.int32 and kept.dtype == torch.int32
    assert ov.is_cuda and of.is_cuda and kept.is_cuda
    assert ov.shape == rv.shape and of.shape == rf.shape and kept.shape == rk.shape, kw
    assert np.array_equal(ov.cpu().numpy().view(np.uint32), rv.view(np.uint32)), kw
    assert np.array_equal(of.cpu().numpy(), rf), kw
    assert np.array_equal(kept.cpu().numpy(), rk), kw
    return ov, of, kept


@pytest.mark.parametrize("F", [0, 1, 10, 300, 700, 1000, 3000])
def test_random_face_soups(F):
    V = 1000
    for seed in range(3):
        g = torch.Generator().manual_seed(100 * F + seed)
        faces = torch.randint(0, V, (F, 3), generator=g, dtype=torch.int32)
        if F >= 10:
            faces[: F // 10, 1] = faces[: F // 10, 0]             # some degenerate faces
        verts = torch.randn(V, 3, generator=g)
        verts[::97, seed] = math.nan
        f, v = faces.to(DEV), verts.to(DEV)
        _same_labels(f, V)
        for kw in GRID:
            _same_clean(v, f, **kw)


def _random_volume_mesh(shape, seed, iso):
    g = torch.Generator().manual_seed(seed)
    vol = torch.randn(shape, generator=g)
    vol = (vol + vol.roll(1, 0) + vol.roll(1, 1) + vol.roll(1, 2)) / 2     # some blobs grow large, most stay small
    return Mh.marching_cubes(vol.to(DEV), iso)


@pytest.mark.parametrize("shape,seed", [((20, 22, 24), 0), ((40, 33, 29), 1), ((64, 64, 64), 2)])
def test_marching_cubes_meshes_of_random_volumes(shape, seed):
    v, f = _random_volume_mesh(shape, seed, 1.2)
    lab = _same_labels(f, len(v))
    assert len(torch.unique(lab)) > 20                              # many components
    for kw in GRID:
        _same_clean(v, f, **kw)
    # the defaults are the identity on a marching-cubes mesh: every vertex is referenced
    ov, of, kept = Mh.clean_mesh(v, f)
    assert torch.equal(kept, torch.arange(len(v), dtype=torch.int32, device=DEV))
    assert torch.equal(of, f) and torch.equal(ov.view(torch.int32), v.view(torch.int32))


@pytest.fixture(scope="module")
def object_meshes():
    g = _object_group()
    occ128, _, _ = extract_fields(g, 128, 16)
    iso = 0.5 * float(occ128.max())
    out = {128: Mh.marching_cubes(occ128, iso)}
    del occ128
    occ256, _, _ = extract_fields(g, 256, 16)
    out[256] = Mh.marching_cubes(occ256, iso)
    return out


@pytest.mark.parametrize("R", [128, 256])
def test_object_meshes(object_meshes, R):
    v, f = object_meshes[R]
    assert len(f) > 100_000
    lab = _same_labels(f, len(v))
    for kw in (dict(), dict(min_faces=64, min_diameter=0.1), dict(keep_largest=True), dict(min_diameter=0.05)):
        _same_clean(v, f, **kw)
    ov, of, kept = Mh.clean_mesh(v, f)
    assert torch.equal(kept, torch.arange(len(v), dtype=torch.int32, device=DEV))
    assert torch.equal(of, f) and torch.equal(ov.view(torch.int32), v.view(torch.int32))
    # two calls give the same bits
    assert torch.equal(Mh.mesh_components(f, len(v)), lab)
    a = Mh.clean_mesh(v, f, min_faces=64, min_diameter=0.1)
    b = Mh.clean_mesh(v, f, min_faces=64, min_diameter=0.1)
    assert all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(a, b))


def test_a_long_permuted_strip_is_one_component():
    """One triangle strip over 1 M vertices, its indices randomly permuted, so the union-find's trees start as long
    chains in no index order.  A correctness case, run once."""
    V = 1_000_000
    g = torch.Generator().manual_seed(7)
    perm = torch.randperm(V, generator=g).to(torch.int32)
    i = torch.arange(V - 2, dtype=torch.int64)
    faces = perm[torch.stack([i, i + 1, i + 2], 1)].to(DEV)
    lab = Mh.mesh_components(faces, V)
    assert int(lab.max()) == 0 and int(lab.min()) == 0
    verts = torch.randn(V, 3, generator=g).to(DEV)
    ov, of, kept = Mh.clean_mesh(verts, faces, keep_largest=True)
    assert torch.equal(kept, torch.arange(V, dtype=torch.int32, device=DEV))
    assert torch.equal(of, faces) and torch.equal(ov, verts)


def _index_grid(R):
    ax = torch.arange(R, dtype=torch.float64, device=DEV)
    return torch.stack(torch.meshgrid(ax, ax, ax, indexing="ij"), -1)


def test_ellipsoid_among_blobs_cleans_to_the_ellipsoid_alone():
    """max(ellipsoid, blobs): the blobs are compact (exactly 0 beyond their radius) and sit in the grid's corners, far
    from the ellipsoid's crossing edges, so those edges see the ellipsoid's values only.  Cleaning away the blobs
    leaves marching_cubes(ellipsoid) exactly: clean_mesh keeps vertices and faces in input order."""
    R, iso = 64, 0.3
    p = _index_grid(R)
    centre = torch.tensor([31.3, 30.6, 32.2], dtype=torch.float64, device=DEV)
    sigma = torch.tensor([9.0, 6.0, 7.5], dtype=torch.float64, device=DEV)
    ell = (0.9 * torch.exp(-0.5 * (((p - centre) / sigma) ** 2).sum(-1))).float()
    blobs = torch.zeros_like(ell, dtype=torch.float64)
    for c, rho in (((5.2, 5.7, 6.1), 3.0), ((57.4, 6.3, 55.8), 2.2), ((6.6, 56.1, 57.3), 1.6), ((57.0, 57.0, 5.5), 2.8),
                   ((5.5, 30.0, 58.0), 1.3)):
        r2 = ((p - torch.tensor(c, dtype=torch.float64, device=DEV)) ** 2).sum(-1)
        blobs = torch.maximum(blobs, 0.9 * torch.clamp(1 - r2 / rho ** 2, min=0))
    vol = torch.maximum(ell, blobs.float())
    ve, fe = Mh.marching_cubes(ell, iso)
    va, fa = Mh.marching_cubes(vol, iso)
    assert len(torch.unique(Mh.mesh_components(fa, len(va)))) == 6
    ok, chi = _topology(ve, fe)
    assert ok and chi == 2
    counts = torch.bincount(Mh.mesh_components(fa, len(va))[fa[:, 0].long()]).sort().values
    for kw in (dict(keep_largest=True), dict(min_diameter=0.2), dict(min_faces=int(counts[-2]) + 1)):
        ov, of, kept = _same_clean(va, fa, **kw)
        assert torch.equal(of, fe) and torch.equal(ov.view(torch.int32), ve.view(torch.int32)), kw
        assert torch.equal(va[kept.long()], ov)
        ok, chi = _topology(ov, of)
        assert ok and chi == 2, kw


def test_refusals_on_the_device():
    v, f = _random_volume_mesh((16, 16, 16), 3, 1.0)
    V = len(v)
    for bad in (V, -1, 2**31 - 1):
        g = f.clone()
        g[len(g) // 2, 1] = bad
        with pytest.raises(ValueError, match="outside"):
            Mh.mesh_components(g, V)
        with pytest.raises(ValueError, match="outside"):
            Mh.clean_mesh(v, g)
        # the next valid call still succeeds
        _same_clean(v, f, min_faces=8)
    with pytest.raises(ValueError, match="outside"):
        Mh.clean_mesh(v[:0], f)
    e = Mh.clean_mesh(v[:0], f[:0])
    assert [tuple(x.shape) for x in e] == [(0, 3), (0, 3), (0,)]
    with pytest.raises(ValueError, match="device|CUDA"):
        Mh.clean_mesh(v.cpu(), f)
    torch.cuda.synchronize()
    graph, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    with torch.cuda.stream(s):
        graph.capture_begin()
        try:
            with pytest.raises(RuntimeError, match="CUDA graph"):
                Mh.clean_mesh(v, f)
            with pytest.raises(RuntimeError, match="CUDA graph"):
                Mh.mesh_components(f, V)
        finally:
            graph.capture_end()
    torch.cuda.synchronize()
