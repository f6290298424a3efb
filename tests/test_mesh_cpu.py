"""CPU-only checks of marching cubes (include/b200gsr_mesh.h, dreamscene_b200.mesh): the signature table agrees with the
header and binds; the library's cube table is the one the face rule generates (harness/mesh_ref.py), uses exactly each
case's crossing edges and is bounded by exactly the face rule's segments; the library refuses bad arguments before
touching a device (made-up device addresses, never dereferenced); and the restatement the GPU tests compare against
gives closed, consistently oriented 2-manifolds."""
import ctypes as C
import math
import os
import re
from collections import Counter

import numpy as np
import pytest
import torch

from dreamscene_b200 import _lib
from dreamscene_b200 import mesh as Mh
from harness import mesh_ref
from tests import test_abi_binding_cpu as abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "b200gsr_mesh.h")


def _prototypes():
    src = re.sub(r"/\*.*?\*/", " ", open(HEADER).read(), flags=re.S)
    return {name: (ret, [" ".join(a.split()) for a in args.split(",")])
            for ret, name, args in re.findall(r"(\bint)\s+(b200gsr_\w+)\s*\(([^)]*)\)\s*;", src)}


def _library_table():
    counts, edges = (C.c_uint8 * 256)(), (C.c_int8 * (256 * _lib.MESH_TABLE_WIDTH))()
    assert _lib.load().b200gsr_mesh_table(counts, edges) == 0
    return np.frombuffer(counts, np.uint8).copy(), np.frombuffer(edges, np.int8).reshape(256, -1).copy()


def test_mesh_signature_table_matches_the_header_and_binds(monkeypatch):
    monkeypatch.setitem(abi._STRUCTS, "b200gsr_mesh_layout", _lib.MeshLayout)
    protos = _prototypes()
    assert list(protos) == list(_lib.MESH_SIGNATURES) == ["b200gsr_mesh_table", "b200gsr_mesh_layout_query",
                                                          "b200gsr_mesh_count", "b200gsr_mesh_emit"]
    assert abi._mismatches(_lib.MESH_SIGNATURES, protos) == []
    assert _lib.MESH_SIGNATURES["b200gsr_mesh_table"][1] == [C.POINTER(C.c_uint8), C.POINTER(C.c_int8)]
    text = open(HEADER).read()
    for name, value in (("MAX_TRIANGLES", _lib.MESH_MAX_TRIANGLES), ("TABLE_WIDTH", _lib.MESH_TABLE_WIDTH)):
        assert re.search(rf"#define B200GSR_MESH_{name} (\d+)", text).group(1) == str(value)
    assert _lib.MESH_TABLE_WIDTH == 3 * _lib.MESH_MAX_TRIANGLES == mesh_ref.TABLE.shape[1]
    body = re.search(r"typedef struct \{([^}]*)\}\s*b200gsr_mesh_layout;", text).group(1)
    names = re.findall(r"\b(\w+);", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert names == [n for n, _ in _lib.MeshLayout._fields_] and C.sizeof(_lib.MeshLayout) == 24
    lib = _lib.load()
    for name, (restype, argtypes) in _lib.MESH_SIGNATURES.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and tuple(fn.argtypes) == tuple(argtypes), name
    others = (set(_lib.SIGNATURES) | set(_lib.SCENE_SIGNATURES) | set(_lib.STEP_SIGNATURES) |
              set(_lib.LOSS_SIGNATURES) | set(_lib.FROZEN_SIGNATURES) | set(_lib.STATS_SIGNATURES) |
              set(_lib.RESERVE_SIGNATURES) | set(_lib.FRAMES_SIGNATURES) | set(_lib.VIEWS_FROZEN_SIGNATURES) |
              set(_lib.VIEWS_STATS_SIGNATURES) | set(_lib.FIELDS_SIGNATURES))
    assert not set(_lib.MESH_SIGNATURES) & others


def test_library_table_is_the_generated_table():
    counts, edges = _library_table()
    assert np.array_equal(counts, mesh_ref.COUNTS)
    assert np.array_equal(edges, mesh_ref.TABLE)
    # triangles per case: 0..5 for 2 / 16 / 50 / 80 / 76 / 32 cases; unused slots are -1
    assert np.bincount(counts, minlength=6).tolist() == [2, 16, 50, 80, 76, 32]
    for case in range(256):
        assert (edges[case, 3 * counts[case]:] == -1).all() and (edges[case, :3 * counts[case]] >= 0).all()


def test_edge_numbering():
    # x 0..3 from corners 0, 2, 4, 6; y 4..7 from 0, 1, 4, 5; z 8..11 from 0, 1, 2, 3
    assert mesh_ref.EDGES == [(0, 0), (0, 2), (0, 4), (0, 6), (1, 0), (1, 1), (1, 4), (1, 5),
                              (2, 0), (2, 1), (2, 2), (2, 3)]


def test_each_case_uses_exactly_its_crossing_edges():
    _, edges = _library_table()
    for case in range(256):
        crossing = {e for e, (a, b) in enumerate(mesh_ref.EDGES) if (case >> b & 1) != (case >> (b | 1 << a) & 1)}
        used = set(edges[case][edges[case] >= 0].tolist())
        assert used == crossing, case


def _boundary(tris):
    """Directed edges of the triangles whose reverse is not among them, as a multiset."""
    d = Counter((t[i], t[(i + 1) % 3]) for t in tris for i in range(3))
    out = Counter()
    for (a, b), n in d.items():
        k = n - d.get((b, a), 0)
        if k > 0:
            out[(a, b)] = k
    return out


def test_each_case_is_bounded_by_the_face_rule_segments():
    counts, edges = _library_table()
    for case in range(256):
        tris = [tuple(edges[case, 3 * t:3 * t + 3].tolist()) for t in range(counts[case])]
        assert len(set(map(frozenset, tris))) == len(tris) and all(len(set(t)) == 3 for t in tris), case
        assert _boundary(tris) == Counter(mesh_ref.face_segments(case)), case
        # no triangle lies in a cube face: its three edges never all belong to one face
        assert not any(set(t) <= f for t in tris for f in mesh_ref.FACE_EDGES), case


def test_neighbouring_cells_make_opposite_segments_on_their_shared_face():
    """Cell A's face (axis n, side 1) is cell B's face (axis n, side 0): whatever the other corners, the two segment
    sets there are each other's reverses, edge for edge (an edge of A's face is the same grid edge as the edge of B's
    face with bit n of its corner cleared)."""
    for n in range(3):
        top = mesh_ref.FACE_EDGES[2 * n + 1]
        bottom = mesh_ref.FACE_EDGES[2 * n]
        to_b = {e: mesh_ref.EDGE_OF[(b & ~(1 << n), (b | 1 << a) & ~(1 << n))]
                for e, (a, b) in enumerate(mesh_ref.EDGES) if e in top}
        rng = np.random.default_rng(n)
        for face_bits in range(16):
            corners = [c for c in range(8) if c >> n & 1]
            for _ in range(8):
                ca = int(rng.integers(256)) & ~sum(1 << c for c in corners)
                cb = int(rng.integers(256)) & ~sum(1 << (c & ~(1 << n)) for c in corners)
                for k, c in enumerate(corners):
                    if face_bits >> k & 1:
                        ca |= 1 << c
                        cb |= 1 << (c & ~(1 << n))
                sa = {(to_b[x], to_b[y]) for x, y in mesh_ref.face_segments(ca) if x in top and y in top}
                sb = {(y, x) for x, y in mesh_ref.face_segments(cb) if x in bottom and y in bottom}
                assert sa == sb, (n, ca, cb)


def _topology(v, f):
    """(directed edges that do not appear exactly once with their reverse exactly once, repeated faces, V - E + F)."""
    d = Counter((a, b) for t in f.tolist() for a, b in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0])))
    bad = sum(1 for (a, b), n in d.items() if n != 1 or d.get((b, a), 0) != 1)
    repeated = len(f) - len({frozenset(t) for t in f.tolist()})
    return bad, repeated, len(v) - len(d) // 2 + len(f)


def _walled(vol, low=-5.0):
    vol = vol.copy()
    vol[[0, -1]] = low
    vol[:, [0, -1]] = low
    vol[:, :, [0, -1]] = low
    return vol


@pytest.mark.parametrize("shape", [(7, 9, 11), (12, 12, 12), (20, 15, 9), (5, 6, 5)])
def test_restatement_is_a_closed_oriented_manifold_on_random_volumes(shape):
    rng = np.random.default_rng(sum(shape))
    for trial in range(12):
        vol = rng.standard_normal(shape).astype(np.float32)
        if trial % 3 == 1:
            vol = np.round(vol * 2) / 2                         # many values exactly at iso 0
        if trial % 3 == 2:
            vol = (vol > 0.3).astype(np.float32)               # binary: every crossing at t = 0 or 1
        v, f = mesh_ref.marching_cubes(_walled(vol), 0.0)
        assert len(f) > 0
        bad, repeated, _ = _topology(v, f)
        assert bad == 0 and repeated == 0, (trial, bad, repeated)
        assert len(np.unique(f)) == len(v)                    # every vertex is used


def _ellipsoid(shape, centre, sigma):
    g = [np.arange(n, dtype=np.float64) for n in shape]
    X, Y, Z = np.meshgrid(*g, indexing="ij")
    q = sum(((c - m) / s) ** 2 for c, m, s in zip((X, Y, Z), centre, sigma))
    return np.exp(-0.5 * q).astype(np.float32)


def test_restatement_of_a_convex_blob_is_a_sphere_turned_outwards():
    vol = _ellipsoid((24, 20, 22), (11.3, 9.6, 10.2), (3.9, 3.2, 3.5))
    iso = 0.3
    v, f = mesh_ref.marching_cubes(vol, iso)
    bad, repeated, chi = _topology(v, f)
    assert bad == 0 and repeated == 0 and chi == 2
    a, b, c = (v[f[:, k]].astype(np.float64) for k in range(3))
    signed = np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6
    r = math.sqrt(2 * math.log(1 / iso))
    exact = 4 / 3 * math.pi * 3.9 * 3.2 * 3.5 * r ** 3
    assert 0.97 * exact < signed < 1.01 * exact                # positive: the normals point outwards


def test_restatement_vertices_and_order_on_a_small_grid():
    vol = np.zeros((2, 3, 2), np.float32)
    vol[0, 1, 0] = 4.0                                         # one inside point: three crossing edges
    v, f = mesh_ref.marching_cubes(vol, np.float32(1.0))
    # point (0,0,0)'s +y edge (t = 1/4), then point (0,1,0)'s +x, +y and +z edges (t = -3 / -4)
    assert v.tolist() == [[0, 0.25, 0], [0.75, 1, 0], [0, 1.75, 0], [0, 1, 0.75]]
    # cell (0,0,0) cuts off its corner 2, cell (0,1,0) its corner 0
    assert sorted(map(sorted, f.tolist())) == [[0, 1, 3], [1, 2, 3]]
    for va, vb, vc in v[f]:
        n = np.cross(vb - va, vc - va)
        assert np.dot(n, (va + vb + vc) / 3 - np.array([0, 1, 0])) > 0     # away from the inside point
    assert [len(x) for x in mesh_ref.marching_cubes(np.ones((1, 5, 5), np.float32), 0.5)] == [0, 0]
    assert [len(x) for x in mesh_ref.marching_cubes(vol, np.float32(4.0))] == [0, 0]   # nothing is > 4


def test_library_refuses_bad_mesh_arguments():
    lib = _lib.load()
    out = _lib.MeshLayout()
    assert lib.b200gsr_mesh_layout_query(7, 9, 11, C.byref(out)) == 0
    assert out.points == 693 and out.cells == 6 * 8 * 10 and out.total >= 693 * 10
    assert lib.b200gsr_mesh_layout_query(1, 5, 5, C.byref(out)) == 0 and out.cells == 0
    assert lib.b200gsr_mesh_layout_query(512, 512, 512, C.byref(out)) == 0
    for dims, msg in (((0, 4, 4), "dimension"), ((4, 1025, 4), "dimension"), ((4, 4, -1), "dimension"),
                      ((1024, 1024, 1024), "too large"), ((1024, 1024, 683), "too large")):
        assert lib.b200gsr_mesh_layout_query(*dims, C.byref(out)) == _lib.ERR_BAD_ARG, dims
        assert msg in _lib.last_error(), dims
    # with every dimension at most 1024 the triangle bound is the tighter one: 5 * 1023^2 * 410 < 2^31 <= 5 * 1023^2 * 411
    assert lib.b200gsr_mesh_layout_query(1024, 1024, 411, C.byref(out)) == 0
    assert lib.b200gsr_mesh_layout_query(1024, 1024, 412, C.byref(out)) == _lib.ERR_BAD_ARG
    assert "cells is too large" in _lib.last_error()
    assert lib.b200gsr_mesh_layout_query(4, 4, 4, None) == _lib.ERR_BAD_ARG
    assert lib.b200gsr_mesh_table(None, (C.c_int8 * 3840)()) == _lib.ERR_BAD_ARG
    assert lib.b200gsr_mesh_table((C.c_uint8 * 256)(), None) == _lib.ERR_BAD_ARG

    assert lib.b200gsr_mesh_layout_query(7, 9, 11, C.byref(out)) == 0
    vol, totals, scr, verts, faces = (C.c_void_p(0x100000 * (k + 1)) for k in range(5))

    def count(X=7, Y=9, Z=11, v=vol, iso=0.5, t=totals, s=scr, n=out.total):
        return lib.b200gsr_mesh_count(X, Y, Z, v, iso, t, s, n, None)

    def emit(X=7, Y=9, Z=11, v=vol, iso=0.5, s=scr, n=out.total, vp=verts, V=10, fp=faces, F=10):
        return lib.b200gsr_mesh_emit(X, Y, Z, v, iso, s, n, vp, V, fp, F, None)

    for call in (count, emit):
        for kw, msg in ((dict(X=0), "dimension"), (dict(Z=2000), "dimension"), (dict(iso=math.inf), "finite"),
                        (dict(iso=-math.inf), "finite"), (dict(iso=math.nan), "finite"), (dict(v=None), "null"),
                        (dict(s=None), "null"), (dict(n=out.total - 1), "scratch holds"),
                        (dict(s=C.c_void_p(0x100080)), "256-byte"), (dict(v=C.c_void_p(0x100002)), "4-byte"),
                        (dict(X=1024, Y=1024, Z=1024), "too large")):
            assert call(**kw) == _lib.ERR_BAD_ARG and msg in _lib.last_error(), (call.__name__, kw)
    assert count(t=None) == _lib.ERR_BAD_ARG and "null" in _lib.last_error()
    assert count(t=C.c_void_p(0x100002)) == _lib.ERR_BAD_ARG and "4-byte" in _lib.last_error()
    for kw, msg in ((dict(vp=None), "null"), (dict(fp=None), "null"), (dict(V=-1), "V = -1"), (dict(F=-1), "F = -1"),
                    (dict(fp=C.c_void_p(0x100001)), "4-byte")):
        assert emit(**kw) == _lib.ERR_BAD_ARG and msg in _lib.last_error(), kw
    # an iso that is finite as a double but not as a float32
    assert count(iso=1e39) == _lib.ERR_BAD_ARG and "finite" in _lib.last_error()


def test_marching_cubes_refusals():
    with pytest.raises(ValueError, match="CUDA tensor"):
        Mh.marching_cubes(torch.zeros(4, 4, 4), 0.5)
    with pytest.raises(ValueError, match="torch tensor"):
        Mh.marching_cubes(np.zeros((4, 4, 4), np.float32), 0.5)
    for bad in (torch.zeros(4, 4), torch.zeros(2, 4, 4, 4)):
        with pytest.raises(ValueError, match="3-D"):
            Mh.marching_cubes(bad, 0.5)
    with pytest.raises(ValueError, match="float32"):
        Mh.marching_cubes(torch.zeros(4, 4, 4, dtype=torch.float64), 0.5)
    with pytest.raises(ValueError, match="CUDA tensor"):
        Mh.extract_mesh({k: torch.zeros(4, n) for k, n in (("_xyz", 3), ("_opacity", 1), ("_scaling", 3),
                                                            ("_rotation", 4))}, 16, 1.0, 4)
