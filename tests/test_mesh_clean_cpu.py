"""CPU-only checks of the mesh components and cleaning (include/b200gsr_mesh_clean.h, dreamscene_b200.mesh.mesh_components
and clean_mesh): the signature table agrees with the header and binds; the library refuses bad arguments before
touching a device (made-up device addresses, never dereferenced); the Python entry points refuse what they cannot take;
and the restatement the GPU tests compare against (harness/mesh_ref.py) gives what the definition gives on hand-made
meshes."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import torch

from dreamscene_b200 import _lib
from dreamscene_b200 import mesh as Mh
from harness import mesh_ref
from tests import test_abi_binding_cpu as abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "b200gsr_mesh_clean.h")
F_MAX = (2**31 - 1) // 3                 # the largest F with 3 F < 2^31


def _prototypes():
    src = re.sub(r"/\*.*?\*/", " ", open(HEADER).read(), flags=re.S)
    return {name: (ret, [" ".join(a.split()) for a in args.split(",")])
            for ret, name, args in re.findall(r"(\bint)\s+(b200gsr_\w+)\s*\(([^)]*)\)\s*;", src)}


def test_mesh_clean_signature_table_matches_the_header_and_binds(monkeypatch):
    monkeypatch.setitem(abi._SCALARS, "double", C.c_double)
    protos = _prototypes()
    assert list(protos) == list(_lib.MESH_CLEAN_SIGNATURES) == ["b200gsr_mesh_clean_layout_query",
                                                                "b200gsr_mesh_components", "b200gsr_mesh_clean_count",
                                                                "b200gsr_mesh_clean_emit"]
    assert abi._mismatches(_lib.MESH_CLEAN_SIGNATURES, protos) == []
    assert _lib.MESH_CLEAN_SIGNATURES["b200gsr_mesh_clean_layout_query"][1][2] == C.POINTER(C.c_size_t)
    # count and emit take the same leading arguments, the scratch's pointer then its size
    count, emit = (_lib.MESH_CLEAN_SIGNATURES[n][1] for n in ("b200gsr_mesh_clean_count", "b200gsr_mesh_clean_emit"))
    assert count[:7] == emit[:7] and count[8:10] == emit[7:9]
    lib = _lib.load()
    for name, (restype, argtypes) in _lib.MESH_CLEAN_SIGNATURES.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and tuple(fn.argtypes) == tuple(argtypes), name
    others = (set(_lib.SIGNATURES) | set(_lib.SCENE_SIGNATURES) | set(_lib.STEP_SIGNATURES) |
              set(_lib.LOSS_SIGNATURES) | set(_lib.FROZEN_SIGNATURES) | set(_lib.STATS_SIGNATURES) |
              set(_lib.RESERVE_SIGNATURES) | set(_lib.FRAMES_SIGNATURES) | set(_lib.VIEWS_FROZEN_SIGNATURES) |
              set(_lib.VIEWS_STATS_SIGNATURES) | set(_lib.FIELDS_SIGNATURES) | set(_lib.MESH_SIGNATURES) |
              set(_lib.MESH_COLOUR_SIGNATURES))
    assert not set(_lib.MESH_CLEAN_SIGNATURES) & others


def _query(V, F):
    n = C.c_size_t(0)
    return _lib.load().b200gsr_mesh_clean_layout_query(V, F, C.byref(n)), int(n.value)


def test_layout_query():
    rc, small = _query(1, 0)
    assert rc == 0 and small > 0
    rc, n = _query(950_830, 1_757_596)
    assert rc == 0 and n >= 950_830 * 38 + 1_757_596 * 4 and n % 256 == 0
    assert _query(2**31 - 1, F_MAX)[0] == 0                 # the limits themselves: sizes only, nothing allocated
    for V, F, msg in ((0, 0, "V = 0"), (-1, 5, "V = -1"), (10, -1, "F = -1"), (10, F_MAX + 1, "3 F")):
        assert _query(V, F)[0] == _lib.ERR_BAD_ARG and msg in _lib.last_error(), (V, F)
    assert _lib.load().b200gsr_mesh_clean_layout_query(10, 10, None) == _lib.ERR_BAD_ARG


def test_library_refuses_bad_arguments():
    lib = _lib.load()
    V, F = 100, 150
    _, nbytes = _query(V, F)
    verts, faces, labels, bad, totals, scr, ov, of, kept = (C.c_void_p(0x100000 * (k + 1)) for k in range(9))
    common = ((dict(V=0), "V = 0"), (dict(V=-3), "V = -3"), (dict(F=-1), "F = -1"), (dict(F=F_MAX + 1), "3 F"),
              (dict(f=None), "null"), (dict(s=None), "null"), (dict(f=C.c_void_p(0x200002)), "4-byte"),
              (dict(s=C.c_void_p(0x600080)), "256-byte"), (dict(n=nbytes - 1), "scratch holds"))

    def components(V=V, F=F, f=faces, lab=labels, b=bad, s=scr, n=nbytes):
        return lib.b200gsr_mesh_components(V, F, f, lab, b, s, n, None)

    def count(V=V, F=F, v=verts, f=faces, mf=1, md=0.0, kl=0, t=totals, s=scr, n=nbytes):
        return lib.b200gsr_mesh_clean_count(V, F, v, f, mf, md, kl, t, s, n, None)

    def emit(V=V, F=F, v=verts, f=faces, mf=1, md=0.0, kl=0, s=scr, n=nbytes, o=ov, g=of, k=kept, Vo=10, Fo=10):
        return lib.b200gsr_mesh_clean_emit(V, F, v, f, mf, md, kl, s, n, o, g, k, Vo, Fo, None)

    for call in (components, count, emit):
        for kw, msg in common:
            assert call(**kw) == _lib.ERR_BAD_ARG and msg in _lib.last_error(), (call.__name__, kw)
    assert components(F=0, f=None, s=None) == _lib.ERR_BAD_ARG and "null" in _lib.last_error()   # past faces
    for kw, msg in ((dict(lab=None), "null"), (dict(b=None), "null"), (dict(lab=C.c_void_p(0x300001)), "4-byte"),
                    (dict(b=C.c_void_p(0x400002)), "4-byte")):
        assert components(**kw) == _lib.ERR_BAD_ARG and msg in _lib.last_error(), kw
    thresholds = ((dict(v=None), "null"), (dict(v=C.c_void_p(0x100002)), "4-byte"), (dict(mf=-1), "min_faces = -1"),
                  (dict(md=-0.5), "min_diameter"), (dict(md=-1e-300), "min_diameter"), (dict(md=math.inf), "min_diameter"),
                  (dict(md=math.nan), "min_diameter"))
    for call in (count, emit):
        for kw, msg in thresholds:
            assert call(**kw) == _lib.ERR_BAD_ARG and msg in _lib.last_error(), (call.__name__, kw)
    for kw, msg in ((dict(t=None), "null"), (dict(t=C.c_void_p(0x500001)), "4-byte")):
        assert count(**kw) == _lib.ERR_BAD_ARG and msg in _lib.last_error(), kw
    for kw, msg in ((dict(o=None), "null"), (dict(g=None), "null"), (dict(k=None), "null"),
                    (dict(o=C.c_void_p(0x700002)), "4-byte"), (dict(g=C.c_void_p(0x800001)), "4-byte"),
                    (dict(k=C.c_void_p(0x900003)), "4-byte"), (dict(Vo=-1), "V_out = -1"), (dict(Fo=-1), "F_out = -1")):
        assert emit(**kw) == _lib.ERR_BAD_ARG and msg in _lib.last_error(), kw


def test_python_refusals_without_a_device():
    v, f = torch.zeros(4, 3), torch.tensor([[0, 1, 2]], dtype=torch.int32)
    with pytest.raises(ValueError, match="CUDA tensor"):
        Mh.clean_mesh(v, f)
    with pytest.raises(ValueError, match="CUDA tensor"):
        Mh.mesh_components(f, 4)
    with pytest.raises(ValueError, match="torch tensor"):
        Mh.clean_mesh(v.numpy(), f)
    with pytest.raises(ValueError, match="torch tensor"):
        Mh.mesh_components(f.numpy(), 4)
    with pytest.raises(ValueError, match=r"\[V,3\]"):
        Mh.clean_mesh(torch.zeros(4, 2), f)
    with pytest.raises(ValueError, match=r"\[F,3\]"):
        Mh.clean_mesh(v, f.view(-1))
    with pytest.raises(ValueError, match="float32"):
        Mh.clean_mesh(v.double(), f)
    with pytest.raises(ValueError, match="int32"):
        Mh.clean_mesh(v, f.long())
    with pytest.raises(ValueError, match="int32"):
        Mh.mesh_components(f.long(), 4)
    for bad in (-1, 2**31, 1.5, True, None):
        with pytest.raises(ValueError, match="min_faces"):
            Mh.clean_mesh(v, f, min_faces=bad)
    for bad in (-0.1, math.inf, math.nan, "0.1", True):
        with pytest.raises(ValueError, match="min_diameter"):
            Mh.clean_mesh(v, f, min_diameter=bad)
    with pytest.raises(ValueError, match="keep_largest"):
        Mh.clean_mesh(v, f, keep_largest=1)
    for bad in (-1, 2**31, 4.0, None):
        with pytest.raises(ValueError, match="num_vertices"):
            Mh.mesh_components(f, bad)


# ---- the restatement on hand-made meshes -------------------------------------------------------------------------

def _tetra(base):
    """A closed tetrahedron on vertices base .. base + 3, turned outwards."""
    return [[base, base + 2, base + 1], [base, base + 1, base + 3], [base, base + 3, base + 2],
            [base + 1, base + 2, base + 3]]


def _clean(v, f, **kw):
    return mesh_ref.clean_mesh(np.asarray(v, np.float32), np.asarray(f, np.int32).reshape(-1, 3), **kw)


TETRA = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)


def test_two_disjoint_tetrahedra():
    v = np.concatenate([TETRA, TETRA * 3 + 5])
    f = np.array(_tetra(0) + _tetra(4), np.int32)
    assert mesh_ref.components(f, 8).tolist() == [0] * 4 + [4] * 4
    ov, of, kept = _clean(v, f)
    assert kept.tolist() == list(range(8)) and np.array_equal(of, f) and np.array_equal(ov.view(np.uint32),
                                                                                        v.view(np.uint32))
    ov, of, kept = _clean(v, f, keep_largest=True)          # a tie at 4 faces: the smaller label
    assert kept.tolist() == [0, 1, 2, 3] and of.tolist() == _tetra(0)
    # diagonals sqrt 3 and 3 sqrt 3 of a whole 8 sqrt 3: 0.3 of it lies between the two
    ov, of, kept = _clean(v, f, min_diameter=0.3)
    assert kept.tolist() == [4, 5, 6, 7] and of.tolist() == _tetra(0)      # renumbered into the kept vertices
    assert np.array_equal(ov, v[4:])
    assert [len(x) for x in _clean(v, f, min_faces=5)] == [0, 0, 0]


def test_a_bowtie_is_one_component():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [-1, 0, 0], [0, -1, 0]], np.float32)
    f = np.array([[0, 1, 2], [0, 3, 4]], np.int32)                   # sharing vertex 0 only
    assert mesh_ref.components(f, 5).tolist() == [0] * 5
    _, of, kept = _clean(v, f, min_faces=2)
    assert kept.tolist() == list(range(5)) and np.array_equal(of, f)


def test_an_isolated_vertex_is_dropped():
    v = np.concatenate([TETRA[:2], [[9, 9, 9]], TETRA[2:]])        # vertex 2 referenced by no face
    f = np.array([[0, 3, 1], [0, 1, 4], [0, 4, 3], [1, 3, 4]], np.int32)
    assert mesh_ref.components(f, 5).tolist() == [0, 0, 2, 0, 0]
    for kw in (dict(), dict(min_faces=0), dict(keep_largest=True), dict(min_diameter=0.01)):
        ov, of, kept = _clean(v, f, **kw)
        assert kept.tolist() == [0, 1, 3, 4], kw
        assert of.tolist() == [[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], kw
        assert 9 not in ov, kw


def test_a_degenerate_face_is_an_ordinary_face():
    v = np.concatenate([TETRA, [[5, 5, 5], [6, 6, 6]]])
    f = np.array(_tetra(0) + [[4, 4, 5]], np.int32)                # connects 4 and 5, one face
    assert mesh_ref.components(f, 6).tolist() == [0, 0, 0, 0, 4, 4]
    _, of, kept = _clean(v, f)
    assert kept.tolist() == list(range(6)) and np.array_equal(of, f)
    _, of, kept = _clean(v, f, min_faces=2)
    assert kept.tolist() == [0, 1, 2, 3] and of.tolist() == _tetra(0)
    f1 = np.array([[2, 2, 2]], np.int32)                           # one vertex, one face: referenced, one face
    _, of, kept = _clean(v, f1)
    assert kept.tolist() == [2] and of.tolist() == [[0, 0, 0]]


def test_no_faces():
    v = TETRA
    assert mesh_ref.components(np.zeros((0, 3), np.int32), 4).tolist() == [0, 1, 2, 3]
    for kw in (dict(), dict(min_faces=0), dict(keep_largest=True), dict(min_diameter=0.3)):
        ov, of, kept = _clean(v, np.zeros((0, 3), np.int32), **kw)
        assert ov.shape == (0, 3) and of.shape == (0, 3) and kept.shape == (0,), kw


def test_diameter_and_face_count_thresholds_are_inclusive():
    # component A: a unit tetrahedron (diagonal sqrt 3); B: a tetrahedron at 10 scaled by s
    s = 4.0
    v = np.concatenate([TETRA, TETRA * s + 10]).astype(np.float32)
    f = np.array(_tetra(0) + _tetra(4) + _tetra(4)[:2], np.int32)  # B has 6 faces
    lo, hi = v.min(0).astype(np.float64), v.max(0).astype(np.float64)
    d_all = math.sqrt(float(np.sum((hi - lo) ** 2)))
    d_a = math.sqrt(3.0)
    frac = d_a / d_all                                              # min_diameter * d_all rounds back to d_a?
    while frac * d_all > d_a:
        frac = np.nextafter(frac, 0)
    while frac * d_all < d_a:
        frac = np.nextafter(frac, 1)
    assert frac * d_all == d_a
    assert _clean(v, f, min_diameter=float(frac))[2].tolist() == list(range(8))       # exactly equal: kept
    assert _clean(v, f, min_diameter=float(np.nextafter(frac, 1)))[2].tolist() == [4, 5, 6, 7]
    assert _clean(v, f, min_faces=4)[2].tolist() == list(range(8))                   # A has exactly 4
    assert _clean(v, f, min_faces=5)[2].tolist() == [4, 5, 6, 7]
    assert _clean(v, f, min_faces=6)[2].tolist() == [4, 5, 6, 7]
    assert _clean(v, f, min_faces=7)[2].tolist() == []
    # keep_largest among those passing: B has the most faces; with B filtered out by size, A
    assert _clean(v, f, keep_largest=True)[2].tolist() == [4, 5, 6, 7]
    assert _clean(v, f, keep_largest=True, min_diameter=1.0)[2].tolist() == []


def test_keep_largest_tie_goes_to_the_smaller_label():
    v = np.concatenate([TETRA + 7, TETRA, TETRA - 7])
    f = np.array(_tetra(8) + _tetra(4) + _tetra(0), np.int32)      # faces listed from the largest label down
    _, of, kept = _clean(v, f, keep_largest=True)
    assert kept.tolist() == [0, 1, 2, 3] and of.tolist() == _tetra(0)
    f2 = np.concatenate([f, [[8, 9, 10]]])                          # now label 8 has one face more
    assert _clean(v, f2, keep_largest=True)[2].tolist() == [8, 9, 10, 11]


def test_nan_coordinates_are_skipped():
    v = np.concatenate([TETRA, TETRA * 2 + 3]).astype(np.float32)
    v[1, 0] = np.nan                                                # A: x from 0 .. 0 (the 1 is gone), y, z 0 .. 1
    v[4:, 2] = np.nan                                               # B: z all NaN, extent 0
    f = np.array(_tetra(0) + _tetra(4), np.int32)
    ov, of, kept = _clean(v, f)
    assert kept.tolist() == list(range(8)) and np.array_equal(ov.view(np.uint32), v.view(np.uint32))
    # d_A = sqrt(0 + 1 + 1), d_B = sqrt(4 + 4 + 0); the whole box: x 0 .. 5, y 0 .. 5, z 0 .. 1
    d_all = math.sqrt(25 + 25 + 1)
    for frac, expect in ((math.sqrt(2) / d_all, list(range(8))), (np.nextafter(math.sqrt(8) / d_all, 0), [4, 5, 6, 7]),
                         (np.nextafter(math.sqrt(8) / d_all, 1), [])):
        assert _clean(v, f, min_diameter=float(frac))[2].tolist() == expect, frac
    allnan = np.full((4, 3), np.nan, np.float32)
    assert _clean(allnan, _tetra(0), min_diameter=0.5)[2].tolist() == [0, 1, 2, 3]   # d = 0 >= 0.5 * 0: kept
    assert _clean(allnan, _tetra(0), min_diameter=0.5, min_faces=5)[2].tolist() == []


def test_out_of_range_indices_are_refused_by_the_restatement():
    for bad in ([[0, 1, 4]], [[0, -1, 2]]):
        with pytest.raises(ValueError, match="outside"):
            mesh_ref.components(np.array(bad), 4)
