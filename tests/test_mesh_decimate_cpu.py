"""CPU-only checks of the mesh decimation (include/b200gsr_mesh_decimate.h, dreamscene_b200.mesh.decimate_mesh): the
signature table agrees with the header and binds; the library refuses bad arguments before touching a device (made-up
device addresses, never dereferenced); the Python entry point refuses what it cannot take; and the restatement the GPU
tests compare against (harness/mesh_ref.py) gives what the definition gives on hand-made meshes."""
import ctypes as C
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
HEADER = os.path.join(ROOT, "include", "b200gsr_mesh_decimate.h")
F_MAX = (2**31 - 1) // 3


def _header():
    return re.sub(r"/\*.*?\*/", " ", open(HEADER).read(), flags=re.S)


def test_mesh_decimate_signature_table_matches_the_header_and_binds():
    src = _header()
    protos = {name: (ret, [" ".join(a.split()) for a in args.split(",")])
              for ret, name, args in re.findall(r"(\bint)\s+(b200gsr_\w+)\s*\(([^)]*)\)\s*;", src)}
    assert list(protos) == list(_lib.MESH_DECIMATE_SIGNATURES) == [
        "b200gsr_mesh_decimate_layout_query", "b200gsr_mesh_decimate_begin", "b200gsr_mesh_decimate_rounds",
        "b200gsr_mesh_decimate_emit"]
    assert abi._mismatches(_lib.MESH_DECIMATE_SIGNATURES, protos) == []
    assert _lib.MESH_DECIMATE_SIGNATURES["b200gsr_mesh_decimate_layout_query"][1][2] == C.POINTER(C.c_size_t)
    defines = dict(re.findall(r"#define\s+(B200GSR_DECIMATE_\w+)\s+(\S+)", src))
    assert int(defines["B200GSR_DECIMATE_MAX_VALENCE"]) == _lib.DECIMATE_MAX_VALENCE == mesh_ref.DEC_MAX_VALENCE
    assert int(defines["B200GSR_DECIMATE_STATUS_WORDS"]) == _lib.DECIMATE_STATUS_WORDS
    assert float(defines["B200GSR_DECIMATE_DET_TOL"]) == mesh_ref.DEC_DET_TOL
    lib = _lib.load()
    for name, (restype, argtypes) in _lib.MESH_DECIMATE_SIGNATURES.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and tuple(fn.argtypes) == tuple(argtypes), name
    others = (set(_lib.SIGNATURES) | set(_lib.SCENE_SIGNATURES) | set(_lib.STEP_SIGNATURES) |
              set(_lib.LOSS_SIGNATURES) | set(_lib.FROZEN_SIGNATURES) | set(_lib.STATS_SIGNATURES) |
              set(_lib.RESERVE_SIGNATURES) | set(_lib.FRAMES_SIGNATURES) | set(_lib.VIEWS_FROZEN_SIGNATURES) |
              set(_lib.VIEWS_STATS_SIGNATURES) | set(_lib.FIELDS_SIGNATURES) | set(_lib.MESH_SIGNATURES) |
              set(_lib.MESH_COLOUR_SIGNATURES) | set(_lib.MESH_CLEAN_SIGNATURES))
    assert not set(_lib.MESH_DECIMATE_SIGNATURES) & others


def _query(V, F):
    n = C.c_size_t(0)
    return _lib.load().b200gsr_mesh_decimate_layout_query(V, F, C.byref(n)), int(n.value)


def test_layout_query():
    rc, small = _query(1, 0)
    assert rc == 0 and small > 0 and small % 256 == 0
    rc, n = _query(950_830, 1_757_596)
    assert rc == 0 and n >= 950_830 * 190 + 1_757_596 * 76 and n % 256 == 0
    assert _query(2**31 - 1, F_MAX)[0] == 0                 # the limits themselves: sizes only, nothing allocated
    for V, F, msg in ((0, 0, "V = 0"), (-1, 5, "V = -1"), (10, -1, "F = -1"), (10, F_MAX + 1, "3 F")):
        assert _query(V, F)[0] == _lib.ERR_BAD_ARG and msg in _lib.last_error(), (V, F)
    assert _lib.load().b200gsr_mesh_decimate_layout_query(10, 10, None) == _lib.ERR_BAD_ARG


def test_library_refuses_bad_arguments():
    lib = _lib.load()
    V, F = 100, 150
    _, nbytes = _query(V, F)
    verts, faces, status, scr, ov, of, kept = (C.c_void_p(0x100000 * (k + 1)) for k in range(7))
    sizes = ((dict(V=0), "V = 0"), (dict(V=-3), "V = -3"), (dict(F=-1), "F = -1"), (dict(F=F_MAX + 1), "3 F"),
             (dict(s=None), "null"), (dict(s=C.c_void_p(0x600080)), "256-byte"), (dict(n=nbytes - 1), "scratch holds"))

    def begin(V=V, F=F, v=verts, f=faces, t=10, o=1, st=status, s=scr, n=nbytes):
        return lib.b200gsr_mesh_decimate_begin(V, F, v, f, t, o, st, s, n, None)

    def rounds(V=V, F=F, r=8, st=status, s=scr, n=nbytes):
        return lib.b200gsr_mesh_decimate_rounds(V, F, r, st, s, n, None)

    def emit(V=V, F=F, v=verts, s=scr, n=nbytes, o=ov, g=of, k=kept, Vo=10, Fo=10):
        return lib.b200gsr_mesh_decimate_emit(V, F, v, s, n, o, g, k, Vo, Fo, None)

    for call in (begin, rounds, emit):
        for kw, msg in sizes:
            assert call(**kw) == _lib.ERR_BAD_ARG and msg in _lib.last_error(), (call.__name__, kw)
    for call in (begin, rounds):
        for kw, msg in ((dict(st=None), "null"), (dict(st=C.c_void_p(0x300002)), "4-byte")):
            assert call(**kw) == _lib.ERR_BAD_ARG and msg in _lib.last_error(), (call.__name__, kw)
    for kw, msg in ((dict(v=None), "null"), (dict(f=None), "null"), (dict(v=C.c_void_p(0x100002)), "4-byte"),
                    (dict(f=C.c_void_p(0x200001)), "4-byte"), (dict(t=-1), "target_faces = -1")):
        assert begin(**kw) == _lib.ERR_BAD_ARG and msg in _lib.last_error(), kw
    assert begin(F=0, f=None, s=None) == _lib.ERR_BAD_ARG and "null" in _lib.last_error()   # faces may be null
    assert rounds(r=-1) == _lib.ERR_BAD_ARG and "rounds = -1" in _lib.last_error()
    for kw, msg in ((dict(v=None), "null"), (dict(o=None), "null"), (dict(g=None), "null"), (dict(k=None), "null"),
                    (dict(o=C.c_void_p(0x700002)), "4-byte"), (dict(g=C.c_void_p(0x800001)), "4-byte"),
                    (dict(k=C.c_void_p(0x900003)), "4-byte"), (dict(Vo=-1), "V_out = -1"), (dict(Fo=-1), "F_out = -1")):
        assert emit(**kw) == _lib.ERR_BAD_ARG and msg in _lib.last_error(), kw


def test_python_refusals_without_a_device():
    v, f = torch.zeros(4, 3), torch.tensor([[0, 1, 2]], dtype=torch.int32)
    with pytest.raises(ValueError, match="CUDA tensor"):
        Mh.decimate_mesh(v, f, 1)
    with pytest.raises(ValueError, match="torch tensor"):
        Mh.decimate_mesh(v.numpy(), f, 1)
    with pytest.raises(ValueError, match=r"\[V,3\]"):
        Mh.decimate_mesh(torch.zeros(4, 2), f, 1)
    with pytest.raises(ValueError, match=r"\[F,3\]"):
        Mh.decimate_mesh(v, f.view(-1), 1)
    with pytest.raises(ValueError, match="float32"):
        Mh.decimate_mesh(v.double(), f, 1)
    with pytest.raises(ValueError, match="int32"):
        Mh.decimate_mesh(v, f.long(), 1)
    for bad in (-1, 2**31, 1.5, True, None, "10"):
        with pytest.raises(ValueError, match="target_faces"):
            Mh.decimate_mesh(v, f, bad)
    with pytest.raises(ValueError, match="optimal_placement"):
        Mh.decimate_mesh(v, f, 1, optimal_placement=1)


# ---- the restatement on hand-made meshes -------------------------------------------------------------------------

def _dec(v, f, target, optimal=True):
    return mesh_ref.decimate_mesh(np.asarray(v, np.float32), np.asarray(f, np.int32).reshape(-1, 3), target, optimal,
                                  return_rounds=True)


def _outward(v, f):
    """Faces turned so their normals point away from the centroid (convex shapes)."""
    v = np.asarray(v, np.float64)
    out = []
    for t in f:
        p = v[list(t)]
        n = np.cross(p[1] - p[0], p[2] - p[0])
        out.append(list(t) if np.dot(n, p.mean(0) - v.mean(0)) > 0 else [t[0], t[2], t[1]])
    return np.array(out, np.int32)


def _euler(v, f):
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
    return len(v) - len(np.unique(e[:, 0] * (len(v) + 1) + e[:, 1])) + len(f)


def _closed_manifold(f):
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]).astype(np.int64)
    key, rev = e[:, 0] * 2**32 + e[:, 1], e[:, 1] * 2**32 + e[:, 0]
    return len(np.unique(key)) == len(key) and np.isin(rev, key).all()


TETRA_V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
TETRA_F = _outward(TETRA_V, [[0, 1, 2], [0, 1, 3], [0, 2, 3], [1, 2, 3]])
OCTA_V = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float32)
OCTA_F = _outward(OCTA_V, [[x, y, z] for x in (0, 1) for y in (2, 3) for z in (4, 5)])


def _same_as_clean(out, v, f):
    ov, of, kept, rounds = out
    cv, cf, ck = mesh_ref.clean_mesh(np.asarray(v, np.float32), np.asarray(f, np.int32))
    assert rounds == 0 and np.array_equal(ov.view(np.uint32), cv.view(np.uint32))
    assert np.array_equal(of, cf) and np.array_equal(kept, ck)


def test_a_tetrahedron_never_collapses():
    for t in (0, 1, 2, 3):
        for opt in (True, False):
            _same_as_clean(_dec(TETRA_V, TETRA_F, t, opt), TETRA_V, TETRA_F)     # valences 3 + 3 - 4 < 3


def test_an_octahedron_stops_at_a_tetrahedron():
    """deg 4 + 4 - 4 = 4 and two common neighbours: an octahedron edge may collapse (to a triangular bipyramid), and
    that to a tetrahedron, which never collapses: the closed surface stays a sphere (chi = 2) with 4 faces."""
    for opt in (True, False):
        ov, of, kept, rounds = _dec(OCTA_V, OCTA_F, 0, opt)
        assert len(of) == 4 and len(ov) == 4 and rounds == 2 and _closed_manifold(of) and _euler(ov, of) == 2
        _same_as_clean(_dec(OCTA_V, OCTA_F, 8, opt), OCTA_V, OCTA_F)           # F <= target: clean_mesh's result
        ov, of, kept, rounds = _dec(OCTA_V, OCTA_F, 6, opt)
        assert len(of) == 6 and rounds == 1 and _closed_manifold(of)


def _sphere(levels=2):
    v, f = OCTA_V.astype(np.float64), OCTA_F
    for _ in range(levels):
        vs, idx, nf = list(map(tuple, v)), {}, []

        def mid(a, b):
            k = (min(a, b), max(a, b))
            if k not in idx:
                m = (np.array(vs[a]) + np.array(vs[b])) / 2
                idx[k] = len(vs)
                vs.append(tuple(m / np.linalg.norm(m)))
            return idx[k]
        for a, b, c in f:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            nf += [[a, ab, ca], [b, bc, ab], [c, ca, bc], [ab, bc, ca]]
        v, f = np.array(vs), np.array(nf, np.int32)
    return v.astype(np.float32), f


def test_overshoot_round_lands_on_target_and_target_minus_one():
    v, f = _sphere()                                          # 66 vertices, 128 faces
    for opt in (True, False):
        for target in (100, 99, 64, 63, 20, 5):
            ov, of, kept, rounds = _dec(v, f, target, opt)
            assert len(of) in (target, target - 1) and rounds >= 1, (target, opt)
            assert _closed_manifold(of) and _euler(ov, of) == 2
            assert np.all(np.diff(kept) > 0)
        _same_as_clean(_dec(v, f, 128, opt), v, f)


def test_a_valence_3_vertex():
    """A vertex of valence 3 on a sphere (a cap raised over one face): the edges to it may collapse (3 + deg - 4 >=
    3 when deg >= 4) and the surface stays a sphere."""
    v, f = _sphere(1)                                          # 18 vertices, 32 faces
    c = f[0]
    apex = (v[c].mean(0) * 1.3).astype(np.float32)
    v2 = np.concatenate([v, apex[None]])
    f2 = np.concatenate([f[1:], [[c[0], c[1], 18], [c[1], c[2], 18], [c[2], c[0], 18]]]).astype(np.int32)
    assert _closed_manifold(f2)
    for opt in (True, False):
        ov, of, kept, rounds = _dec(v2, f2, 30, opt)
        assert len(of) in (30, 29) and _closed_manifold(of) and _euler(ov, of) == 2


def _grid(n):
    xs = np.arange(n + 1, dtype=np.float32)
    v = np.stack(np.meshgrid(xs, xs, indexing="ij"), -1).reshape(-1, 2)
    v = np.concatenate([v, np.zeros((len(v), 1), np.float32)], 1)
    f = []
    for i in range(n):
        for j in range(n):
            a, b, c, d = i * (n + 1) + j, (i + 1) * (n + 1) + j, (i + 1) * (n + 1) + j + 1, i * (n + 1) + j + 1
            f += [[a, b, c], [a, c, d]]
    return v, np.array(f, np.int32)


def test_an_open_square_patch_keeps_its_boundary():
    v, f = _grid(6)                                            # 49 vertices, 72 faces, 24 on the boundary
    boundary = np.flatnonzero((v[:, 0] == 0) | (v[:, 0] == 6) | (v[:, 1] == 0) | (v[:, 1] == 6))
    for opt in (True, False):
        ov, of, kept, rounds = _dec(v, f, 0, opt)
        assert rounds >= 1 and len(of) < len(f)
        assert set(boundary) <= set(kept.tolist())
        bi = np.searchsorted(kept, boundary)
        assert np.array_equal(ov[bi].view(np.uint32), v[boundary].view(np.uint32))   # boundary vertices never move
        assert _euler(ov, of) == 1 and np.all(ov[:, 2] == 0)                          # a flat disc stays flat


def test_two_tetrahedra_joined_non_manifold():
    """Two tetrahedra sharing an edge (four faces on it) and two sharing only a vertex (a pinch): no vertex of either
    join is regular, and a tetrahedron never collapses, so nothing changes."""
    v = np.concatenate([TETRA_V, TETRA_V[[1, 2]] * 0 + [[0, 0, -1], [-1, -1, -1]]]).astype(np.float32)
    f_edge = np.concatenate([TETRA_F, _outward(v[[0, 1, 4, 5]], [[0, 1, 2], [0, 1, 3], [0, 2, 3], [1, 2, 3]])])
    f_edge[4:] = np.array([[0, 1, 4, 5][i] for i in f_edge[4:].reshape(-1)]).reshape(-1, 3)
    for opt in (True, False):
        _same_as_clean(_dec(v, f_edge, 0, opt), v, f_edge)
    v2 = np.concatenate([TETRA_V, -TETRA_V[1:]]).astype(np.float32)                  # vertex 0 shared
    f2 = np.concatenate([TETRA_F, _outward(v2[[0, 4, 5, 6]], [[0, 1, 2], [0, 1, 3], [0, 2, 3], [1, 2, 3]])])
    f2[4:] = np.array([[0, 4, 5, 6][i] for i in f2[4:].reshape(-1)]).reshape(-1, 3)
    start, ev, ef, p, q = mesh_ref._fans(f2.astype(np.int64), np.ones(len(f2), bool), 7)
    k = mesh_ref._regular(start, ev, ef, p, q, f2.astype(np.int64), 7)
    assert k[0] == 0 and (k[1:] == 3).all()                                          # the pinch is not regular
    for opt in (True, False):
        _same_as_clean(_dec(v2, f2, 0, opt), v2, f2)


def test_a_collapse_that_would_flip_a_face_is_rejected():
    """A flat fan around vertex 0 with a sliver face (0, 5, 6) just below edge (0, 1): moving 0 onto 1 turns the sliver
    over, so when the quadric puts the survivor at vertex 1's place edge (0, 1) is no candidate."""
    v = np.array([[0, 0, 0], [1, 0, 0], [0.5, 1, 0], [-0.5, 1, 0], [-1, 0, 0], [-0.5, -1, 0], [0.6, -0.05, 0]],
                 np.float32)
    # the sliver face (0, 6, 5) lies just below edge (0, 1); the fan is closed by a tent under it
    ring = [1, 2, 3, 4, 5, 6]
    f = [[0, ring[i], ring[(i + 1) % 6]] for i in range(6)]
    apex = len(v)
    v = np.concatenate([v, [[0, 0, -1]]]).astype(np.float32)
    f += [[apex, ring[(i + 1) % 6], ring[i]] for i in range(6)]
    f = np.array(f, np.int32)
    assert _closed_manifold(f)
    start, ev, ef, p, q = mesh_ref._fans(f.astype(np.int64), np.ones(len(f), bool), len(v))
    k = mesh_ref._regular(start, ev, ef, p, q, f.astype(np.int64), len(v))
    pos = v.astype(np.float64)
    Q = np.zeros((len(v), 10))
    a, b = np.array([0]), np.array([1])
    ok, x, c = mesh_ref._candidates(a, b, k, start, p, q, pos, Q, False, len(v))
    # with a zero quadric every placement costs 0: a is chosen, so vertex 1 moves onto 0 and face (1, 6, apex) ...
    assert x[0].tolist() == pos[0].tolist()
    # ... while moving 0 onto 1 would put face (0, 5, 6) over: check the flip rule directly on that move
    nb = mesh_ref._cross(pos[5] - pos[0], pos[6] - pos[0])
    na = mesh_ref._cross(pos[5] - pos[1], pos[6] - pos[1])
    assert mesh_ref._dot(nb, na) < 0
    Qb = np.zeros((len(v), 10))
    Qb[0, 0] = 1.0                                            # x^2 from vertex 0's quadric: x = 0 costs 0 only at a
    okb, xb, _ = mesh_ref._candidates(np.array([0]), np.array([6]), k, start, p, q, pos, Qb, False, len(v))
    assert okb[0] and xb[0].tolist() == pos[0].tolist()
    Qc = np.zeros((len(v), 10))
    Qc[1, 0], Qc[1, 3], Qc[1, 9] = 1.0, -1.0, 1.0              # (x - 1)^2: only x = 1 (vertex 1's place) costs 0
    okc, xc, _ = mesh_ref._candidates(a, b, k, start, p, q, pos, Qc, False, len(v))
    assert xc[0].tolist() == pos[1].tolist() and not okc[0]   # the move that turns (0, 5, 6) over is refused


def test_a_tie_between_equal_costs_goes_to_the_smaller_edge():
    """A flat square patch: every face lies in z = 0, so every placement in the plane costs exactly 0 and the key order
    falls to (a, b).  One collapse (target F - 2) takes the smallest candidate edge, removes its larger endpoint and
    leaves the survivor where it was (with a singular quadric the first of a, b, midpoint wins the tie)."""
    v, f = _grid(4)
    fl = f.astype(np.int64)
    start, ev, ef, p, q = mesh_ref._fans(fl, np.ones(len(f), bool), len(v))
    k = mesh_ref._regular(start, ev, ef, p, q, fl, len(v))
    seg, idx = mesh_ref._segments(start[:-1], k)
    e = (seg < p[idx]) & (k[p[idx]] > 0)
    a, b = seg[e], p[idx][e]
    for opt in (True, False):
        ok, x, c = mesh_ref._candidates(a, b, k, start, p, q, v.astype(np.float64), np.zeros((len(v), 10)), opt, len(v))
        first = np.lexsort((b[ok], a[ok]))[0]
        ov, of, kept, rounds = _dec(v, f, len(f) - 2, opt)
        assert rounds == 1 and len(of) == len(f) - 2
        assert set(range(len(v))) - set(kept.tolist()) == {int(b[ok][first])}, opt
        assert np.array_equal(ov, v[kept])


def test_two_calls_and_both_placements():
    v, f = _sphere()
    a = _dec(v, f, 40, True)
    b = _dec(v, f, 40, True)
    assert all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(a, b))
    c = _dec(v, f, 40, False)
    assert len(c[1]) in (40, 39) and not np.array_equal(a[0], c[0])


def test_out_of_range_indices_are_refused_by_the_restatement():
    for bad in ([[0, 1, 4]], [[0, -1, 2]]):
        with pytest.raises(ValueError, match="outside"):
            mesh_ref.decimate_mesh(TETRA_V, np.array(bad), 0)
