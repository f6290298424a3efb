"""CPU-only checks of the opacity field (include/b200gsr_fields.h, dreamscene_b200.fields): the signature table
agrees with the header and binds; the library refuses bad arguments before touching a device (made-up device
addresses, never dereferenced); extract_fields refuses what it cannot take; and the restatement the GPU tests compare
against (harness/fields_ref.py) agrees with a brute-force evaluation of every grid point, also where the resolution is
not a multiple of num_blocks."""
import ctypes as C
import math
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from dreamscene_b200 import _lib
from dreamscene_b200 import fields as Fd
from harness import fields_ref
from tests import test_abi_binding_cpu as abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "b200gsr_fields.h")


def _prototypes():
    src = re.sub(r"/\*.*?\*/", " ", open(HEADER).read(), flags=re.S)
    return {name: (ret, [" ".join(a.split()) for a in args.split(",")])
            for ret, name, args in re.findall(r"(\bint)\s+(b200gsr_\w+)\s*\(([^)]*)\)\s*;", src)}


def test_fields_signature_table_matches_the_header_and_binds(monkeypatch):
    monkeypatch.setitem(abi._SCALARS, "double", C.c_double)
    monkeypatch.setitem(abi._STRUCTS, "b200gsr_fields_layout", _lib.FieldsLayout)
    # info is a device pointer, bound as void*; the layout is a host struct, bound as a pointer to its mirror
    protos = _prototypes()
    assert list(protos) == list(_lib.FIELDS_SIGNATURES) == ["b200gsr_fields_layout_query", "b200gsr_fields"]
    assert abi._mismatches(_lib.FIELDS_SIGNATURES, protos) == []
    text = open(HEADER).read()
    for name, value in (("MAX_R", _lib.FIELDS_MAX_R), ("MAX_CHUNKS", _lib.FIELDS_MAX_CHUNKS)):
        assert re.search(rf"#define B200GSR_FIELDS_{name} (\d+)", text).group(1) == str(value)
    # the two structs, field by field, in the header's order
    for struct, cls in (("b200gsr_fields_layout", _lib.FieldsLayout), ("b200gsr_fields_info", _lib.FieldsInfo)):
        body = re.search(r"typedef struct \{([^}]*)\}\s*" + struct + ";", text).group(1)
        names = re.findall(r"\b(\w+)(?:\[\d+\])?;", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
        assert names == [n for n, _ in cls._fields_], struct
    assert C.sizeof(_lib.FieldsInfo) == 40 and C.sizeof(_lib.FieldsLayout) == 24
    lib = _lib.load()
    for name, (restype, argtypes) in _lib.FIELDS_SIGNATURES.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and tuple(fn.argtypes) == tuple(argtypes), name
    others = (set(_lib.SIGNATURES) | set(_lib.SCENE_SIGNATURES) | set(_lib.STEP_SIGNATURES) |
              set(_lib.LOSS_SIGNATURES) | set(_lib.FROZEN_SIGNATURES) | set(_lib.STATS_SIGNATURES) |
              set(_lib.RESERVE_SIGNATURES) | set(_lib.FRAMES_SIGNATURES) | set(_lib.VIEWS_FROZEN_SIGNATURES) |
              set(_lib.VIEWS_STATS_SIGNATURES))
    assert not set(_lib.FIELDS_SIGNATURES) & others


def _coords(R):
    t = torch.linspace(-1, 1, R)
    return t, C.c_void_p(t.data_ptr())


def _query(P=1000, R=128, nb=16, rr=1.5, coords=None):
    t, p = _coords(R)
    out = _lib.FieldsLayout()
    rc = _lib.load().b200gsr_fields_layout_query(P, R, nb, rr, p if coords is None else coords, C.byref(out))
    return rc, out


def test_layout_query_sizes_the_default_grid():
    rc, out = _query()
    assert rc == 0
    assert out.blocks_per_axis == 16
    assert out.max_blocks_per_axis == 4          # boxes 7/127 * 2 + 2 * 0.1875 wide, 16/127 apart
    assert out.max_pairs == 1000 * 4 ** 3
    rc, out = _query(R=10, nb=4)                 # chunks of 2: five per axis, the reference's split
    assert rc == 0 and out.blocks_per_axis == 5
    rc, out = _query(rr=-1.0)                    # empty boxes: nothing can be a member
    assert rc == 0 and out.max_pairs == 0


def test_library_refuses_bad_field_arguments():
    lib = _lib.load()
    for kw, msg in ((dict(P=0), "at least one row"), (dict(R=0), "resolution"), (dict(R=1025), "resolution"),
                    (dict(nb=0), "num_blocks"), (dict(R=8, nb=9), "num_blocks"), (dict(R=4, nb=3), "multiple"),
                    (dict(R=128, nb=128), "chunks per axis"), (dict(rr=math.inf), "finite"),
                    (dict(rr=math.nan), "finite"), (dict(P=40_000_000), "too large")):
        rc, _ = _query(**kw)
        assert rc == _lib.ERR_BAD_ARG and msg in _lib.last_error(), kw
    assert _query(coords=C.c_void_p(0))[0] == _lib.ERR_BAD_ARG and "coords" in _lib.last_error()
    bad = torch.linspace(-1, 1, 16)
    bad[3] = math.nan
    assert _query(R=16, nb=4, coords=C.c_void_p(bad.data_ptr()))[0] == _lib.ERR_BAD_ARG
    assert lib.b200gsr_fields_layout_query(10, 16, 4, 1.5, _coords(16)[1], None) == _lib.ERR_BAD_ARG

    t, cp = _coords(16)
    rc, lay = _query(P=10, R=16, nb=4)
    assert rc == 0
    dev = [C.c_void_p(0x100000 * (k + 1)) for k in range(7)]      # xyz, opacity, scaling, rotation, occ, info, scratch

    def call(ptrs=dev, P=10, R=16, nb=4, nbytes=lay.total):
        x, o, s, r, occ, info, scr = ptrs
        return lib.b200gsr_fields(P, x, o, s, r, R, nb, 1.5, cp, occ, info, scr, nbytes, None)

    for k in range(7):
        ptrs = list(dev)
        ptrs[k] = None
        assert call(ptrs) == _lib.ERR_BAD_ARG and "null" in _lib.last_error()
    for k, what in ((3, "rotation"), (5, "info"), (6, "scratch")):
        ptrs = list(dev)
        ptrs[k] = C.c_void_p(0x100008 if k == 3 else 0x100004 if k == 5 else 0x100080)
        assert call(ptrs) == _lib.ERR_BAD_ARG and what in _lib.last_error()
    assert call(nbytes=lay.total - 1) == _lib.ERR_BAD_ARG and "scratch holds" in _lib.last_error()
    assert call(R=16, nb=3) == _lib.ERR_BAD_ARG and "multiple" in _lib.last_error()
    assert call(P=-1) == _lib.ERR_BAD_ARG


def _group(P, seed=0, device="cpu", std=0.05):
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(P, 3, generator=g)
    d /= d.norm(dim=1, keepdim=True)
    xyz = 0.5 * torch.rand(P, 1, generator=g) ** (1 / 3) * d
    leaves = dict(_xyz=xyz, _opacity=1.5 * torch.randn(P, 1, generator=g),
                  _scaling=math.log(std) + 0.3 * torch.randn(P, 3, generator=g), _rotation=torch.randn(P, 4, generator=g))
    return {k: v.to(device) for k, v in leaves.items()}


def test_extract_fields_refusals():
    g = _group(50)
    with pytest.raises(ValueError, match="CUDA tensors"):
        Fd.extract_fields(g, 16, 4)
    with pytest.raises(ValueError, match="multiple of the block size"):
        Fd.extract_fields(g, 4, 3)
    for nb in (0, -2, 17):
        with pytest.raises(ValueError, match="num_blocks"):
            Fd.extract_fields(g, 16, nb)
    with pytest.raises(ValueError, match="_rotation has shape"):
        Fd.extract_fields(dict(g, _rotation=g["_rotation"][:, :3]), 16, 4)
    with pytest.raises(ValueError, match="empty"):
        Fd.extract_fields({k: v[:0] for k, v in g.items()}, 16, 4)
    with pytest.raises(TypeError, match="ReservedGroup"):
        Fd.extract_fields(SimpleNamespace(_reserved_rows=True, **g), 16, 4)
    # the reference's assert, restated: resolution % (2 / num_blocks) with Python floats
    with pytest.raises(AssertionError):
        fields_ref.chunks(4, 3)


def _brute_force(group, R, nb, rr):
    """Every grid point on its own, in float64 numpy: its block from the chunking, the block's members by the float32
    box test of the reference, and each member's weight from numpy's inverse of the float64 covariance."""
    n = fields_ref.normalise(group)
    keep = n["mask"].numpy()
    xyz32 = n["xyz"].numpy()
    center = n["center"].double().numpy()
    xyz = (group["_xyz"].double().numpy()[keep] - center) * n["scale"]
    stds = np.exp(group["_scaling"].double().numpy()[keep]) * n["scale"]
    q = group["_rotation"].double().numpy()[keep]
    q = q / np.linalg.norm(q, axis=1, keepdims=True)
    opa = 1.0 / (1.0 + np.exp(-group["_opacity"].double().numpy()[keep, 0]))
    r, x, y, z = q.T
    Rm = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], -1),
                   np.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], -1),
                   np.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1)], 1)
    L = Rm * stds[:, None, :]
    inv = np.linalg.inv(L @ L.transpose(0, 2, 1))
    coords = torch.linspace(-1, 1, R).numpy()
    split = R // nb
    r32 = np.float32((2 / nb) * rr)
    lo = [np.float32(coords[c:c + split].min() - r32) for c in range(0, R, split)]
    hi = [np.float32(coords[c:c + split].max() + r32) for c in range(0, R, split)]
    occ = np.zeros((R, R, R))
    for i in range(R):
        for j in range(R):
            for k in range(R):
                b = [i // split, j // split, k // split]
                inside = np.ones(len(xyz32), bool)
                for a in range(3):
                    inside &= (xyz32[:, a] > lo[b[a]]) & (xyz32[:, a] < hi[b[a]])
                d = np.array([coords[i], coords[j], coords[k]], np.float64)[None] - xyz[inside]
                power = -0.5 * np.einsum("ni,nij,nj->n", d, inv[inside], d)
                occ[i, j, k] = (opa[inside] * np.where(power > 0, 0.0, np.exp(power))).sum()
    return occ


@pytest.mark.parametrize("R,nb", [(8, 2), (10, 4), (9, 2)])
def test_restatement_matches_a_brute_force_evaluation(R, nb):
    """(10, 4) and (9, 2) cut the axis into chunks of 2 and 4 with a shorter last one: five and three chunks."""
    g = _group(60, seed=R, std=0.15)
    ref = _brute_force(g, R, nb, 1.5)
    occ64, center, scale = fields_ref.extract_fields(g, R, nb, 1.5, dtype=torch.float64)
    occ32, _, _ = fields_ref.extract_fields(g, R, nb, 1.5)
    assert len(fields_ref.chunks(R, nb)) == -(-R // (R // nb))
    assert ref.max() > 0.5
    np.testing.assert_allclose(occ64.numpy(), ref, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(occ32.double().numpy(), ref, rtol=1e-4, atol=1e-5)
    assert center.dtype == torch.float32 and isinstance(scale, float)


def test_member_counts_follow_the_widened_boxes():
    g = _group(200, seed=3)
    counts = fields_ref.member_counts(g, 16, 4, 1.5)
    xyz = fields_ref.normalise(g)["xyz"]
    # chunks of 4 points 2/15 apart, widened by (2 / 4) * 1.5 = 0.75 on each side: box c is
    # (-1 + 8c/15 - 0.75, -1 + (8c + 6)/15 + 0.75), and a row is in every box its three coordinates fall into
    lo = torch.tensor([-1 + 8 * c / 15 - 0.75 for c in range(4)])
    hi = torch.tensor([-1 + (8 * c + 6) / 15 + 0.75 for c in range(4)])
    per_axis = ((xyz[:, :, None] > lo) & (xyz[:, :, None] < hi)).sum(1)      # [K, 4]: rows per chunk and axis
    expect = torch.einsum("ki,kj,kl->ijl", *[((xyz[:, a, None] > lo) & (xyz[:, a, None] < hi)).long() for a in range(3)])
    assert counts.shape == (4, 4, 4) and torch.equal(counts, expect)
    assert int(per_axis.sum()) >= 3 * len(xyz)
