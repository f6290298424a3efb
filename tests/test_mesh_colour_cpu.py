"""CPU-only checks of the mesh colour (include/b200gsr_mesh_colour.h, dreamscene_b200.fields.extract_fields_rgb,
dreamscene_b200.mesh.marching_cubes(attributes=) and extract_coloured_mesh): the signature table agrees with the header
and binds; the library refuses bad arguments before touching a device (made-up device addresses, never dereferenced);
the Python entry points refuse what they cannot take; and the restatements the GPU tests compare against
(harness/fields_ref.py, harness/mesh_ref.py) give the colours the definition gives on hand-made cases."""
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
from dreamscene_b200 import mesh as Mh
from harness import fields_ref, mesh_ref
from tests import test_abi_binding_cpu as abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "b200gsr_mesh_colour.h")
R_MAX = 894                      # the largest R with 3 R^3 < 2^31


def _prototypes():
    src = re.sub(r"/\*.*?\*/", " ", open(HEADER).read(), flags=re.S)
    return {name: (ret, [" ".join(a.split()) for a in args.split(",")])
            for ret, name, args in re.findall(r"(\bint)\s+(b200gsr_\w+)\s*\(([^)]*)\)\s*;", src)}


def test_mesh_colour_signature_table_matches_the_header_and_binds(monkeypatch):
    monkeypatch.setitem(abi._SCALARS, "double", C.c_double)
    monkeypatch.setitem(abi._STRUCTS, "b200gsr_fields_layout", _lib.FieldsLayout)
    protos = _prototypes()
    assert list(protos) == list(_lib.MESH_COLOUR_SIGNATURES) == ["b200gsr_fields_rgb_layout_query",
                                                                 "b200gsr_fields_rgb", "b200gsr_mesh_attributes"]
    assert abi._mismatches(_lib.MESH_COLOUR_SIGNATURES, protos) == []
    # the query takes exactly what the opacity field's query takes
    assert (_lib.MESH_COLOUR_SIGNATURES["b200gsr_fields_rgb_layout_query"] ==
            _lib.FIELDS_SIGNATURES["b200gsr_fields_layout_query"])
    lib = _lib.load()
    for name, (restype, argtypes) in _lib.MESH_COLOUR_SIGNATURES.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and tuple(fn.argtypes) == tuple(argtypes), name
    others = (set(_lib.SIGNATURES) | set(_lib.SCENE_SIGNATURES) | set(_lib.STEP_SIGNATURES) |
              set(_lib.LOSS_SIGNATURES) | set(_lib.FROZEN_SIGNATURES) | set(_lib.STATS_SIGNATURES) |
              set(_lib.RESERVE_SIGNATURES) | set(_lib.FRAMES_SIGNATURES) | set(_lib.VIEWS_FROZEN_SIGNATURES) |
              set(_lib.VIEWS_STATS_SIGNATURES) | set(_lib.FIELDS_SIGNATURES) | set(_lib.MESH_SIGNATURES))
    assert not set(_lib.MESH_COLOUR_SIGNATURES) & others


def _coords(R):
    t = torch.linspace(-1, 1, R)
    return t, C.c_void_p(t.data_ptr())


def _queries(P=1000, R=128, nb=16, rr=1.5, coords=None):
    """(rc, layout) of the opacity field's query and of the colour field's, for the same arguments."""
    t, p = _coords(R)
    lib, out = _lib.load(), []
    for q in (lib.b200gsr_fields_layout_query, lib.b200gsr_fields_rgb_layout_query):
        lay = _lib.FieldsLayout()
        rc = q(P, R, nb, rr, p if coords is None else coords, C.byref(lay))
        out.append((rc, [getattr(lay, f) for f, _ in lay._fields_], _lib.last_error() if rc else ""))
    return out


def test_rgb_layout_query_is_the_field_query_with_one_more_limit():
    for kw in (dict(), dict(R=10, nb=4), dict(rr=-1.0), dict(P=5, R=R_MAX, nb=2), dict(P=77, R=64, nb=8)):
        (rc, lay, _), (rc_rgb, lay_rgb, _) = _queries(**kw)
        assert rc == rc_rgb == 0 and lay == lay_rgb, kw
    # the same refusals, with the same messages
    for kw in (dict(P=0), dict(R=0), dict(R=1025), dict(nb=0), dict(R=8, nb=9), dict(R=4, nb=3), dict(R=128, nb=128),
               dict(rr=math.inf), dict(rr=math.nan), dict(P=40_000_000), dict(coords=C.c_void_p(0))):
        (rc, _, msg), (rc_rgb, _, msg_rgb) = _queries(**kw)
        assert rc == rc_rgb == _lib.ERR_BAD_ARG and msg == msg_rgb, kw
    # 3 R^3 < 2^31: R = 895 is a grid the opacity field takes and the colour field does not
    (rc, _, _), (rc_rgb, _, msg) = _queries(P=5, R=R_MAX + 1, nb=2)
    assert rc == 0 and rc_rgb == _lib.ERR_BAD_ARG and "3 R^3" in msg
    assert 3 * R_MAX ** 3 < 2 ** 31 <= 3 * (R_MAX + 1) ** 3
    assert _lib.load().b200gsr_fields_rgb_layout_query(10, 16, 4, 1.5, _coords(16)[1], None) == _lib.ERR_BAD_ARG


def test_library_refuses_bad_colour_field_arguments():
    lib = _lib.load()
    t, cp = _coords(16)
    lay = _lib.FieldsLayout()
    assert lib.b200gsr_fields_rgb_layout_query(10, 16, 4, 1.5, cp, C.byref(lay)) == 0
    # xyz, opacity, scaling, rotation, features_dc, occ, rgb, info, scratch
    dev = [C.c_void_p(0x100000 * (k + 1)) for k in range(9)]

    def call(ptrs=dev, P=10, R=16, nb=4, nbytes=lay.total):
        x, o, s, r, dc, occ, rgb, info, scr = ptrs
        return lib.b200gsr_fields_rgb(P, x, o, s, r, dc, R, nb, 1.5, cp, occ, rgb, info, scr, nbytes, None)

    for k in range(9):
        ptrs = list(dev)
        ptrs[k] = None
        assert call(ptrs) == _lib.ERR_BAD_ARG and "null" in _lib.last_error(), k
    for k, what in ((3, "rotation"), (4, "features_dc"), (6, "rgb"), (7, "info"), (8, "scratch")):
        ptrs = list(dev)
        ptrs[k] = C.c_void_p(dev[k].value + (8 if k == 3 else 2 if k in (4, 6) else 4 if k == 7 else 0x80))
        assert call(ptrs) == _lib.ERR_BAD_ARG and what in _lib.last_error(), k
    assert call(nbytes=lay.total - 1) == _lib.ERR_BAD_ARG and "scratch holds" in _lib.last_error()
    assert call(R=16, nb=3) == _lib.ERR_BAD_ARG and "multiple" in _lib.last_error()
    assert call(P=-1) == _lib.ERR_BAD_ARG
    big, bp = _coords(R_MAX + 1)
    assert (lib.b200gsr_fields_rgb(10, *dev[:5], R_MAX + 1, 2, 1.5, bp, *dev[5:], 1 << 40, None) == _lib.ERR_BAD_ARG
            and "3 R^3" in _lib.last_error())


def test_library_refuses_bad_attribute_arguments():
    lib = _lib.load()
    out = _lib.MeshLayout()
    assert lib.b200gsr_mesh_layout_query(7, 9, 11, C.byref(out)) == 0
    vol, scr, attr, dst = (C.c_void_p(0x100000 * (k + 1)) for k in range(4))

    def call(X=7, Y=9, Z=11, v=vol, iso=0.5, s=scr, n=out.total, a=attr, o=dst, V=10):
        return lib.b200gsr_mesh_attributes(X, Y, Z, v, iso, s, n, a, o, V, None)

    # marching cubes' refusals, then the attribute pass's own
    for kw, msg in ((dict(X=0), "dimension"), (dict(Z=2000), "dimension"), (dict(iso=math.inf), "finite"),
                    (dict(iso=math.nan), "finite"), (dict(iso=1e39), "finite"), (dict(v=None), "null"),
                    (dict(s=None), "null"), (dict(n=out.total - 1), "scratch holds"),
                    (dict(s=C.c_void_p(0x100080)), "256-byte"), (dict(v=C.c_void_p(0x100002)), "4-byte"),
                    (dict(X=1024, Y=1024, Z=1024), "too large"), (dict(a=None), "null"), (dict(o=None), "null"),
                    (dict(a=C.c_void_p(0x300001)), "4-byte"), (dict(o=C.c_void_p(0x400002)), "4-byte"),
                    (dict(V=-1), "V = -1")):
        assert call(**kw) == _lib.ERR_BAD_ARG and msg in _lib.last_error(), kw


def _group(P, seed=0, device="cpu", std=0.05):
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(P, 3, generator=g)
    d /= d.norm(dim=1, keepdim=True)
    xyz = 0.5 * torch.rand(P, 1, generator=g) ** (1 / 3) * d
    leaves = dict(_xyz=xyz, _opacity=1.5 * torch.randn(P, 1, generator=g),
                  _scaling=math.log(std) + 0.3 * torch.randn(P, 3, generator=g), _rotation=torch.randn(P, 4, generator=g),
                  _features_dc=torch.randn(P, 1, 3, generator=g))
    return {k: v.to(device) for k, v in leaves.items()}


def test_python_refusals_without_a_device():
    g = _group(50)
    with pytest.raises(ValueError, match="CUDA tensors"):
        Fd.extract_fields_rgb(g, 16, 4)
    with pytest.raises(ValueError, match="multiple of the block size"):
        Fd.extract_fields_rgb(g, 4, 3)
    for nb in (0, 17):
        with pytest.raises(ValueError, match="num_blocks"):
            Fd.extract_fields_rgb(g, 16, nb)
    with pytest.raises(ValueError, match="_rotation has shape"):
        Fd.extract_fields_rgb(dict(g, _rotation=g["_rotation"][:, :3]), 16, 4)
    with pytest.raises(TypeError, match="ReservedGroup"):
        Fd.extract_fields_rgb(SimpleNamespace(_reserved_rows=True, **g), 16, 4)
    with pytest.raises(ValueError, match="CUDA tensors"):
        Mh.extract_coloured_mesh(g, 16, 1.0, 4)
    with pytest.raises(ValueError, match="CUDA tensor"):
        Mh.marching_cubes(torch.zeros(4, 4, 4), 0.5, torch.zeros(4, 4, 4, 3))


def test_sh2rgb_is_torchs_float32_expression_clamped_at_zero():
    dc = torch.tensor([[[-10.0, -1.7724539, 0.0]], [[1.0, 1e-8, -1.77245]], [[math.nan, 3.5, -1e30]]])
    c = fields_ref.sh2rgb(dc)
    x = dc.numpy()[:, 0].astype(np.float32)
    expect = np.maximum(x * np.float32(fields_ref.SH_C0) + np.float32(0.5), np.float32(0))   # two roundings
    expect[np.isnan(x)] = np.nan
    assert c.dtype == torch.float32 and c.shape == (3, 3)
    np.testing.assert_array_equal(c.numpy(), expect)
    assert float(c[0, 0]) == 0.0 and float(c[2, 2]) == 0.0 and math.isnan(float(c[2, 0]))    # negative -> 0, NaN kept
    assert float(c[0, 2]) == 0.5 and float(c[1, 0]) == np.float32(np.float32(fields_ref.SH_C0) + np.float32(0.5))


def test_restated_field_of_a_single_colour_group_is_that_colour():
    g = _group(80, seed=1, std=0.15)
    colour = torch.tensor([0.25, 0.8, 1.3])                                 # above 1 is kept: no clamp there
    g["_features_dc"] = ((colour - 0.5) / fields_ref.SH_C0).view(1, 1, 3).repeat(80, 1, 1)
    c = fields_ref.sh2rgb(g["_features_dc"])
    assert ((c - colour).abs() < 1e-6).all()
    for dtype, tol in ((torch.float64, 1e-12), (torch.float32, 1e-6)):
        occ, rgb, _, _ = fields_ref.extract_fields_rgb(g, 10, 2, 1.5, dtype=dtype)
        on = occ > 0
        assert rgb.shape == (10, 10, 10, 3) and rgb.dtype == dtype and int(on.sum()) > 500
        assert ((rgb[on] - c[0].to(dtype)).abs() <= tol * (1 + c[0].to(dtype).abs())).all()
        assert (rgb[~on] == 0).all()
    occ32, _, _ = fields_ref.extract_fields(g, 10, 2, 1.5)
    assert torch.equal(fields_ref.extract_fields_rgb(g, 10, 2, 1.5)[0], occ32)


def test_restated_negative_colours_contribute_zero():
    """Half the Gaussians have a red SH2RGB below 0: they count as red 0, so the red field is the other half's red
    times their share of occ, which a field of only those Gaussians gives."""
    g = _group(60, seed=2, std=0.15)
    dc = g["_features_dc"].clone()
    dc[::2, 0, 0] = -5.0                                     # 0.5 - 1.41 < 0
    dc[1::2, 0, 0] = (0.6 - 0.5) / fields_ref.SH_C0
    g["_features_dc"] = dc
    assert (fields_ref.sh2rgb(dc)[::2, 0] == 0).all()
    occ, rgb, _, _ = fields_ref.extract_fields_rgb(g, 8, 2, 1.5, dtype=torch.float64)
    # the same group with the negative ones at red exactly 0
    zero = dict(g, _features_dc=torch.where(torch.arange(60).view(-1, 1, 1) % 2 == 0,
                                            torch.full_like(dc, -0.5 / fields_ref.SH_C0), dc))
    assert (fields_ref.sh2rgb(zero["_features_dc"])[::2, 0].abs() < 1e-7).all()
    occ_z, rgb_z, _, _ = fields_ref.extract_fields_rgb(zero, 8, 2, 1.5, dtype=torch.float64)
    assert torch.equal(occ, occ_z)
    assert ((rgb[..., 0] - rgb_z[..., 0]).abs() < 1e-7).all()
    on = occ > 0
    assert float(rgb[..., 0][on].min()) >= 0 and float(rgb[..., 0][on].max()) <= 0.6 + 1e-12
    assert float(rgb[..., 0][on].max()) > 0.1


def test_restated_field_matches_a_per_point_sum():
    """Every grid point on its own, in float64: members by the reference's box test on the float32 centres, weights
    from the float64 restatement's covariances, and the colour as sum(op w c) / sum(op w)."""
    g = _group(40, seed=3, std=0.2)
    R, nb, rr = 6, 2, 1.5
    occ, rgb, _, _ = fields_ref.extract_fields_rgb(g, R, nb, rr, dtype=torch.float64)
    occ_f, _, _ = fields_ref.extract_fields(g, R, nb, rr, dtype=torch.float64)
    assert torch.equal(occ, occ_f)
    n = fields_ref.normalise(g)
    keep = n["mask"]
    xyz = (g["_xyz"][keep].double() - n["center"].double()) * n["scale"]
    covs = fields_ref.covariance(torch.exp(g["_scaling"][keep].double()) * n["scale"], g["_rotation"][keep].double())
    opa = torch.sigmoid(g["_opacity"][keep].double())[:, 0]
    col = fields_ref.sh2rgb(g["_features_dc"])[keep].double()
    boxes = fields_ref.block_boxes(R, nb, rr, "cpu")
    X = torch.linspace(-1, 1, R)
    split = R // nb
    for i, j, k in [(0, 0, 0), (2, 3, 1), (5, 5, 5), (3, 2, 4), (1, 4, 2)]:
        vmin, vmax = boxes[(i // split, j // split, k // split)]
        member = (n["xyz"] < vmax).all(-1) & (n["xyz"] > vmin).all(-1)
        p = torch.tensor([X[i], X[j], X[k]], dtype=torch.float64)
        w = fields_ref.gaussian_3d_coeff(p - xyz[member], covs[member])
        o = (opa[member] * w).sum()
        expect = (opa[member, None] * w[:, None] * col[member]).sum(0) / o
        assert abs(float(occ[i, j, k] - o)) <= 1e-12 and float(o) > 0
        assert torch.allclose(rgb[i, j, k], expect, rtol=1e-10, atol=1e-12), (i, j, k)


def test_restated_attributes_at_t_0_and_1_are_the_endpoints():
    """Values equal to iso put vertices at t = 0 (the outside point is at iso) and t = 1 (the inside point's neighbour
    is at iso); attributes on a 1/256 grid keep a + t (b - a) exact there."""
    rng = np.random.default_rng(4)
    vol = rng.integers(0, 2, (6, 7, 5)).astype(np.float32)         # 0 and 1 with iso 0: every t is 0 or 1
    attr = (rng.integers(0, 256, (6, 7, 5, 3)) / 256).astype(np.float32)
    v, f = mesh_ref.marching_cubes(vol, np.float32(0.0))
    a = mesh_ref.vertex_attributes(vol, np.float32(0.0), attr)
    assert a.dtype == np.float32 and a.shape == (len(v), 3) and len(v) > 20
    frac = v - np.floor(v)
    assert set(np.unique(frac)) <= {0.0}                            # t in {0, 1}: every vertex on a grid point
    idx = v.astype(np.int64)
    np.testing.assert_array_equal(a, attr[idx[:, 0], idx[:, 1], idx[:, 2]])
    # every vertex sits on the edge's outside end, which is at iso: the start (t = 0) or the end (t = 1), and both occur
    assert (vol[idx[:, 0], idx[:, 1], idx[:, 2]] == 0).all()
    inside = vol > 0
    starts_out = sum(int((~inside[sl0] & inside[sl1]).sum()) for sl0, sl1 in (
        (np.s_[:-1], np.s_[1:]), (np.s_[:, :-1], np.s_[:, 1:]), (np.s_[:, :, :-1], np.s_[:, :, 1:])))
    assert 0 < starts_out < len(v)


def test_restated_attributes_are_the_vertex_interpolation():
    """Attribute channel 0 equal to the volume itself puts iso on every vertex, to rounding; a channel equal to a grid
    coordinate reproduces that vertex coordinate bit for bit when the coordinate is the vertex's axis."""
    rng = np.random.default_rng(5)
    vol = rng.standard_normal((9, 8, 7)).astype(np.float32)
    ii, jj, kk = np.meshgrid(*[np.arange(n, dtype=np.float32) for n in vol.shape], indexing="ij")
    attr = np.stack([vol, ii, kk], -1)
    v, _ = mesh_ref.marching_cubes(vol, np.float32(0.2))
    a = mesh_ref.vertex_attributes(vol, np.float32(0.2), attr)
    assert np.abs(a[:, 0] - 0.2).max() < 1e-5
    np.testing.assert_array_equal(a[:, 1], v[:, 0])          # i + t (i + 1 - i) on x edges, i elsewhere
    np.testing.assert_array_equal(a[:, 2], v[:, 2])
    nan = vol.copy()
    nan[4, 3, 2] = math.nan
    vn, _ = mesh_ref.marching_cubes(nan, np.float32(0.0))
    an = mesh_ref.vertex_attributes(nan, np.float32(0.0), attr)
    assert np.array_equal(np.isnan(an).any(1), np.isnan(vn).any(1)) and np.isnan(an).any()
    assert mesh_ref.vertex_attributes(np.ones((1, 4, 4), np.float32), 0.5, np.ones((1, 4, 4, 3))).shape == (0, 3)
