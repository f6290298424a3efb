"""CPU-only checks of render_scene (dreamscene_b200.scene) and its C entry points (include/b200gsr_scene.h): the
signature table agrees with the header, the library refuses bad arguments before touching a device, the Python side
refuses what the kernels cannot take and normalises its per-view flags, and the group table is packed as the
kernels read it."""
import ctypes as C
import os
import re

import pytest
import torch

from dreamscene_b200 import _lib
from dreamscene_b200 import scene as S
from tests.test_abi_binding_cpu import _mismatches

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCENE_HEADER = os.path.join(ROOT, "include", "b200gsr_scene.h")


def _scene_prototypes():
    src = re.sub(r"/\*.*?\*/", " ", open(SCENE_HEADER).read(), flags=re.S)
    out = {}
    for ret, name, args in re.findall(r"(\bint)\s+(b200gsr_\w+)\s*\(([^)]*)\)\s*;", src):
        out[name] = (ret, [" ".join(a.split()) for a in args.split(",")])
    return out


def test_scene_signature_table_matches_the_header():
    protos = _scene_prototypes()
    assert list(protos) == list(_lib.SCENE_SIGNATURES) == ["b200gsr_forward_scene", "b200gsr_backward_scene"]
    assert _mismatches(_lib.SCENE_SIGNATURES, protos) == []
    for name, (restype, argtypes) in _lib.SCENE_SIGNATURES.items():      # the check sees a single wrong entry
        for i, t in enumerate(argtypes):
            if t is C.c_void_p:
                bad = argtypes[:i] + [C.c_uint64] + argtypes[i + 1:]
                assert _mismatches({name: (restype, bad)}, {name: protos[name]}) != [], (name, i)


def test_library_exports_and_binds_the_scene_entry_points():
    lib = _lib.load()
    for name, (restype, argtypes) in _lib.SCENE_SIGNATURES.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and tuple(fn.argtypes) == tuple(argtypes), name
    assert lib.b200gsr_version() == _lib.ABI_VERSION == 3
    assert not set(_lib.SCENE_SIGNATURES) & set(_lib.SIGNATURES)


def _fake_call(B=2, P=10, M=4, score=0, sh_degree=1, bg_step=3, groups_n=(6, 4), rot_offset=0, noise=True):
    """Call b200gsr_forward_scene with made-up (never dereferenced) device addresses: validation runs before any
    CUDA call, so the refusals are observable without a GPU."""
    lib = _lib.load()
    bg = 0x10000
    prm = (_lib.Params * B)(*[_lib.Params(P, M, sh_degree, 64, 64, 0.5, 0.5, 1.0, 0, score, bg + 4 * bg_step * v,
                                          0x20000, 0x30000, 0x40000) for v in range(B)])
    groups = (_lib.Group * len(groups_n))()
    for k, n in enumerate(groups_n):
        groups[k] = _lib.Group(0x100000, 0x100000, 0x100000, 0x100000 + rot_offset, 0x100000, 0x100000, n)
    c = (C.c_float * B)(*([0.447] * B))
    rc = lib.b200gsr_forward_scene(B, prm, len(groups_n), groups, c if noise else None, c, 1, None, C.c_void_p(0x50000),
                                   C.c_void_p(0x60000), C.c_void_p(0x70000), C.c_void_p(0x80000), 1 << 20,
                                   C.c_void_p(0x90000), 1 << 20, 1 << 20, 0, None, 0, None)
    return rc, _lib.last_error()


@pytest.mark.parametrize("kwargs,code,msg", [
    (dict(score=1), -4, "score_flag"),
    (dict(P=11), -1, "groups hold 10 rows"),
    (dict(B=0), -4, "number of views"),
    (dict(B=17), -4, "number of views"),
    (dict(bg_step=4), -1, "contiguous"),
    (dict(sh_degree=2), -1, "inconsistent with sh_degree"),
    (dict(rot_offset=4), -1, "16-byte aligned"),
    (dict(noise=False), -1, "host arrays"),
    (dict(groups_n=(6, -1), P=5), -1, "negative size"),
    (dict(groups_n=(1,) * 25, P=25), -4, "num_groups"),
])
def test_forward_scene_refuses_bad_arguments_before_any_device_work(kwargs, code, msg):
    rc, err = _fake_call(**kwargs)
    assert rc == code and msg in err, (rc, err)


def test_backward_scene_refuses_missing_gradient_destinations():
    lib = _lib.load()
    prm = (_lib.Params * 1)(_lib.Params(4, 1, 0, 32, 32, 0.5, 0.5, 1.0, 0, 0, 0x10000, 0x20000, 0x30000, 0x40000))
    groups = (_lib.Group * 1)(_lib.Group(0x100000, 0x100000, 0x100000, 0x100000, 0x100000, None, 4))
    grads = (_lib.GroupGrad * 1)(_lib.GroupGrad(0x200000, 0x200000, None, 0x200000, 0x200000, None))
    c = (C.c_float * 1)(0.0)
    rc = lib.b200gsr_backward_scene(1, prm, 1, groups, grads, c, c, 0, None, None, None, None, None, None, 0, 1 << 20,
                                    None, 0, None)
    assert rc == -1 and "group 0: null gradient pointer" in _lib.last_error()
    grads[0].scaling = 0x200000
    rc = lib.b200gsr_backward_scene(1, prm, 1, groups, grads, c, c, 0, None, None, None, None, None, None, 0, 1 << 20,
                                    None, 8, None)
    assert rc == -1 and "unknown flags" in _lib.last_error()


def _groups(sizes, M, device="cpu"):
    return [{"_xyz": torch.zeros(n, 3, device=device), "_opacity": torch.zeros(n, 1, device=device),
             "_scaling": torch.zeros(n, 3, device=device), "_rotation": torch.zeros(n, 4, device=device),
             "_features_dc": torch.zeros(n, 1, 3, device=device), "_features_rest": torch.zeros(n, M - 1, 3, device=device)}
            for n in sizes]


def _settings(B, H=32, W=32, score=False):
    from dreamscene_b200 import GaussianRasterizationSettings
    return [GaussianRasterizationSettings(H, W, 0.5, 0.5, torch.ones(3), 1.0, torch.eye(4), torch.eye(4), 1,
                                          torch.zeros(3), False, score) for _ in range(B)]


def test_render_scene_refusals(monkeypatch):
    g = _groups([5, 3], 4)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        S.render_scene(g, _settings(2))
    with pytest.raises(ValueError, match="same number of SH coefficients"):
        S.render_scene(_groups([5], 4) + _groups([3], 9), _settings(2))
    mixed = _settings(1) + _settings(1, H=48)
    with pytest.raises(ValueError, match="image size"):
        S.render_scene(g, mixed)
    with pytest.raises(ValueError, match="score_flag"):
        S.render_scene(g, _settings(2, score=True))
    with pytest.raises(ValueError, match="views"):
        S.render_scene(g, _settings(17))
    with pytest.raises(ValueError, match="groups"):
        S.render_scene(_groups([1] * 25, 4), _settings(1))
    with pytest.raises(ValueError, match="shs_aug"):
        S.render_scene(g, _settings(2), shs_aug=[True, False, True])
    monkeypatch.setattr(S, "_check_device", lambda flat: None)      # lets the count check run on CPU tensors
    with pytest.raises(ValueError, match="means2D"):
        S.render_scene(g, _settings(2), means2D=[torch.zeros(8, 3)])


def test_render_scene_refuses_in_backward_rank_reduction(monkeypatch):
    from dreamscene_b200 import parallel
    monkeypatch.setattr(parallel, "reduction_active", lambda: True)
    with pytest.raises(RuntimeError, match="all_reduce_gradients"):
        S.render_scene(_groups([5], 4), _settings(1))


def test_per_view_flags_are_normalised():
    import numpy as np
    assert S._view_flags(True, 3, "x") == (True, True, True)
    assert S._view_flags(False, 2, "x") == (False, False)
    assert S._view_flags(np.bool_(True), 2, "x") == (True, True)
    assert S._view_flags(torch.tensor(False), 2, "x") == (False, False)
    assert S._view_flags([1, 0, True], 3, "x") == (True, False, True)
    assert S._view_flags((False,), 1, "x") == (False,)
    with pytest.raises(ValueError, match="expected a bool or 2"):
        S._view_flags([True], 2, "x")


def test_group_table_packs_pointers_and_sizes_in_order():
    g = _groups([5, 0, 1, 130], 1) + _groups([2], 1)
    raw = [[S._get(x, n) for n in S._FIELDS] for x in g]
    arr = S._group_table(raw)
    assert [arr[k].n for k in range(len(g))] == [5, 0, 1, 130, 2]
    for k, ts in enumerate(raw):
        for name, t in zip(("xyz", "opacity", "scaling", "rotation", "f_dc", "f_rest"), ts):
            want = t.data_ptr() if t.numel() else None
            assert getattr(arr[k], name) == want, (k, name)
    assert arr[0].f_rest is None                     # M = 1: no _features_rest rows
    flat, M, P = S._scene_groups(_groups([5, 0, 7], 16))
    assert M == 16 and P == 12 and len(flat) == 18 and flat[6] is not None
