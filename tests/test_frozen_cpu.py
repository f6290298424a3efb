"""CPU-only checks of the frozen-group backwards (include/b200gsr_frozen.h) and of the `frozen` arguments of
render_scene and StepGraph: the signature table agrees with the header and overlaps no other table, the library
refuses bad masks and missing gradient destinations before any device work (made-up device addresses, never
dereferenced), and the Python side refuses what it cannot honour before touching a device."""
import ctypes as C
import os
import re

import pytest
import torch

from dreamscene_b200 import _lib
from dreamscene_b200 import graph as G
from dreamscene_b200 import scene as S
from tests.test_abi_binding_cpu import _mismatches
from tests.test_scene_render_cpu import _groups, _settings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FROZEN_HEADER = os.path.join(ROOT, "include", "b200gsr_frozen.h")


def _frozen_prototypes():
    src = re.sub(r"/\*.*?\*/", " ", open(FROZEN_HEADER).read(), flags=re.S)
    out = {}
    for ret, name, args in re.findall(r"(\bint)\s+(b200gsr_\w+)\s*\(([^)]*)\)\s*;", src):
        out[name] = (ret, [" ".join(a.split()) for a in args.split(",")])
    return out


def test_frozen_signature_table_matches_the_header():
    protos = _frozen_prototypes()
    assert list(protos) == list(_lib.FROZEN_SIGNATURES) == ["b200gsr_backward_scene_frozen",
                                                            "b200gsr_backward_scene_dyn_frozen"]
    assert _mismatches(_lib.FROZEN_SIGNATURES, protos) == []
    for name, (restype, argtypes) in _lib.FROZEN_SIGNATURES.items():      # the check sees a single wrong entry
        for i, t in enumerate(argtypes):
            if t is C.c_void_p:
                bad = argtypes[:i] + [C.c_uint64] + argtypes[i + 1:]
                assert _mismatches({name: (restype, bad)}, {name: protos[name]}) != [], (name, i)
    # the plain entry points' arguments, then the mask before the stream
    for name, base in (("b200gsr_backward_scene_frozen", _lib.SCENE_SIGNATURES["b200gsr_backward_scene"]),
                       ("b200gsr_backward_scene_dyn_frozen", _lib.STEP_SIGNATURES["b200gsr_backward_scene_dyn"])):
        argtypes = _lib.FROZEN_SIGNATURES[name][1]
        assert argtypes == base[1][:-1] + [C.c_uint32, C.c_void_p], name


def test_library_binds_the_frozen_entry_points_and_the_table_overlaps_no_other():
    lib = _lib.load()
    for name, (restype, argtypes) in _lib.FROZEN_SIGNATURES.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and tuple(fn.argtypes) == tuple(argtypes), name
    others = (set(_lib.SIGNATURES) | set(_lib.SCENE_SIGNATURES) | set(_lib.STEP_SIGNATURES) |
              set(_lib.LOSS_SIGNATURES))
    assert not set(_lib.FROZEN_SIGNATURES) & others
    assert lib.b200gsr_version() == _lib.ABI_VERSION == 3


def _fake_backward(dyn, mask, groups_n=(6, 4), null_grad_group=None, B=2, M=4):
    """One of the frozen backwards with made-up device addresses: validation runs before any CUDA call, and the
    saved-state pointers are null, so a call that passes validation stops at their check."""
    lib = _lib.load()
    P = sum(groups_n)
    prm = (_lib.Params * B)(*[_lib.Params(P, M, 1, 64, 64, 0.5, 0.5, 1.0, 0, 0, 0x10000 + 12 * v, 0x20000, 0x30000,
                                          0x40000) for v in range(B)])
    groups = (_lib.Group * len(groups_n))()
    grads = (_lib.GroupGrad * len(groups_n))()
    for k, n in enumerate(groups_n):
        groups[k] = _lib.Group(*([0x100000] * 6), n)
        grads[k] = _lib.GroupGrad(*([None] * 6 if k == null_grad_group else [0x200000] * 6))
    if dyn:
        rc = lib.b200gsr_backward_scene_dyn_frozen(B, prm, len(groups_n), groups, grads, C.c_void_p(0xA0000),
                                                   C.c_void_p(0xB0000), None, None, None, None, None, None, 0,
                                                   1 << 20, None, 0, mask, None)
    else:
        c = (C.c_float * B)(*([0.447] * B))
        rc = lib.b200gsr_backward_scene_frozen(B, prm, len(groups_n), groups, grads, c, c, 1, None, None, None, None,
                                               None, None, 0, 1 << 20, None, 0, mask, None)
    return rc, _lib.last_error()


@pytest.mark.parametrize("dyn", [False, True])
def test_frozen_backward_refusals_before_any_device_work(dyn):
    # a mask bit at or above num_groups
    for mask in (0b100, 0x80000000, 0b111):
        rc, err = _fake_backward(dyn, mask)
        assert rc == -1 and "frozen mask" in err and "num_groups 2" in err, (mask, rc, err)
    # a trainable group still needs every gradient pointer
    rc, err = _fake_backward(dyn, 0b01, null_grad_group=1)
    assert rc == -1 and "group 1: null gradient pointer" in err, (rc, err)
    rc, err = _fake_backward(dyn, 0, null_grad_group=0)
    assert rc == -1 and "group 0: null gradient pointer" in err, (rc, err)
    # a frozen group's pointers may be null: validation passes and stops at the (null) saved state
    for mask, null in ((0b10, 1), (0b01, 0), (0b11, 0)):
        rc, err = _fake_backward(dyn, mask, null_grad_group=null)
        assert rc == -1 and "null saved-state/gradient pointer" in err, (mask, rc, err)
    # 24 groups, the highest one frozen
    rc, err = _fake_backward(dyn, 1 << 23, groups_n=(1,) * 24, null_grad_group=23)
    assert rc == -1 and "null saved-state/gradient pointer" in err, (rc, err)


def test_frozen_mask_from_flags():
    assert S._frozen_mask(None, 3, "x") == 0
    assert S._frozen_mask([True, False, True], 3, "x") == 0b101
    assert S._frozen_mask((0, 1), 2, "x") == 0b10
    assert S._frozen_mask([k != "env" for k in ("env", "floor", "obj")], 3, "x") == 0b110
    with pytest.raises(ValueError, match="one bool per group"):
        S._frozen_mask([True], 2, "x")


def test_render_scene_refuses_a_frozen_list_of_the_wrong_length():
    g = _groups([5, 3], 4)
    for frozen in ([True], [True, False, False], []):
        with pytest.raises(ValueError, match=r"render_scene: frozen must hold one bool per group \(2\)"):
            S.render_scene(g, _settings(2), frozen=frozen)


def _opts(groups):
    from dreamscene_b200 import GaussianAdam
    for g in groups:
        for t in g.values():
            t.requires_grad_(True)
    return [GaussianAdam([t for t in g.values()], lr=0.0, eps=1e-15) for g in groups]


def test_step_graph_frozen_refusals(monkeypatch):
    groups = _groups([5, 3], 4)
    opts = _opts(groups)
    with pytest.raises(ValueError, match="StepGraph: frozen must hold one bool per group"):
        G.StepGraph(groups, opts, views=2, height=32, width=32, frozen=[True])
    monkeypatch.setattr(S, "_check_device", lambda flat: None)      # lets the host checks run on CPU tensors
    # an optimizer over a frozen group's leaf would never step: refused before any device work
    sg = G.StepGraph(groups, opts, views=2, height=32, width=32, frozen=[False, True])
    with pytest.raises(ValueError, match="leaf of frozen group 1"):
        sg.render(_settings(2))
    sg.frozen = [True, True, True]                                  # reassigned: checked again at render()
    with pytest.raises(ValueError, match="one bool per group"):
        sg.render(_settings(2))
    sg = G.StepGraph(groups, opts[:1], views=2, height=32, width=32, frozen=[False, True])
    assert sg._frozen_key() == 0b10
    sg._check_frozen_leaves([t for g in groups for t in g.values()], sg._frozen_key())   # env-only optimizer: fine
    sg.frozen = None
    assert sg._frozen_key() == 0
