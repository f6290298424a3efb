"""CPU-only checks of the backwards that gather the densification statistics (include/b200gsr_stats.h) and of the
`densify_stats` arguments of render_scene and StepGraph: the signature table agrees with the header, overlaps no
other table and binds; the library refuses a bad view, half a statistics record and statistics on a frozen group
before any device work (made-up device addresses, never dereferenced); the Python side refuses bad statistics
tensors before touching a device."""
import ctypes as C
import os
import re

import pytest
import torch

from dreamscene_b200 import _lib
from dreamscene_b200 import graph as G
from dreamscene_b200 import scene as S
from tests.test_abi_binding_cpu import _mismatches, _prototypes
from tests.test_frozen_cpu import _opts
from tests.test_scene_render_cpu import _groups, _settings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STATS_HEADER = os.path.join(ROOT, "include", "b200gsr_stats.h")


def _stats_prototypes():
    src = re.sub(r"/\*.*?\*/", " ", open(STATS_HEADER).read(), flags=re.S)
    out = {}
    for ret, name, args in re.findall(r"(\bint)\s+(b200gsr_\w+)\s*\(([^)]*)\)\s*;", src):
        out[name] = (ret, [" ".join(a.split()) for a in args.split(",")])
    return out


def test_stats_signature_table_matches_the_header():
    protos = _stats_prototypes()
    assert list(protos) == list(_lib.STATS_SIGNATURES) == ["b200gsr_backward_scene_stats",
                                                           "b200gsr_backward_scene_dyn_stats"]
    assert _mismatches(_lib.STATS_SIGNATURES, protos) == []
    for name, (restype, argtypes) in _lib.STATS_SIGNATURES.items():      # the check sees a single wrong entry
        for i, t in enumerate(argtypes):
            if t is C.c_void_p:
                bad = argtypes[:i] + [C.c_uint64] + argtypes[i + 1:]
                assert _mismatches({name: (restype, bad)}, {name: protos[name]}) != [], (name, i)
        # the statistics records are passed as b200gsr_group_stats
        k = protos[name][1].index("const b200gsr_group_stats* stats")
        assert argtypes[k] is C.POINTER(_lib.GroupStats)
    # the _frozen entry points' arguments up to frozen_groups, then the statistics and the view before the stream
    for name, base, view in (("b200gsr_backward_scene_stats", "b200gsr_backward_scene_frozen", C.c_int32),
                             ("b200gsr_backward_scene_dyn_stats", "b200gsr_backward_scene_dyn_frozen", C.c_void_p)):
        argtypes = _lib.STATS_SIGNATURES[name][1]
        assert argtypes == _lib.FROZEN_SIGNATURES[base][1][:-1] + [C.POINTER(_lib.GroupStats), view, C.c_void_p], name


def test_group_stats_layout():
    assert C.sizeof(_lib.GroupStats) == 24
    assert [f for f, _ in _lib.GroupStats._fields_] == ["xyz_gradient_accum", "denom", "max_radii2D"]


def test_library_binds_the_stats_entry_points_and_the_table_overlaps_no_other():
    lib = _lib.load()
    for name, (restype, argtypes) in _lib.STATS_SIGNATURES.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and tuple(fn.argtypes) == tuple(argtypes), name
    others = (set(_lib.SIGNATURES) | set(_lib.SCENE_SIGNATURES) | set(_lib.STEP_SIGNATURES) |
              set(_lib.LOSS_SIGNATURES) | set(_lib.FROZEN_SIGNATURES))
    assert not set(_lib.STATS_SIGNATURES) & others
    assert lib.b200gsr_version() == _lib.ABI_VERSION == 3
    assert list(_prototypes()) == _lib.EXPORTS          # b200gsr.h is unchanged


def _fake_backward(dyn, stats, view=-1, mask=0, groups_n=(6, 4), B=2, M=4, d_means2D=None):
    """One of the statistics backwards with made-up device addresses: validation runs before any CUDA call, and the
    saved-state pointers are null, so a call that passes validation stops at their check."""
    lib = _lib.load()
    P = sum(groups_n)
    prm = (_lib.Params * B)(*[_lib.Params(P, M, 1, 64, 64, 0.5, 0.5, 1.0, 0, 0, 0x10000 + 12 * v, 0x20000, 0x30000,
                                          0x40000) for v in range(B)])
    groups = (_lib.Group * len(groups_n))()
    grads = (_lib.GroupGrad * len(groups_n))()
    for k, n in enumerate(groups_n):
        groups[k] = _lib.Group(*([0x100000] * 6), n)
        grads[k] = _lib.GroupGrad(*([0x200000] * 6))
    arr = None
    if stats is not None:
        arr = (_lib.GroupStats * len(groups_n))()
        for k, e in enumerate(stats):
            if e is not None:
                arr[k] = _lib.GroupStats(*e)
    if dyn:
        rc = lib.b200gsr_backward_scene_dyn_stats(B, prm, len(groups_n), groups, grads, C.c_void_p(0xA0000),
                                                  C.c_void_p(0xB0000), None, None, None, None, None, None, 0,
                                                  1 << 20, d_means2D, 0, mask, arr, view, None)
    else:
        c = (C.c_float * B)(*([0.447] * B))
        rc = lib.b200gsr_backward_scene_stats(B, prm, len(groups_n), groups, grads, c, c, 1, None, None, None, None,
                                              None, None, 0, 1 << 20, d_means2D, 0, mask, arr, view, None)
    return rc, _lib.last_error()


FULL = (0x300000, 0x310000, 0x320000)
NO_MAX = (0x300000, 0x310000, None)


def test_by_value_view_refusals_before_any_device_work():
    for view in (-2, 2, 7, -(2 ** 31)):
        rc, err = _fake_backward(False, [FULL, None], view=view)
        assert rc == -1 and "stats_view" in err and "not in -1..1" in err, (view, rc, err)
    for view in (-1, 0, 1):             # valid: validation passes and stops at the (null) saved state
        rc, err = _fake_backward(False, [FULL, None], view=view)
        assert rc == -1 and "null saved-state/gradient pointer" in err, (view, rc, err)


@pytest.mark.parametrize("dyn", [False, True])
def test_stats_record_refusals_before_any_device_work(dyn):
    view = C.c_void_p(0xC0000) if dyn else 0
    # accum and denom: both or neither
    for half in ((0x300000, None, None), (None, 0x310000, None), (None, 0x310000, 0x320000)):
        rc, err = _fake_backward(dyn, [None, half], view=view)
        assert rc == -1 and "group 1: xyz_gradient_accum and denom" in err, (half, rc, err)
    rc, err = _fake_backward(dyn, [(None, None, 0x320000), None], view=view)
    assert rc == -1 and "group 0: max_radii2D without" in err, (rc, err)
    # statistics on a frozen group
    for mask, stats, g in ((0b01, [FULL, None], 0), (0b10, [None, NO_MAX], 1), (0b11, [None, FULL], 1)):
        rc, err = _fake_backward(dyn, stats, view=view, mask=mask)
        assert rc == -1 and f"group {g}: statistics on a frozen group" in err, (mask, rc, err)
    # the frozen mask's own check still comes first
    rc, err = _fake_backward(dyn, [FULL, None], view=view, mask=0b100)
    assert rc == -1 and "frozen mask" in err, (rc, err)
    # accepted: statistics on the trainable group, an empty record on the frozen one, no record at all, max_radii2D
    # left out; a null d_means2D passes as well
    for mask, stats in ((0b10, [FULL, None]), (0b01, [None, NO_MAX]), (0, None), (0b11, [None, None]), (0, [FULL, FULL])):
        rc, err = _fake_backward(dyn, stats, view=view, mask=mask)
        assert rc == -1 and "null saved-state/gradient pointer" in err, (mask, stats, rc, err)


def test_dyn_needs_a_view_pointer_only_when_a_group_gathers():
    rc, err = _fake_backward(True, [FULL, None], view=None)
    assert rc == -1 and "stats_view must be a device pointer" in err, (rc, err)
    for stats in (None, [None, None]):
        rc, err = _fake_backward(True, stats, view=None)
        assert rc == -1 and "null saved-state/gradient pointer" in err, (stats, rc, err)


def test_the_frozen_entry_points_still_need_d_means2D():
    """Only the statistics entry points accept a null d_means2D."""
    lib = _lib.load()
    B, P, M = 2, 10, 4
    prm = (_lib.Params * B)(*[_lib.Params(P, M, 1, 64, 64, 0.5, 0.5, 1.0, 0, 0, 0x10000 + 12 * v, 0x20000, 0x30000,
                                          0x40000) for v in range(B)])
    groups = (_lib.Group * 1)(_lib.Group(*([0x100000] * 6), P))
    grads = (_lib.GroupGrad * 1)(_lib.GroupGrad(*([0x200000] * 6)))
    c = (C.c_float * B)(*([0.447] * B))
    ptrs = [C.c_void_p(0x400000 + 0x10000 * k) for k in range(5)]
    rc = lib.b200gsr_backward_scene_frozen(B, prm, 1, groups, grads, c, c, 1, None, *ptrs, 1 << 20, 1 << 20, None, 0, 0,
                                           None)
    assert rc == -1 and "null saved-state/gradient pointer" in _lib.last_error()


# ---- Python ---------------------------------------------------------------------------------------------------------
def _stats_for(groups, **kw):
    out = []
    for g in groups:
        n = int(g["_xyz"].shape[0])
        out.append((torch.zeros(n, 1, **kw), torch.zeros(n, 1, **kw), torch.zeros(n, **kw)))
    return out


def test_densify_stats_validation():
    groups = _groups([5, 3], 4)
    ok = _stats_for(groups)
    assert S._densify_stats(None, groups, 0, "x") is None
    assert S._densify_stats([None, None], groups, 0, "x") is None
    st = S._densify_stats([ok[0], (ok[1][0], ok[1][1], None)], groups, 0, "x")
    assert st[0][0] is ok[0][0] and st[1][2] is None
    with pytest.raises(ValueError, match=r"one entry per group \(2\)"):
        S._densify_stats([ok[0]], groups, 0, "x")
    with pytest.raises(ValueError, match=r"densify_stats\[1\] must be \(xyz_gradient_accum"):
        S._densify_stats([None, (ok[1][0], None, None)], groups, 0, "x")
    with pytest.raises(ValueError, match=r"densify_stats\[0\] denom must be a contiguous float32"):
        S._densify_stats([(ok[0][0], ok[0][1].double(), None), None], groups, 0, "x")
    with pytest.raises(ValueError, match=r"densify_stats\[0\] xyz_gradient_accum must be a contiguous float32"):
        S._densify_stats([(torch.zeros(2, 5)[:, 0], ok[0][1], None), None], groups, 0, "x")
    with pytest.raises(ValueError, match=r"densify_stats\[1\] max_radii2D has 5 elements, group 1 has 3 rows"):
        S._densify_stats([None, (ok[1][0], ok[1][1], ok[0][2])], groups, 0, "x")
    with pytest.raises(ValueError, match=r"frozen group 1"):
        S._densify_stats([None, ok[1]], groups, 0b10, "x")
    S._densify_stats([ok[0], None], groups, 0b10, "x")        # the trained group of a frozen pair: fine
    with pytest.raises(ValueError, match="on the groups' device"):
        S._densify_stats([(ok[0][0].to("meta"), ok[0][1], None), None], groups, 0, "x")


def test_render_scene_refusals():
    groups = _groups([5, 3], 4)
    ok = _stats_for(groups)
    with pytest.raises(ValueError, match="render_scene: densify_stats.*frozen group 0"):
        S.render_scene(groups, _settings(2), densify_stats=ok, frozen=[True, False])
    for view in (2, -2):
        with pytest.raises(ValueError, match=r"render_scene: stats_view must be -1 \(the last view\) or in 0..1"):
            S.render_scene(groups, _settings(2), densify_stats=ok, stats_view=view)


def test_step_graph_stats_refusals_and_layout_key(monkeypatch):
    groups = _groups([5, 3], 4)
    opts = _opts(groups)
    ok = _stats_for(groups)
    with pytest.raises(ValueError, match=r"StepGraph: densify_stats\[1\] gathers statistics for frozen group 1"):
        G.StepGraph(groups, opts[:1], views=2, height=32, width=32, frozen=[False, True], densify_stats=ok)
    sg = G.StepGraph(groups, opts[:1], views=2, height=32, width=32, frozen=[False, True], densify_stats=[ok[0], None])
    k0 = sg._stats_key()
    assert k0 == (((ok[0][0].data_ptr(), ok[0][1].data_ptr(), ok[0][2].data_ptr()), None), True)
    # new tensors (densify) change the key: the next render() re-captures
    sg.densify_stats = [_stats_for(groups)[0], None]
    assert sg._stats_key() != k0
    sg.keep_means2D = False
    assert sg._stats_key()[1] is False
    sg.densify_stats = None
    assert sg._stats_key() == (None, False)
    # reassigned onto a frozen group: refused at render(), before any device work
    monkeypatch.setattr(S, "_check_device", lambda flat: None)
    sg.densify_stats = ok
    with pytest.raises(ValueError, match="frozen group 1"):
        sg.render(_settings(2))
    with pytest.raises(RuntimeError, match="needs a render"):
        sg.step(stats_view=0)
