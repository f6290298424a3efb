"""CPU-only checks of the reserved-row groups (include/b200gsr_reserve.h, dreamscene_b200.reserve): the signature table
agrees with the header and binds; the AdamLive record's layout; the headroom policy; and the refusals - a live count
above the capacity, leaves / moments / statistics of mismatched capacities, the library's bad arguments (made-up
device addresses, never dereferenced) and a reserved group passed to the eager render_scene."""
import ctypes as C
import os
import re
from types import SimpleNamespace

import pytest
import torch

from dreamscene_b200 import _lib
from dreamscene_b200 import reserve as RS
from dreamscene_b200 import scene as S
from tests.test_abi_binding_cpu import _mismatches
from tests.test_scene_render_cpu import _settings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "b200gsr_reserve.h")


def _prototypes():
    src = re.sub(r"/\*.*?\*/", " ", open(HEADER).read(), flags=re.S)
    return {name: (ret, [" ".join(a.split()) for a in args.split(",")])
            for ret, name, args in re.findall(r"(\bint)\s+(b200gsr_\w+)\s*\(([^)]*)\)\s*;", src)}


def test_reserve_signature_table_matches_the_header_and_binds():
    protos = _prototypes()
    assert list(protos) == list(_lib.RESERVE_SIGNATURES)
    assert _mismatches(_lib.RESERVE_SIGNATURES, protos) == []
    # the base entry points' arguments plus the device live counts before the stream
    fwd = _lib.RESERVE_SIGNATURES["b200gsr_forward_scene_dyn_live"][1]
    assert fwd == _lib.STEP_SIGNATURES["b200gsr_forward_scene_dyn"][1][:-1] + [C.c_void_p, C.c_void_p]
    bwd = _lib.RESERVE_SIGNATURES["b200gsr_backward_scene_dyn_live"][1]
    assert bwd == _lib.STATS_SIGNATURES["b200gsr_backward_scene_dyn_stats"][1][:-1] + [C.c_void_p, C.c_void_p]
    adam = _lib.RESERVE_SIGNATURES["b200gsr_adam_step_dyn_live"][1]
    assert adam[:3] == _lib.STEP_SIGNATURES["b200gsr_adam_step_dyn"][1][:3] and adam[3] is C.POINTER(_lib.AdamLive)
    lib = _lib.load()
    for name, (restype, argtypes) in _lib.RESERVE_SIGNATURES.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and tuple(fn.argtypes) == tuple(argtypes), name
    others = (set(_lib.SIGNATURES) | set(_lib.SCENE_SIGNATURES) | set(_lib.STEP_SIGNATURES) |
              set(_lib.LOSS_SIGNATURES) | set(_lib.FROZEN_SIGNATURES) | set(_lib.STATS_SIGNATURES))
    assert not set(_lib.RESERVE_SIGNATURES) & others
    assert lib.b200gsr_version() == _lib.ABI_VERSION == 3


def test_adam_live_layout():
    assert C.sizeof(_lib.AdamLive) == 16
    assert (_lib.AdamLive.rows.offset, _lib.AdamLive.row_floats.offset, _lib.AdamLive.reserved.offset) == (0, 8, 12)


def test_library_refuses_bad_live_arguments():
    lib = _lib.load()
    groups = (_lib.Group * 2)(_lib.Group(*([0x100000] * 6), 6), _lib.Group(*([0x100000] * 6), 4))
    # scale loss: no live array, no group, a bad accumulate
    assert lib.b200gsr_scale_loss_live(2, 2, groups, None, C.c_void_p(0x1000), C.c_void_p(0x2000), None,
                                       C.c_void_p(0x3000), 0, None, 0, None) == _lib.ERR_BAD_ARG
    assert lib.b200gsr_scale_loss_live(2, 0, groups, C.c_void_p(0x10), C.c_void_p(0x1000), C.c_void_p(0x2000), None,
                                       C.c_void_p(0x3000), 0, None, 0, None) == _lib.ERR_BAD_ARG
    assert lib.b200gsr_scale_loss_live(2, 2, groups, C.c_void_p(0x10), C.c_void_p(0x1000), C.c_void_p(0x2000), None,
                                       C.c_void_p(0x3000), 2, None, 0, None) == _lib.ERR_BAD_ARG
    # Adam: a live record whose row size does not divide the tensor
    t = (_lib.AdamTensor * 1)(_lib.AdamTensor(0x1000, 0x2000, 0x3000, 0x4000, 10))
    live = (_lib.AdamLive * 1)(_lib.AdamLive(0x10, 3, 0))
    assert lib.b200gsr_adam_step_dyn_live(1, t, C.c_void_p(0x5000), live, None) == _lib.ERR_BAD_ARG
    assert "row_floats" in _lib.last_error()
    assert lib.b200gsr_adam_step_dyn_live(1, t, C.c_void_p(0x5000), None, None) == _lib.ERR_BAD_ARG
    # the scene entry points: a null live array
    prm = (_lib.Params * 1)(_lib.Params(10, 4, 1, 64, 64, 0.5, 0.5, 1.0, 0, 0, 0x10000, 0x20000, 0x30000, 0x40000))
    rc = lib.b200gsr_forward_scene_dyn_live(1, prm, 2, groups, C.c_void_p(0x50000), C.c_void_p(0x60000), None,
                                            C.c_void_p(0x1), C.c_void_p(0x1), C.c_void_p(0x1), C.c_void_p(0x1), 0,
                                            C.c_void_p(0x1), 0, 1024, 0, None, 0, None, None)
    assert rc == _lib.ERR_BAD_ARG and "live" in _lib.last_error()


def test_headroom_policy():
    assert RS.capacity_for(1000) == 2000                 # DEFAULT_HEADROOM = 1: room to double
    assert RS.capacity_for(1000, 0.5) == 1500
    assert RS.capacity_for(0) == 1 and RS.capacity_for(10, 0.0) == 11
    with pytest.raises(ValueError, match="headroom"):
        RS.capacity_for(10, -0.1)


def _tensors(n, M=4):
    return (torch.randn(n, 3), torch.randn(n, 1, 3), torch.randn(n, M - 1, 3), torch.randn(n, 1), torch.randn(n, 3),
            torch.randn(n, 4))


def test_from_tensors_holds_the_rows_at_capacity_and_rows_are_prefix_views():
    xyz, dc, rest, op, sc, rot = _tensors(10)
    g = RS.ReservedGroup.from_tensors(xyz, dc, rest, op, sc, rot)
    assert g.capacity == 20 and g.live_count == 10 and g.live.dtype == torch.int32 and int(g.live) == 10
    assert g._features_rest.shape == (20, 3, 3) and g.xyz_gradient_accum.shape == (20, 1)
    r = g.rows()
    assert torch.equal(r._xyz, xyz) and r._xyz.data_ptr() == g._xyz.data_ptr() and r.denom.shape == (10, 1)
    assert not g._xyz[10:].any()


def test_growth_moves_the_rows_and_the_optimizer_state():
    xyz, dc, rest, op, sc, rot = _tensors(6)
    g = RS.ReservedGroup.from_tensors(xyz, dc, rest, op, sc, rot, capacity=8)
    opt = torch.optim.Adam(g.param_groups({"xyz": 0.1, "opacity": 0.1}), lr=0.0)
    old = g._xyz
    opt.state[old] = {"step": torch.tensor(3.0), "exp_avg": torch.ones(8, 3), "exp_avg_sq": torch.full((8, 3), 2.0)}
    g._grow(9, opt)
    assert g.capacity == 18 and g._xyz is not old and opt.param_groups[0]["params"] == [g._xyz]
    st = opt.state[g._xyz]
    assert old not in opt.state and float(st["step"]) == 3.0 and st["exp_avg"].shape == (18, 3)
    assert torch.equal(st["exp_avg"][:6], torch.ones(6, 3)) and not st["exp_avg"][6:].any()
    assert torch.equal(g._xyz[:6], xyz) and g.live_count == 6


def test_refusals():
    xyz, dc, rest, op, sc, rot = _tensors(6)
    with pytest.raises(ValueError, match="capacity 4 is below"):
        RS.ReservedGroup.from_tensors(xyz, dc, rest, op, sc, rot, capacity=4)
    g = RS.ReservedGroup.from_tensors(xyz, dc, rest, op, sc, rot, capacity=8)
    leaves = {k: getattr(g, k) for k in S._FIELDS}
    with pytest.raises(ValueError, match="live count 9 not in 0..8"):
        RS.ReservedGroup(leaves, {k: getattr(g, k) for k in RS._STATS}, 9)
    bad = dict(leaves, _opacity=torch.zeros(7, 1))
    with pytest.raises(ValueError, match="_opacity has 7 rows"):
        RS.ReservedGroup(bad, {k: getattr(g, k) for k in RS._STATS}, 6)
    with pytest.raises(ValueError, match="denom has 6 elements"):
        RS.ReservedGroup(leaves, dict({k: getattr(g, k) for k in RS._STATS}, denom=torch.zeros(6, 1)), 6)
    opt = SimpleNamespace(state={g._xyz: {"exp_avg": torch.zeros(6, 3), "exp_avg_sq": torch.zeros(6, 3)}})
    with pytest.raises(ValueError, match="moments of _xyz"):
        g._moments(opt)
    with pytest.raises(ValueError, match="mask has 5 elements"):
        g.prune(torch.zeros(5, dtype=torch.bool))
    with pytest.raises(TypeError, match="rows()"):
        S.render_scene([g], _settings(1))
