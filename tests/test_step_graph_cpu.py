"""CPU-only checks of the graph-replay entry points (include/b200gsr_step.h) and of StepGraph's refusals: the
signature table agrees with the header, the library refuses bad arguments before any launch (made-up device
addresses, never dereferenced), and StepGraph refuses what it cannot replay before touching a device."""
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
STEP_HEADER = os.path.join(ROOT, "include", "b200gsr_step.h")


def _step_prototypes():
    src = re.sub(r"/\*.*?\*/", " ", open(STEP_HEADER).read(), flags=re.S)
    out = {}
    for ret, name, args in re.findall(r"(\bint)\s+(b200gsr_\w+)\s*\(([^)]*)\)\s*;", src):
        out[name] = (ret, [" ".join(a.split()) for a in args.split(",")])
    return out


def test_step_signature_table_matches_the_header():
    protos = _step_prototypes()
    assert list(protos) == list(_lib.STEP_SIGNATURES)
    assert _mismatches(_lib.STEP_SIGNATURES, protos) == []
    for name, (restype, argtypes) in _lib.STEP_SIGNATURES.items():      # the check sees a single wrong entry
        for i, t in enumerate(argtypes):
            if t is C.c_void_p:
                bad = argtypes[:i] + [C.c_uint64] + argtypes[i + 1:]
                assert _mismatches({name: (restype, bad)}, {name: protos[name]}) != [], (name, i)


def test_library_binds_the_step_entry_points_and_the_record_is_32_bytes():
    lib = _lib.load()
    for name, (restype, argtypes) in _lib.STEP_SIGNATURES.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and tuple(fn.argtypes) == tuple(argtypes), name
    assert not set(_lib.STEP_SIGNATURES) & (set(_lib.SIGNATURES) | set(_lib.SCENE_SIGNATURES))
    assert C.sizeof(_lib.StepView) == 32 and _lib.StepView.sh_degree.offset == 16
    assert lib.b200gsr_version() == _lib.ABI_VERSION == 3


def _fake_dyn(B=2, P=10, M=4, score=0, sh_degree=3, bg_step=3, groups_n=(6, 4), views=0xA0000, seed=0xB0000,
              backward=False, grads_ok=True):
    """The _dyn entry points with made-up device addresses: validation runs before any CUDA call.  sh_degree = 3 with
    M = 4 would be refused by the by-value entry points; here the host value is ignored."""
    lib = _lib.load()
    bg = 0x10000
    prm = (_lib.Params * B)(*[_lib.Params(P, M, sh_degree, 64, 64, 0.0, 0.0, 1.0, 0, score, bg + 4 * bg_step * v,
                                          0x20000, 0x30000, 0x40000) for v in range(B)])
    groups = (_lib.Group * len(groups_n))()
    for k, n in enumerate(groups_n):
        groups[k] = _lib.Group(0x100000, 0x100000, 0x100000, 0x100000, 0x100000, 0x100000, n)
    v, s = (C.c_void_p(views) if views else None), (C.c_void_p(seed) if seed else None)
    if backward:
        grads = (_lib.GroupGrad * len(groups_n))()
        for k in range(len(groups_n)):
            grads[k] = _lib.GroupGrad(*([0x200000] * 6 if grads_ok or k else [0x200000, None] + [0x200000] * 4))
        rc = lib.b200gsr_backward_scene_dyn(B, prm, len(groups_n), groups, grads, v, s, None, None, None, None, None,
                                            None, 0, 1 << 20, None, 0, None)
    else:
        rc = lib.b200gsr_forward_scene_dyn(B, prm, len(groups_n), groups, v, s, None, None, C.c_void_p(0x60000),
                                           C.c_void_p(0x70000), C.c_void_p(0x80000), 1 << 20, C.c_void_p(0x90000),
                                           1 << 20, 1 << 20, 0, None, 0, None)
    return rc, _lib.last_error()


@pytest.mark.parametrize("kwargs,code,msg", [
    (dict(views=0), -1, "device pointers to B step records"),
    (dict(seed=0), -1, "device pointers to B step records"),
    (dict(B=0), -4, "number of views"),
    (dict(B=17), -4, "number of views"),
    (dict(score=1), -4, "score_flag"),
    (dict(P=11), -1, "groups hold 10 rows"),
    (dict(bg_step=4), -1, "contiguous"),
    (dict(groups_n=(1,) * 25, P=25), -4, "num_groups"),
    (dict(), -1, "null output/workspace pointer"),          # every argument fine up to the missing out_color
])
def test_forward_scene_dyn_refuses_bad_arguments_before_any_launch(kwargs, code, msg):
    rc, err = _fake_dyn(**kwargs)
    assert rc == code and msg in err, (rc, err)


def test_backward_scene_dyn_refusals():
    rc, err = _fake_dyn(backward=True, views=0)
    assert rc == -1 and "step records" in err
    rc, err = _fake_dyn(backward=True, grads_ok=False)
    assert rc == -1 and "group 0: null gradient pointer" in err
    rc, err = _fake_dyn(backward=True)
    assert rc == -1 and "null saved-state/gradient pointer" in err


def test_adam_step_dyn_and_pair_report_refusals():
    lib = _lib.load()
    t = (_lib.AdamTensor * 1)(_lib.AdamTensor(0x1000, 0x2000, 0x3000, 0x4000, 8))
    assert lib.b200gsr_adam_step_dyn(1, t, None, None) == -1 and "scalars" in _lib.last_error()
    assert lib.b200gsr_adam_step_dyn(33, t, C.c_void_p(0x5000), None) == -4 and "at most 32" in _lib.last_error()
    t[0].grad = None
    assert lib.b200gsr_adam_step_dyn(1, t, C.c_void_p(0x5000), None) == -1 and "null pointer" in _lib.last_error()
    assert lib.b200gsr_adam_step_dyn(0, None, None, None) == 0           # nothing to do, nothing launched
    assert lib.b200gsr_pair_report(None, C.c_void_p(0x1000), None) == -1 and "pair_report" in _lib.last_error()
    assert lib.b200gsr_pair_report(C.c_void_p(0x1000), None, None) == -1


def _graph(monkeypatch, groups=None, B=2):
    from dreamscene_b200 import GaussianAdam
    groups = groups or _groups([5, 3], 4)
    for g in groups:
        for t in g.values():
            t.requires_grad_(True)
    opts = [GaussianAdam([t for t in g.values()], lr=0.0, eps=1e-15) for g in groups]
    monkeypatch.setattr(S, "_check_device", lambda flat: None)      # lets the host checks run on CPU tensors
    return G.StepGraph(groups, opts, views=B, height=32, width=32)


def test_step_graph_refusals(monkeypatch):
    groups = _groups([5, 3], 4)
    with pytest.raises(TypeError, match="GaussianAdam"):
        G.StepGraph(groups, [torch.optim.Adam([torch.zeros(1, requires_grad=True)])], views=1, height=8, width=8)
    with pytest.raises(ValueError, match="views"):
        G.StepGraph(groups, [], views=17, height=8, width=8)
    sg = _graph(monkeypatch)
    with pytest.raises(ValueError, match="score_flag"):
        sg.render(_settings(2, score=True))
    with pytest.raises(ValueError, match="built for 2 views of 32x32"):
        sg.render(_settings(2, H=48))
    with pytest.raises(ValueError, match="built for 2 views"):
        sg.render(_settings(3))
    deg3 = [s._replace(sh_degree=3) for s in _settings(2)]          # M = 4 allows degree 1 at most
    with pytest.raises(ValueError, match="sh_degree 3"):
        sg.render(deg3)
    flat_fov = [s._replace(tanfovx=0.0) for s in _settings(2)]
    with pytest.raises(ValueError, match="tanfovx"):
        sg.render(flat_fov)
    with pytest.raises(ValueError, match="shs_aug"):
        sg.render(_settings(2), shs_aug=[True])
    with pytest.raises(ValueError, match="focal"):
        sg.render(_settings(2), focal=[1.0])
    with pytest.raises(RuntimeError, match="render"):
        sg.step()


def test_step_graph_refuses_view_sharding_and_cpu_tensors(monkeypatch):
    from dreamscene_b200 import GaussianAdam, parallel
    g = _groups([5], 4)
    sg = G.StepGraph(g, [GaussianAdam([t.requires_grad_(True) for t in g[0].values()])], views=2, height=32, width=32)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        sg.render(_settings(2))
    monkeypatch.setattr(parallel, "reduction_active", lambda: True)
    with pytest.raises(RuntimeError, match="view sharding"):
        sg.render(_settings(2))


def test_step_graph_is_exported():
    import dreamscene_b200
    assert dreamscene_b200.StepGraph is G.StepGraph and "StepGraph" in dreamscene_b200.__all__
