"""CPU-only checks of the reconstruction-loss entry points (include/b200gsr_loss.h) and of StepGraph's target mode:
the signature table agrees with the header, the library refuses bad arguments before any launch (made-up device
addresses, never dereferenced), and StepGraph refuses a target or target indices it cannot replay before touching a
device."""
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
LOSS_HEADER = os.path.join(ROOT, "include", "b200gsr_loss.h")


def _loss_prototypes():
    src = re.sub(r"/\*.*?\*/", " ", open(LOSS_HEADER).read(), flags=re.S)
    out = {}
    for ret, name, args in re.findall(r"(\bint|\bsize_t)\s+(b200gsr_\w+)\s*\(([^)]*)\)\s*;", src):
        out[name] = (ret, [" ".join(a.split()) for a in args.split(",")])
    return out


def test_loss_signature_table_matches_the_header():
    protos = _loss_prototypes()
    assert list(protos) == list(_lib.LOSS_SIGNATURES)
    assert _mismatches(_lib.LOSS_SIGNATURES, protos) == []
    for name, (restype, argtypes) in _lib.LOSS_SIGNATURES.items():      # the check sees a single wrong entry
        for i, t in enumerate(argtypes):
            bad = argtypes[:i] + [C.c_uint64 if t is C.c_void_p else C.c_void_p] + argtypes[i + 1:]
            assert _mismatches({name: (restype, bad)}, {name: protos[name]}) != [], (name, i)


def test_library_binds_the_loss_entry_points():
    lib = _lib.load()
    for name, (restype, argtypes) in _lib.LOSS_SIGNATURES.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and tuple(fn.argtypes) == tuple(argtypes), name
    assert not set(_lib.LOSS_SIGNATURES) & (set(_lib.SIGNATURES) | set(_lib.SCENE_SIGNATURES) |
                                            set(_lib.STEP_SIGNATURES))
    assert lib.b200gsr_version() == _lib.ABI_VERSION == 3


def test_scratch_bytes_is_one_double_per_block_and_view():
    lib = _lib.load()
    assert lib.b200gsr_recon_l2_scratch_bytes(1, 1) == 8
    assert lib.b200gsr_recon_l2_scratch_bytes(1, 4096) == 8
    assert lib.b200gsr_recon_l2_scratch_bytes(3, 4097) == 48
    assert lib.b200gsr_recon_l2_scratch_bytes(2, 3 * 512 * 512) == 2 * 192 * 8
    assert lib.b200gsr_recon_l2_scratch_bytes(0, 10) == 0 and lib.b200gsr_recon_l2_scratch_bytes(1, 0) == 0


def _fake(B=2, N=1000, image=0x10000, target=0x20000, half=1, n_targets=2, index=None, grad_out=0x30000,
          loss=0x40000, d_image=0x50000, scratch=0x60000, scratch_bytes=None):
    lib = _lib.load()
    vp = lambda a: C.c_void_p(a) if a else None
    if scratch_bytes is None:
        scratch_bytes = lib.b200gsr_recon_l2_scratch_bytes(max(B, 1), max(N, 1))
    rc = lib.b200gsr_recon_l2(B, N, vp(image), vp(target), half, n_targets, vp(index), 100.0, vp(grad_out), vp(loss),
                              vp(d_image), vp(scratch), scratch_bytes, None)
    return rc, _lib.last_error()


@pytest.mark.parametrize("kwargs,code,msg", [
    (dict(B=0), -1, "must be >= 1"),
    (dict(N=0), -1, "must be >= 1"),
    (dict(n_targets=0), -1, "must be >= 1"),
    (dict(B=70000, n_targets=70000), -4, "at most 65535 views"),
    (dict(half=2), -1, "target_is_half"),
    (dict(image=0), -1, "device pointers"),
    (dict(target=0), -1, "device pointers"),
    (dict(loss=0, d_image=0), -1, "nothing to compute"),
    (dict(grad_out=0), -1, "needs grad_out"),
    (dict(B=3), -1, "B 3 > n_targets 2"),
    (dict(scratch=0), -2, "scratch"),
    (dict(scratch_bytes=8), -2, "scratch"),
    (dict(scratch=0x60004), -2, "8-byte aligned"),
])
def test_recon_l2_refuses_bad_arguments_before_any_launch(kwargs, code, msg):
    rc, err = _fake(**kwargs)
    assert rc == code and msg in err, (rc, err)


def _target_graph(monkeypatch, target, B=1):
    from dreamscene_b200 import GaussianAdam
    groups = _groups([5, 3], 4)
    for g in groups:
        for t in g.values():
            t.requires_grad_(True)
    opts = [GaussianAdam([t for t in g.values()], lr=0.0, eps=1e-15) for g in groups]
    monkeypatch.setattr(S, "_check_device", lambda flat: None)      # lets the host checks run on CPU tensors
    return G.StepGraph(groups, opts, views=B, height=32, width=32, target=target)


@pytest.mark.parametrize("target,exc,msg", [
    (torch.zeros(2, 3, 32, 32, dtype=torch.float64), TypeError, "float16 or float32"),
    (torch.zeros(2, 3, 32, 32, dtype=torch.int32), TypeError, "float16 or float32"),
    (torch.zeros(3, 32, 32, dtype=torch.float16), ValueError, r"\[G,3,32,32\]"),
    (torch.zeros(2, 3, 32, 48, dtype=torch.float16), ValueError, r"\[G,3,32,32\]"),
    (torch.zeros(2, 1, 32, 32, dtype=torch.float16), ValueError, r"\[G,3,32,32\]"),
    (torch.zeros(0, 3, 32, 32, dtype=torch.float16), ValueError, r"\[G,3,32,32\]"),
    (torch.zeros(2, 3, 32, 64, dtype=torch.float16)[..., ::2], ValueError, "contiguous"),
    (torch.zeros(3, 2, 32, 32).transpose(0, 1), ValueError, "contiguous"),
])
def test_step_graph_refuses_a_bad_target(monkeypatch, target, exc, msg):
    with pytest.raises(exc, match=msg):
        _target_graph(monkeypatch, target)


def test_step_graph_refuses_bad_target_indices_and_a_cpu_target(monkeypatch):
    sg = _target_graph(monkeypatch, torch.zeros(3, 3, 32, 32, dtype=torch.float16), B=2)
    S2 = _settings(2)
    with pytest.raises(ValueError, match="needs render"):
        sg.render(S2)
    with pytest.raises(ValueError, match="expected 2 target indices"):
        sg.render(S2, target_index=[0])
    with pytest.raises(ValueError, match="expected 2 target indices"):
        sg.render(S2, target_index=[0, 1, 2])
    with pytest.raises(ValueError, match=r"in 0..2"):
        sg.render(S2, target_index=[0, 3])
    with pytest.raises(ValueError, match=r"in 0..2"):
        sg.render(S2, target_index=[-1, 0])
    with pytest.raises(ValueError, match="CUDA tensor"):       # every index fine: the device check comes last
        sg.render(S2, target_index=[2, 0])
    sg.target = torch.zeros(3, 3, 32, 64, dtype=torch.float16)[..., ::2]      # a reassigned target is checked too
    with pytest.raises(ValueError, match="contiguous"):
        sg.render(S2, target_index=[2, 0])
    sg.target = None
    with pytest.raises(ValueError, match="needs a StepGraph built with target"):
        sg.render(S2, target_index=[0, 1])


def test_step_graph_without_target_refuses_target_index(monkeypatch):
    from dreamscene_b200 import GaussianAdam
    groups = _groups([5], 4)
    opts = [GaussianAdam([t.requires_grad_(True) for t in groups[0].values()])]
    monkeypatch.setattr(S, "_check_device", lambda flat: None)
    sg = G.StepGraph(groups, opts, views=1, height=32, width=32)
    with pytest.raises(ValueError, match="target_index needs"):
        sg.render(_settings(1), target_index=[0])
    with pytest.raises(RuntimeError, match="render"):
        sg.step(optimize=False)


def test_recon_l2_loss_refuses_what_it_cannot_take():
    from dreamscene_b200.losses import recon_l2_loss
    img = torch.zeros(3, 4, 4)
    with pytest.raises(TypeError, match="image must be float32"):
        recon_l2_loss(img.half(), img.half())
    with pytest.raises(TypeError, match="float16 or float32"):
        recon_l2_loss(img, img.double())
    with pytest.raises(ValueError, match="differ in shape"):
        recon_l2_loss(img, torch.zeros(3, 4, 5, dtype=torch.float16))
    with pytest.raises(RuntimeError, match="no CPU"):
        recon_l2_loss(img, img.half())
