"""CPU-only checks of the frozen rows on the two-step scene route (include/b200gsr_views_frozen.h,
multiview.rasterize_views(frozen_rows=), scene.assemble_scene(frozen=), scene.frozen_rows): the signature table and
the range record agree with the header, the library refuses bad ranges, masks and missing gradient destinations
before any device work (made-up device addresses, never dereferenced), and the Python side refuses what the library
would refuse, naming the argument, before touching a device."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

from dreamscene_b200 import _lib
from dreamscene_b200 import multiview as MV
from dreamscene_b200 import scene as S
from tests.test_abi_binding_cpu import _mismatches
from tests.test_scene_render_cpu import _groups, _settings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "b200gsr_views_frozen.h")


def _prototypes():
    src = re.sub(r"/\*.*?\*/", " ", open(HEADER).read(), flags=re.S)
    return {name: (ret, [" ".join(a.split()) for a in args.split(",")])
            for ret, name, args in re.findall(r"(\bint)\s+(b200gsr_\w+)\s*\(([^)]*)\)\s*;", src)}


def test_views_frozen_signature_table_matches_the_header_and_binds():
    protos = _prototypes()
    assert list(protos) == list(_lib.VIEWS_FROZEN_SIGNATURES) == ["b200gsr_backward_views_frozen",
                                                                  "b200gsr_assemble_backward_frozen"]
    assert _mismatches(_lib.VIEWS_FROZEN_SIGNATURES, protos) == []
    for name, (restype, argtypes) in _lib.VIEWS_FROZEN_SIGNATURES.items():      # the check sees a single wrong entry
        for i, t in enumerate(argtypes):
            if t is C.c_void_p:
                bad = argtypes[:i] + [C.c_uint64] + argtypes[i + 1:]
                assert _mismatches({name: (restype, bad)}, {name: protos[name]}) != [], (name, i)
    # the plain entry points' arguments, then the ranges and their count / the mask, before the stream
    views = _lib.VIEWS_FROZEN_SIGNATURES["b200gsr_backward_views_frozen"][1]
    assert views == _lib.SIGNATURES["b200gsr_backward_views_ex"][1][:-1] + [C.POINTER(_lib.RowRange), C.c_int32,
                                                                             C.c_void_p]
    asm = _lib.VIEWS_FROZEN_SIGNATURES["b200gsr_assemble_backward_frozen"][1]
    assert asm == _lib.SIGNATURES["b200gsr_assemble_backward"][1][:-1] + [C.c_uint32, C.c_void_p]
    lib = _lib.load()
    for name, (restype, argtypes) in _lib.VIEWS_FROZEN_SIGNATURES.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and tuple(fn.argtypes) == tuple(argtypes), name
    others = (set(_lib.SIGNATURES) | set(_lib.SCENE_SIGNATURES) | set(_lib.STEP_SIGNATURES) |
              set(_lib.LOSS_SIGNATURES) | set(_lib.FROZEN_SIGNATURES) | set(_lib.STATS_SIGNATURES) |
              set(_lib.RESERVE_SIGNATURES) | set(_lib.FRAMES_SIGNATURES))
    assert not set(_lib.VIEWS_FROZEN_SIGNATURES) & others
    assert lib.b200gsr_version() == _lib.ABI_VERSION == 3


def test_row_range_layout_and_limit_match_the_header(tmp_path):
    """The ctypes RowRange against sizeof / offsetof of b200gsr_row_range, and MAX_FROZEN_RANGES against the
    header's B200GSR_MAX_FROZEN_RANGES, both printed by a host program built from the header."""
    assert C.sizeof(_lib.RowRange) == 8 and (_lib.RowRange.lo.offset, _lib.RowRange.len.offset) == (0, 4)
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    src = tmp_path / "layout.cu"
    src.write_text('#include <cstddef>\n#include <cstdio>\n#include "b200gsr_views_frozen.h"\n'
                   'int main() { std::printf("%zu %zu %zu %d %d\\n", sizeof(b200gsr_row_range), '
                   'offsetof(b200gsr_row_range, lo), offsetof(b200gsr_row_range, len), B200GSR_MAX_FROZEN_RANGES, '
                   '(B200GSR_MAX_GROUPS + 1) / 2); }\n')
    exe = str(tmp_path / "layout")
    subprocess.run([nvcc, "-std=c++17", "-Wno-deprecated-gpu-targets", "-I", os.path.join(ROOT, "include"), "-o", exe,
                    str(src)], check=True, timeout=300)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0, out.stderr
    size, lo, ln, limit, groups_limit = (int(x) for x in out.stdout.split())
    assert (size, lo, ln) == (C.sizeof(_lib.RowRange), _lib.RowRange.lo.offset, _lib.RowRange.len.offset)
    assert limit == groups_limit == _lib.MAX_FROZEN_RANGES


FAKE = 256


def _backward_views(ranges, P=10, B=2, saved=None):
    """b200gsr_backward_views_frozen over made-up addresses; with saved = NULL a call whose ranges pass validation
    stops at the null saved-state check, before any device work."""
    lib = _lib.load()
    prm = (_lib.Params * B)(*[_lib.Params(P, 4, 1, 64, 64, 0.3, 0.3, 1.0, 0, 0, FAKE + 12 * v, FAKE, FAKE, FAKE)
                              for v in range(B)])
    vin = (_lib.ViewInputs * B)(*[_lib.ViewInputs(FAKE, FAKE, None, FAKE, FAKE, FAKE, None) for _ in range(B)])
    out = (_lib.ViewGrads * B)(*[_lib.ViewGrads(FAKE, FAKE, FAKE, None, FAKE, FAKE, FAKE, None, 0) for _ in range(B)])
    if ranges is None:
        arr, n = None, 3
    else:
        arr = (_lib.RowRange * max(len(ranges), 1))(*[_lib.RowRange(lo, ln) for lo, ln in ranges])
        n = len(ranges)
    rc = lib.b200gsr_backward_views_frozen(B, prm, vin, FAKE, FAKE, FAKE, FAKE, saved, 1 << 40, 1 << 20, out, 0, arr, n,
                                           None)
    return rc, _lib.last_error()


@pytest.mark.parametrize("ranges,msg", [
    ([(2, 0)], "frozen range 0 is empty"),
    ([(0, 3), (5, -1)], "frozen range 1 is empty"),
    ([(-1, 2)], "frozen range 0 [-1, 1) is outside [0, P = 10)"),
    ([(8, 3)], "frozen range 0 [8, 11) is outside [0, P = 10)"),
    ([(4, 2), (1, 1)], "frozen range 1 starts at 1, before the end 6 of range 0"),
    ([(1, 3), (3, 2)], "frozen range 1 starts at 3, before the end 4 of range 0"),
    ([(2 * k, 1) for k in range(5)] + [(10, 1)], "outside [0, P = 10)"),
])
def test_backward_views_frozen_refuses_bad_ranges(ranges, msg):
    rc, err = _backward_views(ranges)
    assert rc == _lib.ERR_BAD_ARG and msg in err, (rc, err)


def test_backward_views_frozen_range_count_and_merging():
    P = 40
    # 13 separate ranges are one too many; touching ones merge, so 26 touching ranges in 12 runs pass
    rc, err = _backward_views([(3 * k, 1) for k in range(13)], P=P)
    assert rc == _lib.ERR_BAD_ARG and "more than 12 frozen ranges" in err, err
    runs = [(3 * k, 1) for k in range(12)]
    touching = sorted(runs + [(3 * k + 1, 1) for k in range(12)])
    for ranges in (runs, touching, [(0, P)], [(k, 1) for k in range(P)]):
        rc, err = _backward_views(ranges, P=P)
        assert rc == _lib.ERR_BAD_ARG and "null saved-state/gradient pointer" in err, (ranges, err)
    # a negative count, and ranges missing for a positive count
    rc, err = _backward_views([], P=P)          # count 0: the plain backward, which stops at the null saved state
    assert rc == _lib.ERR_BAD_ARG and "null saved-state/gradient pointer" in err, err
    lib = _lib.load()
    rc, err = _backward_views(None, P=P)
    assert rc == _lib.ERR_BAD_ARG and "frozen is null with num_frozen 3" in err, err
    prm = (_lib.Params * 1)(_lib.Params(P, 4, 1, 64, 64, 0.3, 0.3, 1.0, 0, 0, FAKE, FAKE, FAKE, FAKE))
    vin = (_lib.ViewInputs * 1)(_lib.ViewInputs(FAKE, FAKE, None, FAKE, FAKE, FAKE, None))
    assert lib.b200gsr_backward_views_frozen(1, prm, vin, FAKE, FAKE, FAKE, FAKE, None, 0, 0, None, 0, None, -1,
                                             None) == _lib.ERR_BAD_ARG
    assert "num_frozen -1 is negative" in _lib.last_error()
    # the views' own checks come first, as in b200gsr_backward_views_ex
    assert lib.b200gsr_backward_views_frozen(0, prm, vin, FAKE, FAKE, FAKE, FAKE, None, 0, 0, None, 0, None, 0,
                                             None) != 0
    assert "number of views 0" in _lib.last_error()


def _assemble_backward(mask, groups_n=(6, 4), null_grad_group=None, M=4, d_in=None):
    """b200gsr_assemble_backward_frozen over made-up addresses; with the packed gradient inputs NULL a call that
    passes the group checks stops at them, before any device work."""
    lib = _lib.load()
    groups = (_lib.Group * len(groups_n))()
    grads = (_lib.GroupGrad * len(groups_n))()
    for k, n in enumerate(groups_n):
        groups[k] = _lib.Group(*([0x100000] * 6), n)
        grads[k] = _lib.GroupGrad(*([None] * 6 if k == null_grad_group else [0x200000] * 6))
    d_in = d_in or [None] * 5
    rc = lib.b200gsr_assemble_backward_frozen(len(groups_n), groups, grads, M, 2, 0.447, 0.447, None, None, 1, *d_in,
                                              mask, None)
    return rc, _lib.last_error()


def test_assemble_backward_frozen_refusals_before_any_device_work():
    for mask in (0b100, 0x80000000, 0b111):
        rc, err = _assemble_backward(mask)
        assert rc == _lib.ERR_BAD_ARG and "frozen mask" in err and "num_groups 2" in err, (mask, err)
    # a trainable group still needs every gradient pointer; a frozen one may have none
    rc, err = _assemble_backward(0b01, null_grad_group=1)
    assert rc == _lib.ERR_BAD_ARG and "group 1: null gradient pointer" in err, err
    rc, err = _assemble_backward(0, null_grad_group=0)
    assert rc == _lib.ERR_BAD_ARG and "group 0: null gradient pointer" in err, err
    for mask, null in ((0b10, 1), (0b01, 0), (0b11, 0)):
        rc, err = _assemble_backward(mask, null_grad_group=null)
        assert rc == _lib.ERR_BAD_ARG and "null gradient input" in err, (mask, err)
    rc, err = _assemble_backward(1 << 23, groups_n=(1,) * 24, null_grad_group=23)
    assert rc == _lib.ERR_BAD_ARG and "null gradient input" in err, err


def test_frozen_rows_of_groups():
    g = _groups([5, 0, 3, 4, 0, 2], 4)
    assert S.frozen_rows(g, None) == []
    assert S.frozen_rows(g, [False] * 6) == []
    assert S.frozen_rows(g, [True] * 6) == [(0, 14)]
    assert S.frozen_rows(g, [True, False, True, False, False, True]) == [(0, 8), (12, 14)]   # the empty group merges
    assert S.frozen_rows(g, [False, True, False, True, True, False]) == [(8, 12)]           # empty groups take no row
    assert S.frozen_rows(g, [True, True, False, False, True, True]) == [(0, 5), (12, 14)]
    with pytest.raises(ValueError, match=r"frozen_rows: frozen must hold one bool per group \(6\)"):
        S.frozen_rows(g, [True])
    # the ranges are what rasterize_views takes, merged as the library merges them
    assert MV._frozen_ranges(S.frozen_rows(g, [True, False, False, True, False, True]), 14) == ((0, 5), (8, 6))


def test_frozen_ranges_mirror_the_library():
    P = 20
    assert MV._frozen_ranges(None, P) == ()
    assert MV._frozen_ranges([], P) == ()
    assert MV._frozen_ranges([(0, 3), (3, 5), (7, 9), (9, 20)], P) == ((0, 5), (7, 13))
    assert MV._frozen_ranges([(k, k + 1) for k in range(P)], P) == ((0, P),)
    assert MV._frozen_ranges([(2 * k, 2 * k + 1) for k in range(10)], P) == tuple((2 * k, 1) for k in range(10))
    for bad, msg in ([[(3, 3)], r"frozen_rows\[0\] = \(3, 3\) is empty"],
                     [[(0, 2), (5, 4)], r"frozen_rows\[1\] = \(5, 4\) is empty"],
                     [[(-1, 2)], r"frozen_rows\[0\] = \(-1, 2\) is outside \[0, P = 20\)"],
                     [[(15, 21)], r"frozen_rows\[0\] = \(15, 21\) is outside"],
                     [[(5, 8), (0, 2)], r"frozen_rows\[1\] = \(0, 2\) starts before the end 8 of frozen_rows\[0\]"],
                     [[(0, 8), (7, 9)], r"frozen_rows\[1\] = \(7, 9\) starts before the end 8"],
                     [[(0, 1, 2)], r"frozen_rows\[0\]: expected a \(lo, hi\) pair"],
                     [[(k, k + 1) for k in range(0, 26, 2)][:13], "frozen_rows: 13 ranges after merging"]):
        with pytest.raises(ValueError, match=msg):
            MV._frozen_ranges(bad, 40 if "13 ranges" in msg else P)


def test_rasterize_views_refuses_bad_frozen_rows_before_any_device_work():
    P = 12
    x = torch.zeros(P, 3)
    kw = dict(means3D=x, opacities=torch.zeros(P, 1), shs=torch.zeros(P, 4, 3), scales=torch.zeros(P, 3),
              rotations=torch.zeros(P, 4))
    with pytest.raises(ValueError, match=r"frozen_rows\[0\] = \(10, 13\) is outside \[0, P = 12\)"):
        MV.rasterize_views(_settings(2), frozen_rows=[(10, 13)], **kw)
    with pytest.raises(ValueError, match=r"frozen_rows\[1\] = \(2, 4\) starts before"):
        MV.rasterize_views(_settings(2), frozen_rows=[(3, 5), (2, 4)], **kw)


def test_assemble_scene_refuses_a_frozen_list_of_the_wrong_length():
    g = _groups([5, 3], 4)
    for frozen in ([True], [True, False, False], []):
        with pytest.raises(ValueError, match=r"assemble_scene: frozen must hold one bool per group \(2\)"):
            S.assemble_scene(g, frozen=frozen)
    # the right length gets as far as the device check
    with pytest.raises(RuntimeError, match="must be CUDA tensors"):
        S.assemble_scene(g, frozen=[True, False])
