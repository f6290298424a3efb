"""CPU-only checks of the densification statistics on the two-step scene route (include/b200gsr_views_stats.h,
multiview.rasterize_views(densify_stats=), scene.stats_rows): the signature table and the record agree with the
header, the library refuses bad records and views before any device work (made-up device addresses, never
dereferenced), the older entry points still insist on d_means2D, and the Python side refuses what the library would
refuse, naming the argument, before touching a device."""
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
HEADER = os.path.join(ROOT, "include", "b200gsr_views_stats.h")


def _prototypes():
    src = re.sub(r"/\*.*?\*/", " ", open(HEADER).read(), flags=re.S)
    return {name: (ret, [" ".join(a.split()) for a in args.split(",")])
            for ret, name, args in re.findall(r"(\bint)\s+(b200gsr_\w+)\s*\(([^)]*)\)\s*;", src)}


def test_views_stats_signature_table_matches_the_header_and_binds():
    protos = _prototypes()
    assert list(protos) == list(_lib.VIEWS_STATS_SIGNATURES) == ["b200gsr_backward_views_stats"]
    assert _mismatches(_lib.VIEWS_STATS_SIGNATURES, protos) == []
    for name, (restype, argtypes) in _lib.VIEWS_STATS_SIGNATURES.items():      # the check sees a single wrong entry
        for i, t in enumerate(argtypes):
            if t is C.c_void_p:
                bad = argtypes[:i] + [C.c_uint64] + argtypes[i + 1:]
                assert _mismatches({name: (restype, bad)}, {name: protos[name]}) != [], (name, i)
    # b200gsr_backward_views_frozen's arguments up to num_frozen, then the records, their count and the view
    args = _lib.VIEWS_STATS_SIGNATURES["b200gsr_backward_views_stats"][1]
    assert args == _lib.VIEWS_FROZEN_SIGNATURES["b200gsr_backward_views_frozen"][1][:-1] + [
        C.POINTER(_lib.RowStats), C.c_int32, C.c_int32, C.c_void_p]
    lib = _lib.load()
    fn = lib.b200gsr_backward_views_stats
    assert fn.restype is C.c_int and tuple(fn.argtypes) == tuple(args)
    others = (set(_lib.SIGNATURES) | set(_lib.SCENE_SIGNATURES) | set(_lib.STEP_SIGNATURES) |
              set(_lib.LOSS_SIGNATURES) | set(_lib.FROZEN_SIGNATURES) | set(_lib.STATS_SIGNATURES) |
              set(_lib.RESERVE_SIGNATURES) | set(_lib.FRAMES_SIGNATURES) | set(_lib.VIEWS_FROZEN_SIGNATURES))
    assert not set(_lib.VIEWS_STATS_SIGNATURES) & others
    assert lib.b200gsr_version() == _lib.ABI_VERSION == 3


def test_row_stats_layout_matches_the_header(tmp_path):
    """The ctypes RowStats against sizeof / offsetof of b200gsr_row_stats, printed by a host program built from the
    header."""
    fields = ("lo", "len", "xyz_gradient_accum", "denom", "max_radii2D")
    assert C.sizeof(_lib.RowStats) == 32
    assert tuple(getattr(_lib.RowStats, f).offset for f in fields) == (0, 4, 8, 16, 24)
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    src = tmp_path / "layout.cu"
    offs = ", ".join(f"offsetof(b200gsr_row_stats, {f})" for f in fields)
    src.write_text('#include <cstddef>\n#include <cstdio>\n#include "b200gsr_views_stats.h"\n'
                   'int main() { std::printf("%zu %zu %zu %zu %zu %zu %d\\n", sizeof(b200gsr_row_stats), ' + offs +
                   ', B200GSR_MAX_GROUPS); }\n')
    exe = str(tmp_path / "layout")
    subprocess.run([nvcc, "-std=c++17", "-Wno-deprecated-gpu-targets", "-I", os.path.join(ROOT, "include"), "-o", exe,
                    str(src)], check=True, timeout=300)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0, out.stderr
    vals = [int(x) for x in out.stdout.split()]
    assert vals[0] == C.sizeof(_lib.RowStats)
    assert tuple(vals[1:6]) == tuple(getattr(_lib.RowStats, f).offset for f in fields)
    assert vals[6] == _lib.MAX_GROUPS


FAKE = 256
ACC, DEN, MAXR = 0x10000, 0x20000, 0x30000


def _views(P, B, means2D=True):
    prm = (_lib.Params * B)(*[_lib.Params(P, 4, 1, 64, 64, 0.3, 0.3, 1.0, 0, 0, FAKE + 12 * v, FAKE, FAKE, FAKE)
                              for v in range(B)])
    vin = (_lib.ViewInputs * B)(*[_lib.ViewInputs(FAKE, FAKE, None, FAKE, FAKE, FAKE, None) for _ in range(B)])
    out = (_lib.ViewGrads * B)(*[_lib.ViewGrads(FAKE, FAKE if means2D else None, FAKE, None, FAKE, FAKE, FAKE, None, 0)
                                 for _ in range(B)])
    return prm, vin, out


def _backward_stats(records, view=1, frozen=(), P=40, B=2, means2D=False, count=None):
    """b200gsr_backward_views_stats over made-up addresses, with saved = NULL: a call whose records, ranges and view
    pass validation stops at the null saved-state check, before any device work.  records: (lo, len, accum, denom,
    max_radii2D) tuples, or None for a NULL array."""
    lib = _lib.load()
    prm, vin, out = _views(P, B, means2D)
    rr = (_lib.RowRange * max(len(frozen), 1))(*[_lib.RowRange(lo, n) for lo, n in frozen])
    if records is None:
        rec, n = None, 3 if count is None else count
    else:
        rec = (_lib.RowStats * max(len(records), 1))(*[_lib.RowStats(*r) for r in records])
        n = len(records) if count is None else count
    rc = lib.b200gsr_backward_views_stats(B, prm, vin, FAKE, FAKE, FAKE, FAKE, None, 1 << 40, 1 << 20, out, 0, rr,
                                          len(frozen), rec, n, view, None)
    return rc, _lib.last_error()


NULL_SAVED = "null saved-state/gradient pointer"


@pytest.mark.parametrize("kw,msg", [
    (dict(records=[], view=-2), "stats_view -2 is outside [-1, B = 2)"),
    (dict(records=[], view=2), "stats_view 2 is outside [-1, B = 2)"),
    (dict(records=[], count=-1), "num_stats -1 is outside [0, 24]"),
    (dict(records=[(k, 1, ACC, DEN, None) for k in range(25)]), "num_stats 25 is outside [0, 24]"),
    (dict(records=None), "stats is null with num_stats 3"),
    (dict(records=[(3, 0, ACC, DEN, None)]), "stats record 0 is empty (len 0)"),
    (dict(records=[(0, 3, ACC, DEN, None), (5, -2, ACC, DEN, None)]), "stats record 1 is empty (len -2)"),
    (dict(records=[(-1, 3, ACC, DEN, None)]), "stats record 0 [-1, 2) is outside [0, P = 40)"),
    (dict(records=[(30, 11, ACC, DEN, None)]), "stats record 0 [30, 41) is outside [0, P = 40)"),
    (dict(records=[(10, 5, ACC, DEN, None), (2, 3, ACC, DEN, None)]), "stats record 1 starts at 2, before the end 15"),
    (dict(records=[(0, 6, ACC, DEN, None), (5, 3, ACC, DEN, None)]), "stats record 1 starts at 5, before the end 6"),
    (dict(records=[(0, 4, ACC, None, None)]), "stats record 0: xyz_gradient_accum and denom must both be set"),
    (dict(records=[(0, 4, None, DEN, MAXR)]), "stats record 0: xyz_gradient_accum and denom must both be set"),
    (dict(records=[(0, 4, None, None, MAXR)]), "stats record 0: max_radii2D without xyz_gradient_accum and denom"),
    (dict(records=[(0, 10, ACC, DEN, None)], frozen=[(9, 3)]), "stats record 0 [0, 10) overlaps the frozen rows [9, 12)"),
    (dict(records=[(20, 5, ACC, DEN, None)], frozen=[(0, 5), (5, 16)]),
     "stats record 0 [20, 25) overlaps the frozen rows [0, 21)"),
    (dict(records=[(0, 5, ACC, DEN, None), (30, 10, None, None, None)], frozen=[(35, 1)]), "stats record 1 [30, 40) "
     "overlaps the frozen rows [35, 36)"),
    (dict(records=[], frozen=[(3, 0)]), "frozen range 0 is empty"),
])
def test_backward_views_stats_refusals_before_any_device_work(kw, msg):
    rc, err = _backward_stats(**kw)
    assert rc == _lib.ERR_BAD_ARG and msg in err, (rc, err)


def test_backward_views_stats_accepts_what_the_header_allows():
    ok = [dict(records=[], view=-1), dict(records=[], view=0), dict(records=None, count=0),
          dict(records=[(0, 40, ACC, DEN, MAXR)]),
          dict(records=[(k, 1, ACC + k, DEN + k, None) for k in range(24)], view=0),
          dict(records=[(0, 5, ACC, DEN, None), (5, 5, None, None, None), (10, 30, ACC, DEN, MAXR)]),
          dict(records=[(0, 9, ACC, DEN, None), (12, 28, ACC, DEN, None)], frozen=[(9, 3)]),       # touching
          dict(records=[(0, 10, ACC, DEN, None)], means2D=True)]
    for kw in ok:
        rc, err = _backward_stats(**kw)
        assert rc == _lib.ERR_BAD_ARG and NULL_SAVED in err, (kw, err)


def test_older_entry_points_still_need_d_means2D():
    """A NULL d_means2D is allowed by b200gsr_backward_views_stats only: the other multi-view backwards refuse it
    before any device work (their saved state is a made-up address, so the refusal has to come first)."""
    lib = _lib.load()
    P, B = 40, 2
    prm, vin, out = _views(P, B, means2D=False)
    rc = lib.b200gsr_backward_views_ex(B, prm, vin, FAKE, FAKE, FAKE, FAKE, FAKE, 1 << 40, 1 << 20, out, 0, None)
    assert rc == _lib.ERR_BAD_ARG and "view 0: null gradient output pointer" in _lib.last_error()
    rc = lib.b200gsr_backward_views(B, prm, vin, FAKE, FAKE, FAKE, FAKE, FAKE, 1 << 40, 1 << 20, out, None)
    assert rc == _lib.ERR_BAD_ARG and "view 0: null gradient output pointer" in _lib.last_error()
    rr = (_lib.RowRange * 1)(_lib.RowRange(0, 4))
    for n in (0, 1):
        rc = lib.b200gsr_backward_views_frozen(B, prm, vin, FAKE, FAKE, FAKE, FAKE, FAKE, 1 << 40, 1 << 20, out, 0, rr,
                                               n, None)
        assert rc == _lib.ERR_BAD_ARG and "view 0: null gradient output pointer" in _lib.last_error()
    # only d_means2D is optional in the statistics backward: a missing d_means3D is still refused
    out[1].d_means3D = None
    rc = lib.b200gsr_backward_views_stats(B, prm, vin, FAKE, FAKE, FAKE, FAKE, FAKE, 1 << 40, 1 << 20, out, 0, None, 0,
                                          None, 0, -1, None)
    assert rc == _lib.ERR_BAD_ARG and "view 1: null gradient output pointer" in _lib.last_error()


def _stats(n, with_max=True, device="cpu"):
    return (torch.zeros(n, 1, device=device), torch.zeros(n, 1, device=device),
            torch.zeros(n, device=device) if with_max else None)


def test_stats_rows_of_groups():
    g = _groups([5, 0, 3, 4, 0, 2], 4)
    st = [_stats(int(x["_xyz"].shape[0]), with_max=k != 3) for k, x in enumerate(g)]
    assert S.stats_rows(g, None) == []
    assert S.stats_rows(g, [None] * 6) == []
    rows = S.stats_rows(g, st)
    assert [(lo, hi) for lo, hi, *_ in rows] == [(0, 5), (5, 8), (8, 12), (12, 14)]         # empty groups take no rows
    assert [r[2:] for r in rows] == [tuple(st[k]) for k in (0, 2, 3, 5)]
    assert rows[2][4] is None
    # trained groups beside frozen ones (as a scene stage has them): the records sit between the frozen ranges
    frozen = [True, False, False, True, False, False]
    part = [None if f else s for f, s in zip(frozen, st)]
    rows = S.stats_rows(g, part)
    assert [(lo, hi) for lo, hi, *_ in rows] == [(5, 8), (12, 14)]
    assert S.frozen_rows(g, frozen) == [(0, 5), (8, 12)]
    assert MV._stats_records(rows, 14, torch.device("cpu"), MV._frozen_ranges(S.frozen_rows(g, frozen), 14)) == \
        tuple((lo, hi - lo) + tuple(r) for lo, hi, *r in rows)
    with pytest.raises(ValueError, match=r"stats_rows: densify_stats must hold one entry per group \(6\)"):
        S.stats_rows(g, st[:2])
    with pytest.raises(ValueError, match=r"stats_rows: densify_stats\[2\] denom has 4 elements, group 2 has 3 rows"):
        S.stats_rows(g, [None, None, (torch.zeros(3), torch.zeros(4), None), None, None, None])
    with pytest.raises(ValueError, match=r"stats_rows: densify_stats\[0\] must be \(xyz_gradient_accum, denom"):
        S.stats_rows(g, [(torch.zeros(5), None, None)] + [None] * 5)


def _leaves(P):
    return dict(means3D=torch.zeros(P, 3), opacities=torch.zeros(P, 1), shs=torch.zeros(P, 4, 3),
                scales=torch.zeros(P, 3), rotations=torch.zeros(P, 4))


@pytest.mark.parametrize("stats,kw,msg", [
    ([(0, 12) + _stats(12)], dict(stats_view=2), r"stats_view must be -1 \(the last view\) or in 0..1, got 2"),
    ([(0, 12) + _stats(12)], dict(stats_view=-2), r"stats_view must be -1 \(the last view\) or in 0..1, got -2"),
    ([(0, 6) + _stats(6)], dict(frozen_rows=[(5, 8)]), r"densify_stats\[0\] = \(0, 6\) overlaps the frozen rows \(5, 8\)"),
    ([(0, 4) + _stats(4), (9, 12) + _stats(3)], dict(frozen_rows=[(2, 3), (3, 10)]),
     r"densify_stats\[0\] = \(0, 4\) overlaps the frozen rows \(2, 10\)"),
    ([(4, 4) + _stats(0)], {}, r"densify_stats\[0\] = \(4, 4\) is empty"),
    ([(10, 13) + _stats(3)], {}, r"densify_stats\[0\] = \(10, 13\) is outside \[0, P = 12\)"),
    ([(5, 8) + _stats(3), (0, 2) + _stats(2)], {}, r"densify_stats\[1\] = \(0, 2\) starts before the end 8"),
    ([(0, 3) + _stats(3)] * 25, {}, r"densify_stats: 25 records, at most 24"),
    ([(0, 3, torch.zeros(3), None, None)], {}, r"densify_stats\[0\] must be \(lo, hi, xyz_gradient_accum, denom"),
    ([(0, 3) + _stats(3)[:2]], {}, r"densify_stats\[0\] must be \(lo, hi, xyz_gradient_accum, denom"),
    ([(0, 3, torch.zeros(4), torch.zeros(3), None)], {}, r"densify_stats\[0\] xyz_gradient_accum has 4 elements, "
     r"rows \(0, 3\) are 3"),
    ([(0, 3, torch.zeros(3), torch.zeros(3), torch.zeros(2))], {}, r"densify_stats\[0\] max_radii2D has 2 elements"),
    ([(0, 3, torch.zeros(3, dtype=torch.float64), torch.zeros(3), None)], {},
     r"densify_stats\[0\] xyz_gradient_accum must be a contiguous float32 tensor"),
    ([(0, 3, torch.zeros(3), torch.zeros(3, dtype=torch.int32), None)], {},
     r"densify_stats\[0\] denom must be a contiguous float32 tensor"),
    ([(0, 3, torch.zeros(3), torch.zeros(3, 2)[:, 0], None)], {}, r"densify_stats\[0\] denom must be a contiguous"),
    ([(0, 3, torch.zeros(3), torch.zeros(3), torch.zeros(3, device="meta"))], {},
     r"densify_stats\[0\] max_radii2D must be on the inputs' device \(cpu\)"),
])
def test_rasterize_views_refuses_bad_densify_stats_before_any_device_work(stats, kw, msg):
    with pytest.raises(ValueError, match=msg):
        MV.rasterize_views(_settings(2), densify_stats=stats, **kw, **_leaves(12))


def test_rasterize_views_with_good_densify_stats_gets_as_far_as_the_device_check():
    """Valid records, views and frozen neighbours pass the host checks: the call stops where every CPU call stops,
    at the refusal to run without a GPU (no port is created without means2D)."""
    for stats, kw in (([(0, 12) + _stats(12)], {}), ([], dict(stats_view=0)),
                      ([(0, 4) + _stats(4, False), (8, 12) + _stats(4)], dict(frozen_rows=[(4, 8)], stats_view=-1)),
                      ([(3, 4) + _stats(1)], dict(means2D=[torch.zeros(12, 3) for _ in range(2)]))):
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            MV.rasterize_views(_settings(2), densify_stats=stats, **kw, **_leaves(12))
