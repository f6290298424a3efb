"""CPU-only checks of deterministic mode: the saved-buffer layout grows only at its end, the new entry points are
exported, and the fixed-point helpers round-trip, have the promised headroom and propagate NaN / Inf."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ("header", "tile_start", "work_order", "n_contrib", "keys", "geom", "dgeom", "bwd_items")


def _fields(lay):
    return {f: getattr(lay, f) for f in FIELDS + ("total",)}


@pytest.mark.parametrize("P,H,W", [(1000, 256, 256), (100_000, 512, 512), (7, 33, 17), (0, 16, 16)])
def test_deterministic_layout_appends_after_every_existing_array(P, H, W):
    from dreamscene_b200 import _lib
    cap = 1 << 20
    for with_backward in (True, False):
        base = _lib.saved_layout(P, H, W, cap, with_backward)
        det = _lib.saved_layout(P, H, W, cap, with_backward, deterministic=True)
        assert all(getattr(det, f) == getattr(base, f) for f in FIELDS)           # every offset unchanged
        extra = det.total - base.total
        assert extra >= 8 * P                                                       # fixed-point score
        if with_backward:
            assert extra >= 120 * P + 8 * P                                         # maxima + sums + score


def test_default_layout_is_unchanged():
    """The default layout, byte for byte, as the library computed it before deterministic mode existed."""
    from dreamscene_b200 import _lib
    up = lambda v: (v + 255) // 256 * 256
    P, H, W, cap = 1000, 256, 256, 1 << 20
    tiles = 16 * 16
    want, off = {}, 0
    for name, size in (("header", 64 * 4), ("tile_start", (tiles + 1) * 4), ("work_order", tiles * 4),
                       ("n_contrib", H * W * 4), ("keys", (cap + 2) * 8), ("geom", P * 48), ("dgeom", P * 48),
                       ("bwd_items", 32 * tiles * 8 * 4)):
        want[name] = off
        off = up(off + size)
    want["total"] = off
    assert _fields(_lib.saved_layout(P, H, W, cap)) == want
    nb = _fields(_lib.saved_layout(P, H, W, cap, with_backward=False))
    assert nb["dgeom"] == want["dgeom"] and nb["total"] == nb["bwd_items"] == want["dgeom"]


def test_deterministic_symbols_are_exported():
    from dreamscene_b200 import _build, _lib
    _build.build()
    lib = _lib.load()
    for s in ("b200gsr_backward_views_ex", "b200gsr_disparity_backward_ex"):
        assert s in _lib.EXPORTS and hasattr(lib, s)
    hdr = open(os.path.join(ROOT, "include", "b200gsr.h")).read()
    for name, value in (("B200GSR_FWD_DETERMINISTIC", _lib.FWD_DETERMINISTIC), ("B200GSR_BWD_DETERMINISTIC", _lib.BWD_DETERMINISTIC),
                        ("B200GSR_SAVED_DETERMINISTIC", _lib.SAVED_DETERMINISTIC)):
        assert f"#define {name} {value:#x}" in hdr or f"#define {name} {value}u" in hdr or f"#define {name} {value}" in hdr
    assert lib.b200gsr_version() == 3


def test_fixed_point_helpers_native_check(tmp_path):
    """tests/native/det_check.cu (the common.cuh fixed-point helpers) compiled with nvcc and run on the CPU."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path / "det_check")
    src = os.path.join(ROOT, "tests", "native", "det_check.cu")
    subprocess.run([nvcc, "-std=c++17", "-Wno-deprecated-gpu-targets", "-I", os.path.join(ROOT, "dreamscene_b200", "csrc"),
                    "-I", os.path.join(ROOT, "include"), "-o", exe, src], check=True, timeout=300)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and "helpers ok" in out.stdout, out.stdout + out.stderr
