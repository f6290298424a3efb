"""CPU-only checks of the video frames (include/b200gsr_frames.h, dreamscene_b200.video): the signature table agrees
with the header and binds; the library refuses bad arguments before touching a device (made-up device addresses,
never dereferenced); render_frames refuses what it cannot take; and the quantisation rule b200gsr_frames implements,
restated in numpy, gives the frames of the reference's loop (harness/video_ref.py) on edge values."""
import ctypes as C
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from dreamscene_b200 import _lib
from dreamscene_b200 import video as V
from harness import video_ref
from tests.test_abi_binding_cpu import _mismatches
from tests.test_scene_render_cpu import _groups, _settings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "b200gsr_frames.h")


def _prototypes():
    src = re.sub(r"/\*.*?\*/", " ", open(HEADER).read(), flags=re.S)
    return {name: (ret, [" ".join(a.split()) for a in args.split(",")])
            for ret, name, args in re.findall(r"(\bint)\s+(b200gsr_\w+)\s*\(([^)]*)\)\s*;", src)}


def test_frames_signature_table_matches_the_header_and_binds():
    protos = _prototypes()
    assert list(protos) == list(_lib.FRAMES_SIGNATURES) == ["b200gsr_frames"]
    assert _mismatches(_lib.FRAMES_SIGNATURES, protos) == []
    assert re.search(r"#define B200GSR_FRAMES_STATS_BYTES (\d+)", open(HEADER).read()).group(1) == \
        str(_lib.FRAMES_STATS_BYTES)
    lib = _lib.load()
    for name, (restype, argtypes) in _lib.FRAMES_SIGNATURES.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and tuple(fn.argtypes) == tuple(argtypes), name
    others = (set(_lib.SIGNATURES) | set(_lib.SCENE_SIGNATURES) | set(_lib.STEP_SIGNATURES) |
              set(_lib.LOSS_SIGNATURES) | set(_lib.FROZEN_SIGNATURES) | set(_lib.STATS_SIGNATURES) |
              set(_lib.RESERVE_SIGNATURES))
    assert not set(_lib.FRAMES_SIGNATURES) & others


def test_library_refuses_bad_frames_arguments():
    lib = _lib.load()
    p = [C.c_void_p(0x100000 * (k + 1)) for k in range(6)]      # color, depth_alpha, focal, rgb8, depth8, stats

    def call(B, H, W, ptrs=p):
        return lib.b200gsr_frames(B, H, W, *ptrs, None)

    for B in (0, -1, _lib.MAX_VIEWS + 1):
        assert call(B, 32, 32) == _lib.ERR_BAD_ARG and "B =" in _lib.last_error()
    for H, W in ((0, 32), (32, 0), (-4, 32)):
        assert call(2, H, W) == _lib.ERR_BAD_ARG and "positive" in _lib.last_error()
    for k in range(6):
        ptrs = list(p)
        ptrs[k] = None
        assert call(2, 32, 32, ptrs) == _lib.ERR_BAD_ARG and "null" in _lib.last_error()
    for k in (3, 4):
        ptrs = list(p)
        ptrs[k] = C.c_void_p(0x100002)
        assert call(2, 32, 32, ptrs) == _lib.ERR_BAD_ARG and "aligned" in _lib.last_error()
    assert call(16, 8192, 8192) == _lib.ERR_BAD_ARG and "too large" in _lib.last_error()


def test_render_frames_refusals(monkeypatch):
    g = _groups([5, 3], 4)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        V.render_frames(g, _settings(2))
    with pytest.raises(ValueError, match="image size"):
        V.render_frames(g, _settings(1) + _settings(1, H=48))
    with pytest.raises(ValueError, match="score_flag"):
        V.render_frames(g, _settings(2, score=True))
    for vpp in (0, _lib.MAX_VIEWS + 1):
        with pytest.raises(ValueError, match="views_per_pass"):
            V.render_frames(g, _settings(2), views_per_pass=vpp)
    reserved = SimpleNamespace(_reserved_rows=True, **g[0])
    with pytest.raises(TypeError, match="ReservedGroup"):
        V.render_frames([reserved], _settings(2))
    monkeypatch.setattr(V, "_check_device", lambda flat: None)       # lets the capture check run on CPU tensors
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    with pytest.raises(RuntimeError, match="CUDA graph"):
        V.render_frames(g, _settings(2))


# ---- the quantisation rule of frames_kernel (csrc/postprocess.cu) restated in numpy: fmaxf / fminf return the
# non-NaN operand, __fmul_rn(x, 255.f) and rintf round half to even, the depth is divided (correctly rounded) by the
# view's normalised maximum, disp_norm(M) -----------------------------------------------------------------------------
F0, F1, F255 = np.float32(0.0), np.float32(1.0), np.float32(255.0)


def _kernel_quantise(x):
    return np.rint(np.fmin(np.fmax(x, F0), F1) * F255).astype(np.uint8)


def _disp_norm(d, m, den):
    with np.errstate(divide="ignore", invalid="ignore"):
        t = (d - m) / den
    return np.where(np.isnan(t), t, np.fmin(np.fmax(t, F0), F1))          # NaN passes, as in torch.clamp


def _kernel_depth(d, m, M):
    den = np.float32(M - m)
    with np.errstate(divide="ignore", invalid="ignore"):
        return _kernel_quantise(_disp_norm(d, m, den) / _disp_norm(np.float32(M), m, den))


def _ties():
    """float32 values x in [0, 1] with x * 255 exactly k + 0.5 in float32, and their float32 neighbours."""
    out = []
    for k in range(255):
        x0 = np.float32((k + 0.5) / 255)
        for x in (x0, np.nextafter(x0, F0), np.nextafter(x0, F1)):
            if np.float32(x) * F255 == np.float32(k + 0.5):
                out.append(np.float32(x))
    return np.array(out, np.float32)


def _reference(rgb, disp):
    """harness/video_ref.py over one view: rgb [3,H,W], disp [1,H,W] float32 numpy."""
    img, dep = video_ref.frames(lambda v: (torch.from_numpy(rgb), torch.from_numpy(disp)), [0])
    return img[0], dep[0]


def test_colour_quantisation_matches_the_reference_on_edge_values():
    ties = _ties()
    assert len(ties) > 100 and (ties * F255 % 1 == 0.5).all()
    edge = np.array([0.0, -0.0, 1.0, np.nextafter(F0, -F1), -1e-30, -0.5, np.nextafter(F1, 2 * F1), 1.5, 1e30, -1e30,
                     np.inf, -np.inf, np.nan, 0.5 / 255, 254.5 / 255, 1.0 / 255], np.float32)
    vals = np.concatenate([ties, edge, np.random.RandomState(0).uniform(-0.1, 1.1, 4000).astype(np.float32)])
    vals = np.resize(vals, 3 * 64 * ((len(vals) + 191) // 192)).astype(np.float32)
    rgb = vals.reshape(3, -1, 64)
    disp = np.zeros((1,) + rgb.shape[1:], np.float32)
    with np.errstate(invalid="ignore"):
        img, _ = _reference(rgb, disp)
    np.testing.assert_array_equal(img, _kernel_quantise(rgb).transpose(1, 2, 0))
    # ties round to even, NaN and everything below 0 give 0, everything above 1 gives 255
    assert (_kernel_quantise(ties) % 2 == 0).all()
    assert list(_kernel_quantise(edge[:13])) == [0, 0, 255, 0, 0, 0, 255, 255, 255, 0, 255, 0, 0]


@pytest.mark.parametrize("case", ["random", "masked_min", "ties", "constant", "single_pixel"])
def test_depth_quantisation_matches_the_reference(case):
    rs = np.random.RandomState(1)
    H, W = 24, 40
    d = rs.uniform(0.2, 3.0, (H, W)).astype(np.float32)           # the raw disparity focal / (depth + 10 alpha + 1e-5)
    if case == "masked_min":
        d[5:9, 5:9] = np.float32(0.05)                             # below the masked minimum: clamped to 0
    if case == "ties":
        m, M = np.float32(0.0), np.float32(1.0)
        d = np.resize(np.concatenate([_ties(), [m, M]]), (H, W)).astype(np.float32)
    if case == "constant":
        d[:] = np.float32(1.7)
    if case == "single_pixel":
        d = d[:1, :1]
    m = np.float32(d.min() if case != "masked_min" else d[d > 0.1].min())
    M = np.float32(d.max())
    disp = _disp_norm(d, m, np.float32(M - m))[None]               # what disparity_from_depth_alpha returns
    with np.errstate(invalid="ignore"):
        _, dep = _reference(np.zeros((3,) + d.shape, np.float32), disp)
    np.testing.assert_array_equal(dep[..., 0], _kernel_depth(d, m, M))
    if M == m:                                                     # max == min: the depth frame is all 0
        assert not dep.any()
    else:
        assert dep.max() == 255
