"""CPU checks of the C ABI's refusals: every forward and backward entry point checks its arguments, its image size
and its workspace before the first CUDA call, so each kind of bad argument returns its own error code and message
on a machine without a GPU."""
import ctypes as C

import pytest

FAKE = 256               # a device pointer that is never dereferenced: every call below is refused before a launch
BIG = 1 << 40            # workspace bytes that pass every size check


@pytest.fixture(scope="module")
def lib():
    from dreamscene_b200 import _build, _lib
    _build.build()
    return _lib.load()


def _err():
    from dreamscene_b200 import _lib
    return _lib.last_error()


def _params(P=10, M=16, deg=3, H=64, W=64, score_flag=0, bg=FAKE, vm=FAKE):
    from dreamscene_b200 import _lib
    return _lib.Params(P, M, deg, H, W, 0.3, 0.3, 1.0, 0, score_flag, bg, vm, FAKE, FAKE)


# one Gaussian input set: means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp
SH_SR = (FAKE, FAKE, None, FAKE, FAKE, FAKE, None)


def _forward(lib, prm=None, inputs=SH_SR, outs=(FAKE, FAKE, FAKE, FAKE), scratch_bytes=BIG, saved_bytes=BIG,
             max_pairs=1 << 20, flags=0, null_params=False):
    prm = prm or _params()
    p = None if null_params else C.byref(prm)
    return lib.b200gsr_forward(p, *inputs, *outs, FAKE, scratch_bytes, FAKE, saved_bytes, max_pairs, flags, None, 0, None)


def _backward(lib, prm=None, inputs=SH_SR, saved=FAKE, saved_bytes=BIG, max_pairs=1 << 20, grads=None, stages=3,
              g_range=None, dsh_coefs=0):
    prm = prm or _params()
    grads = grads or (FAKE, FAKE, FAKE, None, FAKE, FAKE, FAKE, None)
    g0, g1 = g_range or (0, prm.P)
    return lib.b200gsr_backward_ex(C.byref(prm), *inputs, FAKE, FAKE, FAKE, FAKE, saved, saved_bytes, None, 0,
                                   max_pairs, *grads, stages, g0, g1, dsh_coefs, None)


def _views(B, mutate=None, P=10, H=64, W=64, inputs=SH_SR, score_flag=0):
    from dreamscene_b200 import _lib
    prm = (_lib.Params * B)()
    vin = (_lib.ViewInputs * B)()
    for v in range(B):
        prm[v] = _params(P=P, H=H, W=W, score_flag=score_flag, bg=FAKE + 12 * v)
        vin[v] = _lib.ViewInputs(*inputs)
    if mutate:
        mutate(prm, vin)
    return prm, vin


def _forward_views(lib, B=2, mutate=None, outs=(FAKE, FAKE, FAKE, FAKE), scratch_bytes=BIG, saved_bytes=BIG,
                   max_pairs=1 << 20, flags=0, **kw):
    prm, vin = _views(B, mutate, **kw)
    return lib.b200gsr_forward_views(B, prm, vin, *outs, FAKE, scratch_bytes, FAKE, saved_bytes, max_pairs, flags,
                                     None, 0, None)


def _view_grads(B, null=None):
    from dreamscene_b200 import _lib
    out = (_lib.ViewGrads * B)()
    for v in range(B):
        out[v] = _lib.ViewGrads(FAKE, FAKE, FAKE, None, FAKE, FAKE, FAKE, None, 0)
    if null is not None:
        setattr(out[null[0]], null[1], None)
    return out


def _backward_views(lib, B=2, mutate=None, saved=FAKE, saved_bytes=BIG, out="grads", flags=0, null_grad=None, **kw):
    prm, vin = _views(B, mutate, **kw)
    out = _view_grads(B, null_grad) if out == "grads" else out
    return lib.b200gsr_backward_views_ex(B, prm, vin, FAKE, FAKE, FAKE, FAKE, saved, saved_bytes, 1 << 20, out, flags,
                                         None)


def _score(lib, B=2, mutate=None, acc=FAKE, scratch_bytes=BIG, saved_bytes=BIG, flags=0, **kw):
    kw.setdefault("inputs", (FAKE, None, None, FAKE, FAKE, FAKE, None))
    prm, vin = _views(B, mutate, score_flag=1, **kw)
    return lib.b200gsr_score_views(B, prm, vin, acc, FAKE, scratch_bytes, FAKE, saved_bytes, 1 << 20, flags, None, 0,
                                   None)


def _set(field, value, view=0, inputs=False):
    def mutate(prm, vin):
        setattr((vin if inputs else prm)[view], field, value)
    return mutate


def _refused(rc, code, text):
    assert rc == code, (rc, _err())
    assert text in _err(), _err()


# ---- inputs checked by validate_inputs (single view) and check_views / check_score_views (stacked views) ------

@pytest.mark.parametrize("field,value,code,text", [("P", -1, -1, "negative size"), ("image_width", -1, -1, "negative size"),
                                                   ("image_height", 65536 * 16, -4, "65535 tiles")])
def test_every_entry_point_refuses_bad_sizes(lib, field, value, code, text):
    prm = _params()
    setattr(prm, field, value)
    _refused(_forward(lib, prm=prm), code, text)
    _refused(_backward(lib, prm=prm), code, text)
    _refused(_forward_views(lib, mutate=_set(field, value)), code, text)
    _refused(_backward_views(lib, mutate=_set(field, value)), code, text)
    _refused(_score(lib, mutate=_set(field, value)), code, text)


def test_single_view_entry_points_refuse_bad_inputs(lib):
    for call in (_forward, _backward):
        _refused(call(lib, prm=_params(bg=None)), -1, "device pointers")
        _refused(call(lib, inputs=(None,) + SH_SR[1:]), -1, "means3D/opacities are required")
        _refused(call(lib, inputs=(FAKE, FAKE, FAKE) + SH_SR[3:]), -1, "excatly one of either SHs")
        _refused(call(lib, inputs=(FAKE, None, None) + SH_SR[3:]), -1, "excatly one of either SHs")
        _refused(call(lib, inputs=SH_SR[:6] + (FAKE,)), -1, "scale/rotation pair or precomputed 3D covariance")
        _refused(call(lib, inputs=SH_SR[:5] + (None, None)), -1, "scale/rotation pair or precomputed 3D covariance")
        _refused(call(lib, prm=_params(deg=4)), -4, "sh_degree 4")
        _refused(call(lib, prm=_params(M=3, deg=1)), -1, "M=3 inconsistent")
    assert lib.b200gsr_forward(None, *([None] * 11), None, 0, None, 0, 1024, 0, None, 0, None) == -1
    assert "params is null" in _err()


def test_forward_refuses_missing_outputs(lib):
    for outs in ((None, FAKE, FAKE, None), (FAKE, None, FAKE, None), (FAKE, FAKE, None, None)):
        _refused(_forward(lib, outs=outs), -1, "null output/workspace pointer")
        _refused(_forward_views(lib, outs=outs), -1, "null output/workspace pointer")
    _refused(_forward(lib, prm=_params(score_flag=1), outs=(FAKE, FAKE, FAKE, None)), -1, "score buffer is null")
    _refused(_forward_views(lib, score_flag=1, outs=(FAKE, FAKE, FAKE, None)), -1, "score buffer is null")


def test_forward_refuses_small_workspaces_and_oversized_deterministic_images(lib):
    from dreamscene_b200 import _lib
    _refused(_forward(lib, scratch_bytes=1024), -2, "workspace too small")
    _refused(_forward(lib, saved_bytes=1024), -2, "workspace too small")
    _refused(_forward(lib, max_pairs=1 << 33), -4, "32 bits")
    _refused(_forward(lib, prm=_params(H=8208, W=8208), flags=_lib.FWD_DETERMINISTIC), -4, "deterministic mode supports")
    _refused(_forward_views(lib, scratch_bytes=1024), -2, "workspace too small")
    _refused(_forward_views(lib, saved_bytes=1024), -2, "workspace too small")
    _refused(_forward_views(lib, max_pairs=1 << 33), -4, "32 bits")
    _refused(_forward_views(lib, H=8208, W=8208, flags=_lib.FWD_DETERMINISTIC), -4, "deterministic mode supports")
    # deterministic mode needs the fixed-point accumulators in `saved`: the size without them is refused
    need = _lib.saved_layout(10, 64, 64, 1 << 20, True, False).total
    _refused(_forward(lib, saved_bytes=need, flags=_lib.FWD_DETERMINISTIC), -2, "workspace too small")


def test_backward_refuses_bad_ranges_and_pointers(lib):
    assert _backward(lib, prm=_params(P=0), saved=None) == 0            # nothing to do: no pointer is needed
    _refused(_backward(lib, g_range=(1, 10)), -1, "bad Gaussian range")
    _refused(_backward(lib, g_range=(0, 11)), -1, "bad Gaussian range")
    _refused(_backward(lib, dsh_coefs=17), -1, "dsh_coefs=17")
    _refused(_backward(lib, inputs=(FAKE, None, FAKE) + SH_SR[3:], dsh_coefs=-1), -1, "needs shs")
    _refused(_backward(lib, saved=None), -1, "null saved-state/gradient pointer")
    _refused(_backward(lib, grads=(None, FAKE, FAKE, None, FAKE, FAKE, FAKE, None)), -1, "null gradient output pointer")
    _refused(_backward(lib, grads=(FAKE, FAKE, FAKE, None, FAKE, FAKE, None, None)), -1, "null gradient output pointer")


def test_backward_refuses_small_saved_buffers_and_oversized_deterministic_images(lib):
    from dreamscene_b200 import _lib
    _refused(_backward(lib, saved_bytes=1024), -2, "saved buffer too small for backward")
    need = _lib.saved_layout(10, 64, 64, 1 << 20, True, False).total
    _refused(_backward(lib, saved_bytes=need, stages=3 | _lib.BWD_DETERMINISTIC), -2, "saved buffer too small")
    _refused(_backward(lib, prm=_params(H=8208, W=8208), stages=3 | _lib.BWD_DETERMINISTIC), -4,
             "deterministic mode supports")
    _refused(_backward_views(lib, saved_bytes=1024), -2, "saved buffer too small for backward")
    _refused(_backward_views(lib, H=8208, W=8208, flags=_lib.BWD_DETERMINISTIC), -4, "deterministic mode supports")


def test_views_entry_points_refuse_inconsistent_views(lib):
    from dreamscene_b200 import _lib
    for call in (_forward_views, _backward_views):
        _refused(call(lib, B=0), -4, "number of views 0")
        _refused(call(lib, B=17), -4, "number of views 17")
        _refused(call(lib, mutate=_set("bg", None, view=1)), -1, "device pointers")
        _refused(call(lib, mutate=_set("P", 11, view=1)), -1, "view 1: P, M, image size and score_flag")
        _refused(call(lib, mutate=_set("score_flag", 1, view=1)), -1, "view 1: P, M, image size and score_flag")
        _refused(call(lib, mutate=_set("bg", FAKE, view=1)), -1, "view 1: backgrounds must be one contiguous")
        _refused(call(lib, mutate=_set("cov3D_precomp", FAKE, view=1, inputs=True)), -1, "exactly one")
        _refused(call(lib, P=1 << 29), -4, "B * P too large")
    kinds = lambda prm, vin: (setattr(vin[1], "shs", None), setattr(vin[1], "colors_precomp", FAKE))
    _refused(_forward_views(lib, mutate=kinds), -1, "view 1: all views must use the same input kinds")
    prm, vin = _views(2)
    assert lib.b200gsr_forward_views(2, None, vin, FAKE, FAKE, FAKE, FAKE, FAKE, BIG, FAKE, BIG, 1 << 20, 0, None, 0,
                                     None) == -1
    assert "null view array" in _err()
    assert _backward_views(lib, P=0, saved=None) == 0
    _refused(_backward_views(lib, saved=None), -1, "null saved-state/gradient pointer")
    _refused(_backward_views(lib, out=None), -1, "null saved-state/gradient pointer")
    assert _lib.BWD_DETERMINISTIC == 4


@pytest.mark.parametrize("view,field", [(0, "d_means3D"), (1, "d_means2D"), (1, "d_shs"), (1, "d_scales")])
def test_views_backward_refuses_a_null_gradient_pointer_before_any_launch(lib, view, field):
    _refused(_backward_views(lib, null_grad=(view, field)), -1, f"view {view}: null gradient output pointer")


def test_score_views_refusals(lib):
    from dreamscene_b200 import _lib
    _refused(_score(lib, B=0), -4, "number of views 0")
    _refused(_score(lib, mutate=_set("viewmatrix", None, view=1)), -1, "view 1: viewmatrix/projmatrix/campos")
    _refused(_score(lib, mutate=_set("image_width", 32, view=1)), -1, "view 1: P and image size")
    _refused(_score(lib, mutate=_set("means3D", None, view=1, inputs=True)), -1, "view 1: means3D/opacities")
    _refused(_score(lib, mutate=_set("rotations", None, view=1, inputs=True)), -1, "exactly one")
    _refused(_score(lib, P=1 << 29), -4, "B * P too large")
    _refused(_score(lib, flags=0x80), -1, "unknown flags 0x80")
    _refused(_score(lib, acc=None), -1, "null accumulator/workspace pointer")
    _refused(_score(lib, scratch_bytes=1024), -2, "workspace too small")
    _refused(_score(lib, saved_bytes=1024), -2, "workspace too small")
    _refused(_score(lib, H=8208, W=8208, B=1, flags=_lib.FWD_DETERMINISTIC), -4, "deterministic mode supports")
    _refused(_score(lib, H=4096, W=4096, B=16, flags=_lib.FWD_DETERMINISTIC), -4, "2^26 pixels")
    # the score pass keeps no deterministic state in `saved`: the plain inference size is enough
    need = _lib.saved_layout(2 * 10, 2 * 64, 64, 1 << 20, False, False).total
    sbytes = _lib.scratch_layout(2 * 10, 2 * 64, 64, 1 << 20).total
    _refused(_score(lib, saved_bytes=need - 1, flags=_lib.FWD_DETERMINISTIC), -2, "workspace too small")
    _refused(_score(lib, scratch_bytes=sbytes - 1), -2, "workspace too small")
