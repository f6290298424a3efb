"""CPU-only checks of the guidance stages' regularisers (b200gsr_tv_loss / b200gsr_scale_loss of
include/b200gsr_loss.h, dreamscene_b200.losses.tv_loss, StepGraph's tv_weight / tv_depth_weight / scale_weight): the
scratch sizes, the refusals before any launch (made-up device addresses, never dereferenced), and the order in which
torch's autograd engine accumulates tv_loss's gradient, which the kernel reproduces."""
import ctypes as C

import pytest
import torch

from dreamscene_b200 import _lib
from dreamscene_b200 import graph as G
from dreamscene_b200 import scene as S
from harness import regularisers_ref as ref
from tests.test_scene_render_cpu import _groups, _settings


def test_tv_scratch_bytes_is_two_doubles_per_block_of_the_scalar_grid():
    lib = _lib.load()
    # 8 warps per block, a warp covers 8 rows x 32 columns of one plane
    assert lib.b200gsr_tv_loss_scratch_bytes(1, 1, 2, 2) == 16
    assert lib.b200gsr_tv_loss_scratch_bytes(2, 3, 37, 29) == 16 * 4              # 6 planes x 5 bands
    assert lib.b200gsr_tv_loss_scratch_bytes(4, 3, 512, 512) == 16 * (12 * 64 * 16 // 8)
    assert lib.b200gsr_tv_loss_scratch_bytes(4, 1, 512, 512) == 16 * (4 * 64 * 16 // 8)
    for bad in ((0, 3, 8, 8), (1, 0, 8, 8), (1, 3, 1, 8), (1, 3, 8, 1), (2, 1, 32768, 32768)):
        assert lib.b200gsr_tv_loss_scratch_bytes(*bad) == 0, bad


def test_scale_scratch_bytes_is_one_double_per_block():
    lib = _lib.load()
    assert lib.b200gsr_scale_loss_scratch_bytes(1) == 8
    assert lib.b200gsr_scale_loss_scratch_bytes(1365) == 8                  # 4095 elements
    assert lib.b200gsr_scale_loss_scratch_bytes(1366) == 16
    assert lib.b200gsr_scale_loss_scratch_bytes(4 * 1200000) == 8 * 3516
    assert lib.b200gsr_scale_loss_scratch_bytes(0) == 0 and lib.b200gsr_scale_loss_scratch_bytes(2 ** 30) == 0


def _vp(a):
    return C.c_void_p(a) if a else None


def _fake_tv(B=2, C_=3, H=16, W=16, x=0x10000, grad_out=0x20000, loss=0x30000, d_x=0x40000, accumulate=0,
             scratch=0x50000, scratch_bytes=None):
    lib = _lib.load()
    if scratch_bytes is None:
        scratch_bytes = lib.b200gsr_tv_loss_scratch_bytes(2, 3, 16, 16)
    rc = lib.b200gsr_tv_loss(B, C_, H, W, _vp(x), _vp(grad_out), _vp(loss), _vp(d_x), accumulate, _vp(scratch),
                             scratch_bytes, None)
    return rc, _lib.last_error()


@pytest.mark.parametrize("kwargs,code,msg", [
    (dict(B=0), -1, "must be >= 1"),
    (dict(C_=0), -1, "must be >= 1"),
    (dict(H=1), -1, "must be >= 2"),
    (dict(W=1), -1, "must be >= 2"),
    (dict(B=2, C_=1, H=32768, W=32768), -4, "2^31 - 1 elements"),
    (dict(accumulate=2), -1, "accumulate"),
    (dict(x=0), -1, "device pointer"),
    (dict(loss=0, d_x=0), -1, "nothing to compute"),
    (dict(grad_out=0), -1, "needs grad_out"),
    (dict(scratch=0), -2, "scratch"),
    (dict(scratch_bytes=16), -2, "scratch"),
    (dict(scratch=0x50004), -2, "8-byte aligned"),
])
def test_tv_loss_refuses_bad_arguments_before_any_launch(kwargs, code, msg):
    rc, err = _fake_tv(**kwargs)
    assert rc == code and msg in err, (rc, err)


def _fake_scale(rows=1000, scales=0x10000, grad_out=0x20000, loss=0x30000, d=0x40000, accumulate=1, scratch=0x50000,
                scratch_bytes=None):
    lib = _lib.load()
    if scratch_bytes is None:
        scratch_bytes = lib.b200gsr_scale_loss_scratch_bytes(1000)
    rc = lib.b200gsr_scale_loss(rows, _vp(scales), _vp(grad_out), _vp(loss), _vp(d), accumulate, _vp(scratch),
                                scratch_bytes, None)
    return rc, _lib.last_error()


@pytest.mark.parametrize("kwargs,code,msg", [
    (dict(rows=0), -1, "must be >= 1"),
    (dict(rows=2 ** 30), -4, "2^31 - 1 elements"),
    (dict(accumulate=-1), -1, "accumulate"),
    (dict(scales=0), -1, "device pointer"),
    (dict(loss=0, d=0), -1, "nothing to compute"),
    (dict(grad_out=0), -1, "needs grad_out"),
    (dict(scratch=0), -2, "scratch"),
    (dict(rows=5000), -2, "scratch"),
    (dict(scratch=0x50001), -2, "8-byte aligned"),
])
def test_scale_loss_refuses_bad_arguments_before_any_launch(kwargs, code, msg):
    rc, err = _fake_scale(**kwargs)
    assert rc == code and msg in err, (rc, err)


def test_tv_loss_refuses_what_it_cannot_take():
    from dreamscene_b200.losses import tv_loss
    with pytest.raises(TypeError, match="float32"):
        tv_loss(torch.zeros(1, 3, 4, 4, dtype=torch.float64))
    with pytest.raises(TypeError, match="float32"):
        tv_loss(torch.zeros(1, 3, 4, 4, dtype=torch.float16))
    for shape in ((3, 4, 4), (1, 1, 3, 4, 4), (1, 3, 1, 4), (1, 3, 4, 1), (0, 3, 4, 4)):
        with pytest.raises(ValueError, match=r"\[B,C,H,W\]"):
            tv_loss(torch.zeros(shape))
    with pytest.raises(RuntimeError, match="no CPU"):
        tv_loss(torch.zeros(1, 3, 2, 2))


def _graph(monkeypatch, **kw):
    from dreamscene_b200 import GaussianAdam
    groups = _groups([5, 3], 4)
    opts = [GaussianAdam([t.requires_grad_(True) for t in g.values()], lr=0.0, eps=1e-15) for g in groups]
    monkeypatch.setattr(S, "_check_device", lambda flat: None)      # lets the host checks run on CPU tensors
    kw.setdefault("height", 32)
    kw.setdefault("width", 32)
    return G.StepGraph(groups, opts, views=1, **kw)


@pytest.mark.parametrize("name", ["tv_weight", "tv_depth_weight", "scale_weight"])
@pytest.mark.parametrize("w", [-1.0, -1e-30, float("nan"), float("inf"), -float("inf")])
def test_step_graph_refuses_bad_weights(monkeypatch, name, w):
    with pytest.raises(ValueError, match=f"{name} must be finite and >= 0"):
        _graph(monkeypatch, **{name: w})


@pytest.mark.parametrize("name", ["tv_weight", "tv_depth_weight", "scale_weight"])
def test_step_graph_refuses_regularisers_with_a_target(monkeypatch, name):
    gt = torch.zeros(2, 3, 32, 32, dtype=torch.float16)
    with pytest.raises(ValueError, match="cannot be combined with target"):
        _graph(monkeypatch, target=gt, **{name: 0.5})
    _graph(monkeypatch, target=gt, **{name: 0.0})       # a weight of 0 is off
    sg = _graph(monkeypatch, target=gt)
    setattr(sg, name, 1.0)                              # a weight set later is checked at render()
    with pytest.raises(ValueError, match="cannot be combined with target"):
        sg.render(_settings(1), target_index=[0])


def test_step_graph_refuses_tv_on_a_single_row_or_column(monkeypatch):
    for hw in (dict(height=1), dict(width=1)):
        with pytest.raises(ValueError, match="height and width >= 2"):
            _graph(monkeypatch, tv_weight=1.0, **hw)
        _graph(monkeypatch, scale_weight=1.0, **hw)     # the scale term has no such limit


def test_weights_are_part_of_the_layout_key(monkeypatch):
    sg = _graph(monkeypatch, tv_weight=1.0, scale_weight=0.5)
    assert sg._reg_key() == (1.0, None, 0.5)
    sg.tv_depth_weight = 2
    assert sg._reg_key() == (1.0, 2.0, 0.5)
    sg.tv_weight = 0.0
    assert sg._reg_key() == (None, 2.0, 0.5)


def _cpu_inputs(shape, scale, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g) * scale
    x.view(-1)[::13] = x.view(-1)[::13].round()          # equal neighbours: differences of +0 and -0 gradients
    return x


@pytest.mark.parametrize("shape", [(4, 3, 37, 29), (2, 1, 16, 16), (1, 1, 2, 2), (3, 3, 5, 64)])
@pytest.mark.parametrize("go", [1.0, 0.5, 0.1, 1 / 3])
@pytest.mark.parametrize("scale", [1e-3, 1.0, 1e3])
def test_autograd_accumulates_the_tv_gradient_in_the_pinned_order(shape, go, scale):
    """On the CPU torch divides by a Python int with an IEEE division, so the restated gradient, with the same
    divisions, must equal autograd's bit for bit (as int32, so the sign of zero counts) - which it does only in the
    order ((w+ + w-) + h-) + h+."""
    x0 = _cpu_inputs(shape, scale, seed=shape[2] * 7 + int(go * 10))
    x = x0.clone().requires_grad_(True)
    ref.tv_loss(x * 1.0).backward(torch.tensor(go))     # through a non-leaf, as the rendered image is
    want = ref.tv_grad(x0, torch.tensor(go))
    assert torch.equal(x.grad.view(torch.int32), want.view(torch.int32))


def test_a_loss_written_first_gets_its_gradient_added_last():
    """The eager step's image gradient is fp32(user + reg) when the user's loss is written before the regulariser
    (StepGraph adds the regulariser's gradient to the user's .grad)."""
    x0 = _cpu_inputs((2, 3, 24, 20), 1.0, seed=3)
    t = torch.randn(x0.shape, generator=torch.Generator().manual_seed(4))
    x = x0.clone().requires_grad_(True)
    img = x * 1.0
    (((img - t) ** 2).mean() + 0.7 * ref.tv_loss(img)).backward()
    u = x0.clone().requires_grad_(True)
    ((u * 1.0 - t) ** 2).mean().backward()
    want = u.grad + ref.tv_grad(x0, torch.tensor(0.7))
    assert torch.equal(x.grad.view(torch.int32), want.view(torch.int32))
