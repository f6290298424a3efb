"""CPU-only checks of dreamscene_b200.optim.GaussianAdam: constructor refusals, the C entry point's export and
argument errors, the per-tensor scalars against what torch's _multi_tensor_adam passes to its foreach kernels, and
the kernel's tensor table (tests/native/optim_check.cu, compiled with nvcc and run on the CPU)."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from dreamscene_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _params():
    return [torch.zeros(4, 3, requires_grad=True), torch.zeros(5, 1, requires_grad=True)]


@pytest.mark.parametrize("kwargs", [dict(amsgrad=True), dict(weight_decay=0.01), dict(maximize=True),
                                    dict(capturable=True), dict(differentiable=True), dict(foreach=True),
                                    dict(foreach=False), dict(fused=True), dict(fused=False),
                                    dict(lr=torch.tensor(0.01)), dict(betas=(torch.tensor(0.9), torch.tensor(0.999)))])
def test_constructor_refuses_what_the_kernel_does_not_compute(kwargs):
    from dreamscene_b200 import GaussianAdam
    with pytest.raises(ValueError):
        GaussianAdam(_params(), **kwargs)


def test_constructor_refuses_per_group_options_and_accepts_the_reference_call():
    from dreamscene_b200 import GaussianAdam
    a, b = _params()
    with pytest.raises(ValueError):
        GaussianAdam([{"params": [a]}, {"params": [b], "amsgrad": True}])
    # gs_renderer.py:653: named one-tensor groups, lr=0.0, eps=1e-15
    opt = GaussianAdam([{"params": [a], "lr": 0.001, "name": "xyz"}, {"params": [b], "lr": 0.05, "name": "opacity"}],
                       lr=0.0, eps=1e-15)
    assert isinstance(opt, torch.optim.Adam)
    assert [g["name"] for g in opt.param_groups] == ["xyz", "opacity"] and opt.param_groups[1]["eps"] == 1e-15
    ref = torch.optim.Adam([{"params": [a]}], lr=0.0, eps=1e-15)
    assert set(ref.param_groups[0]) <= set(opt.param_groups[0])       # same hyper-parameter keys (+ "name")
    opt.add_param_group({"params": [torch.zeros(2, requires_grad=True)], "maximize": True})
    with pytest.raises(ValueError):
        opt.step()


def test_export_and_abi_version():
    import dreamscene_b200
    from dreamscene_b200 import _build
    assert "GaussianAdam" in dreamscene_b200.__all__
    assert "b200gsr_adam_step" in _lib.EXPORTS
    _build.build()
    lib = _lib.load()
    assert hasattr(lib, "b200gsr_adam_step") and lib.b200gsr_version() == _lib.ABI_VERSION == 3
    assert C.sizeof(_lib.AdamTensor) == 64


def _record(ptr=16, n=1):
    return _lib.AdamTensor(ptr, ptr, ptr, ptr, n, 0.1, 0.999, 0.001, 1e-15, -0.01, 0.03)


def test_entry_point_rejects_bad_arguments_without_a_gpu():
    lib = _lib.load()
    arr = lambda recs: (_lib.AdamTensor * len(recs))(*recs)
    assert lib.b200gsr_adam_step(-1, None, None) == -1
    assert lib.b200gsr_adam_step(1, None, None) == -1
    assert lib.b200gsr_adam_step(1, arr([_record(n=-1)]), None) == -1 and "negative" in _lib.last_error()
    assert lib.b200gsr_adam_step(1, arr([_record(ptr=0)]), None) == -1 and "null" in _lib.last_error()
    n = _lib.ADAM_MAX_TENSORS + 1
    assert lib.b200gsr_adam_step(n, arr([_record()] * n), None) == -4 and str(_lib.ADAM_MAX_TENSORS) in _lib.last_error()
    # nothing to update: no launch, no CUDA call
    assert lib.b200gsr_adam_step(0, None, None) == 0
    assert lib.b200gsr_adam_step(2, arr([_record(ptr=0, n=0), _record(ptr=0, n=0)]), None) == 0


def test_launches_split_above_the_table_limit():
    from dreamscene_b200.optim import launches
    L = _lib.ADAM_MAX_TENSORS
    assert launches([]) == []
    for n in (1, 7, L, L + 1, 2 * L + 3):
        parts = launches(list(range(n)))
        assert [x for p in parts for x in p] == list(range(n))
        assert all(1 <= len(p) <= L for p in parts) and len(parts) == (n + L - 1) // L


def test_scalars_equal_what_torch_passes_to_its_foreach_kernels(monkeypatch):
    """Run torch's own _multi_tensor_adam (foreach=True; on the CPU it takes the same Python path) with the foreach
    ops wrapped, and compare the fp32 images of the scalars it passes with adam_scalars."""
    from dreamscene_b200.optim import adam_scalars
    seen = {}

    def wrap(name, grab):
        orig = getattr(torch, name)

        def f(*a, **k):
            v = grab(*a, **k)
            if v is not None:
                seen.setdefault(name, []).append(v)
            return orig(*a, **k)
        monkeypatch.setattr(torch, name, f)

    wrap("_foreach_lerp_", lambda a, b, w: w)
    wrap("_foreach_mul_", lambda a, s: s)
    wrap("_foreach_addcmul_", lambda a, b, c, v: v)
    wrap("_foreach_div_", lambda a, s: list(s))
    wrap("_foreach_add_", lambda a, s, **k: None if isinstance(s, torch.Tensor) else s)
    wrap("_foreach_addcdiv_", lambda a, b, c, s: list(s))
    betas, eps = (0.9, 0.999), 1e-15
    ps = [torch.zeros(7, requires_grad=True), torch.zeros(3, requires_grad=True)]
    opt = torch.optim.Adam([{"params": [ps[0]], "lr": 0.0016}, {"params": [ps[1]], "lr": 0.05}], lr=0.0, eps=eps,
                           betas=betas, foreach=True)
    f32 = np.float32
    for it, jump in enumerate([0, 0, 0, 96, 0, 9899, 0, 2 ** 20]):
        for p in ps:
            p.grad = torch.ones_like(p)
            if jump:
                opt.state[p]["step"] += jump      # counters far into a run
        opt.param_groups[0]["lr"] = 0.0016 * 0.97 ** it
        seen.clear()
        opt.step()
        for gi, group in enumerate(opt.param_groups):
            step = opt.state[group["params"][0]]["step"].item()
            w, b2, omb2, e, step_size, bc2s = (f32(x) for x in adam_scalars(group["lr"], *betas, eps, step))
            assert f32(seen["_foreach_lerp_"][gi]) == w and f32(seen["_foreach_mul_"][gi]) == b2
            assert f32(seen["_foreach_addcmul_"][gi]) == omb2 and f32(seen["_foreach_add_"][gi]) == e
            assert f32(seen["_foreach_div_"][gi][0]) == bc2s
            assert f32(seen["_foreach_addcdiv_"][gi][0]) == step_size
            assert np.float32(step) == np.float32(it + 1 + sum([0, 0, 0, 96, 0, 9899, 0, 2 ** 20][:it + 1]))


def test_tensor_table_native_check(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path / "optim_check")
    src = os.path.join(ROOT, "tests", "native", "optim_check.cu")
    subprocess.run([nvcc, "-std=c++17", "-Wno-deprecated-gpu-targets", "-I", os.path.join(ROOT, "dreamscene_b200", "csrc"),
                    "-I", os.path.join(ROOT, "include"), "-o", exe, src], check=True, timeout=300)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and "adam table ok" in out.stdout, out.stdout + out.stderr
