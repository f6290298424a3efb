"""Adam for the Gaussian parameter groups (DESIGN.md section 0, f6) - one kernel per step, bitwise equal to
torch.optim.Adam.

The reference builds ``torch.optim.Adam(l, lr=0.0, eps=1e-15)`` over seven one-tensor groups
(/root/reference/gs_renderer.py:653) and steps it after every backward.  Without ``foreach`` / ``fused``, torch
runs ``_multi_tensor_adam``: per group lerp, mul, addcmul, sqrt, div, add and addcdiv as separate kernels.
``GaussianAdam`` is a drop-in for that constructor call whose ``step()`` updates every parameter of every group in
one launch (b200gsr_adam_step) and produces the same bits as the default path: parameters, ``exp_avg``,
``exp_avg_sq`` and ``step``.  ``torch.optim.Adam(fused=True)`` rounds differently and so drifts away from the
reference's trajectory.

The state is torch's own (``step`` a CPU float32 scalar tensor, the moments ``zeros_like(p)``), so the
reference's optimizer surgery (``replace_tensor_to_optimizer``, ``_prune_optimizer``,
``cat_tensors_to_optimizer``) and ``state_dict`` / ``load_state_dict`` work unchanged, in both directions between
the two classes.
"""
from __future__ import annotations

import contextlib
from typing import List, Tuple

import torch

from . import _lib

_ONE = torch.tensor(1.0)           # the step-counter increment, as _multi_tensor_adam adds it on the CPU
_REFUSED = (("amsgrad", False), ("weight_decay", 0), ("maximize", False), ("capturable", False),
            ("differentiable", False), ("foreach", None), ("fused", None))


def adam_scalars(lr: float, beta1: float, beta2: float, eps: float, step: float) -> Tuple[float, ...]:
    """The per-tensor scalars of one step, as the double expressions _multi_tensor_adam evaluates (the kernel
    receives their fp32 images): (lerp weight, beta2, 1 - beta2, eps, step_size, bias_correction2_sqrt)."""
    bias_correction1 = 1 - beta1 ** step
    bias_correction2 = 1 - beta2 ** step
    return 1 - beta1, beta2, 1 - beta2, eps, (lr / bias_correction1) * -1, bias_correction2 ** 0.5


def launches(records: list, limit: int = _lib.ADAM_MAX_TENSORS) -> List[list]:
    """Split a step's tensor records into calls of at most `limit` tensors (one launch each)."""
    return [records[i:i + limit] for i in range(0, len(records), limit)]


def _check_group(group: dict) -> None:
    g = group.get
    if (g("amsgrad", False) or g("weight_decay", 0) != 0 or g("maximize", False) or g("capturable", False)
            or g("differentiable", False) or g("foreach") is not None or g("fused") is not None
            or isinstance(group["lr"], torch.Tensor) or isinstance(group["betas"][0], torch.Tensor)
            or isinstance(group["betas"][1], torch.Tensor)):
        for key, allowed in _REFUSED:
            if g(key, allowed) != allowed:
                raise ValueError(f"GaussianAdam: {key}={group[key]!r} is not supported (only {key}={allowed!r})")
        raise ValueError("GaussianAdam: lr and betas must be Python numbers, not tensors")


def _refuse(p, g, m, v, step_t, dev) -> None:
    """Raise the error that explains why (p, grad, exp_avg, exp_avg_sq, step) cannot be stepped."""
    if g.is_sparse:
        raise RuntimeError("GaussianAdam does not support sparse gradients")
    if p.device != dev or g.device != dev or dev.type != "cuda":
        raise RuntimeError("GaussianAdam: all parameters and gradients must be on one CUDA device")
    if p.dtype != torch.float32 or g.dtype != torch.float32:
        raise RuntimeError("GaussianAdam: parameters and gradients must be float32")
    if g.shape != p.shape:
        raise RuntimeError(f"GaussianAdam: gradient shape {tuple(g.shape)} != parameter shape {tuple(p.shape)}")
    if step_t.device.type != "cpu" or step_t.dtype != torch.float32:
        raise RuntimeError("GaussianAdam: state['step'] must be a CPU float32 tensor (torch's default Adam layout)")
    for name, t in (("param", p), ("exp_avg", m), ("exp_avg_sq", v)):
        if not t.is_contiguous() or t.dtype != torch.float32 or t.device != dev or t.shape != p.shape:
            raise RuntimeError(f"GaussianAdam: {name} must be a contiguous float32 tensor shaped and placed like "
                               "its parameter")
    raise RuntimeError("GaussianAdam: unsupported tensor layout")


class GaussianAdam(torch.optim.Adam):
    """torch.optim.Adam with a native single-launch ``step()``; everything else is inherited.

    Supported: the default configuration (any lr, betas, eps; per-group values; lr changed between steps).
    Refused with ValueError: amsgrad, weight_decay != 0, maximize, capturable, differentiable, an explicit
    ``foreach`` or ``fused``, and tensor lr or betas.  Parameters, gradients and moments are fp32 CUDA tensors on
    one device; parameters and moments must be contiguous (updated in place), gradients are made contiguous.
    ``step()`` runs on the current stream and never synchronises with the host.
    """

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, *,
                 foreach=None, maximize=False, capturable=False, differentiable=False, fused=None,
                 decoupled_weight_decay=False):
        defaults = dict(lr=lr, betas=betas, weight_decay=weight_decay, amsgrad=amsgrad, foreach=foreach,
                        maximize=maximize, capturable=capturable, differentiable=differentiable, fused=fused)
        _check_group(defaults)
        super().__init__(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad,
                         foreach=foreach, maximize=maximize, capturable=capturable, differentiable=differentiable,
                         fused=fused, decoupled_weight_decay=decoupled_weight_decay)
        for group in self.param_groups:
            _check_group(group)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        records, steps, dev = [], [], None
        f32, strided = torch.float32, torch.strided
        for group in self.param_groups:
            _check_group(group)
            lr, (beta1, beta2), eps = group["lr"], group["betas"], group["eps"]
            for p in group["params"]:
                g = p.grad
                if g is None:
                    continue
                if dev is None:
                    dev = p.device
                state = self.state[p]
                if len(state) == 0:
                    state["step"] = torch.tensor(0.0, dtype=f32)
                    state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                m, v, step_t = state["exp_avg"], state["exp_avg_sq"], state["step"]
                # one combined test on the hot path; _refuse names the failing condition
                if not (g.layout == strided and p.dtype == g.dtype == m.dtype == v.dtype == step_t.dtype == f32
                        and p.is_contiguous() and m.is_contiguous() and v.is_contiguous()
                        and p.shape == g.shape == m.shape == v.shape and step_t.is_cpu
                        and dev.type == "cuda" and p.device == g.device == m.device == v.device == dev):
                    _refuse(p, g, m, v, step_t, dev)
                if not g.is_contiguous():
                    g = g.contiguous()
                steps.append(step_t)
                records.append((p, g, m, v, lr, beta1, beta2, eps, step_t))
        if not records:
            return loss
        torch._foreach_add_(steps, _ONE, alpha=1.0)      # as torch: the counter first, then the math
        table = [_lib.AdamTensor(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel(),
                                 *adam_scalars(lr, beta1, beta2, eps, step_t.item()))
                 for p, g, m, v, lr, beta1, beta2, eps, step_t in records]
        lib = _lib.load()
        stream = _lib.stream(dev)
        with contextlib.nullcontext() if dev.index == torch.cuda.current_device() else torch.cuda.device(dev):
            for part in launches(table):
                _lib.check(lib.b200gsr_adam_step(len(part), (_lib.AdamTensor * len(part))(*part), stream),
                           "b200gsr_adam_step")
        return loss
