"""Fused depth/alpha -> normalised disparity (SURVEY.md section 8 f1, post-processing half).

``disparity_from_depth_alpha(depth_alpha, focal)`` replaces DreamScene's scene_gaussian.py:871-881

    depth, alpha = torch.chunk(depth_alpha, 2)
    disp  = focal / (depth + (alpha * 10) + 1e-5)
    try:    min_d = disp[alpha <= 0.1].min()
    except: min_d = disp.min()
    disp  = torch.clamp((disp - min_d) / (disp.max() - min_d), 0.0, 1.0)

for one view ([2,H,W]) or a batch ([B,2,H,W]) with two small kernels each way and NO host
synchronisation (the boolean-mask indexing above copies the mask population to the host per view).
Returns (disp [.,1,H,W], alpha [.,1,H,W]), equal bit for bit to torch's evaluation of the expression on CUDA:
`focal / x` rounded as torch's ``x.reciprocal() * focal``, and NaN wherever torch's is NaN (a view whose
``disp.max()`` equals ``min_d`` divides 0 by 0).  Differentiable like the PyTorch expression: outside the pixels
that tie for min_d or disp.max() the gradient is autograd's bit for bit; on those ties it carries the paths through
min_d and disp.max(), sums over the view that agree with autograd's within fp32 rounding.
"""
from __future__ import annotations

import torch

from . import _lib


class _Disparity(torch.autograd.Function):
    @staticmethod
    def forward(ctx, depth_alpha, focal):
        da = _lib.prepare(depth_alpha.detach())
        B, _, H, W = da.shape
        dev = da.device
        out = torch.empty(B, 1, H, W, device=dev)
        stats = torch.empty(B, 8, dtype=torch.int32, device=dev)
        lib = _lib.load()
        with torch.cuda.device(dev):
            rc = lib.b200gsr_disparity_forward(B, H * W, _lib.ptr(da), _lib.ptr(focal), _lib.ptr(out), _lib.ptr(stats),
                                               _lib.stream(dev))
        _lib.check(rc, "b200gsr_disparity_forward")
        alpha = da[:, 1:2].clone()
        ctx.deterministic = torch.are_deterministic_algorithms_enabled()   # the backward runs in the forward's mode
        ctx.save_for_backward(da, focal, stats)
        return out, alpha

    @staticmethod
    def backward(ctx, g_disp, g_alpha):
        da, focal, stats = ctx.saved_tensors
        B, _, H, W = da.shape
        dev = da.device
        g_disp = torch.zeros(B, 1, H, W, device=dev) if g_disp is None else _lib.prepare(g_disp)
        g_alpha = _lib.prepare(g_alpha)
        d_da = torch.empty_like(da)
        st = stats.clone()          # the backward accumulates into the record: keep the forward's pristine
        lib, ptr = _lib.load(), _lib.ptr
        with torch.cuda.device(dev):
            rc = lib.b200gsr_disparity_backward_ex(B, H * W, ptr(da), ptr(focal), ptr(g_disp), ptr(g_alpha), ptr(st),
                                                   ptr(d_da), _lib.BWD_DETERMINISTIC if ctx.deterministic else 0,
                                                   _lib.stream(dev))
        _lib.check(rc, "b200gsr_disparity_backward")
        return d_da, None


def disparity_from_depth_alpha(depth_alpha: torch.Tensor, focal):
    """depth_alpha [2,H,W] or [B,2,H,W] (the rasterizer's second image output); focal = float, or a
    sequence / tensor of B floats = 1 / (2 tan(FoVx/2)) per view.  -> (disp, alpha)."""
    if depth_alpha.device.type != "cuda":
        raise RuntimeError("disparity_from_depth_alpha (b200gsr): CUDA tensors only; there is no CPU fallback")
    single = depth_alpha.dim() == 3
    da = depth_alpha.unsqueeze(0) if single else depth_alpha
    B = da.shape[0]
    if not torch.is_tensor(focal):
        focal = torch.tensor([float(focal)] * B if not hasattr(focal, "__len__") else [float(f) for f in focal],
                             dtype=torch.float32, device=da.device)
    focal = focal.to(da.device, torch.float32).reshape(B).contiguous()
    disp, alpha = _Disparity.apply(da, focal)
    return (disp[0], alpha[0]) if single else (disp, alpha)
