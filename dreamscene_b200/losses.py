"""The reconstruction loss of DreamScene's refine stages (DESIGN.md section 0, f9) and the guidance stages'
total-variation regulariser (f10).

``recon_l2_loss(image, target, weight)`` replaces the reference's

    loss = l2_loss(image.to(torch.float16), gt_images[i]) * 100        # object_trainer.py:646-649, scene_trainer.py

(``l2_loss(a, b) = ((a - b) ** 2).mean()``, utils/system_utils.py:63-64) with one native kernel each way
(include/b200gsr_loss.h).  Same dtype rules as torch: a float16 target gives a float16 loss with every intermediate
in fp16, a float32 target a float32 loss.  The image gradient is bit for bit torch's autograd gradient of the
expression; the loss value is a fixed-order sum, within one fp16 ulp (float16) or 1e-6 relative (float32) of torch's.

``tv_loss(x)`` (f10) replaces the reference's total-variation regulariser of the guidance stages
(utils/system_utils.py:39-47, object_trainer.py:380, scene_trainer.py:869-870) with the same contract: the gradient
bit for bit torch's, the value a fixed-order sum within 1e-6 relative.  StepGraph(tv_weight=...) runs it, and the
scale regulariser, inside its graphs.
"""
from __future__ import annotations

import torch

from . import _lib


class _ReconL2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, target, weight):
        lib, ptr = _lib.load(), _lib.ptr
        N = image.numel()
        dev = image.device
        loss = torch.empty((), dtype=target.dtype, device=dev)
        scratch = torch.empty(lib.b200gsr_recon_l2_scratch_bytes(1, N), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            rc = lib.b200gsr_recon_l2(1, N, ptr(image), ptr(target), int(target.dtype == torch.float16), 1, None,
                                      weight, None, ptr(loss), None, ptr(scratch), scratch.numel(), _lib.stream(dev))
        _lib.check(rc, "b200gsr_recon_l2")
        ctx.weight = weight
        ctx.save_for_backward(image, target)
        return loss

    @staticmethod
    def backward(ctx, grad_out):
        image, target = ctx.saved_tensors
        lib, ptr = _lib.load(), _lib.ptr
        dev = image.device
        go = grad_out.to(target.dtype).contiguous()
        d_image = torch.empty_like(image)
        with torch.cuda.device(dev):
            rc = lib.b200gsr_recon_l2(1, image.numel(), ptr(image), ptr(target), int(target.dtype == torch.float16), 1,
                                      None, ctx.weight, ptr(go), None, ptr(d_image), None, 0, _lib.stream(dev))
        _lib.check(rc, "b200gsr_recon_l2")
        return d_image, None, None


def recon_l2_loss(image: torch.Tensor, target: torch.Tensor, weight: float = 100.0) -> torch.Tensor:
    """weight * mean((image.to(float16) - target) ** 2) as a 0-dim tensor of target's dtype.  image: float32 CUDA;
    target: float16 or float32 CUDA of the same shape."""
    if image.dtype != torch.float32:
        raise TypeError(f"recon_l2_loss: image must be float32, got {image.dtype}")
    if target.dtype not in (torch.float16, torch.float32):
        raise TypeError(f"recon_l2_loss: target must be float16 or float32, got {target.dtype}")
    if image.shape != target.shape:
        raise ValueError(f"recon_l2_loss: image {tuple(image.shape)} and target {tuple(target.shape)} differ in shape")
    if image.device.type != "cuda" or target.device != image.device:
        raise RuntimeError("recon_l2_loss (b200gsr): image and target must be on the same CUDA device; there is no CPU "
                           "fallback")
    if not 0 < image.numel() < 2 ** 31:
        raise ValueError("recon_l2_loss: the image must have between 1 and 2^31 - 1 elements")
    return _ReconL2.apply(image.contiguous(), target.detach().contiguous(), float(weight))


class _TV(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        lib, ptr = _lib.load(), _lib.ptr
        B, C, H, W = x.shape
        loss = torch.empty((), dtype=torch.float32, device=x.device)
        scratch = torch.empty(lib.b200gsr_tv_loss_scratch_bytes(B, C, H, W), dtype=torch.uint8, device=x.device)
        with torch.cuda.device(x.device):
            rc = lib.b200gsr_tv_loss(B, C, H, W, ptr(x), None, ptr(loss), None, 0, ptr(scratch), scratch.numel(),
                                     _lib.stream(x.device))
        _lib.check(rc, "b200gsr_tv_loss")
        ctx.save_for_backward(x)
        return loss

    @staticmethod
    def backward(ctx, grad_out):
        if torch.is_grad_enabled():
            # create_graph=True: the kernel's gradient would carry no history, and a later double backward through it
            # would silently miss x's second-order terms
            raise RuntimeError("tv_loss has no double backward: its gradient kernel is not differentiable "
                               "(backward with create_graph=True)")
        x, = ctx.saved_tensors
        lib, ptr = _lib.load(), _lib.ptr
        go = grad_out.to(torch.float32).contiguous()
        d_x = torch.empty_like(x)
        with torch.cuda.device(x.device):
            rc = lib.b200gsr_tv_loss(*x.shape, ptr(x), ptr(go), None, ptr(d_x), 0, None, 0, _lib.stream(x.device))
        _lib.check(rc, "b200gsr_tv_loss")
        return d_x


def tv_loss(x: torch.Tensor) -> torch.Tensor:
    """The reference's total-variation loss of x [B,C,H,W] (float32 CUDA, H and W >= 2) as a 0-dim float32 tensor:
    2 * (h_tv / (C (H-1) W) + w_tv / (C H (W-1))) / B over the squared differences of adjacent elements.  The forward
    computes the value only (a fixed-order sum, within 1e-6 relative of torch's), the backward the gradient only (bit
    for bit torch's autograd gradient of the expression)."""
    if not torch.is_tensor(x) or x.dtype != torch.float32:
        raise TypeError(f"tv_loss: x must be a float32 tensor, got {getattr(x, 'dtype', type(x))}")
    if x.dim() != 4 or x.shape[2] < 2 or x.shape[3] < 2 or x.shape[0] < 1 or x.shape[1] < 1:
        raise ValueError(f"tv_loss: x must be [B,C,H,W] with B, C >= 1 and H, W >= 2, got {tuple(x.shape)}")
    if x.device.type != "cuda":
        raise RuntimeError("tv_loss (b200gsr): x must be a CUDA tensor; there is no CPU fallback")
    if x.numel() >= 2 ** 31:
        raise ValueError("tv_loss: x must have at most 2^31 - 1 elements")
    return _TV.apply(x.contiguous())
