"""The reconstruction loss of DreamScene's refine stages (DESIGN.md section 0, f9).

``recon_l2_loss(image, target, weight)`` replaces the reference's

    loss = l2_loss(image.to(torch.float16), gt_images[i]) * 100        # object_trainer.py:646-649, scene_trainer.py

(``l2_loss(a, b) = ((a - b) ** 2).mean()``, utils/system_utils.py:63-64) with one native kernel each way
(include/b200gsr_loss.h).  Same dtype rules as torch: a float16 target gives a float16 loss with every intermediate
in fp16, a float32 target a float32 loss.  The image gradient is bit for bit torch's autograd gradient of the
expression; the loss value is a fixed-order sum, within one fp16 ulp (float16) or 1e-6 relative (float32) of torch's.
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
