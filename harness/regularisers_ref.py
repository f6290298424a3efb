"""The guidance stages' regularisers as torch expressions (harness code for the f10 tests and benchmarks).

tv_loss is the reference's total variation (utils/system_utils.py:39-47), restated with the same torch ops in the
same order, so that its autograd graph - and so its gradient - is the reference's:

    2 * (sum((x[:, :, 1:] - x[:, :, :-1]) ** 2) / (C (H-1) W) + sum((x[..., 1:] - x[..., :-1]) ** 2) / (C H (W-1))) / B

scale_loss is the scale regulariser of object_trainer.py:379 / scene_trainer.py:868.  tv_grad restates the gradient
autograd computes for tv_loss term by term, in the order the engine accumulates it; it pins that order on the CPU.
"""
import torch


def tv_loss(x: torch.Tensor) -> torch.Tensor:
    B, C, H, W = x.shape
    # the ops are created in the reference's order (the h term's, then the w term's): the autograd engine's order of
    # accumulation, and so the gradient's rounding, follows it
    h_sq = torch.pow(x[:, :, 1:, :] - x[:, :, :H - 1, :], 2).sum()
    w_sq = torch.pow(x[:, :, :, 1:] - x[:, :, :, :W - 1], 2).sum()
    return 2 * (h_sq / (C * (H - 1) * W) + w_sq / (C * H * (W - 1))) / B


def scale_loss(scales: torch.Tensor) -> torch.Tensor:
    return torch.mean(scales, dim=-1).mean()


def tv_grad(x: torch.Tensor, g: torch.Tensor) -> torch.Tensor:
    """tv_loss(x)'s gradient for the incoming 0-dim gradient g, with the scalar divisions as torch does them on x's
    device: ((w+ + w-) + h-) + h+, the zero-padded contributions of the minuends (+) and subtrahends (-)."""
    B, C, H, W = x.shape
    g2 = 2 * (g / B)
    gh, gw = g2 / (C * (H - 1) * W), g2 / (C * H * (W - 1))
    ch = gh * (2 * (x[:, :, 1:] - x[:, :, :-1]))
    cw = gw * (2 * (x[..., 1:] - x[..., :-1]))
    wp, wm, hp, hm = (torch.zeros_like(x) for _ in range(4))
    wp[..., 1:] = cw
    wm[..., :-1] = -cw
    hp[:, :, 1:] = ch
    hm[:, :, :-1] = -ch
    return ((wp + wm) + hm) + hp
