"""3D Gaussian filtering (SURVEY.md section 8(a) a9) - additive API over b200gsr_score_views.

The reference (/root/reference/scene_gaussian.py:1046-1103) prunes an object in three steps:
  prune_list             48 full score_flag renders from random sphere cameras, scores summed in view order;
  calculate_v_imp_score  the summed score weighted by (volume / kth) ** v_pow, kth = element int(0.9 n) of the
                         volumes sorted in descending order;
  prune_gaussians        drop everything at or below the percent-th element of the sorted weighted score.
Here:
  important_score        the summed score of any number of views, as stacked score-only passes (no SH read, no
                         image, no backward state) adding into one [P] accumulator;
  volume_weighted_score  calculate_v_imp_score with the same elementwise torch ops and the sort replaced by
                         b200gsr_kth_smallest (no host sync);
  gaussian_filtering     both, then densify.prune_by_score; returns what densify.prune_points returns.

Under torch.use_deterministic_algorithms(True) (read at call time) the score is summed in 64-bit fixed point:
bitwise reproducible and independent of views_per_pass.  Its headroom is 2^26 pixels over all views of one call
(256 views of 512 x 512); larger camera sets are refused.
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence, Tuple

import torch

from . import _lib
from . import densify as _densify
from . import rasterizer as R


def view_chunks(n_views: int, views_per_pass: int):
    """[(first, end)] of the stacked passes that cover n_views views, at most views_per_pass each."""
    return [(b, min(b + views_per_pass, n_views)) for b in range(0, n_views, views_per_pass)]


def important_score(settings_list: Sequence[R.GaussianRasterizationSettings], means3D: torch.Tensor,
                    opacities: torch.Tensor, scales: Optional[torch.Tensor] = None,
                    rotations: Optional[torch.Tensor] = None, cov3D_precomp: Optional[torch.Tensor] = None, *,
                    views_per_pass: int = 16) -> torch.Tensor:
    """-> float32 [P]: the sum over the views of settings_list of the important score that
    GaussianRasterizer(settings with score_flag=True) returns (sh_degree, bg and score_flag of the settings are
    irrelevant).  Non-differentiable.  The views run as stacked passes of up to views_per_pass views
    (1..16) adding into one accumulator.  A pass that overflowed its pair capacity adds nothing and is re-issued
    with a larger one, so the result never contains a partial pass."""
    views_per_pass = int(views_per_pass)
    if not 1 <= views_per_pass <= _lib.MAX_VIEWS:
        raise ValueError(f"views_per_pass must be in 1..{_lib.MAX_VIEWS}, got {views_per_pass}")
    if ((scales is None or rotations is None) and cov3D_precomp is None) or \
            ((scales is not None or rotations is not None) and cov3D_precomp is not None):
        raise ValueError("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")
    settings_list = list(settings_list)
    n_views = len(settings_list)
    if n_views:
        H, W = int(settings_list[0].image_height), int(settings_list[0].image_width)
        for s in settings_list:
            if int(s.image_height) != H or int(s.image_width) != W:
                raise ValueError("all views must share the image size")
    else:
        H = W = 0
    det = R.deterministic_mode()
    if det and n_views * H * W > _lib.SCORE_DET_MAX_PIXELS:
        raise ValueError(f"deterministic important score: {n_views} views of {W}x{H} are {n_views * H * W} pixels; the "
                         f"64-bit fixed-point sum has headroom for {_lib.SCORE_DET_MAX_PIXELS} (2^26) pixels")
    dev = means3D.device
    if dev.type != "cuda":
        raise RuntimeError("important_score (b200gsr): inputs must be CUDA tensors; there is no CPU fallback")
    if torch.cuda.is_current_stream_capturing():
        raise RuntimeError("important_score waits for the pair counts of its passes and cannot be captured into a CUDA graph")
    P = int(means3D.shape[0])
    if P == 0 or n_views == 0:
        return torch.zeros(P, dtype=torch.float32, device=dev)
    lib = _lib.load()
    with torch.no_grad(), torch.cuda.device(dev):
        inputs = [_lib.prepare(None if t is None else t.detach())
                  for t in (means3D, None, None, opacities, scales, rotations, cov3D_precomp)]
        d = R._device_state(dev)
        d.resolve()                            # non-blocking overflow check of earlier forwards, as every forward does
        stream = _lib.stream(dev)
        acc = torch.zeros(P, dtype=torch.int64 if det else torch.float32, device=dev)
        flags = _lib.FWD_NO_BACKWARD | (_lib.FWD_DETERMINISTIC if det else 0)
        keep: list = []
        # M = 0 and no background: the score pass reads no colour (nor sh_degree or score_flag)
        params = [R._make_params(s, P, 0, keep, dev, None) for s in settings_list]

        def issue(b0, b1, cap):
            B = b1 - b0
            prm = (_lib.Params * B)(*params[b0:b1])
            vin = R._view_inputs([inputs] * B)

            def launch(cap, flags, scratch, saved, notify_ptr, seq):
                return lib.b200gsr_score_views(B, prm, vin, _lib.ptr(acc), _lib.ptr(scratch), scratch.numel(),
                                               _lib.ptr(saved), saved.numel(), cap, flags, notify_ptr, seq, stream)

            # `saved` holds no deterministic state in the score pass: the accumulator does
            layout = (B * P, _lib.stacked_height(B, H, W), W, False, False)
            _, slot, seq = R._issue_once(d, layout, flags, cap, launch, stream.value, False, "b200gsr_score_views")
            return slot, seq

        def settle(items):
            # A pass that overflowed added nothing to `acc`: it is re-issued as it is, without zeroing anything.
            for b0, b1, key, cap, slot, seq in items:
                d.settle(key, cap, slot, seq, lambda c, b0=b0, b1=b1: issue(b0, b1, c))

        # Every pass is issued without waiting once its shape's capacity is known; the pair counts are read after
        # the last pass is enqueued, and only passes that overflowed (and so added nothing) are issued again.
        pending = []
        for b0, b1 in view_chunks(n_views, views_per_pass):
            key = (b1 - b0, P, H, W)
            cap, known = d.capacity_for(key, (b1 - b0) * P, False)
            item = (b0, b1, key, cap) + issue(b0, b1, cap)
            if known:
                pending.append(item)
                if len(pending) >= 64:              # bound the notify slots held by this call
                    settle(pending)
                    pending = []
            else:
                settle([item])                      # a shape seen for the first time: learn its capacity now
        settle(pending)

        if not det:
            return acc
        score = torch.empty(P, dtype=torch.float32, device=dev)
        _lib.check(lib.b200gsr_score_finish(P, _lib.ptr(acc), _lib.ptr(score), _lib.FWD_DETERMINISTIC, stream),
                   "b200gsr_score_finish")
        return score


def volume_weighted_score(score: torch.Tensor, scaling_raw: torch.Tensor, v_pow: float) -> torch.Tensor:
    """calculate_v_imp_score: score * (volume / kth) ** v_pow with volume = prod(exp(scaling_raw), 1) and kth the
    element int(0.9 n) of the volumes in descending order.  The elementwise ops are the reference's torch ops (so
    bit-identical); the sort is replaced by b200gsr_kth_smallest at rank n - 1 - int(0.9 n) (no host sync)."""
    volume = torch.prod(torch.exp(scaling_raw.detach()), dim=1)
    n = int(volume.numel())
    if n == 0:
        return torch.zeros_like(volume)
    index = int(n * 0.9)
    kth = _densify.kth_smallest(volume, n - 1 - index).reshape(())
    v_list = torch.pow(volume / kth, v_pow)
    return v_list * score.detach()


def gaussian_filtering(params: Dict[str, torch.Tensor], adam: Optional[Dict[str, Tuple[torch.Tensor, torch.Tensor]]],
                       stats: Optional[Dict[str, torch.Tensor]], settings_list: Sequence[R.GaussianRasterizationSettings],
                       v_pow: float, prune_decay: float, prune_percent: float, *, views_per_pass: int = 16,
                       score: Optional[torch.Tensor] = None):
    """The reference's gaussian_filtering on a params dict (raw leaves xyz, opacity, scaling, rotation, ... as in
    densify): important score over settings_list of the activated Gaussians (sigmoid opacity, exp scaling,
    normalised rotation), volume weighting, then prune_by_score at percent prune_decay ** 1 * prune_percent.
    score: a precomputed important score [P] instead of the renders (e.g. one summed over ranks).
    -> (params, adam, stats) of the kept rows, as densify.prune_points."""
    if score is None:
        with torch.no_grad():
            score = important_score(settings_list, params["xyz"], torch.sigmoid(params["opacity"]),
                                    scales=torch.exp(params["scaling"]),
                                    rotations=torch.nn.functional.normalize(params["rotation"]),
                                    views_per_pass=views_per_pass)
    v_list = volume_weighted_score(score, params["scaling"], v_pow)
    return _densify.prune_by_score(params, adam, stats, v_list, (prune_decay ** 1) * prune_percent)
