"""Densification / pruning (SURVEY.md section 8 f4) - additive API over libb200gsr's primitives.

Functional equivalents of the reference's GaussianModel methods (/root/reference/gs_renderer.py):
  add_densification_stats  (:1046-1051 + the max_radii2D update of training/object_trainer.py:385-390)
  densify_and_prune        (:1010-1024 = densify_and_clone :986-1008 + densify_and_split :949-984 + prune)
  prune_points             (:889-903, incl. the Adam-state surgery of _prune_optimizer :868-887)
  prune_by_score           (prune_gaussians :1076-1081: percentile of the important score)
They take and return plain dicts of tensors (names as in the reference's optimizer groups:
xyz, f_dc, f_rest, opacity, scaling, rotation) plus, optionally, the Adam moments
{name: (exp_avg, exp_avg_sq)}; wiring the results back into nn.Parameters / the optimizer is the caller's
(INTEGRATION.md shows the few lines).  Everything index-related runs in a handful of kernels; the only
host synchronisation is reading the new point count to size the output tensors.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch

from . import _lib

PARAM_NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")


def _cuda_device(t: torch.Tensor) -> torch.device:
    if t.device.type != "cuda":
        raise RuntimeError("densify (b200gsr): CUDA tensors only; there is no CPU fallback")
    return t.device


def add_densification_stats(viewspace_grad: torch.Tensor, radii: torch.Tensor, xyz_gradient_accum: torch.Tensor,
                            denom: torch.Tensor, max_radii2D: Optional[torch.Tensor] = None) -> None:
    """In place, for the view just rendered: where radii > 0: accum += |grad[:, :2]|, denom += 1,
    max_radii2D = max(max_radii2D, radii)."""
    dev = _cuda_device(viewspace_grad)
    P = int(viewspace_grad.shape[0])
    g, r = _lib.prepare(viewspace_grad.detach()), radii.detach().to(torch.int32).contiguous()
    for t in (xyz_gradient_accum, denom) + ((max_radii2D,) if max_radii2D is not None else ()):
        assert t.is_contiguous() and t.dtype == torch.float32 and t.numel() == P
    ptr = _lib.ptr
    with torch.cuda.device(dev):
        _lib.check(_lib.load().b200gsr_densify_stats(P, ptr(g), ptr(r), ptr(xyz_gradient_accum), ptr(denom),
                                                     ptr(max_radii2D), _lib.stream(dev)), "b200gsr_densify_stats")


def _gather_all(lib, dev, src_map, n_out, params, adam):
    out_p, out_a = {}, None
    ptr, stream = _lib.ptr, _lib.stream(dev)
    for name, t in params.items():
        t = _lib.prepare(t.detach())
        row = t[0].numel() if t.shape[0] else int(torch.tensor(t.shape[1:]).prod())
        o = torch.empty((n_out,) + tuple(t.shape[1:]), dtype=torch.float32, device=dev)
        _lib.check(lib.b200gsr_gather_rows(n_out, row, ptr(src_map), ptr(t), ptr(o), 0, stream), "b200gsr_gather_rows")
        out_p[name] = o
    if adam is not None:
        out_a = {}
        for name, (m1, m2) in adam.items():
            res = []
            for m in (m1, m2):
                m = _lib.prepare(m.detach())
                row = m[0].numel() if m.shape[0] else int(torch.tensor(m.shape[1:]).prod())
                o = torch.empty((n_out,) + tuple(m.shape[1:]), dtype=torch.float32, device=dev)
                _lib.check(lib.b200gsr_gather_rows(n_out, row, ptr(src_map), ptr(m), ptr(o), 1, stream),
                           "b200gsr_gather_rows")
                res.append(o)
            out_a[name] = tuple(res)
    return out_p, out_a


def densify_and_prune(params: Dict[str, torch.Tensor], adam: Optional[Dict[str, Tuple[torch.Tensor, torch.Tensor]]],
                      xyz_gradient_accum: torch.Tensor, denom: torch.Tensor, max_grad: float, min_opacity: float,
                      extent: float, max_screen_size, percent_dense: float = 0.01, N: int = 2,
                      generator: Optional[torch.Generator] = None, z: Optional[torch.Tensor] = None):
    """-> (new_params, new_adam, info).  Output order and every decision follow the reference:
    [kept originals | clones | N blocks of split children].  The densification statistics of the new set
    are zeros (densification_postfix), returned in info["xyz_gradient_accum" / "denom" / "max_radii2D"].
    z: the standard-normal draws of torch.normal(std=stds) [N * split parents, 3] (drawn here if omitted)."""
    lib = _lib.load()
    dev = _cuda_device(params["xyz"])
    P = int(params["xyz"].shape[0])
    src = {k: _lib.prepare(params[k].detach()) for k in PARAM_NAMES}   # split_children reads rotation as float4
    ptr = _lib.ptr
    with torch.cuda.device(dev):
        stream = _lib.stream(dev)
        scratch = torch.empty(int(lib.b200gsr_densify_scratch_bytes(P)), dtype=torch.uint8, device=dev)
        totals = torch.zeros(5, dtype=torch.int32, device=dev)
        big_ws = 0.1 * extent if max_screen_size else 0.0
        child_div = float(torch.tensor(0.8 * N, dtype=torch.float32))
        _lib.check(lib.b200gsr_densify_plan(P, ptr(_lib.prepare(xyz_gradient_accum.detach())),
                                            ptr(_lib.prepare(denom.detach())), ptr(src["scaling"]),
                                            ptr(src["opacity"]), float(max_grad), float(percent_dense * extent),
                                            float(min_opacity), float(big_ws), child_div, ptr(scratch), ptr(totals), stream),
                   "b200gsr_densify_plan")
        n_keep, n_clone, n_child, n_sel, _ = [int(x) for x in totals.tolist()]       # the one host sync: output sizes
        n_out = n_keep + n_clone + N * n_child
        src_map = torch.empty(max(n_out, 1), dtype=torch.int32, device=dev)
        child_draw = torch.empty(max(N * n_child, 1), dtype=torch.int32, device=dev)
        _lib.check(lib.b200gsr_densify_map(P, N, ptr(scratch), ptr(totals), ptr(src_map), ptr(child_draw), stream),
                   "b200gsr_densify_map")
        new_p, new_a = _gather_all(lib, dev, src_map, n_out, src, adam)
        if z is None:
            z = torch.randn(max(N * n_sel, 1), 3, device=dev, generator=generator)
        z = _lib.prepare(z.detach())
        _lib.check(lib.b200gsr_split_children(n_out, n_keep + n_clone, child_div, ptr(src_map), ptr(child_draw),
                                              ptr(src["xyz"]), ptr(src["scaling"]), ptr(src["rotation"]), ptr(z),
                                              ptr(new_p["xyz"]), ptr(new_p["scaling"]), stream), "b200gsr_split_children")
    info = dict(kept=n_keep, cloned=n_clone, split_parents=n_sel, split_parents_surviving=n_child, points=n_out,
                src_map=src_map[:n_out], xyz_gradient_accum=torch.zeros(n_out, 1, device=dev),
                denom=torch.zeros(n_out, 1, device=dev), max_radii2D=torch.zeros(n_out, device=dev))
    return new_p, new_a, info


def prune_points(params: Dict[str, torch.Tensor], adam, stats: Optional[Dict[str, torch.Tensor]], prune_mask: torch.Tensor):
    """Remove the rows where prune_mask is True from every parameter, Adam moment and statistics array."""
    lib = _lib.load()
    dev = prune_mask.device
    P = int(prune_mask.shape[0])
    keep = (~prune_mask.bool()).to(torch.uint8).contiguous()
    with torch.cuda.device(dev):
        scratch = torch.empty(int(lib.b200gsr_densify_scratch_bytes(P)), dtype=torch.uint8, device=dev)
        count = torch.zeros(1, dtype=torch.int32, device=dev)
        src_map = torch.empty(max(P, 1), dtype=torch.int32, device=dev)
        _lib.check(lib.b200gsr_compact_plan(P, _lib.ptr(keep), _lib.ptr(scratch), _lib.ptr(src_map), _lib.ptr(count),
                                            _lib.stream(dev)), "b200gsr_compact_plan")
        n_out = int(count.item())
        new_p, new_a = _gather_all(lib, dev, src_map, n_out, params, adam)
        new_s = None
        if stats is not None:
            new_s, _ = _gather_all(lib, dev, src_map, n_out, stats, None)
    return new_p, new_a, new_s


def kth_smallest(v: torch.Tensor, k: int) -> torch.Tensor:
    """-> device tensor [1]: the k-th smallest (0-based) element of v (any shape), without a sort or host sync."""
    v = _lib.prepare(v.detach()).reshape(-1)
    dev = v.device
    out = torch.empty(1, dtype=torch.float32, device=dev)
    scratch = torch.empty(2048, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().b200gsr_kth_smallest(int(v.numel()), _lib.ptr(v), int(k), _lib.ptr(scratch), _lib.ptr(out),
                                                    _lib.stream(dev)), "b200gsr_kth_smallest")
    return out


def percentile_threshold(score: torch.Tensor, percent: float) -> torch.Tensor:
    """sorted(score)[int(percent * (n - 1))] without sorting (device scalar, no host sync)."""
    return kth_smallest(score, int(percent * (score.numel() - 1)))


def prune_by_score(params, adam, stats, important_score: torch.Tensor, percent: float):
    """prune_gaussians(percent, important_score): drop everything at or below the percentile."""
    thr = percentile_threshold(important_score, percent)
    return prune_points(params, adam, stats, (important_score.reshape(-1) <= thr))
