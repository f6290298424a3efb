"""Fused multi-view rendering (SURVEY.md section 8 f1) - additive API, the per-view API is untouched.

DreamScene renders the C_batch_size = 4 views of a training step one after the other
(/root/reference/training/scene_trainer.py:801-832): four full passes of the nine rasterizer kernels
over small (512^2) images and four dense gradient tensors per parameter that autograd then sums.
``rasterize_views`` renders B views of the same image size in ONE tile-binning / sort / composite pass
(the views are stacked vertically into one image; view v's Gaussians are the virtual Gaussians
[v*P, (v+1)*P)); only the two per-Gaussian stages run once per view, each with its own camera.  The
backward replays the stacked image once and accumulates the gradient of every parameter tensor that
several views share directly in the kernel, so one dense gradient per shared parameter is written
instead of B.

    outs = rasterize_views(settings_list, means3D, opacities, shs=..., scales=..., rotations=...,
                           means2D=[m2d_0, ..., m2d_{B-1}])
    color_v, radii_v, depth_alpha_v = outs[v]

Frozen rows: ``frozen_rows=[(lo, hi), ...]`` (half-open ranges of the P rows, the same in every view) are rendered as
any other row, but the backward computes no gradient for them: their gradient rows and means2D rows are zeros, and
the other rows' gradients are those of the call without ``frozen_rows`` (bit for bit in deterministic mode).
``scene.frozen_rows(groups, frozen)`` gives the ranges of frozen parameter groups packed by ``scene.assemble_scene``.

Densification statistics: ``densify_stats=[(lo, hi, xyz_gradient_accum, denom, max_radii2D or None), ...]`` makes the
backward do the reference's add_densification_stats for rows [lo, hi) of view ``stats_view`` itself, in place, in the
launch that computes that view's screen-space gradient.  Without ``means2D`` no screen-space gradient is then stored
at all.  ``scene.stats_rows(groups, stats)`` gives the records of the groups packed by ``scene.assemble_scene``.

Every tensor argument is either ONE tensor (shared by all views) or a list of B tensors (per-view
values, e.g. the separately augmented shs / scales of scene_render); `settings_list` holds the B
GaussianRasterizationSettings (cameras, sh_degree, scale_modifier, bg may differ; image size and
score_flag must agree).  Per view the results equal GaussianRasterizer(settings[v])(...) - the
sorted lists are the same lists, bit for bit - and gradients equal the sum over the per-view calls.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Union

import torch

from . import _lib
from . import rasterizer as R

TensorOrList = Union[torch.Tensor, Sequence[torch.Tensor], None]
_NAMES = ("means3D", "shs", "colors_precomp", "opacities", "scales", "rotations", "cov3D_precomp")
_ACC_BIT = {"means3D": 1, "opacities": 2, "shs": 4, "colors_precomp": 4, "scales": 8, "rotations": 16, "cov3D_precomp": 32}
_GRAD_FIELD = {"means3D": "d_means3D", "opacities": "d_opacities", "shs": "d_shs", "colors_precomp": "d_colors",
               "scales": "d_scales", "rotations": "d_rotations", "cov3D_precomp": "d_cov3D"}


def _frozen_ranges(frozen_rows, P: int):
    """None or [(lo, hi), ...] -> the merged (lo, len) pairs that b200gsr_backward_views_frozen takes.  Refuses what
    the library refuses: an empty, out-of-bounds, unsorted or overlapping range, or more than MAX_FROZEN_RANGES after
    merging ranges that touch."""
    if frozen_rows is None:
        return ()
    out: list = []
    end = 0
    for k, r in enumerate(frozen_rows):
        if len(r) != 2:
            raise ValueError(f"frozen_rows[{k}]: expected a (lo, hi) pair, got {r!r}")
        lo, hi = int(r[0]), int(r[1])
        if hi <= lo:
            raise ValueError(f"frozen_rows[{k}] = ({lo}, {hi}) is empty")
        if lo < 0 or hi > P:
            raise ValueError(f"frozen_rows[{k}] = ({lo}, {hi}) is outside [0, P = {P})")
        if k > 0 and lo < end:
            raise ValueError(f"frozen_rows[{k}] = ({lo}, {hi}) starts before the end {end} of frozen_rows[{k - 1}]: "
                             "the ranges must be sorted and must not overlap")
        if out and lo == end:
            out[-1] = (out[-1][0], out[-1][1] + hi - lo)
        else:
            out.append((lo, hi - lo))
        end = hi
    if len(out) > _lib.MAX_FROZEN_RANGES:
        raise ValueError(f"frozen_rows: {len(out)} ranges after merging touching ones, at most "
                         f"{_lib.MAX_FROZEN_RANGES}")
    return tuple(out)


def _stats_records(densify_stats, P: int, dev, frozen):
    """None or [(lo, hi, accum, denom, max_radii2D or None), ...] -> the validated (lo, len, accum, denom, max_radii2D)
    records that b200gsr_backward_views_stats takes.  Refuses what the library refuses - an empty, out-of-bounds,
    unsorted or overlapping record, more than MAX_GROUPS records, a record that overlaps the merged frozen ranges
    `frozen` - and statistics tensors that are not contiguous float32 tensors of hi - lo elements on `dev`."""
    if densify_stats is None:
        return None
    out: list = []
    end = 0
    entries = list(densify_stats)
    if len(entries) > _lib.MAX_GROUPS:
        raise ValueError(f"densify_stats: {len(entries)} records, at most {_lib.MAX_GROUPS}")
    for k, e in enumerate(entries):
        if len(e) != 5 or e[2] is None or e[3] is None:
            raise ValueError(f"densify_stats[{k}] must be (lo, hi, xyz_gradient_accum, denom, max_radii2D or None)")
        lo, hi = int(e[0]), int(e[1])
        if hi <= lo:
            raise ValueError(f"densify_stats[{k}] = ({lo}, {hi}) is empty")
        if lo < 0 or hi > P:
            raise ValueError(f"densify_stats[{k}] = ({lo}, {hi}) is outside [0, P = {P})")
        if k > 0 and lo < end:
            raise ValueError(f"densify_stats[{k}] = ({lo}, {hi}) starts before the end {end} of densify_stats[{k - 1}]: "
                             "the records must be sorted and must not overlap")
        end = hi
        for flo, flen in frozen:
            if lo < flo + flen and flo < hi:
                raise ValueError(f"densify_stats[{k}] = ({lo}, {hi}) overlaps the frozen rows ({flo}, {flo + flen}): "
                                 "the reference gathers statistics for the trained rows only")
        for name, t in zip(("xyz_gradient_accum", "denom", "max_radii2D"), e[2:]):
            if t is None:
                continue
            if not torch.is_tensor(t) or t.dtype != torch.float32 or not t.is_contiguous():
                raise ValueError(f"densify_stats[{k}] {name} must be a contiguous float32 tensor")
            if t.numel() != hi - lo:
                raise ValueError(f"densify_stats[{k}] {name} has {t.numel()} elements, rows ({lo}, {hi}) are {hi - lo}")
            if t.device != dev:
                raise ValueError(f"densify_stats[{k}] {name} must be on the inputs' device ({dev})")
        out.append((lo, hi - lo, e[2], e[3], e[4]))
    return tuple(out)


class _RasterizeViews(torch.autograd.Function):
    @staticmethod
    def forward(ctx, settings, spec, B, frozen, stats, ports, *flat):
        # spec[name] = None | ("shared", idx) | ("list", [idx...]) into `flat`; flat also holds the `ports` means2D
        # ports last: B, or 0 when `stats` = (records, view) is given without them (then no screen-space gradient is
        # stored)
        lib = _lib.load()
        tensors = [_lib.prepare(t) for t in flat]
        get = lambda name, v: None if spec[name] is None else tensors[spec[name][1] if spec[name][0] == "shared" else spec[name][1][v]]
        m0 = get("means3D", 0)
        dev = m0.device
        if dev.type != "cuda":
            raise RuntimeError("rasterize_views (b200gsr): inputs must be CUDA tensors; there is no CPU fallback")
        P = int(m0.shape[0])
        sh0 = get("shs", 0)
        M = int(sh0.shape[1]) if sh0 is not None else 0
        H, W = int(settings[0].image_height), int(settings[0].image_width)
        score_flag = bool(settings[0].score_flag)
        with_backward = any(ctx.needs_input_grad)
        d = R._device_state(dev)
        capturing = torch.cuda.is_current_stream_capturing()
        if not capturing:
            d.resolve()
        keep: list = []
        with torch.cuda.device(dev):
            Hs = _lib.stacked_height(B, H, W)
            bg_all = torch.stack([R._const(s.bg, dev).reshape(3) for s in settings]).contiguous()
            prm = (_lib.Params * B)(*[R._make_params(s, P, M, keep, dev, bg_all, v) for v, s in enumerate(settings)])
            vin = R._view_inputs([[get(name, v) for name in _NAMES] for v in range(B)])
            color = torch.empty(3, Hs, W, dtype=torch.float32, device=dev)
            depth_alpha = torch.empty(2, Hs, W, dtype=torch.float32, device=dev)
            radii = torch.empty(B, P, dtype=torch.int32, device=dev)
            score = torch.zeros(B, P, dtype=torch.float32, device=dev) if score_flag else None
            stream = _lib.stream(dev)
            det = R.deterministic_mode()
            ptr = _lib.ptr

            def launch(cap, flags, scratch, saved, notify_ptr, seq):
                return lib.b200gsr_forward_views(B, prm, vin, ptr(color), ptr(depth_alpha), ptr(radii), ptr(score),
                                                 ptr(scratch), scratch.numel(), ptr(saved), saved.numel(), cap, flags,
                                                 notify_ptr, seq, stream)

            saved, cap = R._issue_with_capacity(d, (B, P, H, W), B * P, Hs, W, with_backward, det, score, launch, capturing,
                                                stream.value)
        ctx.meta = (spec, B, P, W, Hs, cap, with_backward, len(flat), det, frozen)
        ctx.stats = stats
        ctx.ports = ports
        ctx.views = (prm, vin)            # the backward reuses the arrays; `keep` holds their device constants
        ctx.keep = keep
        ctx.saved_buf = saved
        ctx.save_for_backward(radii, depth_alpha, *tensors)
        ctx.mark_non_differentiable(radii)
        ctx.set_materialize_grads(False)
        if score is not None:
            ctx.mark_non_differentiable(score)
            return color, radii, depth_alpha, score
        return color, radii, depth_alpha

    @staticmethod
    def backward(ctx, g_color, _g_radii, g_da, *_):
        spec, B, P, W, Hs, cap, with_backward, nflat, det, frozen = ctx.meta
        prm, vin = ctx.views
        radii, depth_alpha = ctx.saved_tensors[:2]
        tensors = list(ctx.saved_tensors[2:])
        dev = radii.device
        lib = _lib.load()
        if not with_backward:
            raise RuntimeError("b200gsr: backward through a forward that ran without gradient accumulators")
        get = lambda name, v: None if spec[name] is None else tensors[spec[name][1] if spec[name][0] == "shared" else spec[name][1][v]]
        g_color = torch.zeros(3, Hs, W, device=dev) if g_color is None else _lib.prepare(g_color)
        g_da = torch.zeros(2, Hs, W, device=dev) if g_da is None else _lib.prepare(g_da)
        grads: List[Optional[torch.Tensor]] = [None] * nflat
        m2d_base = nflat - ctx.ports
        with torch.cuda.device(dev):
            out = (_lib.ViewGrads * B)()
            for v in range(B):
                acc = 0
                for name in _NAMES:
                    t = get(name, v)
                    if t is None:
                        continue
                    idx = spec[name][1] if spec[name][0] == "shared" else spec[name][1][v]
                    if grads[idx] is None:
                        grads[idx] = torch.empty_like(t)           # first view writing this tensor's gradient
                    else:
                        acc |= _ACC_BIT[name]                      # shared with an earlier view: accumulate in the kernel
                    setattr(out[v], _GRAD_FIELD[name], grads[idx].data_ptr())
                if ctx.ports:
                    g2 = torch.empty(P, 3, dtype=torch.float32, device=dev)
                    grads[m2d_base + v] = g2
                    out[v].d_means2D = g2.data_ptr()
                out[v].accumulate = acc
            ptr = _lib.ptr
            args = (B, prm, vin, ptr(radii), ptr(depth_alpha), ptr(g_color), ptr(g_da), ptr(ctx.saved_buf),
                    ctx.saved_buf.numel(), cap, out, _lib.BWD_DETERMINISTIC if det else 0)
            ranges = (_lib.RowRange * len(frozen))(*[_lib.RowRange(lo, n) for lo, n in frozen]) if frozen else None
            if ctx.stats is not None:
                records, view = ctx.stats
                rec = (_lib.RowStats * len(records))(*[_lib.RowStats(lo, n, *[ptr(t) for t in ts])
                                                       for lo, n, *ts in records]) if records else None
                name = "b200gsr_backward_views_stats"
                rc = lib.b200gsr_backward_views_stats(*args, ranges, len(frozen), rec, len(records), view,
                                                      _lib.stream(dev))
            elif frozen:
                name = "b200gsr_backward_views_frozen"
                rc = lib.b200gsr_backward_views_frozen(*args, ranges, len(frozen), _lib.stream(dev))
            else:
                name = "b200gsr_backward_views"
                rc = lib.b200gsr_backward_views_ex(*args, _lib.stream(dev))
        _lib.check(rc, name)
        return (None,) * 6 + tuple(grads)


def rasterize_views(settings: Sequence[R.GaussianRasterizationSettings], means3D: TensorOrList, opacities: TensorOrList,
                    shs: TensorOrList = None, colors_precomp: TensorOrList = None, scales: TensorOrList = None,
                    rotations: TensorOrList = None, cov3D_precomp: TensorOrList = None,
                    means2D: Optional[Sequence[torch.Tensor]] = None,
                    frozen_rows: Optional[Sequence[Sequence[int]]] = None,
                    densify_stats: Optional[Sequence] = None, stats_view: int = -1):
    """-> list of B tuples (color[3,H,W], radii[P], depth_alpha[2,H,W]) (score first when score_flag), views
    into the stacked outputs.  means2D: optional list of B [P,3] tensors whose .grad receives the per-view
    screen-space gradients (the reference's viewspace_points).  frozen_rows: None, or sorted, non-overlapping,
    non-empty (lo, hi) ranges of the P rows (at most MAX_FROZEN_RANGES once touching ones merge) whose gradient the
    backward does not compute: their rows of every input's gradient and of the means2D gradients are zeros, and the
    other rows get the gradients of the call without frozen_rows.

    densify_stats: None, or sorted, non-overlapping, non-empty records (lo, hi, xyz_gradient_accum, denom, max_radii2D
    or None) of the P rows (at most MAX_GROUPS, none overlapping frozen_rows), each tensor a contiguous float32 tensor
    of hi - lo elements on the inputs' device.  The backward then does the reference's add_densification_stats for
    view `stats_view` inside the render backward, in place: for each row of a record whose radius in that view is
    positive, xyz_gradient_accum[row - lo] += |screen-space gradient[:2]|, denom[row - lo] += 1, max_radii2D[row - lo]
    = max(max_radii2D[row - lo], radius) - bit for bit what densify.add_densification_stats does with that view's
    means2D gradient and radii.  Each backward adds once (a retain_graph second backward adds again); no backward, no
    statistics.  Without means2D no screen-space gradient is stored at all; with it both are produced.
    scene.stats_rows(groups, stats) gives the records of assemble_scene's packed groups.
    stats_view: the view whose statistics are gathered: -1 (default) is the last view, B - 1, as render_scene's."""
    B = len(settings)
    if not 1 <= B <= _lib.MAX_VIEWS:
        raise ValueError(f"need 1..{_lib.MAX_VIEWS} views")
    args = dict(means3D=means3D, shs=shs, colors_precomp=colors_precomp, opacities=opacities, scales=scales,
                rotations=rotations, cov3D_precomp=cov3D_precomp)
    if (shs is None) == (colors_precomp is None):
        raise Exception("Please provide excatly one of either SHs or precomputed colors!")
    if ((scales is None or rotations is None) and cov3D_precomp is None) or \
            ((scales is not None or rotations is not None) and cov3D_precomp is not None):
        raise Exception("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")
    flat: list = []
    spec = {}
    for name in _NAMES:
        a = args[name]
        if a is None:
            spec[name] = None
        elif torch.is_tensor(a):
            spec[name] = ("shared", len(flat)); flat.append(a)
        else:
            if len(a) != B:
                raise ValueError(f"{name}: expected {B} per-view tensors")
            spec[name] = ("list", list(range(len(flat), len(flat) + B))); flat.extend(a)
    P = int((means3D if torch.is_tensor(means3D) else means3D[0]).shape[0])
    dev = (means3D if torch.is_tensor(means3D) else means3D[0]).device
    if means2D is None:
        # with densify_stats no port is needed: the backward then writes no screen-space gradient
        means2D = [] if densify_stats is not None else [torch.zeros(P, 3, device=dev) for _ in range(B)]
    elif len(means2D) != B:
        raise ValueError(f"means2D: expected {B} per-view tensors")
    flat.extend(means2D)
    H = int(settings[0].image_height)
    for s in settings:
        if int(s.image_height) != H or int(s.image_width) != int(settings[0].image_width) or bool(s.score_flag) != bool(settings[0].score_flag):
            raise ValueError("all views must share the image size and score_flag")
    frozen = _frozen_ranges(frozen_rows, P)
    stats = None
    if densify_stats is not None:
        sv = int(stats_view)
        if not -1 <= sv < B:
            raise ValueError(f"rasterize_views: stats_view must be -1 (the last view) or in 0..{B - 1}, got {stats_view}")
        stats = (_stats_records(densify_stats, P, dev, frozen), B - 1 if sv == -1 else sv)
    res = _RasterizeViews.apply(tuple(settings), spec, B, frozen, stats, len(means2D), *flat)
    color, radii, da = res[0], res[1], res[2]
    Hp = color.shape[1] // B
    outs = []
    for v in range(B):
        item = (color[:, v * Hp:v * Hp + H, :], radii[v], da[:, v * Hp:v * Hp + H, :])
        if len(res) == 4:
            item = (res[3][v],) + item
        outs.append(item)
    return outs
