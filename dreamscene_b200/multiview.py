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


class _RasterizeViews(torch.autograd.Function):
    @staticmethod
    def forward(ctx, settings, spec, B, *flat):
        # spec[name] = None | ("shared", idx) | ("list", [idx...]) into `flat`; flat also holds the B means2D ports last
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
        ctx.meta = (spec, B, P, W, Hs, cap, with_backward, len(flat), det)
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
        spec, B, P, W, Hs, cap, with_backward, nflat, det = ctx.meta
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
        m2d_base = nflat - B
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
                g2 = torch.empty(P, 3, dtype=torch.float32, device=dev)
                grads[m2d_base + v] = g2
                out[v].d_means2D = g2.data_ptr()
                out[v].accumulate = acc
            ptr = _lib.ptr
            rc = lib.b200gsr_backward_views_ex(B, prm, vin, ptr(radii), ptr(depth_alpha), ptr(g_color), ptr(g_da),
                                               ptr(ctx.saved_buf), ctx.saved_buf.numel(), cap, out,
                                               _lib.BWD_DETERMINISTIC if det else 0, _lib.stream(dev))
        _lib.check(rc, "b200gsr_backward_views")
        return (None, None, None) + tuple(grads)


def rasterize_views(settings: Sequence[R.GaussianRasterizationSettings], means3D: TensorOrList, opacities: TensorOrList,
                    shs: TensorOrList = None, colors_precomp: TensorOrList = None, scales: TensorOrList = None,
                    rotations: TensorOrList = None, cov3D_precomp: TensorOrList = None,
                    means2D: Optional[Sequence[torch.Tensor]] = None):
    """-> list of B tuples (color[3,H,W], radii[P], depth_alpha[2,H,W]) (score first when score_flag), views
    into the stacked outputs.  means2D: optional list of B [P,3] tensors whose .grad receives the per-view
    screen-space gradients (the reference's viewspace_points)."""
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
        means2D = [torch.zeros(P, 3, device=dev) for _ in range(B)]
    if len(means2D) != B:
        raise ValueError(f"means2D: expected {B} per-view tensors")
    flat.extend(means2D)
    H = int(settings[0].image_height)
    for s in settings:
        if int(s.image_height) != H or int(s.image_width) != int(settings[0].image_width) or bool(s.score_flag) != bool(settings[0].score_flag):
            raise ValueError("all views must share the image size and score_flag")
    res = _RasterizeViews.apply(tuple(settings), spec, B, *flat)
    color, radii, da = res[0], res[1], res[2]
    Hp = color.shape[1] // B
    outs = []
    for v in range(B):
        item = (color[:, v * Hp:v * Hp + H, :], radii[v], da[:, v * Hp:v * Hp + H, :])
        if len(res) == 4:
            item = (res[3][v],) + item
        outs.append(item)
    return outs
